"""Multi-step RNNUqRangeEstimate timings (forecast_steps = 2): predict at B=65536, T=48, F=32, O=16, H=256, one trunk
layer, dropout 0.2 / recurrent dropout 0.1 (MC dropout) at fp32, bf16 and bf16x3, and the fp32 train step at B=4096.
One JSON line per case with the mean ms per call (CUDA events, after warm-up), the card and its power limit as read in
the same run.

    python tools/bench_uq_chain.py [--iters 5] [--warmup 2] [--batch 65536] [--train-batch 4096]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'oracle'))

import lfm_oracle as orc  # noqa: E402
from lfm_quant_b200.engine import ForecastChainEngine  # noqa: E402

T, F, O, H, L, S = 48, 32, 16, 256, 1, 2
DROP = dict(dropout=0.2, recurrent_dropout=0.1, seed=521)


def _power_limit_w():
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader,nounits', '-i',
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:
        return None


def _time(fn, warmup, iters):
    for i in range(warmup):
        fn(i)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(iters):
        fn(warmup + i)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def _engine(B, precision, train):
    eng = ForecastChainEngine(forecast_steps=S, weights=[1.0, 0.5], max_batch=B, seq_len=T, n_inputs=F, n_outputs=O,
                              num_hidden=H, num_layers=L, target_idx=3, precision=precision, train=train,
                              forward_only=not train, uq=True, **DROP)
    # the trunk's weights, then one recurrent layer + both heads per extra stage
    w = orc.init_params(L, F, O, H, init_scale=1.0, seed=521, dtype=np.float32, uq=True)
    for s in range(1, S):
        w += orc.init_params(1, F, O, H, init_scale=1.0, seed=521 + 7 * s, dtype=np.float32, uq=True)
    eng.set_weights(w)
    return eng


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--batch', type=int, default=65536)
    ap.add_argument('--train-batch', type=int, default=4096)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_uq_chain needs a CUDA device')
    card, power = torch.cuda.get_device_name(), _power_limit_w()
    rng = np.random.default_rng(0)
    base = dict(forecast_steps=S, T=T, F=F, O=O, H=H, L=L, card=card, power_limit_w=power, **DROP)
    for prec in ('fp32', 'bf16', 'bf16x3'):
        eng = _engine(a.batch, prec, train=False)
        x = torch.from_numpy(rng.standard_normal((a.batch, T, F), dtype=np.float32)).cuda()
        ms = _time(lambda i: eng.forward(x, step=i), a.warmup, a.iters)
        print(json.dumps(dict(case='uq_chain_predict', precision=prec, B=a.batch, ms=round(ms, 3), **base)), flush=True)
        eng.close()
        del eng, x
        torch.cuda.empty_cache()
    B = a.train_batch
    eng = _engine(B, 'fp32', train=True)
    x = torch.from_numpy(rng.standard_normal((B, T, F), dtype=np.float32)).cuda()
    ys = [torch.from_numpy(rng.standard_normal((B, T, O), dtype=np.float32)).cuda() for _ in range(S)]
    ms = _time(lambda i: eng.train_step(x, ys, i, 0.01), a.warmup, a.iters)
    print(json.dumps(dict(case='uq_chain_train_step', precision='fp32', B=B, ms=round(ms, 3), **base)), flush=True)
    eng.close()


if __name__ == '__main__':
    main()
