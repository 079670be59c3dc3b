"""Forward-only (predict) timings of every cell / head / precision at the predict.py scale: B=65536, T=48, F=32, O=16,
H=256, one layer.  One JSON line per case with the mean ms per forward call (CUDA events, after warm-up), the card and its
power limit as read in the same run.

    python tools/bench_infer.py [--iters 5] [--warmup 2] [--batch 65536]

Cases: {lstm, gru} x {point, uq (dropout 0.2, recurrent dropout 0.1: MC dropout)} x {fp32, bf16, bf16x3}, plus the LSTM
point estimate at bf16 under LFMQ_FORCE_GENERIC=1 (the general stepped path, like for like with the GRU).
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
from lfm_quant_b200.engine import ForecasterEngine  # noqa: E402


def _power_limit_w():
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader,nounits', '-i',
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:
        return None


def run_case(cell, uq, precision, generic, a, card, power):
    T, F, O, H, B = 48, 32, 16, 256, a.batch
    kw = dict(dropout=0.2, recurrent_dropout=0.1, seed=521) if uq else {}
    if generic:
        os.environ['LFMQ_FORCE_GENERIC'] = '1'
    try:
        eng = ForecasterEngine(max_batch=B, seq_len=T, n_inputs=F, n_outputs=O, num_hidden=H, target_idx=3,
                               precision=precision, train=False, forward_only=True, rnn_cell=cell, uq=uq, **kw)
    finally:
        os.environ.pop('LFMQ_FORCE_GENERIC', None)
    rng = np.random.default_rng(0)
    eng.set_weights(orc.init_params(1, F, O, H, init_scale=1.0, seed=521, dtype=np.float32, rnn_cell=cell, uq=uq))
    x = torch.from_numpy(rng.standard_normal((B, T, F), dtype=np.float32)).cuda()
    for i in range(a.warmup):
        eng.forward(x, step=i)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(a.iters):
        eng.forward(x, step=a.warmup + i)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / a.iters
    eng.close()
    del eng, x
    torch.cuda.empty_cache()
    print(json.dumps({'cell': cell, 'head': 'uq' if uq else 'point', 'precision': precision,
                      'path': 'generic-forced' if generic else 'default', 'B': B, 'T': T, 'F': F, 'O': O, 'H': H,
                      'ms_per_forward': round(ms, 3), 'seq_per_s': round(B / ms * 1e3), 'card': card,
                      'power_limit_w': power}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--batch', type=int, default=65536)
    a = ap.parse_args()
    card, power = torch.cuda.get_device_name(), _power_limit_w()
    for cell in ('lstm', 'gru'):
        for uq in (False, True):
            for precision in ('fp32', 'bf16', 'bf16x3'):
                run_case(cell, uq, precision, False, a, card, power)
    run_case('lstm', False, 'bf16', True, a, card, power)


if __name__ == '__main__':
    main()
