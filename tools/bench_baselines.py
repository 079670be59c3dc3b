"""MLPLinearPointEstimate timings on the dense handle: the train step (forward, MLP loss, weight gradient, clip, Adadelta)
at B=4096 and predict (the forward) at B=65536, T=48, F=32, O=16.  One JSON line per case with the mean ms per call
(CUDA events around many calls, after warm-up), the bytes the call must read at least, the achieved GB/s and its share
of the H100 SXM's 3.35 TB/s, and the card and its power limit as read in the same run.

The model reads every byte of x once per pass for O multiply-adds each, so bandwidth bounds it: predict reads
B*T*F*4 bytes, the train step twice that (the forward and the weight gradient each read x).

    python tools/bench_baselines.py [--iters 50] [--warmup 5] [--batch 65536] [--train-batch 4096]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lfm_quant_b200.engine import DenseEngine  # noqa: E402

T, F, O = 48, 32, 16
PEAK_GBS = 3350.0


def _power_limit_w():
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader,nounits', '-i',
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:
        return None


def _time(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--batch', type=int, default=65536)
    ap.add_argument('--train-batch', type=int, default=4096)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_baselines needs a CUDA device')
    card, power = torch.cuda.get_device_name(), _power_limit_w()
    rng = np.random.default_rng(0)
    W = rng.uniform(-0.05, 0.05, size=(T * F, O)).astype(np.float32)
    b = np.zeros(O, dtype=np.float32)

    def line(case, B, ms, nbytes, launches):
        gbs = nbytes / ms / 1e6
        print(json.dumps(dict(case=case, B=B, T=T, F=F, O=O, ms=round(ms, 4), min_bytes=nbytes,
                              achieved_gb_s=round(gbs, 1), share_of_3350_gb_s=round(gbs / PEAK_GBS, 3),
                              launches_per_call=launches, card=card, power_limit_w=power)), flush=True)

    B = a.train_batch
    eng = DenseEngine(max_batch=B, seq_len=T, n_inputs=F, n_outputs=O, target_idx=3, optimizer='Adadelta')
    eng.set_weights([W, b])
    x = torch.randn(B, T * F, device='cuda')
    y = torch.randn(B, O, device='cuda')
    out = torch.empty(2, device='cuda')
    step = [0]

    def train():
        eng.train_step(x, y, step[0], 0.6, out=out)
        step[0] += 1
    n0 = eng.launch_count
    train()
    launches = eng.launch_count - n0
    line('train_step', B, _time(train, a.iters, a.warmup), 2 * B * T * F * 4, launches)
    eng.close()
    del x, y

    B = a.batch
    eng = DenseEngine(max_batch=B, seq_len=T, n_inputs=F, n_outputs=O, target_idx=3, forward_only=True)
    eng.set_weights([W, b])
    x = torch.randn(B, T * F, device='cuda')
    preds = torch.empty(B, O, device='cuda')
    n0 = eng.launch_count
    eng.forward(x, out=preds)
    launches = eng.launch_count - n0
    line('predict', B, _time(lambda: eng.forward(x, out=preds), a.iters, a.warmup), B * T * F * 4, launches)
    eng.close()


if __name__ == '__main__':
    main()
