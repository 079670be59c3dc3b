"""Times the split-conformal kernels on one GPU.

nearest: lfmq_nearest_topk (engine.nearest_topk, the influence top-K kernel's nearest mode: 3xTF32 wgmma with the
top-K kept in the epilogue) at Nq = 16384 queries, Nt = 262144 pool rows, D1 = 257, K = 32, against the torch path a
user would write today: torch.cdist of the queries against column chunks of the pool, torch.topk of each chunk and a
merge with the running list, once with TF32 off and once with it on.
calibrate: lfmq_conformal_calibrate (score pass, one radix sort of every step, rank selection) at Nc = 10^6, S = 3,
Q = 32, then lfmq_conformal_apply of 10^6 query windows, against torch.sort + index and torch.searchsorted.

Inputs are seeded random draws.  Time over CUDA events after a warm-up call; the card's name and power limit are read
in the same run.  Prints one JSON line per case.

usage: python tools/bench_conformal.py [--out FILE] [--reps K] [--cases nearest,calibrate]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lfm_quant_b200.engine import conformal_apply, conformal_calibrate, nearest_topk  # noqa: E402

NQ, NT, D1, K = 16384, 262144, 257, 32
NC, S, Q = 10 ** 6, 3, 32
CHUNK = 32768


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def torch_nearest(a, b, k):
    best_d, best_i = None, None
    for c0 in range(0, b.shape[0], CHUNK):
        d = torch.cdist(a, b[c0:c0 + CHUNK]) ** 2
        v, i = torch.topk(d, min(k, d.shape[1]), dim=1, largest=False)
        i = i + c0
        if best_d is None:
            best_d, best_i = v, i
        else:
            v, j = torch.topk(torch.cat([best_d, v], 1), k, dim=1, largest=False)
            best_i = torch.gather(torch.cat([best_i, i], 1), 1, j)
            best_d = v
    return best_i, best_d


def bench_nearest(reps):
    g = torch.Generator(device='cuda').manual_seed(0)
    b = torch.randn(NT, D1, device='cuda', generator=g) * torch.exp(0.5 * torch.randn(NT, 1, device='cuda', generator=g))
    a = torch.randn(NQ, D1, device='cuda', generator=g)
    value = torch.rand(NT, device='cuda', generator=g)
    ms = timed(lambda: nearest_topk(a, b, K, value=value), reps)
    idx = nearest_topk(a, b, K)[0]
    out = {'case': 'nearest', 'Nq': NQ, 'Nt': NT, 'D1': D1, 'K': K, 'ms': round(ms, 3),
           'tflops': round(2.0 * NQ * NT * D1 / ms / 1e9, 2)}
    for tf32 in (False, True):
        torch.backends.cuda.matmul.allow_tf32 = tf32
        tm = timed(lambda: torch_nearest(a, b, K), max(1, reps // 2))
        ti = torch_nearest(a, b, K)[0]
        key = 'torch_tf32' if tf32 else 'torch_fp32'
        out[key + '_ms'] = round(tm, 3)
        out[key + '_speedup'] = round(tm / ms, 2)
        out[key + '_same_sets'] = round(float(np.mean([len(set(x) & set(y)) / K for x, y in
                                                       zip(idx[:256].tolist(), ti[:256].tolist())])), 4)
    torch.backends.cuda.matmul.allow_tf32 = False
    return out


def bench_calibrate(reps):
    g = torch.Generator(device='cuda').manual_seed(1)
    pred = torch.randn(S, NC, device='cuda', generator=g)
    y = pred + torch.randn(S, NC, device='cuda', generator=g)
    scale = torch.rand(S, NC, device='cuda', generator=g) + 0.5
    levels = list(np.linspace(0.02, 0.99, Q))
    cal = conformal_calibrate(pred, y, levels, scale=scale)
    ms_cal = timed(lambda: conformal_calibrate(pred, y, levels, scale=scale), reps)
    ms_apply = timed(lambda: conformal_apply(pred, cal, y=y, scale=scale), reps)
    lv = torch.tensor(levels, dtype=torch.float64, device='cuda')

    def torch_path():
        r = torch.abs(y - pred) / scale
        srt = torch.sort(r, dim=1)[0]
        rank = torch.ceil((NC + 1) * lv).long().clamp(max=NC) - 1
        qhat = srt[:, rank]
        w = qhat[:, None, :] * scale[:, :, None]
        lo, hi = pred[:, :, None] - w, pred[:, :, None] + w
        ge = NC - torch.searchsorted(srt, r.contiguous())
        return lo, hi, (1 + ge).float() / (NC + 1)
    tm = timed(torch_path, reps)
    return {'case': 'calibrate+apply', 'Nc': NC, 'N': NC, 'S': S, 'Q': Q, 'calibrate_ms': round(ms_cal, 3),
            'apply_ms': round(ms_apply, 3), 'torch_ms': round(tm, 3), 'speedup': round(tm / (ms_cal + ms_apply), 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--cases', default='nearest,calibrate')
    args = ap.parse_args()
    gpu = card()
    lines = []
    for case in args.cases.split(','):
        r = {'nearest': bench_nearest, 'calibrate': bench_calibrate}[case](args.reps)
        r['gpu'] = gpu
        lines.append(json.dumps(r))
        print(lines[-1], flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as fh:
            fh.write('\n'.join(lines) + '\n')


if __name__ == '__main__':
    main()
