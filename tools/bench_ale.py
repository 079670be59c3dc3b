"""Times accumulated local effects on one GPU (ForecastChainEngine.ale, lfmq_chain_ale) against the host loop a user
would write today: per field, the edges and bins found with NumPy, the two edge copies built with torch indexing,
model.predict_device's launches of batch_size rows (lfmq_forward / lfmq_forward_uq, window i at row i), and a NumPy
fold of the local effects into the per-bin means, standard deviations and the centred ALE.

Shapes: N = 16384 windows, T = 48, F = 32, O = 16, H = 256, L = 1, K = 16 bins over the latest quarter of every field
(G = 32, 64 copies).  A point model at fp32 and bf16 and a UQ model at fp32 (dropout 0.2 / recurrent 0.15; J = 2
outputs).  The call runs on a forward-only engine of MC_ROWS = 8192 rows per launch, as NativeForecaster.ale does; the
loop on one of batch_size = 256 rows.  Time over CUDA events after a warm-up call (the loop is timed once after a
warm-up of its engine).  The sort, gather and fold kernels' shares come from a separate torch.profiler run of one call.
The card's name and power limit are read in the same run.  Prints one JSON line per case.

usage: python tools/bench_ale.py [--out FILE] [--reps K] [--cases point-fp32,point-bf16,uq-fp32]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lfm_quant_b200.engine import ForecastChainEngine  # noqa: E402

N, T, F, O, H, L, K = 16384, 48, 32, 16, 256, 1, 16
TI = 3
BATCH, WIDE = 256, 8192
CASES = {'point-fp32': ('fp32', False), 'point-bf16': ('bf16', False), 'uq-fp32': ('fp32', True)}
KERNELS = {'sort': 'DeviceSegmentedRadixSort', 'keys': 'ale_keys_kernel', 'edges': 'ale_edges_kernel',
           'gather': 'ale_gather_kernel', 'pick': 'ale_pick_kernel', 'fold': 'ale_fold_kernel'}


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def timed(fn, reps):
    fn()                                              # warm-up: module load, first launches of this shape
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def engine(rows, prec, uq):
    e = ForecastChainEngine(forecast_steps=1, weights=[1.0], max_batch=rows, seq_len=T, n_inputs=F, n_outputs=O,
                            num_hidden=H, num_layers=L, target_idx=TI, precision=prec, train=False, forward_only=True,
                            uq=uq, dropout=0.2, recurrent_dropout=0.15)
    rng = np.random.RandomState(0)
    e.set_weights([rng.uniform(-0.1, 0.1, size=s[1]) for s in e.stages[0].trainable_specs])
    return e


def host_loop(eng, x, step):
    """What a caller writes without the entry point: per field the type-1 quantile edges and bins in NumPy, both edge
    copies built with torch and forwarded batch by batch as predict_device does, and a NumPy fold."""
    J = 2 if eng.uq else 1
    xs = x[:, T - 1, :].cpu().numpy()
    out = []
    for f in range(F):
        v = xs[:, f]
        s = np.sort(v)
        q = np.concatenate([[s[0]], s[-(-np.arange(1, K + 1) * N // K) - 1]])
        z = np.unique(q)
        b = np.maximum(np.searchsorted(z, v, side='left'), 1)
        zt, bt = torch.from_numpy(z.astype(np.float32)).cuda(), torch.from_numpy(b).cuda()
        f_ = []
        for edge in (zt[bt], zt[bt - 1]):
            xc = x.clone()
            xc[:, T - 1, f] = edge
            outs = [eng.forward(xc[a:a + BATCH], step=step, row0=a) for a in range(0, N, BATCH)]
            f_.append(torch.stack([torch.cat([o[j] for o in outs])[:, -1, TI] for j in range(J)], dim=1))
        d = (f_[0] - f_[1]).cpu().numpy().astype(np.float64)
        n = np.bincount(b, minlength=z.size)[1:]
        mean = np.stack([np.bincount(b, weights=d[:, j], minlength=z.size)[1:] / n for j in range(J)], axis=1)
        sq = np.stack([np.bincount(b, weights=(d[:, j] - mean[b - 1, j]) ** 2, minlength=z.size)[1:] / n
                       for j in range(J)], axis=1)
        acc = np.vstack([np.zeros((1, J)), np.cumsum(mean, axis=0)])
        out.append((acc - (n[:, None] * 0.5 * (acc[:-1] + acc[1:])).sum(axis=0) / N, mean, np.sqrt(sq)))
    return out


def kernel_share(wide, x, cols):
    """Device time of the sort, gather, fold (and the small ALE) kernels and of all kernels in one call, from
    torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        wide.ale(x, cols, K, 1)
        torch.cuda.synchronize()
    got, total = {k: [0.0, 0] for k in KERNELS}, 0.0
    for e in prof.key_averages():
        t = getattr(e, 'device_time_total', None)
        if t is None:
            t = e.cuda_time_total
        if getattr(e, 'device_type', None) is not None and 'CUDA' not in str(e.device_type):
            continue
        total += t
        for k, name in KERNELS.items():
            if name in e.key:
                got[k][0] += t / 1e3
                got[k][1] += e.count
    for k in ('sort', 'gather', 'fold'):
        if got[k][1] == 0:
            raise RuntimeError('%s kernel not found in the trace' % KERNELS[k])
    return got, total / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--reps', type=int, default=1)
    ap.add_argument('--cases', default=','.join(CASES))
    a = ap.parse_args()
    torch.cuda.set_device(0)
    gpu = card()
    rng = np.random.RandomState(1)
    x = torch.from_numpy(rng.normal(size=(N, T, F)).astype(np.float32)).cuda()
    cols = (T - 1) * F + np.arange(F)
    rows = []
    for name in a.cases.split(','):
        prec, uq = CASES[name]
        wide, narrow = engine(WIDE, prec, uq), engine(BATCH, prec, uq)
        call = timed(lambda: wide.ale(x, cols, K, 1), a.reps)
        res = [t.cpu().numpy() for t in wide.ale(x, cols, K, 1)]
        narrow.forward(x[:BATCH], step=1, row0=0)               # the loop's warm-up: its engine's first launches
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ref = host_loop(narrow, x, 1)
        torch.cuda.synchronize()
        loop = (time.perf_counter() - t0) * 1e3
        # the two agree to the fp32 rounding of the forwards (the loop runs narrower launches at the same keys)
        scale = max(np.abs(r[0]).max() for r in ref)
        diff = max(np.abs(res[3][f] - ref[f][0]).max() for f in range(F)) / scale
        got, total = kernel_share(wide, x, cols)
        row = dict(case=name, G=F, K=K, copies=2 * F, N=N, T=T, F=F, O=O, H=H, L=L, call_ms=round(call, 1),
                   host_loop_ms=round(loop, 1), speedup=round(loop / call, 2), max_rel_diff_vs_loop=float('%.2e' % diff),
                   profiled_kernels_ms=round(total, 1), gpu=gpu)
        moved = 2.0 * 2 * F * N * T * F * 4                     # read and write the inputs of every copy once
        for k, (ms, count) in got.items():
            row.update({k + '_ms': round(ms, 3), k + '_share': round(ms / total, 5), k + '_launches': count})
        row['gather_TBps'] = round(moved / (got['gather'][0] * 1e-3) / 1e12, 3)
        print(json.dumps(row), flush=True)
        rows.append(row)
        wide.close()
        narrow.close()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as fh:
            for row in rows:
                fh.write(json.dumps(row) + '\n')


if __name__ == '__main__':
    main()
