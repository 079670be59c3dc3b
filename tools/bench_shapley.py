"""Times Shapley attributions on one GPU (ForecastChainEngine.shapley, lfmq_chain_shapley) against the host loop a user
would write today: per coalition copy, the inputs built with torch indexing, model.predict_device's launches of
batch_size rows (lfmq_forward / lfmq_forward_uq, sample m of window i at row m * N + i), and a torch fold of the
explained outputs into phi, f_x and f_bg.

Shapes: N = 16384 windows, T = 48, F = 32, O = 16, H = 256, L = 1, M = 8 samples (4 antithetic pairs); the field
partition (G = 32, 264 copies) and the quarter partition (G = 48, 392 copies).  A point model at fp32 and bf16 and a UQ
model at fp32 (dropout 0.2 / recurrent 0.15; K = 2 outputs).  The call runs on a forward-only engine of MC_ROWS = 8192
rows per launch, as NativeForecaster.shapley does; the loop on one of batch_size = 256 rows.  Time over CUDA events
after a warm-up call (the loop, which takes tens of seconds, is timed once after a warm-up of its engine).  The gather
and fold kernels' share comes from a separate torch.profiler run of one call on the field partition.  The card's name
and power limit are read in the same run.  Prints one JSON line per case.

usage: python tools/bench_shapley.py [--out FILE] [--reps K] [--cases point-fp32,point-bf16,uq-fp32]"""
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

N, T, F, O, H, L, M = 16384, 48, 32, 16, 256, 1, 8
TI = 3
BATCH, WIDE = 256, 8192
CASES = {'point-fp32': ('fp32', False), 'point-bf16': ('bf16', False), 'uq-fp32': ('fp32', True)}


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


def host_loop(eng, x, groups, seed, step):
    """What a caller writes without the entry point: every coalition copy built with torch, forwarded batch by batch
    as predict_device does, and its explained outputs folded with torch."""
    G = int(groups.max()) + 1
    gcol = torch.from_numpy(groups.astype(np.int64)).cuda()
    gen = torch.Generator(device='cuda')
    gen.manual_seed(seed)
    flat = x.view(N, T * F)
    K = 2 if eng.uq else 1
    phi = torch.zeros(N, K, G, device='cuda')
    f_x, f_bg = torch.zeros(N, K, device='cuda'), torch.zeros(N, K, device='cuda')
    for m in range(M):
        if m % 2 == 0:
            donor = flat[torch.randperm(N, device='cuda', generator=gen)]
            order = torch.randperm(G, device='cuda', generator=gen)
        else:
            order = order.flip(0)
        rank = torch.empty_like(order)
        rank[order] = torch.arange(G, device='cuda')
        prev = None
        for k in range(G + 1):
            xc = torch.where(rank[gcol] >= k, donor, flat).view(N, T, F) if k < G else x
            outs = [eng.forward(xc[a:a + BATCH], step=step, row0=m * N + a) for a in range(0, N, BATCH)]
            v = torch.stack([torch.cat([o[j] for o in outs])[:, -1, TI] for j in range(K)], dim=1)
            if k == 0:
                f_bg += v
            else:
                phi[:, :, order[k - 1]] += v - prev
            if k == G:
                f_x += v
            prev = v
    return phi / M, f_x / M, f_bg / M


def kernel_share(wide, x, groups):
    """Device time of the gather and fold kernels and of all kernels in one call, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        wide.shapley(x, groups, M, 7, 1)
        torch.cuda.synchronize()
    got, total = {}, 0.0
    for e in prof.key_averages():
        t = getattr(e, 'device_time_total', None)
        if t is None:
            t = e.cuda_time_total
        if getattr(e, 'device_type', None) is not None and 'CUDA' not in str(e.device_type):
            continue
        total += t
        for name in ('perm_importance_gather', 'shapley_fold'):
            if name in e.key:
                got[name] = (t / 1e3, e.count)
    for name in ('perm_importance_gather', 'shapley_fold'):
        if name not in got:
            raise RuntimeError('%s kernel not found in the trace' % name)
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
    cols = np.arange(T * F)
    rows = []
    for name in a.cases.split(','):
        prec, uq = CASES[name]
        wide, narrow = engine(WIDE, prec, uq), engine(BATCH, prec, uq)
        for part, groups in (('fields', (cols % F).astype(np.int32)), ('quarters', (cols // F).astype(np.int32))):
            G = int(groups.max()) + 1
            call = timed(lambda: wide.shapley(x, groups, M, 7, 1), a.reps)
            narrow.forward(x[:BATCH], step=1, row0=0)          # the loop's warm-up: its engine's first launches
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            host_loop(narrow, x, groups, 7, 1)
            torch.cuda.synchronize()
            loop = (time.perf_counter() - t0) * 1e3
            row = dict(case=name, partition=part, G=G, copies=M * (G + 1), N=N, T=T, F=F, O=O, H=H, L=L, M=M,
                       call_ms=round(call, 1), host_loop_ms=round(loop, 1), speedup=round(loop / call, 2), gpu=gpu)
            if part == 'fields':
                got, total = kernel_share(wide, x, groups)
                moved = 2.0 * M * G * N * T * F * 4            # read and write the inputs of every gathered copy once
                g_ms, f_ms = got['perm_importance_gather'][0], got['shapley_fold'][0]
                row.update(profiled_kernels_ms=round(total, 1), gather_ms=round(g_ms, 2),
                           gather_share=round(g_ms / total, 4), gather_TBps=round(moved / (g_ms * 1e-3) / 1e12, 3),
                           fold_ms=round(f_ms, 2), fold_share=round(f_ms / total, 4),
                           fold_launches=got['shapley_fold'][1])
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
