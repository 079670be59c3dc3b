"""Times permutation importance on one GPU (ForecastChainEngine.permutation_importance,
lfmq_chain_permutation_importance) against the host loop a user would write today: per copy, the permuted inputs built
with torch indexing, model.predict_device's launches of batch_size rows (lfmq_forward / lfmq_forward_uq at row0 = the
batch's first window), and the loss entry point over the copy.

Shapes: N = 16384 held-out windows, T = 48, F = 32, O = 16, H = 256, L = 1, R = 2 repeats; the field partition
(G = 32, 65 copies) and the quarter partition (G = 48, 97 copies).  A point model at fp32 and bf16 and a UQ model at fp32
(dropout 0.2 / recurrent 0.15).  The call runs on a forward-only engine of MC_ROWS = 8192 rows per launch, as
NativeForecaster.permutation_importance does; the loop on one of batch_size = 256 rows.  Time over CUDA events after a
warm-up call.  The gather kernel's time comes from a separate torch.profiler run of one call, with the bytes it must
move (read and write each copy's N x T x F inputs once).  The card's name and power limit are read in the same run.
Prints one JSON line per case.

usage: python tools/bench_importance.py [--out FILE] [--reps K]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lfm_quant_b200.engine import ForecastChainEngine  # noqa: E402

N, T, F, O, H, L, R = 16384, 48, 32, 16, 256, 1, 2
BATCH, WIDE = 256, 8192


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
                            num_hidden=H, num_layers=L, target_idx=3, precision=prec, train=False, forward_only=True,
                            uq=uq, dropout=0.2, recurrent_dropout=0.15)
    rng = np.random.RandomState(0)
    e.set_weights([rng.uniform(-0.1, 0.1, size=s[1]) for s in e.stages[0].trainable_specs])
    return e


def host_loop(eng, x, y, groups, seed, step):
    """What a caller writes without the entry point: every copy built, forwarded batch by batch and reduced."""
    G = int(groups.max()) + 1
    cols = [torch.from_numpy(groups == g).cuda() for g in range(G)]
    gen = torch.Generator(device='cuda')
    gen.manual_seed(seed)
    flat = x.view(N, T * F)
    out = []
    for xc in [x] + [None] * (G * R):
        if xc is None:
            g = (len(out) - 1) // R
            perm = torch.randperm(N, device='cuda', generator=gen)
            xc = torch.where(cols[g], flat[perm], flat).view(N, T, F)
        preds = [eng.forward(xc[a:a + BATCH], step=step, row0=a) for a in range(0, N, BATCH)]
        preds = [torch.cat([p[k] for p in preds]) for k in range(len(preds[0]))]
        out.append(eng.loss_uq(preds[0::2], preds[1::2], [y]) if eng.uq else eng.loss(preds, [y]))
    return out


def gather_ms(wide, x, y, groups):
    """Device time of the gather kernel in one call, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        wide.permutation_importance(x, [y], groups, R, 7, 1)
        torch.cuda.synchronize()
    for e in prof.key_averages():
        if 'perm_importance_gather' in e.key:
            total = getattr(e, 'device_time_total', None)
            if total is None:
                total = e.cuda_time_total
            return total / 1e3, e.count
    raise RuntimeError('perm_importance_gather_kernel not found in the trace')


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--reps', type=int, default=3)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    gpu = card()
    rng = np.random.RandomState(1)
    x = torch.from_numpy(rng.normal(size=(N, T, F)).astype(np.float32)).cuda()
    y = torch.from_numpy(rng.normal(size=(N, T, O)).astype(np.float32)).cuda()
    cols = np.arange(T * F)
    rows = []
    for name, prec, uq in (('point-fp32', 'fp32', False), ('point-bf16', 'bf16', False), ('uq-fp32', 'fp32', True)):
        wide, narrow = engine(WIDE, prec, uq), engine(BATCH, prec, uq)
        for part, groups in (('fields', (cols % F).astype(np.int32)), ('quarters', (cols // F).astype(np.int32))):
            G = int(groups.max()) + 1
            call = timed(lambda: wide.permutation_importance(x, [y], groups, R, 7, 1), a.reps)
            loop = timed(lambda: host_loop(narrow, x, y, groups, 7, 1), 1)
            g_ms, g_n = gather_ms(wide, x, y, groups)
            moved = 2.0 * G * R * N * T * F * 4                # read and write each permuted copy once
            row = dict(case=name, partition=part, G=G, copies=1 + G * R, N=N, T=T, F=F, O=O, H=H, L=L, R=R,
                       call_ms=round(call, 2), host_loop_ms=round(loop, 2), speedup=round(loop / call, 2),
                       gather_ms=round(g_ms, 3), gather_launches=g_n, gather_TBps=round(moved / (g_ms * 1e-3) / 1e12, 3),
                       gpu=gpu)
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
