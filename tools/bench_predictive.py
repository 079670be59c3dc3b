"""Times predictive quantiles and scores on one GPU (ForecastChainEngine.forward_dist, lfmq_chain_forward_uq_dist)
against the Monte-Carlo moments alone (forward_mc) and against the host route a user would take today: one
forward of batch_size rows per launch for every sample (lfmq_forward_uq, sample m of window b at row m * N + b, as
predict_device launches them), the samples copied to the host, and a vectorised fp64 NumPy pass over the mixtures
(quantiles by 64 bisection steps inside the component-quantile bracket, the closed-form CRPS with its M^2 pair sum,
the log score by logsumexp, the PIT).

Shapes: N = 16384 windows, T = 48, F = 32, O = 16, H = 256, L = 1, Q = 5 levels, a UQ model (dropout 0.2 / recurrent
0.15) at fp32 and bf16, M in {8, 32, 128} samples.  forward_mc and forward_dist run on a forward-only engine of
MC_ROWS = 8192 rows per launch, as NativeForecaster.predict_mc and predict_dist do; the host route on one of
batch_size = 256 rows.  Each is timed once after a warm-up call (host clock around work that ends in a device
synchronise).  The error check compares forward_dist's outputs at the timed size with the fp64 pass on the samples of
the host route (the same rows and dropout masks).  At M = 128 a separate torch.profiler run of one forward_dist call
gives the device time of the gather and the distribution kernels.  The card's name and power limit are read in the
same run.  Prints one JSON line per case.

usage: python tools/bench_predictive.py [--out FILE] [--cases fp32,bf16] [--samples 8,32,128]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
from scipy import special

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lfm_quant_b200.engine import ForecastChainEngine  # noqa: E402

N, T, F, O, H, L, TI = 16384, 48, 32, 16, 256, 1, 3
BATCH, WIDE = 256, 8192
LEVELS = [0.05, 0.25, 0.5, 0.75, 0.95]
STEP = 3


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def engine(rows, prec):
    e = ForecastChainEngine(forecast_steps=1, weights=[1.0], max_batch=rows, seq_len=T, n_inputs=F, n_outputs=O,
                            num_hidden=H, num_layers=L, target_idx=TI, precision=prec, train=False, forward_only=True,
                            uq=True, dropout=0.2, recurrent_dropout=0.15)
    rng = np.random.RandomState(0)
    e.set_weights([rng.uniform(-0.1, 0.1, size=s[1]) for s in e.stages[0].trainable_specs])
    return e


def once(fn):
    fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, out


def host_samples(eng, x, M):
    """(mu, v) [N, M] of every sample from launches of batch_size rows keyed by the tiled rows."""
    mu = torch.empty(M, N, device='cuda')
    v = torch.empty(M, N, device='cuda')
    for m in range(M):
        for a in range(0, N, BATCH):
            p, var = eng.forward(x[a:a + BATCH], step=STEP, row0=m * N + a)
            mu[m, a:a + BATCH] = p[:, -1, TI]
            v[m, a:a + BATCH] = var[:, -1, TI]
    return mu.T.double().cpu().numpy(), v.T.double().cpu().numpy()


def host_dist(mu, v, y, chunk=256):
    """fp64 quantiles [N,Q] and {crps, nll, pit} [N,3] of every window's mixture, vectorised over windows."""
    sd = np.sqrt(v)
    Nw, M = mu.shape
    q = np.empty((Nw, len(LEVELS)))
    for k, tau in enumerate(LEVELS):
        comp = mu + sd * special.ndtri(tau)
        lo, hi = comp.min(axis=1), comp.max(axis=1)
        for _ in range(64):
            mid = 0.5 * (lo + hi)
            below = special.ndtr((mid[:, None] - mu) / sd).mean(axis=1) < tau
            lo, hi = np.where(below, mid, lo), np.where(below, hi, mid)
        q[:, k] = 0.5 * (lo + hi)

    def A(m, var):
        s = np.sqrt(var)
        z = m / s
        return 2.0 * s * np.exp(-0.5 * z * z) / np.sqrt(2.0 * np.pi) + m * special.erf(z / np.sqrt(2.0))
    sc = np.empty((Nw, 3))
    yy = y[:, None]
    for a in range(0, Nw, chunk):
        m_, v_ = mu[a:a + chunk], v[a:a + chunk]
        pairs = A(m_[:, :, None] - m_[:, None, :], v_[:, :, None] + v_[:, None, :]).mean(axis=(1, 2))
        sc[a:a + chunk, 0] = A(m_ - yy[a:a + chunk], v_).mean(axis=1) - 0.5 * pairs
    logs = -0.5 * (yy - mu) ** 2 / v - 0.5 * np.log(v) - 0.5 * np.log(2 * np.pi)
    sc[:, 1] = -(special.logsumexp(logs, axis=1) - np.log(M))
    sc[:, 2] = special.ndtr((yy - mu) / sd).mean(axis=1)
    return q, sc


def kernel_ms(fn):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {'gather': 0.0, 'dist': 0.0, 'all': 0.0}
    for e in prof.key_averages():
        t = e.device_time_total / 1e3 if hasattr(e, 'device_time_total') else e.cuda_time_total / 1e3
        out['all'] += t
        if 'dist_gather_kernel' in e.key:
            out['gather'] += t
        elif 'dist_kernel' in e.key:
            out['dist'] += t
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--cases', default='fp32,bf16')
    ap.add_argument('--samples', default='8,32,128')
    args = ap.parse_args()
    torch.cuda.set_device(0)
    name = card()
    rng = np.random.RandomState(1)
    x = torch.from_numpy(rng.normal(size=(N, T, F)).astype(np.float32)).cuda()
    y = torch.from_numpy(rng.normal(scale=0.05, size=(N, T, O)).astype(np.float32)).cuda()
    y_last = y[:, -1, TI].double().cpu().numpy()
    lines = []
    for prec in args.cases.split(','):
        wide, narrow = engine(WIDE, prec), engine(BATCH, prec)
        for M in [int(m) for m in args.samples.split(',')]:
            t_mc, _ = once(lambda: wide.forward_mc(x, M, step=STEP))
            t_dist, (_, q, sc) = once(lambda: wide.forward_dist(x, M, LEVELS, ys=[y], step=STEP))
            t0 = time.perf_counter()
            mu, v = host_samples(narrow, x, M)
            t_fwd = (time.perf_counter() - t0) * 1e3
            t0 = time.perf_counter()
            hq, hsc = host_dist(mu, v, y_last)
            t_np = (time.perf_counter() - t0) * 1e3
            q, sc = q[0].double().cpu().numpy(), sc[0].double().cpu().numpy()
            std = np.sqrt(v.mean(axis=1) + mu.var(axis=1))
            row = dict(case='uq-%s' % prec, M=M, N=N, T=T, F=F, O=O, H=H, Q=len(LEVELS), card=name,
                       forward_mc_ms=round(t_mc, 2), forward_dist_ms=round(t_dist, 2),
                       dist_over_mc_ms=round(t_dist - t_mc, 2), host_forward_ms=round(t_fwd, 1),
                       host_numpy_ms=round(t_np, 1), host_total_ms=round(t_fwd + t_np, 1),
                       speedup_vs_host=round((t_fwd + t_np) / t_dist, 2),
                       err_q_over_std=float(np.max(np.abs(q - hq) / std[:, None])),
                       err_crps_rel=float(np.max(np.abs(sc[:, 0] - hsc[:, 0]) / np.abs(hsc[:, 0]))),
                       err_nll_abs=float(np.max(np.abs(sc[:, 1] - hsc[:, 1]))),
                       err_pit_abs=float(np.max(np.abs(sc[:, 2] - hsc[:, 2]))),
                       pair_terms=N * M * (M + 1) // 2)
            if M == max(int(m) for m in args.samples.split(',')):
                k = kernel_ms(lambda: wide.forward_dist(x, M, LEVELS, ys=[y], step=STEP))
                row.update(profiled_gather_ms=round(k['gather'], 3), profiled_dist_kernel_ms=round(k['dist'], 3),
                           profiled_all_kernels_ms=round(k['all'], 2))
            print(json.dumps(row), flush=True)
            lines.append(row)
        wide.close()
        narrow.close()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as fh:
            for r in lines:
                fh.write(json.dumps(r) + '\n')


if __name__ == '__main__':
    main()
