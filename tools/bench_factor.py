"""Times the lookahead factor backtest (lfmq_factor_eval) on one GPU.

Size: N = 2^20 rows over D = 600 monthly dates (about 1750 companies a date), G = 3 factor scores, M = 2 measures,
Q = 10 buckets; 10 % of the scores are quantised to 4 significant digits, so ties are common, and 3 % of the scores
and measures are NaN.  Two library times are reported: call_ms, lfmq_factor_eval alone with its outputs and work
allocated once, and lib_ms, the engine.factor_eval wrapper, which also reads D back from the device (a host
synchronisation) and allocates the outputs on every call.  They are timed against two alternatives that compute the
same outputs, each timed up to its device outputs (no copy to the host):
  pandas: groupby(date).rank(method='average') and NumPy, what a user would write on the host;
  torch:  the same steps on the GPU with torch.sort (stable) and scatter_add.
Each result is checked against tests/factor_oracle.py at that size (integers exactly, fp64 within 1e-12 of the
oracle or of the measure's scale).  GPU times are CUDA-event means after a warm-up call; the pandas path runs once.  The
card's name and power limit are read in the same run.  Prints one JSON line.

usage: python tools/bench_factor.py [--out FILE] [--reps K]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import pandas as pd
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
import factor_oracle as fo  # noqa: E402
from lfm_quant_b200 import _native as N_  # noqa: E402
from lfm_quant_b200.engine import factor_eval  # noqa: E402

N, D, G, M, Q = 2 ** 20, 600, 3, 2, 10


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


def problem(seed=0):
    rng = np.random.RandomState(seed)
    companies = 2000
    pairs = rng.choice(D * companies, size=N, replace=False)
    date, company = (pairs // companies).astype(np.int32), (pairs % companies).astype(np.int32)
    score = rng.lognormal(0, 1, size=(G, N)) * rng.choice([-1, 1], size=(G, N), p=[0.2, 0.8])
    t = rng.uniform(size=(G, N)) < 0.1
    score[t] = np.array([float('%.3e' % v) for v in score[t]])
    score[rng.uniform(size=(G, N)) < 0.03] = np.nan
    measure = 0.05 * np.tanh(score[:M]) + rng.standard_t(4, size=(M, N)) * 0.1
    measure[rng.uniform(size=(M, N)) < 0.03] = np.nan
    return date, company, score, measure


# ---- pandas / NumPy --------------------------------------------------------------------------------------------
def pandas_eval(date, company, score, measure):
    out = dict(n=np.zeros((G, D), np.int32), bucket_n=np.zeros((G, D, Q), np.int32),
               n_pair=np.zeros((G, M, D), np.int32), ic=np.full((G, M, D), np.nan),
               bucket_mean=np.full((G, M, D, Q), np.nan), spread=np.full((G, M, D), np.nan),
               turnover=np.full((G, D), np.nan))
    for g in range(G):
        df = pd.DataFrame({'date': date, 'company': company, 's': score[g]})
        grp = df.groupby('date')['s']
        r, n = grp.rank(method='average'), grp.transform('count')
        df['b'] = np.floor((r - 0.5) * Q / n) + 1
        fin = df['b'].notna()
        nb = df[fin].groupby(['date', 'b']).size()
        out['n'][g] = grp.count().reindex(range(D), fill_value=0).to_numpy()
        out['bucket_n'][g][nb.index.get_level_values(0), nb.index.get_level_values(1).astype(int) - 1] = nb.to_numpy()
        top = df[df['b'] == Q][['date', 'company']]
        prev = set(zip(top['date'] + 1, top['company']))
        top_n = top.groupby('date').size()
        fresh = top[[(d, c) not in prev for d, c in zip(top['date'], top['company'])]].groupby('date').size()
        tv = (fresh.reindex(top_n.index, fill_value=0) / top_n)
        tv = tv[tv.index > 0]
        out['turnover'][g][tv.index.to_numpy()] = tv.to_numpy()
        for m in range(M):
            df['y'] = measure[m]
            bm = df[fin & df['y'].notna()].groupby(['date', 'b'])['y'].mean()
            out['bucket_mean'][g, m][bm.index.get_level_values(0),
                                     bm.index.get_level_values(1).astype(int) - 1] = bm.to_numpy()
            pair = df[df['s'].notna() & df['y'].notna()].copy()
            pg = pair.groupby('date')
            pair['rx'], pair['ry'] = pg['s'].rank(method='average'), pg['y'].rank(method='average')
            stats = pair.groupby('date').apply(lambda f: pd.Series(
                {'n': len(f), 'ic': np.corrcoef(f['rx'], f['ry'])[0, 1] if len(f) >= 3 and f['rx'].std() > 0
                 and f['ry'].std() > 0 else np.nan}), include_groups=False)
            out['n_pair'][g, m][stats.index.to_numpy()] = stats['n'].to_numpy()
            out['ic'][g, m][stats.index.to_numpy()] = stats['ic'].to_numpy()
        out['spread'][g] = out['bucket_mean'][g, :, :, Q - 1] - out['bucket_mean'][g, :, :, 0]
    return out


# ---- torch on the GPU ------------------------------------------------------------------------------------------
def _avg_rank(date, v):
    """(order, average rank in order) of the finite v within each date: a stable sort by v, then by date."""
    o1 = torch.sort(v, stable=True)[1]
    o = o1[torch.sort(date[o1], stable=True)[1]]
    d, x = date[o], v[o]
    n = x.shape[0]
    new = torch.ones(n, dtype=torch.bool, device=v.device)
    new[1:] = (d[1:] != d[:-1]) | (x[1:] != x[:-1])
    pos = torch.arange(n, device=v.device)
    run_start = torch.cummax(torch.where(new, pos, torch.zeros_like(pos)), 0)[0]
    seg_new = torch.ones(n, dtype=torch.bool, device=v.device)
    seg_new[1:] = d[1:] != d[:-1]
    seg_start = torch.cummax(torch.where(seg_new, pos, torch.zeros_like(pos)), 0)[0]
    end = torch.ones(n, dtype=torch.bool, device=v.device)
    end[:-1] = new[1:]
    run_end = torch.flip(torch.cummin(torch.flip(torch.where(end, pos, torch.full_like(pos, n)), [0]), 0)[0], [0])
    return o, (run_start - seg_start + run_end - seg_start + 2).double() / 2


def torch_eval(date, company, score, measure):
    dev = score.device
    out = dict(n=torch.zeros(G, D, dtype=torch.int64, device=dev),
               bucket_n=torch.zeros(G, D * Q, dtype=torch.int64, device=dev),
               n_pair=torch.zeros(G, M, D, dtype=torch.int64, device=dev),
               ic=torch.full((G, M, D), float('nan'), dtype=torch.float64, device=dev),
               bucket_mean=torch.full((G, M, D * Q), float('nan'), dtype=torch.float64, device=dev),
               turnover=torch.full((G, D), float('nan'), dtype=torch.float64, device=dev))
    date = date.long()
    pred_key = company.long() * D + date
    ok = torch.sort(pred_key)
    pk, po = ok
    pred = torch.full((N,), -1, dtype=torch.int64, device=dev)
    hit = pk[1:] == pk[:-1] + 1
    pred[po[1:][hit]] = po[:-1][hit]
    one = lambda k: torch.ones(k, dtype=torch.float64, device=dev)     # noqa: E731
    for g in range(G):
        fin = torch.isfinite(score[g])
        idx = torch.nonzero(fin).squeeze(1)
        o, r = _avg_rank(date[idx], score[g, idx])
        rows, d = idx[o], date[idx][o]
        n = torch.zeros(D, dtype=torch.float64, device=dev).scatter_add_(0, d, one(len(d)))
        b = torch.floor((r - 0.5) * Q / n[d]).long() + 1
        out['n'][g] = n.long()
        out['bucket_n'][g].scatter_add_(0, d * Q + b - 1, torch.ones_like(b))
        bq = torch.zeros(N, dtype=torch.int64, device=dev)
        bq[rows] = b
        top = rows[b == Q]
        p = pred[top]
        fresh = (p < 0) | (bq[p.clamp(min=0)] != Q)
        tn = torch.zeros(D, dtype=torch.float64, device=dev).scatter_add_(0, date[top], one(len(top)))
        fn = torch.zeros(D, dtype=torch.float64, device=dev).scatter_add_(0, date[top], fresh.double())
        tv = fn / tn
        tv[0] = float('nan')
        out['turnover'][g] = tv
        for m in range(M):
            y = measure[m, rows]
            fy = torch.isfinite(y)
            key = d * Q + b - 1
            s = torch.zeros(D * Q, dtype=torch.float64, device=dev).scatter_add_(0, key[fy], y[fy])
            c = torch.zeros(D * Q, dtype=torch.float64, device=dev).scatter_add_(0, key[fy], one(int(fy.sum())))
            out['bucket_mean'][g, m] = s / c
            pr = torch.nonzero(fin & torch.isfinite(measure[m])).squeeze(1)
            ox, rx = _avg_rank(date[pr], score[g, pr])
            oy, ry = _avg_rank(date[pr], measure[m, pr])
            xr = torch.empty(len(pr), dtype=torch.float64, device=dev)
            yr = torch.empty_like(xr)
            xr[ox], yr[oy] = rx, ry
            dp = date[pr]
            acc = lambda v: torch.zeros(D, dtype=torch.float64, device=dev).scatter_add_(0, dp, v)  # noqa: E731
            npair = acc(one(len(pr)))
            mx, my = acc(xr) / npair, acc(yr) / npair
            cx, cy = xr - mx[dp], yr - my[dp]
            sxx, syy, sxy = acc(cx * cx), acc(cy * cy), acc(cx * cy)
            ic = sxy / torch.sqrt(sxx * syy)
            ic[(npair < 3) | (sxx == 0) | (syy == 0)] = float('nan')
            out['n_pair'][g, m], out['ic'][g, m] = npair.long(), ic
    return out


def to_host(out):
    res = {k: v.cpu().numpy() for k, v in out.items()}
    res['bucket_n'] = res['bucket_n'].reshape(G, D, Q)
    res['bucket_mean'] = res['bucket_mean'].reshape(G, M, D, Q)
    res['spread'] = res['bucket_mean'][..., Q - 1] - res['bucket_mean'][..., 0]
    return res


def raw_call(dd, cc, ss, mm):
    """lfmq_factor_eval alone: outputs and work allocated once, no host synchronisation inside the timed calls."""
    lib = N_.load()
    n = C.c_uint64(0)
    N_.check(lib.lfmq_factor_eval_work_bytes(N, D, G, M, Q, C.byref(n)))
    work = torch.empty(n.value, dtype=torch.uint8, device='cuda')
    i32, f64 = dict(dtype=torch.int32, device='cuda'), dict(dtype=torch.float64, device='cuda')
    out = [torch.empty(G * D, **i32), torch.empty(G * D * Q, **i32), torch.empty(G * M * D, **i32),
           torch.empty(G * M * D, **f64), torch.empty(G * M * D * Q, **f64), torch.empty(G * M * D, **f64),
           torch.empty(G * D, **f64)]
    p = lambda t: C.c_void_p(t.data_ptr())       # noqa: E731
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    return lambda: N_.check(lib.lfmq_factor_eval(p(dd), p(cc), N, D, p(ss), G, p(mm), M, Q, *[p(t) for t in out],
                                                p(work), n.value, stream))


def check(got, want, measure):
    """max deviations from the oracle: integers must match; fp64 within 1e-12 relative (ic, turnover) or of the
    measure's scale (bucket means, spread)."""
    for k in ('n', 'bucket_n', 'n_pair'):
        if not np.array_equal(np.asarray(got[k], np.int64), want[k]):
            return False, k
    scale = np.nanmax(np.abs(measure))
    for k in ('ic', 'turnover', 'bucket_mean', 'spread'):
        g, w = np.asarray(got[k]), want[k]
        if not np.array_equal(np.isnan(g), np.isnan(w)):
            return False, k + ' NaN'
        f = ~np.isnan(w)
        tol = 1e-12 * (np.abs(w[f]) if k in ('ic', 'turnover') else scale)
        if not np.all(np.abs(g[f] - w[f]) <= np.maximum(tol, 1e-300)):
            return False, '%s max dev %.3g' % (k, float(np.max(np.abs(g[f] - w[f]))))
    return True, ''


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out')
    ap.add_argument('--reps', type=int, default=20)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    date, company, score, measure = problem()
    cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()      # noqa: E731
    dd, cc, ss, mm = cu(date), cu(company), cu(score), cu(measure)
    want = fo.evaluate(date, company, score, measure, Q, D=D)
    call_ms = timed(raw_call(dd, cc, ss, mm), args.reps)
    lib_ms = timed(lambda: factor_eval(dd, cc, ss, mm, Q), args.reps)
    lib_ok = check({k: v.cpu().numpy() for k, v in factor_eval(dd, cc, ss, mm, Q).items()}, want, measure)
    torch_ms = timed(lambda: torch_eval(dd, cc, ss, mm), max(1, args.reps // 4))
    torch_ok = check(to_host(torch_eval(dd, cc, ss, mm)), want, measure)
    t0 = time.perf_counter()
    pd_out = pandas_eval(date, company, score, measure)
    pandas_ms = (time.perf_counter() - t0) * 1e3
    pandas_ok = check(pd_out, want, measure)
    res = {'case': 'factor_eval', 'N': N, 'D': D, 'G': G, 'M': M, 'Q': Q, 'card': card(),
           'call_ms': round(call_ms, 3), 'lib_ms': round(lib_ms, 3), 'torch_ms': round(torch_ms, 3), 'pandas_ms': round(pandas_ms, 1),
           'lib_matches_oracle': lib_ok[0], 'torch_matches_oracle': torch_ok[0], 'pandas_matches_oracle': pandas_ok[0],
           'mismatch': {k: v[1] for k, v in (('lib', lib_ok), ('torch', torch_ok), ('pandas', pandas_ok)) if not v[0]}}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, 'a') as fh:
            fh.write(line + '\n')


if __name__ == '__main__':
    main()
