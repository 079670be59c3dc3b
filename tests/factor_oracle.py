"""fp64 NumPy / SciPy restatement of the lookahead factor backtest (DESIGN.md section 5k): lfmq_factor_eval's per-date
outputs, the summary over dates with the Newey-West lag rule, the factor and measure builders and forward_returns,
written date by date from the definitions, independently of lfm_quant_b200.scripts.predict."""
import math

import numpy as np
import scipy.stats


def evaluate(date_idx, company, score, measure, Q, D=None):
    """The outputs of lfmq_factor_eval, as engine.factor_eval names them, by loops over the factors and dates."""
    date_idx, company = np.asarray(date_idx), np.asarray(company)
    score, measure = np.atleast_2d(np.asarray(score, np.float64)), np.atleast_2d(np.asarray(measure, np.float64))
    G, M = len(score), len(measure)
    D = int(date_idx.max()) + 1 if D is None else D
    out = dict(n=np.zeros((G, D), np.int32), bucket_n=np.zeros((G, D, Q), np.int32),
               n_pair=np.zeros((G, M, D), np.int32), ic=np.full((G, M, D), np.nan),
               bucket_mean=np.full((G, M, D, Q), np.nan), spread=np.full((G, M, D), np.nan),
               turnover=np.full((G, D), np.nan))
    order = np.argsort(date_idx, kind='stable')
    by_date = np.split(order, np.searchsorted(date_idx[order], np.arange(1, D)))
    for g in range(G):
        top_prev = None
        for d in range(D):
            rows = by_date[d]
            s = score[g, rows]
            fin = np.isfinite(s)
            u = rows[fin]
            n = len(u)
            out['n'][g, d] = n
            bucket = np.zeros(0, np.int64)
            if n:
                r = scipy.stats.rankdata(score[g, u], method='average')
                bucket = np.floor((r - 0.5) * Q / n).astype(np.int64) + 1
                out['bucket_n'][g, d] = np.bincount(bucket - 1, minlength=Q)
            top = set(company[u[bucket == Q]].tolist())
            if d > 0 and top:
                out['turnover'][g, d] = len(top - top_prev) / len(top)
            top_prev = top
            for m in range(M):
                y = measure[m, u]
                for q in range(1, Q + 1):
                    v = y[(bucket == q) & np.isfinite(y)]
                    if len(v):
                        out['bucket_mean'][g, m, d, q - 1] = math.fsum(v) / len(v)
                out['spread'][g, m, d] = out['bucket_mean'][g, m, d, Q - 1] - out['bucket_mean'][g, m, d, 0]
                both = np.isfinite(y)
                out['n_pair'][g, m, d] = both.sum()
                out['ic'][g, m, d] = spearman(score[g, u[both]], y[both])
    return out


def spearman(x, y):
    """Spearman's rho by exact integer rank moments (NaN when n < 3 or a rank variance is 0), as the library forms it."""
    n = len(x)
    if n < 3:
        return np.nan
    cx = np.rint(2 * scipy.stats.rankdata(x, method='average')).astype(np.int64) - (n + 1)
    cy = np.rint(2 * scipy.stats.rankdata(y, method='average')).astype(np.int64) - (n + 1)
    if n < 2 ** 20:          # n^3 < 2^63: exact in int64
        sxy, sxx, syy = int(cx @ cy), int(cx @ cx), int(cy @ cy)
    else:
        cx, cy = [int(v) for v in cx], [int(v) for v in cy]
        sxy = sum(a * b for a, b in zip(cx, cy))
        sxx, syy = sum(a * a for a in cx), sum(b * b for b in cy)
    if sxx == 0 or syy == 0:
        return np.nan
    return float(sxy) / math.sqrt(float(sxx) * float(syy))


def months(dates):
    d = np.asarray(dates, np.int64)
    ym = np.where(d >= 10 ** 7, d // 100, d)
    return (ym // 100) * 12 + ym % 100 - 1


def nw_lag(dates, horizon):
    m = sorted(set(months(dates).tolist()))
    if len(m) < 2:
        return 0
    spacing = min(b - a for a, b in zip(m, m[1:]))
    return max(0, -(-horizon // spacing) - 1)


def nw_t(x, lag):
    """Newey-West t with Bartlett weights over the finite entries, by the textbook double loop."""
    x = [v for v in np.asarray(x, np.float64) if np.isfinite(v)]
    n = len(x)
    if n < 2:
        return np.nan
    mu = sum(x) / n
    gamma = lambda k: sum((x[t] - mu) * (x[t - k] - mu) for t in range(k, n)) / n     # noqa: E731
    var = gamma(0) + 2 * sum((1 - k / (lag + 1)) * gamma(k) for k in range(1, min(lag, n - 1) + 1))
    return mu / math.sqrt(var / n) if var > 0 else np.nan


def summary(dates, out, Q, horizons):
    """{(g, m): {column: value}} of factor.dat."""
    res = {}
    G, M, _ = out['ic'].shape
    for g in range(G):
        for m in range(M):
            ic = out['ic'][g, m]
            f = ic[np.isfinite(ic)]
            sp = out['spread'][g, m]
            fs = sp[np.isfinite(sp)]
            lag = nw_lag(dates, horizons[m])
            tv = out['turnover'][g]
            row = dict(n_dates=len(f), mean_ic=f.mean() if len(f) else np.nan,
                       sd_ic=f.std(ddof=1) if len(f) > 1 else np.nan, hit=(f > 0).mean() if len(f) else np.nan,
                       t_ic=nw_t(ic, lag), mean_spread=fs.mean() if len(fs) else np.nan,
                       sd_spread=fs.std(ddof=1) if len(fs) > 1 else np.nan, t_spread=nw_t(sp, lag),
                       mean_turnover=tv[np.isfinite(tv)].mean() if np.isfinite(tv).any() else np.nan, nw_lag=lag)
            row['ir'] = row['mean_ic'] / row['sd_ic'] if row['sd_ic'] > 0 else np.nan
            for q in range(Q):
                b = out['bucket_mean'][g, m, :, q]
                row['mean_q%d' % (q + 1)] = b[np.isfinite(b)].mean() if np.isfinite(b).any() else np.nan
            res[(g, m)] = row
    return res


def forward_returns(rows, date, gvkey, horizon):
    """ret from a dict {(gvkey, yyyymm month index): r} of the datafile, row by row."""
    out = []
    for d, g in zip(months(date), gvkey):
        p = 1.0
        for k in range(1, horizon + 1):
            r = rows.get((str(g), int(d) + k), np.nan)
            if not np.isfinite(r):
                p = np.nan
                break
            p *= 1.0 + r
        out.append(p - 1.0)
    return np.array(out)


def scores(df, steps, uq):
    """{name: score} of a preds.dat frame."""
    sn = df['seq_norm'].to_numpy(np.float64)
    res = {'lfm_%d' % s: df['preds_%d' % s].to_numpy(np.float64) / sn for s in range(1, steps + 1)}
    res['qfm'] = df['inp_t0'].to_numpy(np.float64) / sn
    if uq:
        for s in range(1, steps + 1):
            v = df['variance_%d' % s].to_numpy(np.float64)
            with np.errstate(invalid='ignore', divide='ignore'):
                pv = df['preds_%d' % s].to_numpy(np.float64) / np.sqrt(v)
            res['lfm_risk_%d' % s] = np.where(np.isfinite(v) & (v > 0), pv, np.nan) / sn
    return res
