"""NumPy reference of the split-conformal intervals (DESIGN.md section 5j): the scores in float32 arithmetic (the bits
lfmq_conformal_* form), the rank rule with its +inf, the p-values, and exact fp64 k-nearest neighbours with d(x)."""
import numpy as np


def scores(pred, y, scale=None):
    """r = |y - pred| / scale in float32, each operation rounded once; NaN where y is not finite."""
    pred, y = np.asarray(pred, dtype=np.float32), np.asarray(y, dtype=np.float32)
    with np.errstate(invalid='ignore'):
        r = np.abs(y - pred)
        if scale is not None:
            r = r / np.asarray(scale, dtype=np.float32)
    return np.where(np.isfinite(y), r, np.float32(np.nan)).astype(np.float32)


def rank(n, level):
    """ceil((n + 1) l) in fp64, as the library forms it from its fp64 levels."""
    return int(np.ceil((n + 1) * np.float64(level)))


def calibrate(pred, y, levels, scale=None):
    """(n_valid [S], sorted [S][Nc] ascending with NaN last, qhat [S][Q]) of calibration arrays [S][Nc]."""
    r = scores(pred, y, scale)
    S = r.shape[0]
    n_valid = np.zeros(S, dtype=np.int32)
    srt = np.sort(r, axis=1)               # NaN last
    qhat = np.full((S, len(levels)), np.inf, dtype=np.float32)
    for s in range(S):
        n = int((~np.isnan(r[s])).sum())
        n_valid[s] = n
        for k, level in enumerate(levels):
            kk = rank(n, level)
            if kk <= n:
                qhat[s, k] = srt[s, kk - 1]
    return n_valid, srt, qhat


def apply(pred, n_valid, srt, qhat, y=None, scale=None):
    """(lower, upper [S][N][Q], pvalue [S][N]): pred -/+ qhat * scale in float32, and (1 + #{r_i >= r}) / (n + 1)."""
    pred = np.asarray(pred, dtype=np.float32)
    sc = np.ones_like(pred) if scale is None else np.asarray(scale, dtype=np.float32)
    w = qhat[:, None, :] * sc[:, :, None]
    lower, upper = pred[:, :, None] - w, pred[:, :, None] + w
    pv = np.full(pred.shape, np.nan, dtype=np.float32)
    if y is not None:
        r = scores(pred, y, scale)
        for s in range(pred.shape[0]):
            n = int(n_valid[s])
            v = srt[s, :n]
            ok = ~np.isnan(r[s])
            ge = n - np.searchsorted(v, r[s][ok], side='left')
            pv[s, ok] = np.float32(1 + ge) / np.float32(n + 1)
    return lower.astype(np.float32), upper.astype(np.float32), pv


def knn(a, b, K, value=None):
    """Exact fp64 k-nearest rows of b [Nt][D] for every a [Nq][D]: (idx [Nq][K], d2 [Nq][K], mean [Nq] or None), ties
    to the lower index, -1 / +inf past Nt; mean is the mean of value over the listed rows."""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    d2 = (a * a).sum(1)[:, None] + (b * b).sum(1)[None, :] - 2.0 * a @ b.T
    d2 = np.maximum(d2, 0.0)
    k = min(K, b.shape[0])
    order = np.argsort(d2, axis=1, kind='stable')[:, :k]
    idx = np.full((a.shape[0], K), -1, dtype=np.int64)
    dd = np.full((a.shape[0], K), np.inf)
    idx[:, :k] = order
    dd[:, :k] = np.take_along_axis(d2, order, axis=1)
    mean = None
    if value is not None:
        mean = np.asarray(value, dtype=np.float64)[order].mean(axis=1)
    return idx, dd, mean


def knn_scale(d, resid_pool):
    """d(x) + beta, beta = 0.1 x the mean absolute training residual."""
    return d + 0.1 * float(np.mean(resid_pool))
