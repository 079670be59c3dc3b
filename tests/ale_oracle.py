"""fp64 oracle of accumulated local effects (lfmq_chain_ale, DESIGN.md section 5h).  TEST INFRASTRUCTURE ONLY.  The
edges and bins of one column, the two edge copies and the per-bin fold over any forward callable f(x, m) -> [N,J]
(tests/shapley_oracle.py gives them for every model kind; m = 0 keys window i's dropout masks as row i)."""
import numpy as np


def bins(v, K):
    """(z, bin_of): the edges z_0 < .. < z_Kg of the finite values of v (type-1 quantiles q_0 = v_(1),
    q_k = v_(ceil(k N' / K)), repeats dropped; empty when N' = 0) and each window's 1-based bin (0: non-finite, or
    fewer than two distinct values)."""
    v = np.asarray(v, dtype=np.float32).astype(np.float64)
    fin = np.isfinite(v)
    s = np.sort(v[fin], kind='stable')
    n = s.size
    if n == 0:
        return np.empty(0), np.zeros(v.size, dtype=np.int64)
    q = [s[0]] + [s[-(-k * n // K) - 1] for k in range(1, K + 1)]
    z = [q[0]]
    for a in q[1:]:
        if a > z[-1]:
            z.append(a)
    z = np.array(z)
    b = np.zeros(v.size, dtype=np.int64)
    if z.size > 1:
        b[fin] = np.maximum(np.searchsorted(z, v[fin], side='left'), 1)
    return z, b


def with_column(x, col, values):
    """x [N,T,F] or [N,T*F] with flattened column `col` of window i set to values[i]."""
    N = x.shape[0]
    out = np.array(x, copy=True).reshape(N, -1)
    out[:, col] = values
    return out.reshape(x.shape)


def ale(x, cols, K, outputs):
    """The outputs of lfmq_chain_ale in fp64 as a dict: n_bins [G], edges [G,K+1], counts [G,K], ale [G,K+1,J],
    local_mean and local_sd [G,K,J] (NaN where the library writes NaN), and d [G] of per-window local effects [N,J]
    (NaN for a window without a bin).  outputs(x_copy, m) -> [N,J]."""
    x = np.asarray(x, dtype=np.float64)
    N, G = x.shape[0], len(cols)
    flat = x.reshape(N, -1)
    res = None
    for g, c in enumerate(cols):
        z, b = bins(flat[:, c], K)
        Kg = max(z.size - 1, 0)
        if Kg:
            lo, hi = np.where(b > 0, b - 1, 0), np.where(b > 0, b, 0)
            d = np.asarray(outputs(with_column(x, c, z[hi]), 0), dtype=np.float64) - \
                np.asarray(outputs(with_column(x, c, z[lo]), 0), dtype=np.float64)
        else:
            d = np.asarray(outputs(x, 0), dtype=np.float64) * np.nan
        J = d.shape[1]
        if res is None:
            res = dict(n_bins=np.zeros(G, dtype=np.int64), edges=np.full((G, K + 1), np.nan),
                       counts=np.zeros((G, K), dtype=np.int64), ale=np.full((G, K + 1, J), np.nan),
                       local_mean=np.full((G, K, J), np.nan), local_sd=np.full((G, K, J), np.nan), d=[])
        res['n_bins'][g] = Kg
        res['edges'][g, :z.size] = z
        d[b == 0] = np.nan
        res['d'].append(d)
        if not Kg:
            continue
        n = np.array([(b == k).sum() for k in range(1, Kg + 1)])
        res['counts'][g, :Kg] = n
        mean = np.stack([d[b == k].mean(axis=0) for k in range(1, Kg + 1)])
        res['local_mean'][g, :Kg] = mean
        res['local_sd'][g, :Kg] = np.stack([d[b == k].std(axis=0) for k in range(1, Kg + 1)])
        acc = np.vstack([np.zeros((1, J)), np.cumsum(mean, axis=0)])                 # g(z_0) .. g(z_Kg)
        centre = (n[:, None] * 0.5 * (acc[:-1] + acc[1:])).sum(axis=0) / n.sum()
        res['ale'][g, :Kg + 1] = acc - centre
    return res
