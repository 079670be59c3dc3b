"""fp64 reference of lfmq_chain_forward_uq_dist's distribution pass (DESIGN.md section 5g): the Gaussian mixture
F(q) = (1/M) sum_s Phi((q - mu_s) / sigma_s) of one window's M Monte-Carlo samples (mu_s, sigma_s^2 = v_s), its
quantiles by scipy.optimize.brentq (or, for many windows at once, by bisection), and the CRPS, log score and PIT of a
target."""
import numpy as np
from scipy import optimize, special, stats


def _mv(mu, v):
    return np.asarray(mu, dtype=np.float64).ravel(), np.asarray(v, dtype=np.float64).ravel()


def cdf(q, mu, v):
    mu, v = _mv(mu, v)
    return float(np.mean(special.ndtr((q - mu) / np.sqrt(v))))


def std(mu, v):
    """The mixture's standard deviation: sqrt(E[v] + Var[mu])."""
    mu, v = _mv(mu, v)
    return float(np.sqrt(v.mean() + mu.var()))


def quantiles(mu, v, levels):
    """The q with F(q) = tau for each level, by brentq inside [min_s, max_s] of the component quantiles."""
    mu, v = _mv(mu, v)
    sd = np.sqrt(v)
    out = []
    for tau in levels:
        comp = mu + sd * special.ndtri(tau)
        lo, hi = comp.min(), comp.max()
        if hi - lo <= 0:
            out.append(lo)
            continue
        lo, hi = lo - 1e-9 * (abs(lo) + 1), hi + 1e-9 * (abs(hi) + 1)
        out.append(optimize.brentq(lambda q: cdf(q, mu, v) - tau, lo, hi, xtol=1e-14, rtol=1e-15, maxiter=500))
    return np.array(out)


def quantiles_batch(mu, v, levels, iters=200):
    """quantiles for many windows at once: mu, v [N,M] -> q [N,Q] by bisection over every (window, level) together,
    inside [min_s, max_s] of the component quantiles.  Above the median it solves the upper tail
    mean_s Phi(-(q - mu_s) / sigma_s) = 1 - tau, which fp64 resolves relative to 1 - tau; below it F(q) = tau."""
    mu, v = np.asarray(mu, dtype=np.float64), np.asarray(v, dtype=np.float64)
    tau = np.asarray(levels, dtype=np.float64)
    sd = np.sqrt(v)
    comp = mu[:, None, :] + sd[:, None, :] * special.ndtri(tau)[None, :, None]       # [N,Q,M]
    lo, hi = comp.min(axis=2), comp.max(axis=2)
    upper = tau > 0.5
    target = np.where(upper, 1.0 - tau, tau)[None, :]
    sign = np.where(upper, -1.0, 1.0)[None, :, None]
    for _ in range(iters):
        mid = 0.5 * (lo + hi)
        done = ~((mid > lo) & (mid < hi))                                            # adjacent doubles
        if done.all():
            break
        tail = special.ndtr(sign * (mid[:, :, None] - mu[:, None, :]) / sd[:, None, :]).mean(axis=2)
        below = np.where(upper[None, :], tail > target, tail < target)               # F(mid) < tau
        lo = np.where(below & ~done, mid, lo)
        hi = np.where(~below & ~done, mid, hi)
    return 0.5 * (lo + hi)


def abs_moment(m, var):
    """E|Z| for Z ~ N(m, var)."""
    s = np.sqrt(var)
    z = m / s
    return 2.0 * s * stats.norm.pdf(z) + m * (2.0 * special.ndtr(z) - 1.0)


def crps(mu, v, y):
    """E|X - y| - E|X - X'| / 2 of the mixture in closed form (Grimit et al. 2006), the full M^2 pair sum."""
    mu, v = _mv(mu, v)
    first = abs_moment(mu - y, v).mean()
    pairs = abs_moment(mu[:, None] - mu[None, :], v[:, None] + v[None, :]).mean()
    return float(first - 0.5 * pairs)


def crps_gaussian(m, s, y):
    """Gneiting & Raftery's one-Gaussian form s [z (2 Phi(z) - 1) + 2 phi(z) - 1 / sqrt(pi)], z = (y - m) / s."""
    z = (y - m) / s
    return float(s * (z * (2.0 * special.ndtr(z) - 1.0) + 2.0 * stats.norm.pdf(z) - 1.0 / np.sqrt(np.pi)))


def nll(mu, v, y):
    """-log f(y) by logsumexp."""
    mu, v = _mv(mu, v)
    logs = -0.5 * (y - mu) ** 2 / v - 0.5 * np.log(v) - 0.5 * np.log(2.0 * np.pi)
    return float(-(special.logsumexp(logs) - np.log(len(mu))))


def pit(mu, v, y):
    return cdf(y, mu, v)


def window(mu, v, y, levels):
    """(quantiles [Q], [crps, nll, pit]) of one window; NaN scores for a NaN target."""
    q = quantiles(mu, v, levels)
    if not np.isfinite(y):
        return q, np.full(3, np.nan)
    return q, np.array([crps(mu, v, y), nll(mu, v, y), pit(mu, v, y)])
