"""The host side of tests/test_gpu_analyses_at_scale.py: the vectorized fp64 quantile solver of
tests/predictive_oracle.py against its brentq one, at the levels and mixtures that test runs (tails down to 1e-4 and
up to 0.9999, multimodal mixtures, variances on the 1e-6 floor)."""
import numpy as np
import pytest

import predictive_oracle as pdo

LEVELS = np.array([1e-4, 5e-4, 1e-3, 0.005, 0.01, 0.025, 0.05, 0.075, 0.1, 0.15, 0.2, 0.25, 0.3, 0.35, 0.4, 0.45, 0.5,
                   0.55, 0.6, 0.65, 0.7, 0.75, 0.8, 0.85, 0.9, 0.95, 0.975, 0.99, 0.995, 0.999, 0.9995, 0.9999])


def _mixtures(kind, N, M, seed):
    rng = np.random.RandomState(seed)
    if kind == 'unimodal':
        mu = rng.normal(size=(N, 1)) + 0.1 * rng.normal(size=(N, M))
        v = np.exp(rng.normal(size=(N, M)) * 0.3)
    elif kind == 'multimodal':
        mu = rng.normal(size=(N, M)) * 300.0
        v = np.exp(rng.normal(size=(N, M)) * 0.3)
    else:                                                   # every variance on the floor, means O(1)
        mu = rng.normal(size=(N, M)) * 0.01 + rng.normal(size=(N, 1))
        v = np.full((N, M), 1e-6)
    return mu, v


@pytest.mark.parametrize('kind,M', [('unimodal', 1), ('unimodal', 8), ('unimodal', 33), ('multimodal', 7),
                                    ('floor', 7)])
def test_vectorized_quantiles_match_brentq(kind, M):
    N = 12
    mu, v = _mixtures(kind, N, M, seed=M)
    levels = LEVELS.astype(np.float32).astype(np.float64)
    got = pdo.quantiles_batch(mu, v, levels)
    assert got.shape == (N, len(levels))
    worst = 0.0
    for b in range(N):
        ref = pdo.quantiles(mu[b], v[b], levels)
        sd = pdo.std(mu[b], v[b])
        worst = max(worst, np.abs(got[b] - ref).max() / sd)
        assert (np.diff(got[b]) > 0).all()
    assert worst < 1e-9, worst


def test_vectorized_quantiles_hit_their_levels_in_the_tails():
    """F(q) = tau to fp64 relative accuracy, in the upper tail too (where 1 - F is what carries the information)."""
    from scipy import special
    mu, v = _mixtures('unimodal', 20, 8, seed=3)
    levels = LEVELS.astype(np.float32).astype(np.float64)
    q = pdo.quantiles_batch(mu, v, levels)
    for b in range(20):
        z = (q[b][:, None] - mu[b][None, :]) / np.sqrt(v[b])[None, :]
        lower, upper = special.ndtr(z).mean(axis=1), special.ndtr(-z).mean(axis=1)
        err = np.where(levels > 0.5, np.abs(upper - (1.0 - levels)) / (1.0 - levels),
                       np.abs(lower - levels) / levels)
        assert err.max() < 1e-10, (b, err.max())
