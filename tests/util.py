"""Shared helpers for the parity tests (oracle = checker only)."""
import numpy as np

import lfm_oracle as orc


def make_problem(B, T, F, O, H, L, seed=0, zero_rows=True, init_scale=0.5, rnn_cell='lstm'):
    rng = np.random.RandomState(seed)
    params = orc.init_params(L, F, O, H, init_scale=init_scale, seed=seed + 1, dtype=np.float64, rnn_cell=rnn_cell)
    for l in range(L):
        params[5 * l + 2] = params[5 * l + 2] + rng.normal(size=params[5 * l + 2].shape) * 0.1
        params[5 * l + 3] = params[5 * l + 3] + rng.normal(size=H) * 0.1
        params[5 * l + 4] = params[5 * l + 4] + rng.normal(size=H) * 0.1
    params[5 * L + 1] = params[5 * L + 1] + rng.normal(size=O) * 0.1
    params = [p.astype(np.float32).astype(np.float64) for p in params]   # exactly representable in fp32
    x = rng.normal(size=(B, T, F)).astype(np.float32)
    y = rng.normal(size=(B, T, O)).astype(np.float32)
    if zero_rows and B > 1 and T > 2:
        y[0, :2, :] = 0.0       # zero-padded steps -> loss mask 0 (losses.py:72)
        y[B - 1, 0, :] = 0.0
    return params, x, y


def make_uq_problem(B, T, F, O, H, L, seed, cell):
    """Weights of RNNUqRangeEstimate (target and variance heads) and inputs."""
    rng = np.random.RandomState(seed)
    params = orc.init_params(L, F, O, H, init_scale=0.5, seed=seed + 1, dtype=np.float64, rnn_cell=cell, uq=True)
    for l in range(L):
        params[5 * l + 2] = params[5 * l + 2] + rng.normal(size=params[5 * l + 2].shape) * 0.1
    params[-1] = rng.normal(size=O) * 0.5
    params[-3] = rng.normal(size=O) * 0.5
    params = [p.astype(np.float32).astype(np.float64) for p in params]
    x = rng.normal(size=(B, T, F)).astype(np.float32)
    return params, x


def rel_err(a, b):
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-30))


def cosine(a, b):
    a = np.asarray(a, dtype=np.float64).ravel()
    b = np.asarray(b, dtype=np.float64).ravel()
    return float(np.dot(a, b) / (np.linalg.norm(a) * np.linalg.norm(b) + 1e-30))


PATTERNS = ('all', 't0', 'last', 'ends')    # which steps of a probe row have nonzero targets


def target_row(rng, T, O, pattern):
    """Targets of one probe row: normal values at the steps `pattern` names, zeros (masked steps) elsewhere."""
    y = rng.normal(size=(T, O)).astype(np.float32)
    keep = np.zeros(T, dtype=bool)
    if pattern == 'all':
        keep[:] = True
    if pattern in ('t0', 'ends'):
        keep[0] = True
    if pattern in ('last', 'ends'):
        keep[-1] = True
    y[~keep] = 0.0
    return y


def probe_rows(B, unit, extra=()):
    """Rows 0 and B-1, both sides of every multiple of `unit`, and `extra`."""
    rows = {0, B - 1} | set(extra)
    for k in range(unit, B, unit):
        rows |= {k - 1, k}
    return sorted(r for r in rows if 0 <= r < B)


def make_engine(B, T, F, O, H, L, **kw):
    from lfm_quant_b200.engine import ForecasterEngine
    return ForecasterEngine(max_batch=B, seq_len=T, n_inputs=F, n_outputs=O, num_hidden=H, num_layers=L, **kw)
