"""Row-by-row checks of the tensor-core paths at the batch sizes they run at.

The tensor-core paths lay rows out differently from one another (128-row tiles and 64-row half tiles in rounds of
co-resident clusters on the cluster path, 128-row tiles in one or two chains on the general path), and those layouts
change with the batch size.  Whole-batch sums dilute a fault in a few rows, so these tests check rows one at a time:

1. Row invariance, bit for bit.  Every per-element operation is row-local (GEMM rows, cell update, head rows), so a row's
   prediction does not depend on where it sits in the batch or how large the batch is: forward(x[perm]) equals
   forward(x)[perm] (paths without row-keyed dropout), and forward(x[a:b], row0=R+a) equals forward(x, row0=R)[a:b]
   (every path; dropout masks are keyed by the global row).  Each small slice is checked against the fp64 oracle, so
   invariance plus the slice check covers the whole batch row by row.
2. Gradient probes.  A target row of zeros is masked (losses.py:72), so a backward at full B in which one row r has
   nonzero targets is the gradient of that row alone (with the full batch's denominators).  Loss, mse_0 and every
   gradient tensor are compared with the oracle on that one row, at rows on both sides of every 64-row (cluster path) or
   128-row (general path) boundary, with targets at every step, at t=0 only (dU must be exactly zero), at t=T-1 only and
   at both ends.  A neighbouring row's oracle gradients must miss the bound by far, so a row mix-up would be seen.
3. Exact zeros and handle reuse: all targets masked give exactly zero gradients and loss; a smaller batch after a larger
   one on the same handle computes what a fresh handle computes.

Per-row gradient errors (max-norm relative, cosine) against the fp64 oracle, worst over all probes, measured on an
H100 SXM (80 GB) and the bounds set from them are listed at ROW_BOUNDS.
"""
import os
import time

import numpy as np
import pytest
import torch

import lfm_oracle as orc
from util import PATTERNS, cosine, make_engine, make_problem, make_uq_problem, probe_rows, rel_err, target_row

pytestmark = pytest.mark.gpu

BF16_TOL = 3e-2
X3_TOL = 1e-4
HEAD_TOL = 1e-5          # relative to the tensor's largest entry: fp32 atomics summed in another order
F, O = 32, 16
TARGET = O - 1
STEP = 3


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()


def _engine(B, T, H, L, env=None, **kw):
    """make_engine with environment switches that lfmq_create reads (LFMQ_FORCE_GENERIC)."""
    env = env or {}
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return make_engine(B, T, F, O, H, L, target_idx=TARGET, **kw)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


# ---- 1. row invariance of predictions ---------------------------------------------------------------------------------
INV_T = 8
INV_BATCHES = [1, 65, 1920, 1921, 3841, 4096]
BIG = 65536
FWD = dict(train=False, forward_only=True)
DROP = dict(dropout=0.2, recurrent_dropout=0.1, seed=77)

# name: (H, L, cell, engine keywords, environment, also at B=65536)
INV_PATHS = {
    'cluster': (256, 1, 'lstm', dict(precision='bf16', **FWD), None, True),
    'cluster-train': (256, 1, 'lstm', dict(precision='bf16'), None, False),
    'cluster-train-dropout': (256, 1, 'lstm', dict(precision='bf16', dropout=0.2, seed=77), None, False),
    'gen-h64-l1': (64, 1, 'lstm', dict(precision='bf16', **FWD), None, False),
    'gen-h64-l2': (64, 2, 'lstm', dict(precision='bf16', **FWD), None, False),
    'gen-h128-l1': (128, 1, 'lstm', dict(precision='bf16', **FWD), None, False),
    'gen-h128-l2': (128, 2, 'lstm', dict(precision='bf16', **FWD), None, False),
    'gen-h512-l1': (512, 1, 'lstm', dict(precision='bf16', **FWD), None, False),
    'gen-h512-l2': (512, 2, 'lstm', dict(precision='bf16', **FWD), None, False),
    'gen-h256-forced': (256, 1, 'lstm', dict(precision='bf16', **FWD), {'LFMQ_FORCE_GENERIC': '1'}, False),
    'gen-h512-l2-train-dropout': (512, 2, 'lstm', dict(precision='bf16', **DROP), None, False),
    'lstm-x3': (256, 1, 'lstm', dict(precision='bf16x3', **FWD), None, True),
    'gru-bf16': (128, 2, 'gru', dict(precision='bf16', **FWD), None, True),
    'gru-x3': (256, 1, 'gru', dict(precision='bf16x3', **FWD), None, True),
    'uq-lstm-bf16': (128, 2, 'lstm', dict(precision='bf16', uq=True, **FWD, **DROP), None, False),
    'uq-lstm-x3': (256, 1, 'lstm', dict(precision='bf16x3', uq=True, **FWD, **DROP), None, True),
    'uq-gru-bf16': (64, 1, 'gru', dict(precision='bf16', uq=True, **FWD, **DROP), None, False),
    'uq-gru-x3': (128, 2, 'gru', dict(precision='bf16x3', uq=True, **FWD, **DROP), None, True),
}

# slice ends on and off 64-row units, 128-row tiles, the general backward's split (1024 of 1921 rows, 2048 of 4096), the
# cluster forward's rounds (3840 = 30 tiles) and the half-tile last round (the last 256 rows at B=65536)
CUTS = (64, 128, 1024, 1920, 2048, 3840, 32768)


def _slices(B):
    ends = {p for p in CUTS if p < B} | {p for p in (B - 256, B - 128, B - 64, B - 1) if p > 0}
    small = sorted({(max(0, p - 37), min(B, p + 27)) for p in ends}) or [(0, B)]
    large = sorted({(a, b) for a, b in ((1, B), (65, B), (0, B - 1), (B // 2 - 1, B)) if 0 <= a and b - a > 64})
    return small, large


def _perm(B):
    """reversal composed with a roll by 65: every row moves across unit and tile boundaries"""
    return np.roll(np.arange(B)[::-1], 65).copy()


def _outputs(eng, x, row0):
    out = eng.forward(x, step=STEP, row0=row0)
    return tuple(o.cpu().numpy() for o in out) if eng.uq else (out.cpu().numpy(),)


@pytest.mark.parametrize('path', list(INV_PATHS))
def test_predictions_are_row_invariant(path):
    H, L, cell, kw, env, big = INV_PATHS[path]
    uq = kw.get('uq', False)
    stochastic = uq or not kw.get('forward_only', False)
    dropout_kw = {k: kw[k] for k in ('dropout', 'recurrent_dropout', 'seed') if k in kw} if stochastic else {}
    keyed = bool(dropout_kw.get('dropout') or dropout_kw.get('recurrent_dropout'))
    tol = X3_TOL if kw['precision'] == 'bf16x3' else BF16_TOL
    batches = INV_BATCHES + ([BIG] if big else [])
    Bmax = batches[-1]
    if uq:
        params, x = make_uq_problem(Bmax, INV_T, F, O, H, L, seed=41, cell=cell)
    else:
        params, x, _ = make_problem(Bmax, INV_T, F, O, H, L, seed=41, init_scale=0.5, rnn_cell=cell)
    eng = _engine(Bmax, INV_T, H, L, env=env, rnn_cell=cell, **kw)
    eng.set_weights(params)
    xd_all = _cuda(x)
    R = 5000
    worst = 0.0

    def oracle(a, b):
        xs = x[a:b].astype(np.float64)
        if uq:
            p, v, _ = orc.forward_uq(params, xs, num_layers=L, rnn_cell=cell, step=STEP, row0=R + a, **dropout_kw)
            return p, v
        p, _ = orc.forward(params, xs, num_layers=L, rnn_cell=cell, training=stochastic, step=STEP, row0=R + a,
                           **dropout_kw)
        return (p,)

    for B in batches:
        xd = xd_all[:B]
        full = _outputs(eng, xd, R)
        for o in full:
            assert np.isfinite(o).all(), (path, B)
        if not keyed:
            perm = _perm(B)
            got = _outputs(eng, xd[torch.from_numpy(perm).cuda()].contiguous(), R)
            for g, f in zip(got, full):
                assert np.array_equal(g, f[perm]), (path, B, 'permutation', float(np.max(np.abs(g - f[perm]))))
        small, large = _slices(B)
        for a, b in small + large:
            got = _outputs(eng, xd[a:b], R + a)
            for g, f in zip(got, full):
                assert np.array_equal(g, f[a:b]), (path, B, (a, b), float(np.max(np.abs(g - f[a:b]))))
            if (a, b) in small:
                for g, r in zip(got, oracle(a, b)):
                    err = rel_err(g, r)
                    worst = max(worst, err)
                    assert err < tol, (path, B, (a, b), err)
    print('row invariance %s: batches %s, worst slice error vs oracle %.3e' % (path, batches, worst))
    eng.close()
    del eng
    torch.cuda.empty_cache()


# ---- 2. gradient probes on isolated rows --------------------------------------------------------------------------------
# Per-row bounds (max-norm relative error, minimum cosine) per path and tensor kind.  Each bound is the worst value over
# all probes of the path, measured on an H100 SXM (80 GB, 400 W power limit) and given in the comment, times at least
# 1.5 (for the cosine: 1 - cos times at least 1.5), rounded up to one significant digit.  The probed rows' arithmetic does
# not depend on the batch layout (test_predictions_are_row_invariant), so these values are reproducible.
ROW_BOUNDS = {
    'cluster': {                                 # H=256, L=1; T=48 at B=4096, T=16 otherwise; dropout 0 and 0.2
        'kernel': (3e-2, 0.99994),               # worst 1.75e-2, cos 0.9999658
        'recurrent_kernel': (3e-2, 0.99994),     # 1.67e-2, 0.9999604
        'bias': (3e-2, 0.99995),                 # 1.69e-2, 0.9999689
        'gamma': (3e-2, 0.99997),                # 1.43e-2, 0.9999861
        'beta': (5e-3, 0.999995),                # 3.10e-3, 0.9999968
        'OUTPUT_1/kernel': (2e-2, 0.99998),      # 8.22e-3, 0.9999908
        'OUTPUT_1/bias': (6e-3, 0.999995),       # 3.95e-3, 0.9999970
    },
    'general': {                                 # T=48; H=512, L=2 with both dropouts; H=128, L=1 (both layers' worst)
        'kernel': (5e-2, 0.9998),                # 2.74e-2, 0.9999115
        'recurrent_kernel': (4e-2, 0.9998),      # 2.44e-2, 0.9999052
        'bias': (4e-2, 0.9998),                  # 2.62e-2, 0.9999084
        'gamma': (3e-2, 0.9998),                 # 1.87e-2, 0.9999208
        'beta': (2e-2, 0.9998),                  # 1.33e-2, 0.9999248
        'OUTPUT_1/kernel': (3e-2, 0.99996),      # 1.97e-2, 0.9999756
        'OUTPUT_1/bias': (9e-3, 0.99998),        # 5.58e-3, 0.9999875
    },
}
LOSS_TOL = 1e-2          # loss of the probe row, relative (worst 4.0e-3)


def _kind(name):
    return name if name.startswith('OUTPUT') else name.split('/')[-1]


def _oracle_row(params, x_row, y_row, L, row0, B, okw):
    preds, fc = orc.forward(params, x_row[None].astype(np.float64), num_layers=L, training=True, step=STEP, row0=row0,
                            **okw)
    loss, mse, dpred, _ = orc.loss_point_estimate(y_row[None].astype(np.float64), preds, target_idx=TARGET,
                                                  target_lambda=0.5, rnn_lambda=0.7, batch_global=B)
    return loss, mse, preds, orc.backward(dpred, fc, num_layers=L)


def _run_probes(path, B, T, H, L, rows, okw):
    params, x, _ = make_problem(B, T, F, O, H, L, seed=51, init_scale=0.3)
    eng = make_engine(B, T, F, O, H, L, target_idx=TARGET, precision='bf16', **okw)
    eng.set_weights(params)
    names = [s[0] for s in eng.trainable_specs]
    nt = eng.n_trainable
    bounds = ROW_BOUNDS[path]
    xd = _cuda(x)
    yd = torch.zeros(B, T, O, dtype=torch.float32, device='cuda')
    row0 = 7000
    rng = np.random.RandomState(B + T)
    worst = {n: [0.0, 1.0] for n in names}     # max-norm relative error, cosine
    worst_loss, least_miss = 0.0, np.inf
    t_gpu = time.time()
    for i, r in enumerate(rows):
        pattern = PATTERNS[i % len(PATTERNS)]
        y_row = target_row(rng, T, O, pattern)
        yd[r] = _cuda(y_row)
        eng.backward(xd, yd, step=STEP, row0=row0)
        grads = eng.grads_list()
        tail = eng.grads[nt:nt + 2].cpu().numpy()
        yd[r] = 0.0
        loss, mse, preds, ref = _oracle_row(params, x[r], y_row, L, row0 + r, B, okw)
        where = (path, B, okw, r, pattern)
        err = abs(tail[0] - loss) / abs(loss)
        worst_loss = max(worst_loss, err)
        assert err < LOSS_TOL, where + ('loss', tail[0], loss)
        # mse_0 = (pred - y)^2 / B of one element: compare |pred - y| at the forward tolerance
        assert abs(np.sqrt(tail[1] * B) - np.sqrt(mse * B)) <= BF16_TOL * np.abs(preds).max(), \
            where + ('mse_0', tail[1], mse)
        if pattern == 't0':
            assert tail[1] == 0.0, where       # the last step is masked
        for name, g, rf in zip(names, grads, ref):
            assert np.isfinite(g).all(), where + (name,)
            if pattern == 't0' and _kind(name) == 'recurrent_kernel':
                assert not np.any(g), where + (name, 'dU of a row with a target at t=0 only is exactly zero')
            if not np.any(rf):
                assert not np.any(g), where + (name,)
                continue
            e, c = rel_err(g, rf), cosine(g, rf)
            worst[name][0] = max(worst[name][0], e)
            worst[name][1] = min(worst[name][1], c)
            tol, cmin = bounds[_kind(name)]
            assert e < tol and c > cmin, where + (name, e, c)
        if pattern == 'all':
            # the bounds see a row mix-up: the neighbour row's gradients miss them by at least 10x
            nb = r + 1 if r + 1 < B else r - 1
            _, _, _, ref_nb = _oracle_row(params, x[nb], y_row, L, row0 + nb, B, okw)
            for name, g, rf in zip(names, grads, ref_nb):
                if _kind(name) in ('kernel', 'recurrent_kernel', 'bias'):
                    miss = rel_err(g, rf) / bounds[_kind(name)][0]
                    least_miss = min(least_miss, miss)
                    assert miss > 10, where + (name, 'neighbour', miss)
    print('row probes %s B=%d T=%d H=%d L=%d %s: %d probes in %.1f s, loss %.2e, neighbour miss >= %.1fx bound'
          % (path, B, T, H, L, okw, len(rows), time.time() - t_gpu, worst_loss, least_miss))
    for name in names:
        print('    %-40s worst rel %.3e  cos %.7f' % (name, worst[name][0], worst[name][1]))
    eng.close()
    del eng
    torch.cuda.empty_cache()


@pytest.mark.parametrize('dropout', [0.0, 0.2])
@pytest.mark.parametrize('B,T', [(4096, 48), (4500, 16), (3841, 16), (1000, 16)])
def test_cluster_gradient_probes(B, T, dropout):
    """Cluster path (H=256, L=1): rows on both sides of every 64-row unit boundary, whatever the co-resident cluster
    count makes of the rounds."""
    _run_probes('cluster', B, T, 256, 1, probe_rows(B, 64), dict(dropout=dropout, seed=123))


GEN_DROP = dict(dropout=0.2, recurrent_dropout=0.1, seed=123)


@pytest.mark.parametrize('B,H,L,okw', [
    (4096, 512, 2, GEN_DROP),     # two backward chains of 16 row tiles
    (2100, 512, 2, GEN_DROP),     # 17 tiles: chains of 9 and 8
    (1920, 512, 2, GEN_DROP),     # 15 tiles: one chain
    (4096, 128, 1, {}),           # persistent forward
])
def test_general_gradient_probes(B, H, L, okw):
    """General path: rows on both sides of every 128-row tile boundary and of the split between the two chains."""
    nrt = (B + 127) // 128
    n_a = (nrt + 1) // 2 if nrt >= 16 else nrt
    rows = probe_rows(B, 128, extra=(128 * n_a - 1, 128 * n_a))
    _run_probes('general', B, 48, H, L, rows, okw)


# ---- 3. exact zeros and handle reuse -----------------------------------------------------------------------------------
@pytest.mark.parametrize('path,B,H,L,okw', [
    ('cluster', 4500, 256, 1, {}), ('cluster', 4500, 256, 1, dict(dropout=0.2, seed=5)),
    ('general', 2100, 512, 2, {}), ('general', 2100, 512, 2, GEN_DROP),
])
def test_all_masked_targets_give_exact_zeros(path, B, H, L, okw):
    """Every target zero: nothing contributes to the loss, so every gradient and the loss are exactly 0.0, also right
    after a full-batch backward on the same handle (nothing of it may survive in the head partials or dz)."""
    T = 8
    params, x, y = make_problem(B, T, F, O, H, L, seed=61, init_scale=0.3)
    eng = make_engine(B, T, F, O, H, L, target_idx=TARGET, precision='bf16', **okw)
    eng.set_weights(params)
    xd = _cuda(x)
    eng.backward(xd, _cuda(y), step=1, row0=0)
    assert np.abs(eng.grads[:eng.n_trainable].cpu().numpy()).max() > 0
    denom = torch.tensor([float(B), 1.0], dtype=torch.float32, device='cuda')
    eng.backward(xd, torch.zeros(B, T, O, dtype=torch.float32, device='cuda'), step=2, row0=0, denom=denom)
    g = eng.grads[:eng.n_trainable + 2].cpu().numpy()
    assert not np.any(g), [s[0] for s in eng.trainable_specs if np.any(g[s[2]:s[2] + int(np.prod(s[1]))])]
    eng.close()


def _grads_at(eng, xd, yd):
    eng.backward(xd, yd, step=STEP, row0=11)
    return eng.grads_list(), eng.grads[eng.n_trainable:eng.n_trainable + 2].cpu().numpy()


def _assert_same_gradients(got, fresh, names, n_lstm, where):
    (g1, t1), (g0, t0) = got, fresh
    for name, a, b in zip(names[:n_lstm], g1[:n_lstm], g0[:n_lstm]):
        if _kind(name) in ('kernel', 'recurrent_kernel', 'bias'):
            assert np.array_equal(a, b), where + (name, float(np.max(np.abs(a - b))))
    for name, a, b in zip(names, g1, g0):
        scale = max(float(np.max(np.abs(b))), 1e-30)
        assert float(np.max(np.abs(a - b))) <= HEAD_TOL * scale, where + (name,)
    np.testing.assert_allclose(t1, t0, rtol=HEAD_TOL)


@pytest.mark.parametrize('path,H,L,okw,seq', [
    ('cluster', 256, 1, {}, (4096, 1000)),
    ('cluster', 256, 1, dict(dropout=0.2, seed=5), (4096, 1000)),
    ('general', 512, 2, GEN_DROP, (4096, 2100, 1000)),
])
def test_smaller_batch_after_larger_on_one_handle(path, H, L, okw, seq):
    """The dz rows, dLoss/dpred tiles, head partials and the ragged last tile are shared between calls on a handle: a
    smaller batch after a larger one must compute what a fresh handle with the same configuration computes (LSTM W, U, b
    gradients bit for bit; head gradients and the loss to the order of the head's fp32 atomics)."""
    Bmax, T = seq[0], 16
    params, x, y = make_problem(Bmax, T, F, O, H, L, seed=71, init_scale=0.3)
    xd, yd = _cuda(x), _cuda(y)
    eng = make_engine(Bmax, T, F, O, H, L, target_idx=TARGET, precision='bf16', **okw)
    eng.set_weights(params)
    names = [s[0] for s in eng.trainable_specs]
    n_lstm = 5 * L
    got = {B: _grads_at(eng, xd[:B], yd[:B]) for B in seq}
    eng.close()
    for B in seq[1:]:
        fresh = make_engine(Bmax, T, F, O, H, L, target_idx=TARGET, precision='bf16', **okw)
        fresh.set_weights(params)
        _assert_same_gradients(got[B], _grads_at(fresh, xd[:B], yd[:B]), names, n_lstm, (path, okw, B))
        fresh.close()
