"""GPU tests at the shapes the tensor-core paths accept but the other suites do not train: every piece of the general
path's backward that depends on H, F or L, the cluster path at its narrowest inputs and outputs, the fp32 path at three
layers, and non-default BatchNormalization moving statistics on every path.

1. General path, bf16 training (gen_supported: H a multiple of 64 up to 512, any L, F <= 1024, O <= 16).  Per shape:
   loss, mse_0 and every gradient tensor against the fp64 oracle, then two Adadelta steps with a MaxNorm bound that
   clips columns in every layer.  What each shape reaches in csrc/rnn_tc.cu is listed at GEN_TRAIN.
2. Forward-only at the shapes of 1 that are new for the forward (F = 300 / 1024, L = 3, H = 384 / 448, O = 1), bf16
   and bf16x3, and one GRU at F = 300, H = 448, L = 3.
3. Cluster path (H = 256, L = 1) at F = 16 (one 16-wide input k-block, k16_x = 1), F = 1 and O = 1: forward and
   gradients; predictions at B = 1921 and F = 16 are row-invariant bit for bit.
4. fp32 path at L = 3 (gradients, one train step), and moving mean / variance away from (0, 1), different in every
   layer, on the fp32, cluster, general bf16 and bf16x3 paths.

Tolerances against the fp64 oracle are those of the other suites: bf16 outputs / loss 3e-2; bf16 gradients per tensor
max-norm relative 6e-2 and cosine 0.999 at T <= 8, 5e-2 and 0.9995 at T = 48 (an oracle tensor that is exactly zero,
dU at T = 1, must come out below 1e-6); bf16 weights after the steps 3e-2; bf16x3 outputs and everything on the fp32
path 1e-4.
"""
import numpy as np
import pytest
import torch

import lfm_oracle as orc
from util import cosine, make_engine, make_problem, rel_err

pytestmark = pytest.mark.gpu

BF16_TOL = 3e-2
X3_TOL = 1e-4
TOL32 = 1e-4
GRAD_T8 = (6e-2, 0.999)        # (max-norm relative, minimum cosine) at T <= 8
GRAD_T48 = (5e-2, 0.9995)      # at T = 48
W_TOL = 3e-2
LR = 0.6


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()


def _init_scale(F):
    """0.3 at F <= 32 and 0.3 sqrt(32 / F) above: the first layer's pre-activations stay O(1), as at F = 32, instead of
    saturating the gates."""
    return 0.3 * min(1.0, np.sqrt(32.0 / F))


def _bn_stats(L, H, seed):
    """Moving mean ~ N(0, 0.3), moving variance ~ U(0.25, 4), drawn per layer (fp32-representable)."""
    rng = np.random.RandomState(seed)
    return [(rng.normal(0.0, 0.3, H).astype(np.float32), rng.uniform(0.25, 4.0, H).astype(np.float32))
            for _ in range(L)]


def _oracle_bn(bn):
    if bn is None:
        return {}
    return dict(bn_mean=[m.astype(np.float64) for m, _ in bn], bn_var=[v.astype(np.float64) for _, v in bn])


def _oracle_grads(params, x, y, O, L, bn=None, **kw):
    preds, fc = orc.forward(params, x.astype(np.float64), num_layers=L, **_oracle_bn(bn), **kw)
    loss, mse, dpred, _ = orc.loss_point_estimate(y.astype(np.float64), preds, target_idx=O - 1, target_lambda=0.5,
                                                  rnn_lambda=0.7)
    return loss, mse, orc.backward(dpred, fc, num_layers=L)


def _check_grads(eng, ref, rel_tol, cos_min, where):
    """Every gradient tensor against the oracle; returns the worst (relative error, cosine) for the log."""
    worst = [0.0, 1.0]
    for (name, _, _, _), g, r in zip(eng.trainable_specs, eng.grads_list(), ref):
        assert np.isfinite(g).all(), where + (name,)
        if np.abs(r).max() == 0.0:            # dU at T = 1 (h_prev = 0)
            assert np.abs(g).max() < 1e-6, where + (name,)
            continue
        e, c = rel_err(g, r), cosine(g, r)
        worst = [max(worst[0], e), min(worst[1], c)]
        assert e < rel_tol, where + (name, e)
        if cos_min is not None:
            assert c > cos_min, where + (name, c)
    return worst


def _backward_vs_oracle(eng, params, x, y, O, L, loss_tol, rel_tol, cos_min, where, bn=None, drop=None):
    """lfmq_backward at (step 5, row 512) against the oracle: loss, mse_0, every gradient tensor."""
    drop = drop or {}
    eng.backward(_cuda(x), _cuda(y), step=5, row0=512)
    tail = eng.grads[eng.n_trainable:eng.n_trainable + 2].cpu().numpy()
    loss, mse, ref = _oracle_grads(params, x, y, O, L, bn=bn, training=True, step=5, row0=512, **drop)
    assert tail[0] == pytest.approx(loss, rel=loss_tol), where + ('loss', tail[0], loss)
    assert tail[1] == pytest.approx(mse, rel=loss_tol), where + ('mse_0', tail[1], mse)
    return _check_grads(eng, ref, rel_tol, cos_min, where)


def _max_norm_that_clips(params, L):
    """A MaxNorm bound below the median column norm of every layer's kernel, so the constraint clips columns in each
    layer (its column count is 4H, its row count F or H)."""
    med = min(float(np.median(np.linalg.norm(params[5 * l], axis=0))) for l in range(L))
    return round(0.9 * med, 4)


def _train_steps_vs_oracle(eng, params, x, y, O, L, max_norm, n_steps, loss_tol, w_tol, where, drop=None):
    """n_steps lfmq_train_step (clip 50, Adadelta, MaxNorm) against the oracle's Train._train_step_point."""
    drop = drop or {}
    cfg = dict(num_layers=L, target_idx=O - 1, target_lambda=0.5, rnn_lambda=0.7, max_grad_norm=50.0,
               optimizer='Adadelta', max_norm=max_norm, train=True, dropout=drop.get('dropout', 0.0),
               recurrent_dropout=drop.get('recurrent_dropout', 0.0), seed=drop.get('seed', 521))
    p = [q.copy() for q in params]
    slots = orc.zero_slots('Adadelta', p)
    xc, yc = _cuda(x), _cuda(y)
    for it in range(n_steps):
        out = eng.train_step(xc, yc, it, LR).cpu().numpy()
        p, mse, loss, _, _ = orc.train_step(p, slots, x.astype(np.float64), y.astype(np.float64), it, cfg, lr=LR)
        assert out[0] == pytest.approx(loss, rel=loss_tol), where + ('loss', it)
        assert out[1] == pytest.approx(mse, rel=loss_tol), where + ('mse_0', it)
    worst = 0.0
    got = eng.get_weights()
    for (name, _, _, _), w, r in zip(eng.trainable_specs, got, p):
        e = rel_err(w, r)
        worst = max(worst, e)
        assert e < w_tol, where + (name, e)
    for l in range(L):
        # the bound is below the initial column norms of every layer (so MaxNorm clipped there), and no column of the
        # engine's kernels is above it
        assert np.linalg.norm(params[5 * l], axis=0).max() > max_norm, where + (l, 'MaxNorm did not clip')
        assert np.linalg.norm(got[5 * l], axis=0).max() <= max_norm * (1 + 1e-5), where + (l, 'MaxNorm')
    return worst


# ---- 1. general path, bf16 training ------------------------------------------------------------------------------------
D2 = dict(dropout=0.2, seed=77)
D21 = dict(dropout=0.2, recurrent_dropout=0.1, seed=77)

# (B, T, F, O, H, L), dropout keywords.  BNU = hidden units per backward tile (64 when H % 128 != 0, else 128); the
# backward step runs H / BNU column tiles per row tile; the first layer's db comes out of its dW GEMM (a constant-one
# input column at F) when F % 64 != 0, else from gcolsum_kernel.
GEN_TRAIN = {
    # BNU = 64, 3 column tiles; dU GEMM M = 192 (ragged second 128-row tile); gbn_drop_bwd with 10 rows per CTA
    'h192-l1': ((200, 6, 32, 16, 192, 1), {}),
    # tile_gemm_kernel<64, EPI_STORE> (dz W^T for layer 0); 5 column tiles; recurrent-dropout state under BNU = 64
    'h320-l2-drop': ((160, 5, 20, 7, 320, 2), dict(dropout=0.25, recurrent_dropout=0.2, seed=99)),
    # the ones column at F = 70 (second 64-wide box); dW GEMM M = 71; 7 column tiles
    'h448-l2-f70': ((130, 4, 70, 5, 448, 2), D2),
    # layer 0 with F % 64 == 0: db from gcolsum_kernel; BNU = 128 with 3 column tiles; 5 rows per CTA in gbn_drop_bwd
    'h384-f64': ((140, 5, 64, 16, 384, 1), {}),
    # L = 3: the middle layer reads dy and then overwrites it; F = 300: 5 input k-blocks; dW GEMM M = 301
    'h128-l3-f300': ((129, 4, 300, 16, 128, 3), D21),
    # F at its limit of 1024 (gcolsum db); <64, EPI_STORE> with one column tile
    'h64-l2-f1024': ((64, 3, 1024, 16, 64, 2), {}),
    # one row, one output
    'h192-l2-b1-o1': ((1, 3, 32, 1, 192, 2), {}),
    # T = 48 with 3 column tiles (persistent backward steps)
    'h192-l2-t48': ((256, 48, 32, 16, 192, 2), D21),
    # 17 row tiles: the backward runs as two chains (9 + 8 row tiles) on two streams, each with 3 column tiles
    'h192-l2-split': ((2100, 8, 32, 16, 192, 2), D21),
}


@pytest.mark.parametrize('name', list(GEN_TRAIN))
def test_general_training_matches_oracle(name):
    (B, T, F, O, H, L), drop = GEN_TRAIN[name]
    params, x, y = make_problem(B, T, F, O, H, L, seed=21, init_scale=_init_scale(F))
    max_norm = _max_norm_that_clips(params, L)
    eng = make_engine(B, T, F, O, H, L, target_idx=O - 1, precision='bf16', optimizer='Adadelta', max_norm=max_norm,
                      **drop)
    eng.set_weights(params)
    rel_tol, cos_min = GRAD_T48 if T > 8 else GRAD_T8
    where = (name,)
    g = _backward_vs_oracle(eng, params, x, y, O, L, BF16_TOL, rel_tol, cos_min, where, drop=drop)
    w = _train_steps_vs_oracle(eng, params, x, y, O, L, max_norm, 2, BF16_TOL, W_TOL, where, drop=drop)
    print('%s: worst gradient rel %.3e cos %.6f; weights after 2 steps rel %.3e' % (name, g[0], g[1], w))
    eng.close()


# ---- 2. forward-only at the new shapes ---------------------------------------------------------------------------------
FWD_NEW = {
    'h128-l3-f300': (129, 4, 300, 16, 128, 3),
    'h64-l2-f1024': (64, 3, 1024, 16, 64, 2),
    'h384-f64': (140, 5, 64, 16, 384, 1),
    'h448-l2-f70': (130, 4, 70, 5, 448, 2),
    'h192-l2-b1-o1': (1, 3, 32, 1, 192, 2),
}


def _forward_vs_oracle(shape, precision, cell):
    B, T, F, O, H, L = shape
    params, x, _ = make_problem(B, T, F, O, H, L, seed=8, init_scale=_init_scale(F), rnn_cell=cell)
    eng = make_engine(B, T, F, O, H, L, train=False, forward_only=True, precision=precision, target_idx=O - 1,
                      rnn_cell=cell)
    eng.set_weights(params)
    preds = eng.forward(_cuda(x)).cpu().numpy()
    eng.close()
    ref, _ = orc.forward(params, x.astype(np.float64), num_layers=L, rnn_cell=cell)
    assert np.isfinite(preds).all()
    return rel_err(preds, ref)


@pytest.mark.parametrize('precision', ['bf16', 'bf16x3'])
@pytest.mark.parametrize('name', list(FWD_NEW))
def test_general_forward_at_new_shapes(name, precision):
    err = _forward_vs_oracle(FWD_NEW[name], precision, 'lstm')
    print('%s %s: rel err %.3e' % (name, precision, err))
    assert err < (X3_TOL if precision == 'bf16x3' else BF16_TOL)


@pytest.mark.parametrize('precision', ['bf16', 'bf16x3'])
def test_gru_forward_f300_h448_l3(precision):
    err = _forward_vs_oracle((130, 4, 300, 5, 448, 3), precision, 'gru')
    print('gru %s: rel err %.3e' % (precision, err))
    assert err < (X3_TOL if precision == 'bf16x3' else BF16_TOL)


# ---- 3. cluster path at narrow inputs and outputs -----------------------------------------------------------------------
CLUSTER = {
    'f16': ((300, 6, 16, 16), dict(dropout=0.2, seed=13)),   # k16_x = 1
    'f1': ((129, 5, 1, 4), {}),                              # a single input feature
    'o1': ((200, 4, 8, 1), {}),                              # a single output
}


@pytest.mark.parametrize('name', list(CLUSTER))
def test_cluster_narrow_inputs_outputs(name):
    (B, T, F, O), drop = CLUSTER[name]
    H, L = 256, 1
    params, x, y = make_problem(B, T, F, O, H, L, seed=12, init_scale=0.3)
    fwd = make_engine(B, T, F, O, H, L, train=False, forward_only=True, precision='bf16', target_idx=O - 1)
    fwd.set_weights(params)
    preds = fwd.forward(_cuda(x)).cpu().numpy()
    fwd.close()
    ref, _ = orc.forward(params, x.astype(np.float64), num_layers=L)
    assert np.isfinite(preds).all()
    assert rel_err(preds, ref) < BF16_TOL, (name, rel_err(preds, ref))
    eng = make_engine(B, T, F, O, H, L, target_idx=O - 1, precision='bf16', **drop)
    eng.set_weights(params)
    g = _backward_vs_oracle(eng, params, x, y, O, L, BF16_TOL, *GRAD_T8, (name,), drop=drop)
    print('cluster %s: forward rel %.3e, worst gradient rel %.3e cos %.6f' % (name, rel_err(preds, ref), g[0], g[1]))
    eng.close()


def test_cluster_f16_predictions_are_row_invariant():
    """B = 1921 at F = 16 (15 full 128-row tiles and a one-row 64-row unit): a permuted batch gives the permuted
    predictions and a slice across the last tile boundary, called with its row offset, gives the slice, bit for bit; the
    slice also matches the oracle."""
    B, T, F, O, H, L = 1921, 8, 16, 16, 256, 1
    params, x, _ = make_problem(B, T, F, O, H, L, seed=41, init_scale=0.5)
    eng = make_engine(B, T, F, O, H, L, train=False, forward_only=True, precision='bf16', target_idx=O - 1)
    eng.set_weights(params)
    xd = _cuda(x)
    R = 5000
    full = eng.forward(xd, step=3, row0=R).cpu().numpy()
    assert np.isfinite(full).all()
    perm = np.roll(np.arange(B)[::-1], 65).copy()
    got = eng.forward(xd[torch.from_numpy(perm).cuda()].contiguous(), step=3, row0=R).cpu().numpy()
    assert np.array_equal(got, full[perm]), float(np.max(np.abs(got - full[perm])))
    a, b = 1883, 1921
    part = eng.forward(xd[a:b].contiguous(), step=3, row0=R + a).cpu().numpy()
    assert np.array_equal(part, full[a:b]), float(np.max(np.abs(part - full[a:b])))
    ref, _ = orc.forward(params, x[a:b].astype(np.float64), num_layers=L)
    assert rel_err(part, ref) < BF16_TOL
    eng.close()


# ---- 4. fp32 at three layers; BatchNormalization moving statistics -----------------------------------------------------
def test_fp32_three_layers_gradients_and_step():
    B, T, F, O, H, L = 40, 6, 12, 5, 24, 3
    drop = dict(dropout=0.2, recurrent_dropout=0.1, seed=31)
    params, x, y = make_problem(B, T, F, O, H, L, seed=6)
    max_norm = _max_norm_that_clips(params, L)
    eng = make_engine(B, T, F, O, H, L, target_idx=O - 1, optimizer='Adadelta', max_norm=max_norm, **drop)
    eng.set_weights(params)
    where = ('fp32-l3',)
    _backward_vs_oracle(eng, params, x, y, O, L, TOL32, TOL32, None, where, drop=drop)
    _train_steps_vs_oracle(eng, params, x, y, O, L, max_norm, 1, TOL32, TOL32, where, drop=drop)
    eng.close()


# path: (B, T, F, O, H, L), engine keywords, forward tolerance, gradient tolerances (None: forward only)
BN_PATHS = {
    'fp32-l2': ((40, 6, 12, 5, 24, 2), dict(precision='fp32', dropout=0.2, recurrent_dropout=0.1, seed=3), TOL32,
                (TOL32, None)),
    'cluster': ((300, 6, 32, 16, 256, 1), dict(precision='bf16', dropout=0.2, seed=3), BF16_TOL, GRAD_T8),
    'general-l2': ((130, 4, 20, 7, 192, 2), dict(precision='bf16', dropout=0.2, recurrent_dropout=0.1, seed=3),
                   BF16_TOL, GRAD_T8),
    'bf16x3-l2': ((130, 5, 20, 7, 128, 2), dict(precision='bf16x3', train=False, forward_only=True), X3_TOL, None),
}


@pytest.mark.parametrize('path', list(BN_PATHS))
def test_bn_moving_statistics(path):
    """Moving mean / variance away from (0, 1) and different in every layer: a path that ignored the mean, used the
    variance for the standard deviation or read another layer's statistics would miss the oracle by far more than the
    tolerance."""
    (B, T, F, O, H, L), kw, ftol, gtol = BN_PATHS[path]
    params, x, y = make_problem(B, T, F, O, H, L, seed=17, init_scale=0.3)
    bn = _bn_stats(L, H, seed=19)
    eng = make_engine(B, T, F, O, H, L, target_idx=O - 1, **kw)
    eng.set_weights(params, bn_stats=bn)
    drop = {k: kw[k] for k in ('dropout', 'recurrent_dropout', 'seed') if k in kw}
    training = kw.get('train', True)
    preds = eng.forward(_cuda(x), step=2, row0=64).cpu().numpy()
    ref, _ = orc.forward(params, x.astype(np.float64), num_layers=L, training=training, step=2, row0=64,
                         **_oracle_bn(bn), **drop)
    ref0, _ = orc.forward(params, x.astype(np.float64), num_layers=L, training=training, step=2, row0=64, **drop)
    err = rel_err(preds, ref)
    print('bn statistics %s: forward rel %.3e (the statistics move the outputs by %.3e)' % (path, err,
                                                                                          rel_err(ref0, ref)))
    assert err < ftol, (path, err)
    if gtol is not None:
        _backward_vs_oracle(eng, params, x, y, O, L, ftol, *gtol, (path,), bn=bn, drop=drop)
    eng.close()
