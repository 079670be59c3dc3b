"""GPU tests of the bf16 tensor-core paths against an oracle that rounds where the kernels round (tests/bf16_oracle.py).

The other suites hold LFMQ_PREC_BF16 to the fp64 oracle at 3e-2 (outputs, loss) and 5e-2 / 6e-2 (gradients): the
distance of bf16 arithmetic from fp64, large enough to hide any kernel fault of about 1e-3.  The emulated oracle rounds
x, h, the packed weights, the folded head weights, the saved gates and cell states, dz, dLoss/dpred and dLoss/dh where
the kernels do, so what separates it from a kernel is only fp32 summation order and the tanh.approx nonlinearities.

1. Per path (cluster: lstm_tc.cu; general: rnn_tc.cu, incl. H = 256 through LFMQ_FORCE_GENERIC; forward-only GRU and
   RNNUqRangeEstimate on the general path), at shapes the other suites run, with BatchNormalization moving statistics
   away from (0, 1): predictions (and variance), loss, mse_0, every gradient tensor and the weights after two Adadelta
   steps with a MaxNorm bound that clips, against the path's emulated oracle at the bounds of BOUNDS.  Every test also
   requires the kernel to be closer (by RATIO) to the emulated oracle than to the fp64 oracle on its outputs, so a bound
   cannot pass while the emulation models nothing.
2. Exact state: after k train steps a handle's forward equals, bit for bit, the forward of a fresh handle loaded with
   the trained weights (the bf16 weight copies are repacked after every update), and so does a forward after
   set_weights changed only the BN moving statistics (on the cluster path those live only in the folded head weights).
"""
import os

import numpy as np
import pytest
import torch

import bf16_oracle as bo
import lfm_oracle as orc
from util import make_engine, make_problem, make_uq_problem, rel_err

pytestmark = pytest.mark.gpu

LR = 0.6
STEP, ROW0 = 5, 512
# The kernel is closer to the emulated oracle than to the fp64 oracle on predictions and variances by at least this factor
# (worst measured 1.6, uq LSTM H=128 L=2; 2.4 to 7.0 elsewhere).  It is not 5: tanh.approx.f32 in the cell updates
# (relative error up to 2^-11) is not modelled and leaves a residual of the size of the bf16 rounding of h.  The loss
# is not held to a ratio: its fp64 error is a sum of squares whose bf16 terms cancel (measured 0.1x to 230x).
RATIO = 1.25
HEAD_TOL = 1e-5          # relative to the tensor's largest entry: fp32 atomics summed in another order

# Max-norm relative error against the emulated oracle, per path and quantity: at least 1.5x the worst value over the
# path's cases below, measured on an H100 80GB HBM3 (700 W power limit), rounded up to one significant digit, except
# where an entry says "below 1.5x"; the worst value is in the comment.  The fp64 bounds the other suites hold the same
# quantities to are 3e-2 (outputs, loss, weights after steps) and 5e-2 / 6e-2 (gradients).  Gradients on the general path stay within 3x of those (worst
# 1.54e-2, H=512 at T=48): the backward's tanh(c) is tanh.approx.bf16x2, off the rounded exact tanh by about one bf16
# ulp, and that enters every dz; the emulated oracle is no closer to the kernel than the fp64 oracle there (ratio 0.7 to
# 1.3).  The h512-l2-t48 gradients come within 1.3x of their bounds (and test_gpu_general_schedules.py's b2100 within
# 1.4x); they were not loosened, since the kernels compute them deterministically (no atomics), so a run cannot drift
# past a bound it once met.
BOUNDS = {
    'cluster': {
        'pred': 2e-3,                 # 7.09e-4 (t48-f32)
        'loss': 5e-5,                 # 2.94e-5, train steps included
        'mse_0': 9e-5,                # 5.79e-5
        'kernel': 9e-3,               # 5.74e-3
        'recurrent_kernel': 4e-3,     # 2.57e-3
        'bias': 3e-3,                 # 1.88e-3
        'gamma': 4e-4,                # 2.24e-4
        'beta': 3e-5,                 # 1.89e-5
        'OUTPUT_1/kernel': 4e-4,      # 2.24e-4
        'OUTPUT_1/bias': 4e-5,        # 2.39e-5
        'weights': 2e-4,              # 1.20e-4, after two Adadelta steps
    },
    'general': {
        'pred': 3e-3,                 # 1.90e-3 (h192-l2-t48)
        'loss': 1e-4,                 # 6.01e-5
        'mse_0': 2e-4,                # 9.55e-5 (h512-l2-t48)
        'kernel': 2e-2,               # 1.54e-2 (h512-l2-t48), below 1.5x
        'recurrent_kernel': 2e-2,     # 1.35e-2 (h512-l2-t48), below 1.5x with b2100's 1.45e-2
        'bias': 2e-2,                 # 1.09e-2 (h512-l2-t48), below 1.5x with b2100's 1.46e-2
        'gamma': 2e-2,                # 8.60e-3
        'beta': 2e-2,                 # 1.38e-2 (h512-l2-t48)
        'OUTPUT_1/kernel': 8e-4,      # 4.84e-4 (H=512: CASE_BOUNDS)
        'OUTPUT_1/bias': 2e-4,        # 1.04e-4
        'weights': 3e-3,              # 1.34e-3
    },
    'gru': {'pred': 4e-3},            # 2.53e-3 (H=512, L=3)
    'uq': {'pred': 4e-3, 'var': 2e-3},   # 2.42e-3, 8.80e-4
}


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()


def _bn_stats(L, H, seed):
    """Moving mean ~ N(0, 0.3), moving variance ~ U(0.25, 4), drawn per layer (as test_gpu_train_shapes._bn_stats)."""
    rng = np.random.RandomState(seed)
    return [(rng.normal(0.0, 0.3, H).astype(np.float32), rng.uniform(0.25, 4.0, H).astype(np.float32))
            for _ in range(L)]


def _bn_kw(bn):
    return dict(bn_mean=[m.astype(np.float64) for m, _ in bn], bn_var=[v.astype(np.float64) for _, v in bn])


def _kind(name):
    return name if name.startswith('OUTPUT') else name.split('/')[-1]


def _engine(B, T, F, O, H, L, env=None, **kw):
    env = env or {}
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return make_engine(B, T, F, O, H, L, **kw)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _max_norm_that_clips(params, L):
    med = min(float(np.median(np.linalg.norm(params[5 * l], axis=0))) for l in range(L))
    return round(0.9 * med, 4)


class _Report:
    """Worst error per quantity against the emulated oracle, its bound and the ratio of the fp64-oracle error to it.
    Everything is printed before anything is asserted, so a failing case still reports all its numbers."""

    def __init__(self, path, case, bounds=None):
        self.path, self.case = path, case
        self.bounds = dict(BOUNDS[path], **(bounds or {}))      # `bounds`: per quantity or kind, over BOUNDS[path]
        self.rows = []

    def check(self, what, kind, got, emu, ref, ratio=False):
        assert np.isfinite(got).all(), (self.case, what)
        bound = self.bounds.get(what, self.bounds[kind])
        self.rows.append((what, rel_err(got, emu), bound, rel_err(got, ref), ratio))

    def done(self):
        for what, e, bound, e64, _ in self.rows:
            print('%-8s %-22s %-26s emulated %.3e  bound %.0e  fp64 %.3e  (x%.1f)'
                  % (self.path, self.case, what, e, bound, e64, e64 / max(e, 1e-30)))
        for what, e, bound, e64, ratio in self.rows:
            assert e < bound, (self.case, what, e, bound)
            if ratio:
                assert e64 >= RATIO * e, (self.case, what, 'emulated %.3e vs fp64 %.3e' % (e, e64))


def _loss_tail(eng):
    return eng.grads[eng.n_trainable:eng.n_trainable + 2].cpu().numpy()


def _run_training_case(path, case, shape, drop, env=None, bounds=None):
    B, T, F, O, H, L = shape
    params, x, y = make_problem(B, T, F, O, H, L, seed=21, init_scale=0.3 * min(1.0, np.sqrt(32.0 / F)))
    bn = _bn_stats(L, H, seed=19)
    bkw = _bn_kw(bn)
    max_norm = _max_norm_that_clips(params, L)
    eng = _engine(B, T, F, O, H, L, env=env, target_idx=O - 1, precision='bf16', optimizer='Adadelta',
                  max_norm=max_norm, **drop)
    eng.set_weights(params, bn_stats=bn)
    rep = _Report(path, case, bounds)
    emu_p, exact_p = bo.Plan(path), bo.Plan(path, bo.identity)
    x64, y64 = x.astype(np.float64), y.astype(np.float64)
    fkw = dict(num_layers=L, training=True, step=STEP, row0=ROW0, **bkw, **drop)
    lkw = dict(target_idx=O - 1, target_lambda=0.5, rnn_lambda=0.7)

    # predictions
    preds = eng.forward(_cuda(x), step=STEP, row0=ROW0).cpu().numpy()
    emu, fc = bo.forward(emu_p, params, x64, **fkw)
    ref, rfc = orc.forward(params, x64, **fkw)
    rep.check('pred', 'pred', preds, emu, ref, ratio=True)

    # loss, mse_0, gradients
    eng.backward(_cuda(x), _cuda(y), step=STEP, row0=ROW0)
    tail = _loss_tail(eng)
    loss_e, mse_e, dpred_e, _ = orc.loss_point_estimate(y64, emu, **lkw)
    loss_r, mse_r, dpred_r, _ = orc.loss_point_estimate(y64, ref, **lkw)
    rep.check('loss', 'loss', tail[0], loss_e, loss_r)
    rep.check('mse_0', 'mse_0', tail[1], mse_e, mse_r)
    g_emu = bo.backward(emu_p, dpred_e, fc)
    g_ref = orc.backward(dpred_r, rfc, num_layers=L)
    for (name, _, _, _), g, ge, gr in zip(eng.trainable_specs, eng.grads_list(), g_emu, g_ref):
        rep.check(name, _kind(name), g, ge, gr)

    # two Adadelta steps (clip 50, MaxNorm that clips), then the weights
    cfg = dict(num_layers=L, target_idx=O - 1, target_lambda=0.5, rnn_lambda=0.7, max_grad_norm=50.0,
               optimizer='Adadelta', max_norm=max_norm, train=True, dropout=drop.get('dropout', 0.0),
               recurrent_dropout=drop.get('recurrent_dropout', 0.0), seed=drop.get('seed', 521))
    pe, pr = [q.copy() for q in params], [q.copy() for q in params]
    se, sr = orc.zero_slots('Adadelta', pe), orc.zero_slots('Adadelta', pr)
    xc, yc = _cuda(x), _cuda(y)
    for it in range(2):
        out = eng.train_step(xc, yc, it, LR).cpu().numpy()
        pe, mse_e, loss_e, _ = bo.train_step(emu_p, pe, se, x64, y64, it, cfg, LR, **bkw)
        pr, mse_r, loss_r, _ = bo.train_step(exact_p, pr, sr, x64, y64, it, cfg, LR, **bkw)
        rep.check('step %d loss' % it, 'loss', out[0], loss_e, loss_r)
        rep.check('step %d mse_0' % it, 'mse_0', out[1], mse_e, mse_r)
    for (name, _, _, _), w, we, wr in zip(eng.trainable_specs, eng.get_weights(), pe, pr):
        rep.check('weights ' + name, 'weights', w, we, wr)
    rep.done()
    eng.close()


D2 = dict(dropout=0.2, seed=77)
D21 = dict(dropout=0.2, recurrent_dropout=0.1, seed=77)

# (B, T, F, O, H, L), dropout keywords; shapes of test_gpu_train_shapes.py / test_gpu_bf16.py
CLUSTER_CASES = {
    't8-f32': ((300, 8, 32, 16, 256, 1), {}),
    't8-f32-drop': ((300, 8, 32, 16, 256, 1), D2),
    't8-f16': ((300, 8, 16, 16, 256, 1), {}),
    't8-f16-drop': ((300, 8, 16, 16, 256, 1), D2),
    't48-f32': ((256, 48, 32, 16, 256, 1), {}),
    't48-f32-drop': ((256, 48, 32, 16, 256, 1), D2),
    't48-f16': ((256, 48, 16, 16, 256, 1), {}),
    't48-f16-drop': ((256, 48, 16, 16, 256, 1), D2),
}


@pytest.mark.parametrize('case', list(CLUSTER_CASES))
def test_cluster_matches_emulated_oracle(case):
    shape, drop = CLUSTER_CASES[case]
    _run_training_case('cluster', case, shape, drop)


# (B, T, F, O, H, L), dropout keywords, environment
GENERAL_CASES = {
    'h64-l1-f20': ((200, 6, 20, 7, 64, 1), {}, None),
    'h64-l2-f300': ((129, 4, 300, 16, 64, 2), D21, None),
    'h192-l2-f20': ((160, 5, 20, 7, 192, 2), D21, None),
    'h192-l1-f300': ((129, 4, 300, 16, 192, 1), D2, None),
    'h192-l2-t48': ((256, 48, 32, 16, 192, 2), D21, None),
    'h512-l2-t48': ((256, 48, 32, 16, 512, 2), D21, None),        # cfg3's model (test_gpu_general_schedules.py)
    'h512-l2-f20': ((130, 4, 20, 7, 512, 2), D21, None),
    'h512-l1-f300': ((129, 4, 300, 16, 512, 1), {}, None),
    'h256-forced': ((300, 6, 32, 16, 256, 1), D2, {'LFMQ_FORCE_GENERIC': '1'}),
}


# Bounds looser than BOUNDS['general'], per case and quantity; worst values measured on an H100 80GB HBM3 (700 W power
# limit) in the comments.
# * OUTPUT_1/kernel at H=512 (here, and b2100 in test_gpu_general_schedules.py: 1.09e-3).  What is established: the
#   kernel is closer to the emulated oracle than to the fp64 one (x3.4, b2100 x1.4); the predictions it is computed
#   from, and every other gradient, stay within BOUNDS['general']; the error follows neither the number of rows summed
#   (cfg3, B T = 65536, has 3.26e-4) nor the size of the prediction error (h192-l2-t48, pred 1.90e-3, stays under
#   4.84e-4).  Its cause is not isolated.  A forward fault of 2^-7 in h at H=512 moves it to 2.7e-2 to 4.7e-2.
# * The loss and mse_0 after the first Adadelta step follow from the first step's gradients, 1.5e-2 from both oracles
#   (tanh.approx.bf16x2, above; ratio 0.8); the first step's own loss and mse_0 stay within BOUNDS['general'].
CASE_BOUNDS = {
    'h512-l2-t48': {
        'OUTPUT_1/kernel': 2e-3,      # 1.11e-3
        'step 1 loss': 5e-4,          # 3.18e-4
        'step 1 mse_0': 4e-4,         # 2.05e-4
    },
}


@pytest.mark.parametrize('case', list(GENERAL_CASES))
def test_general_matches_emulated_oracle(case):
    shape, drop, env = GENERAL_CASES[case]
    _run_training_case('general', case, shape, drop, env, CASE_BOUNDS.get(case))


# test_gpu_infer_cells.py shapes
GRU_SHAPES = [(200, 5, 20, 7, 64, 1), (130, 4, 33, 16, 128, 2), (300, 6, 32, 3, 256, 1), (129, 3, 9, 16, 512, 3),
              (140, 5, 70, 5, 192, 2)]


@pytest.mark.parametrize('shape', GRU_SHAPES)
def test_gru_forward_matches_emulated_oracle(shape):
    B, T, F, O, H, L = shape
    params, x, _ = make_problem(B, T, F, O, H, L, seed=5, init_scale=0.5, rnn_cell='gru')
    bn = _bn_stats(L, H, seed=19)
    eng = make_engine(B, T, F, O, H, L, train=False, forward_only=True, precision='bf16', target_idx=O - 1,
                      rnn_cell='gru')
    eng.set_weights(params, bn_stats=bn)
    preds = eng.forward(_cuda(x)).cpu().numpy()
    eng.close()
    kw = dict(num_layers=L, rnn_cell='gru', **_bn_kw(bn))
    emu, _ = bo.forward(bo.Plan('general'), params, x.astype(np.float64), **kw)
    ref, _ = orc.forward(params, x.astype(np.float64), **kw)
    rep = _Report('gru', 'x'.join(map(str, shape)))
    rep.check('pred', 'pred', preds, emu, ref, ratio=True)
    rep.done()


UQ_KW = dict(dropout=0.2, recurrent_dropout=0.1, seed=521)


@pytest.mark.parametrize('shape,cell', [((200, 6, 20, 7, 128, 2), 'lstm'), ((300, 5, 32, 16, 256, 1), 'lstm'),
                                        ((150, 6, 33, 5, 64, 1), 'gru'), ((130, 4, 32, 16, 256, 2), 'gru')])
def test_uq_forward_matches_emulated_oracle(shape, cell):
    B, T, F, O, H, L = shape
    params, x = make_uq_problem(B, T, F, O, H, L, seed=13, cell=cell)
    bn = _bn_stats(L, H, seed=19)
    eng = make_engine(B, T, F, O, H, L, target_idx=O - 1, uq=True, rnn_cell=cell, train=False, forward_only=True,
                      precision='bf16', **UQ_KW)
    eng.set_weights(params, bn_stats=bn)
    pred, var = eng.forward(_cuda(x), step=4, row0=64)
    pred, var = pred.cpu().numpy(), var.cpu().numpy()
    eng.close()
    kw = dict(num_layers=L, rnn_cell=cell, step=4, row0=64, **_bn_kw(bn), **UQ_KW)
    ep, ev, _ = bo.forward(bo.Plan('general'), params, x.astype(np.float64), uq=True, **kw)
    rp, rv, _ = orc.forward_uq(params, x.astype(np.float64), **kw)
    rep = _Report('uq', '%s-%s' % (cell, 'x'.join(map(str, shape))))
    rep.check('pred', 'pred', pred, ep, rp, ratio=True)
    rep.check('var', 'var', var, ev, rv, ratio=True)
    rep.done()


# ---- exact state: the bf16 weight copies follow every update ----------------------------------------------------------
STATE_CASES = {
    'cluster': ((300, 8, 32, 16, 256, 1), {}),
    'cluster-drop': ((300, 8, 32, 16, 256, 1), D2),
    'general-l2-drop': ((160, 5, 20, 7, 192, 2), D21),
}


def _flat_from(eng, arrays):
    """The flat parameter vector of eng's layout filled from get_weights(trainable_only=False) of another handle."""
    flat = np.zeros(eng.n_total, dtype=np.float32)
    for (name, shp, off, _), a in zip(eng.specs, arrays):
        flat[off:off + int(np.prod(shp))] = np.asarray(a, dtype=np.float32).ravel()
    return flat


def _fresh_like(shape, drop, max_norm, arrays):
    B, T, F, O, H, L = shape
    e = make_engine(B, T, F, O, H, L, target_idx=O - 1, precision='bf16', optimizer='Adadelta', max_norm=max_norm,
                    **drop)
    e.set_flat(_flat_from(e, arrays))
    return e


def _assert_same_gradients(g1, g0, t1, t0, names, where):
    for name, a, b in zip(names, g1, g0):
        scale = max(float(np.max(np.abs(b))), 1e-30)
        assert float(np.max(np.abs(a - b))) <= HEAD_TOL * scale, where + (name, float(np.max(np.abs(a - b))) / scale)
    np.testing.assert_allclose(t1, t0, rtol=HEAD_TOL)


@pytest.mark.parametrize('k', [1, 3])
@pytest.mark.parametrize('case', list(STATE_CASES))
def test_forward_after_train_steps_uses_the_updated_weights(case, k):
    """After k train steps the handle's forward and next backward are a fresh handle's with the trained weights: the
    bf16 copies (packed weights, folded head) were repacked after the last update, not left one step behind."""
    shape, drop = STATE_CASES[case]
    B, T, F, O, H, L = shape
    params, x, y = make_problem(B, T, F, O, H, L, seed=31, init_scale=0.3)
    bn = _bn_stats(L, H, seed=19)
    max_norm = _max_norm_that_clips(params, L)
    eng = make_engine(B, T, F, O, H, L, target_idx=O - 1, precision='bf16', optimizer='Adadelta', max_norm=max_norm,
                      **drop)
    eng.set_weights(params, bn_stats=bn)
    xc, yc = _cuda(x), _cuda(y)
    for it in range(k):
        eng.train_step(xc, yc, it, LR)
    got = eng.forward(xc, step=k, row0=ROW0).cpu().numpy()
    eng.backward(xc, yc, step=k, row0=ROW0)
    g1, t1 = eng.grads_list(), _loss_tail(eng)
    names = [s[0] for s in eng.trainable_specs]
    trained = eng.get_weights(trainable_only=False)
    assert max(rel_err(w, p) for w, p in zip(eng.get_weights(), params)) > 1e-4    # the steps moved the weights
    eng.close()
    fresh = _fresh_like(shape, drop, max_norm, trained)
    want = fresh.forward(xc, step=k, row0=ROW0).cpu().numpy()
    assert np.array_equal(got, want), (case, k, float(np.max(np.abs(got - want))))
    fresh.backward(xc, yc, step=k, row0=ROW0)
    _assert_same_gradients(g1, fresh.grads_list(), t1, _loss_tail(fresh), names, (case, k))
    fresh.close()


@pytest.mark.parametrize('case', list(STATE_CASES))
def test_set_weights_of_bn_statistics_alone_reaches_the_forward(case):
    """set_weights that changes only the (non-trainable) BN moving statistics changes the next forward to what a fresh
    handle with those statistics computes, bit for bit (on the cluster path they live only in the folded head)."""
    shape, drop = STATE_CASES[case]
    B, T, F, O, H, L = shape
    params, x, _ = make_problem(B, T, F, O, H, L, seed=32, init_scale=0.3)
    bn0, bn1 = _bn_stats(L, H, seed=19), _bn_stats(L, H, seed=20)
    eng = make_engine(B, T, F, O, H, L, target_idx=O - 1, precision='bf16', **drop)
    eng.set_weights(params, bn_stats=bn0)
    xc = _cuda(x)
    before = eng.forward(xc, step=2, row0=ROW0).cpu().numpy()
    eng.set_weights(params, bn_stats=bn1)
    got = eng.forward(xc, step=2, row0=ROW0).cpu().numpy()
    eng.close()
    fresh = make_engine(B, T, F, O, H, L, target_idx=O - 1, precision='bf16', **drop)
    fresh.set_weights(params, bn_stats=bn1)
    want = fresh.forward(xc, step=2, row0=ROW0).cpu().numpy()
    fresh.close()
    assert rel_err(before, want) > 1e-2          # the statistics matter
    assert np.array_equal(got, want), (case, float(np.max(np.abs(got - want))))
