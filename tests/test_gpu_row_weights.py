"""Row weights of the training loss (lfmq_set_row_weights, DESIGN.md section 6d) on every training path.

1. Weights of 1 give the same bits as no weights: the loss tail, every gradient and the parameters after lfmq_apply.
   The bf16 heads sum their loss terms and head gradients through fp32 shared-memory atomics, whose order varies from
   run to run, so there the recurrent-layer gradients are compared bit for bit and the head's to HEAD_TOL.
2. Random weights, zeros included, against the fp64 weighted oracle (tests/row_weights_oracle.py): fp32 within 1e-4,
   tf32 within 1.1e-2.  bf16 is held to the error its unweighted step has against the same oracle.
3. At fp32 without dropout, weight 2 on a row equals duplicating the row and weight 0 equals removing it.
"""
import numpy as np
import pytest
import torch

import row_weights_oracle as rwo
from util import make_problem, rel_err

pytestmark = pytest.mark.gpu

F, O, TARGET = 12, 6, 2
HEAD_TOL = 2e-5
CFG = dict(target_idx=TARGET, target_lambda=0.5, rnn_lambda=0.7)


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _engine(B, T, H, L, **kw):
    from lfm_quant_b200.engine import ForecasterEngine
    return ForecasterEngine(max_batch=B, seq_len=T, n_inputs=F, n_outputs=O, num_hidden=H, num_layers=L,
                            target_idx=TARGET, **kw)


def _chain(B, T, H, L, S, **kw):
    from lfm_quant_b200.engine import ForecastChainEngine
    return ForecastChainEngine(forecast_steps=S, weights=[1.0] * S, max_batch=B, seq_len=T, n_inputs=F, n_outputs=O,
                               num_hidden=H, num_layers=L, target_idx=TARGET, **kw)


def _dense(B, T):
    from lfm_quant_b200.engine import DenseEngine
    return DenseEngine(max_batch=B, seq_len=T, n_inputs=F, n_outputs=O, target_idx=TARGET)


def _weights(B, seed, zeros=True):
    rng = np.random.RandomState(seed)
    w = rng.uniform(0.0, 3.0, size=B).astype(np.float32)
    if zeros:
        w[rng.choice(B, size=max(1, B // 8), replace=False)] = 0.0
    return w


# ---- the paths --------------------------------------------------------------------------------------------------------
# name -> (B, T, H, L, engine kwargs)
POINT = {
    'fp32-lstm': (256, 8, 64, 1, dict(precision='fp32')),
    'fp32-gru': (256, 8, 64, 2, dict(precision='fp32', rnn_cell='gru')),
    'tf32-lstm': (256, 8, 64, 1, dict(precision='tf32')),
    'tf32-gru': (256, 8, 64, 1, dict(precision='tf32', rnn_cell='gru')),
}
BF16 = {
    'bf16-cluster': (4096, 48, 256, 1, dict(precision='bf16')),
    'bf16-general': (2100, 16, 512, 2, dict(precision='bf16', dropout=0.2, recurrent_dropout=0.1, seed=7)),
}


def _run(eng, x, y, w, step=3, apply=True):
    """One backward (+ apply) on eng with row weights w (None: unweighted): (gradient + tail, parameters after)."""
    wd = None if w is None else _cuda(w)
    eng.set_row_weights(wd)
    eng.backward(x, y, step=step, row0=0)
    g = eng.grads[:eng.n_trainable + 2].cpu().numpy().copy()
    p = None
    if apply:
        eng.apply(0.5, step)
        p = np.concatenate([a.ravel() for a in eng.get_weights()])
    torch.cuda.synchronize()
    return g, p


@pytest.mark.parametrize('name', list(POINT) + ['dense'])
def test_ones_give_the_unweighted_bits(name):
    if name == 'dense':
        B, T = 300, 5
        rng = np.random.RandomState(3)
        x = rng.normal(size=(B, T, F)).astype(np.float32)
        y = rng.normal(size=(B, O)).astype(np.float32)
        y[::7] = 0.0
        make = lambda: _dense(B, T)  # noqa: E731
        params = None
    else:
        B, T, H, L, kw = POINT[name]
        params, x, y = make_problem(B, T, F, O, H, L, seed=11, init_scale=0.3, rnn_cell=kw.get('rnn_cell', 'lstm'))
        make = lambda: _engine(B, T, H, L, **kw)  # noqa: E731
    out = []
    for w in (None, np.ones(B, np.float32)):
        eng = make()
        if params is not None:
            eng.set_weights(params)
        else:
            eng.set_weights([np.random.RandomState(5).normal(size=a.shape).astype(np.float32) * 0.1
                             for a in eng.get_weights()])
        out.append(_run(eng, _cuda(x), _cuda(y), w))
        eng.close()
    (g0, p0), (g1, p1) = out
    assert np.array_equal(g0, g1), float(np.max(np.abs(g0 - g1)))
    assert np.array_equal(p0, p1), float(np.max(np.abs(p0 - p1)))


@pytest.mark.parametrize('S', [1, 2])
def test_uq_ones_give_the_unweighted_bits(S):
    B, T, H, L = 256, 8, 64, 1
    rng = np.random.RandomState(21)
    x = _cuda(rng.normal(size=(B, T, F)).astype(np.float32))
    ys = [_cuda(rng.normal(size=(B, T, O)).astype(np.float32)) for _ in range(S)]
    params, res = None, []
    for w in (None, np.ones(B, np.float32)):
        eng = _chain(B, T, H, L, S, uq=True, dropout=0.1, seed=3)
        if params is None:
            params = eng.get_weights()
        eng.set_weights(params)
        eng.set_row_weights(None if w is None else _cuda(w))
        out = eng.train_step(x, ys, 2, 0.5)
        torch.cuda.synchronize()
        res.append((np.concatenate([g.ravel() for g in eng.grads_list()]),
                    np.asarray([float(v) for v in out]),
                    np.concatenate([a.ravel() for a in eng.get_weights()])))
        eng.close()
    for a, b in zip(res[0], res[1]):
        assert np.array_equal(a, b)


@pytest.mark.parametrize('name', list(BF16))
def test_bf16_ones_give_the_unweighted_bits(name):
    B, T, H, L, kw = BF16[name]
    params, x, y = make_problem(B, T, F, O, H, L, seed=13, init_scale=0.3)
    xd, yd = _cuda(x), _cuda(y)
    eng = _engine(B, T, H, L, **kw)
    eng.set_weights(params)
    g0, _ = _run(eng, xd, yd, None, apply=False)
    g1, _ = _run(eng, xd, yd, np.ones(B, np.float32), apply=False)
    for s in eng.trainable_specs:
        a, b = g0[s[2]:s[2] + int(np.prod(s[1]))], g1[s[2]:s[2] + int(np.prod(s[1]))]
        if s[0].startswith('lstm') and s[0].split('/')[-1] in ('kernel', 'recurrent_kernel', 'bias'):
            assert np.array_equal(a, b), s[0]
        else:
            assert rel_err(b, a) <= HEAD_TOL, (s[0], rel_err(b, a))
    np.testing.assert_allclose(g1[-2:], g0[-2:], rtol=HEAD_TOL)
    eng.close()


# ---- 2. random weights against the oracle --------------------------------------------------------------------------------
@pytest.mark.parametrize('name', list(POINT))
def test_random_weights_match_the_oracle(name):
    B, T, H, L, kw = POINT[name]
    tol = 1e-4 if kw['precision'] == 'fp32' else 1.1e-2
    params, x, y = make_problem(B, T, F, O, H, L, seed=17, init_scale=0.3, rnn_cell=kw.get('rnn_cell', 'lstm'))
    w = _weights(B, 1)
    eng = _engine(B, T, H, L, **kw)
    eng.set_weights(params)
    g, _ = _run(eng, _cuda(x), _cuda(y), w, apply=False)
    loss, mse, ref = rwo.point_grads(params, x, y, w.astype(np.float64),
                                     dict(CFG, num_layers=L, rnn_cell=kw.get('rnn_cell', 'lstm')))
    worst = 0.0
    for s, r in zip(eng.trainable_specs, ref):
        e = rel_err(g[s[2]:s[2] + int(np.prod(s[1]))], r.ravel())
        worst = max(worst, e)
        assert e <= tol, (s[0], e)
    assert abs(g[-2] - loss) <= tol * abs(loss) and abs(g[-1] - mse) <= tol * abs(mse)
    print('%s: worst gradient error %.2e (bound %.1e)' % (name, worst, tol))
    eng.close()


@pytest.mark.parametrize('name', list(BF16))
def test_bf16_random_weights_match_the_oracle(name):
    """bf16 with random weights is as close to the fp64 weighted oracle as the unweighted step is to the unweighted
    oracle (no dropout, so the oracle's forward is the handle's)."""
    B, T, H, L, kw = BF16[name]
    kw = dict(precision='bf16')
    params, x, y = make_problem(B, T, F, O, H, L, seed=19, init_scale=0.3)
    eng = _engine(B, T, H, L, **kw)
    eng.set_weights(params)
    w = _weights(B, 2)
    errs = {}
    for key, wv in (('unweighted', None), ('weighted', w)):
        g, _ = _run(eng, _cuda(x), _cuda(y), wv, apply=False)
        _, _, ref = rwo.point_grads(params, x, y, None if wv is None else wv.astype(np.float64),
                                    dict(CFG, num_layers=L))
        errs[key] = max(rel_err(g[s[2]:s[2] + int(np.prod(s[1]))], r.ravel())
                        for s, r in zip(eng.trainable_specs, ref))
    print(name, errs)
    assert errs['weighted'] <= 2.0 * errs['unweighted'] + 1e-3, errs
    eng.close()


# ---- 3. weight 2 = a duplicated row, weight 0 = a removed row -----------------------------------------------------------
def _dup_remove(make, x, y, j, k, prepare=None):
    """Gradients of (w[j] = 2, w[k] = 0, else 1) on x, y and of the unweighted batch with row j repeated and row k
    dropped."""
    B = x.shape[0]
    w = np.ones(B, np.float32)
    w[j], w[k] = 2.0, 0.0
    rows = [i for i in range(B) if i != k] + [j]
    out = []
    for xx, yy, ww in ((x, y, w), (x[rows], y[rows], None)):
        eng = make(len(rows) if ww is None else B)
        if prepare:
            prepare(eng)
        g, _ = _run(eng, _cuda(xx), _cuda(yy), ww, apply=False)
        out.append(g)
        eng.close()
    return out


@pytest.mark.parametrize('cell', ['lstm', 'gru'])
def test_weight_two_duplicates_and_zero_removes_a_row(cell):
    B, T, H, L = 200, 8, 64, 1
    params, x, y = make_problem(B, T, F, O, H, L, seed=23, init_scale=0.3, rnn_cell=cell)
    gw, gd = _dup_remove(lambda b: _engine(b, T, H, L, precision='fp32', rnn_cell=cell), x, y, 5, 77,
                         lambda e: e.set_weights(params))
    assert rel_err(gw, gd) <= 1e-5, rel_err(gw, gd)


def test_uq_weight_two_duplicates_and_zero_removes_a_row():
    B, T, H, L = 200, 8, 64, 1
    rng = np.random.RandomState(29)
    x = rng.normal(size=(B, T, F)).astype(np.float32)
    y = rng.normal(size=(B, T, O)).astype(np.float32)
    params = None

    def prep(e):
        nonlocal params
        if params is None:
            params = e.get_weights()
        e.set_weights(params)
    gw, gd = _dup_remove(lambda b: _engine(b, T, H, L, precision='fp32', uq=True), x, y, 9, 123, prep)
    # the uq tail is {uq_loss, mse_0}: both and every gradient
    assert rel_err(gw, gd) <= 1e-5, rel_err(gw, gd)


def test_dense_weight_two_duplicates_and_zero_removes_a_row():
    B, T = 300, 5
    rng = np.random.RandomState(31)
    x = rng.normal(size=(B, T, F)).astype(np.float32)
    y = rng.normal(size=(B, O)).astype(np.float32)
    y[::9] = 0.0
    params = [rng.normal(size=a.shape).astype(np.float32) * 0.1 for a in _dense_shapes(T)]
    gw, gd = _dup_remove(lambda b: _dense(b, T), x, y, 4, 150, lambda e: e.set_weights(params))
    assert rel_err(gw, gd) <= 1e-5, rel_err(gw, gd)


def _dense_shapes(T):
    return [np.zeros((T * F, O)), np.zeros(O)]


def test_dense_random_weights_match_the_oracle():
    B, T = 300, 5
    rng = np.random.RandomState(37)
    x = rng.normal(size=(B, T, F)).astype(np.float32)
    y = rng.normal(size=(B, O)).astype(np.float32)
    y[::9] = 0.0
    W = (rng.normal(size=(T * F, O)) * 0.1).astype(np.float32)
    b = (rng.normal(size=O) * 0.1).astype(np.float32)
    w = _weights(B, 3)
    eng = _dense(B, T)
    eng.set_weights([W, b])
    g, _ = _run(eng, _cuda(x), _cuda(y), w, apply=False)
    xf = x.reshape(B, -1).astype(np.float64)
    pred = xf @ W + b
    loss, mse, dpred = rwo.loss_dense(y.astype(np.float64), pred, w.astype(np.float64), target_idx=TARGET,
                                      target_lambda=0.5)
    assert rel_err(g[:T * F * O], (xf.T @ dpred).ravel()) <= 1e-4
    assert rel_err(g[T * F * O:T * F * O + O], dpred.sum(0)) <= 1e-4
    assert abs(g[-2] - loss) <= 1e-4 * loss and abs(g[-1] - mse) <= 1e-4 * mse
    eng.close()


def test_all_zero_weights_give_zero_loss_and_gradient():
    B, T, H, L = 128, 8, 64, 1
    params, x, y = make_problem(B, T, F, O, H, L, seed=41, init_scale=0.3)
    eng = _engine(B, T, H, L, precision='fp32')
    eng.set_weights(params)
    g, _ = _run(eng, _cuda(x), _cuda(y), np.zeros(B, np.float32), apply=False)
    assert not np.any(g)
    eng.close()


def test_loss_entry_points_stay_unweighted():
    """lfmq_loss ignores the handle's row weights: validation is unweighted."""
    B, T, H, L = 128, 8, 64, 1
    params, x, y = make_problem(B, T, F, O, H, L, seed=43, init_scale=0.3)
    eng = _engine(B, T, H, L, precision='fp32')
    eng.set_weights(params)
    p = eng.forward(_cuda(x), step=0)
    a = eng.loss(p, _cuda(y)).cpu().numpy()
    eng.set_row_weights(_cuda(_weights(B, 4)))
    b = eng.loss(p, _cuda(y)).cpu().numpy()
    assert np.array_equal(a, b)
    eng.close()
