"""CPU tests of the bf16-rounding oracle (tests/bf16_oracle.py): its rounding is torch's bf16 conversion bit for bit (NaN
payloads aside), each path's plan is the fp64 oracle's arithmetic when the rounding is switched off, and with it on the
plans round something."""
import numpy as np
import pytest
import torch

import bf16_oracle as bo
import lfm_oracle as orc
from util import make_problem, make_uq_problem


def _torch_bits(a):
    t = torch.from_numpy(np.asarray(a, dtype=np.float32)).to(torch.bfloat16).float()
    return t.numpy().view(np.uint32)


def _bits(a):
    return np.asarray(a, dtype=np.float32).view(np.uint32)


def _f32(bits):
    return np.array(bits, dtype=np.uint32).view(np.float32)


def test_rb_matches_torch_bit_for_bit_at_the_edges():
    vals = _f32([
        0x3F808000,   # tie, even below (1.0 + half an ulp): stays 1.0
        0x3F818000,   # tie, odd below: rounds up to 0x3F82
        0xBF808000, 0xBF818000,            # the same ties, negative
        0x3F808001, 0x3F807FFF,            # just above / below a tie
        0x00000001, 0x00008000, 0x00018000, 0x0000FFFF, 0x807FFFFF,    # fp32 subnormals, incl. ties
        0x7F7F0000, 0x7F7F7FFF,            # bf16 max, just below the rounding threshold
        0x7F7F8000, 0x7F7FFFFF, 0xFF7FFFFF,  # ties / values above bf16 max: overflow to +-inf
        0x7F800000, 0xFF800000,            # +-inf
        0x7FC00000, 0x7F800001, 0xFFC00001,  # NaNs
        0x00000000, 0x80000000,
    ])
    rng = np.random.RandomState(0)
    rand = _f32(rng.randint(0, 2 ** 32, size=20000, dtype=np.uint64).astype(np.uint32))
    for v in (vals, rand):
        got = _bits(bo.rb(v))
        want = _torch_bits(v)
        nan = np.isnan(v)
        assert np.array_equal(got[~nan], want[~nan])
        # NaN stays NaN; its payload is the kernels' canonical 0x7FFF (torch's CPU conversion picks another)
        assert np.isnan(bo.rb(v)[nan]).all() and np.all(got[nan] == 0x7FFF0000)
    # spot checks of the rule itself
    assert bo.rb(_f32([0x3F808000]))[0] == 1.0
    assert _bits(bo.rb(_f32([0x3F818000])))[0] == 0x3F820000
    assert np.isinf(bo.rb(_f32([0x7F7F8000]))[0])
    assert _bits(bo.rb(_f32([0x7F7F7FFF])))[0] == 0x7F7F0000


def _bn(L, H, seed):
    rng = np.random.RandomState(seed)
    return [rng.normal(0.0, 0.3, H) for _ in range(L)], [rng.uniform(0.25, 4.0, H) for _ in range(L)]


def _close(a, b, tol=1e-12):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.max(np.abs(a - b))) <= tol * max(float(np.max(np.abs(b))), 1e-30)


# path, (B, T, F, O, H, L), dropout keywords (training)
IDENTITY_CASES = [
    ('cluster', (5, 4, 6, 3, 256, 1), {}),
    ('cluster', (4, 3, 5, 2, 256, 1), dict(dropout=0.25, seed=9)),
    ('general', (5, 4, 6, 3, 64, 1), {}),
    ('general', (4, 5, 7, 3, 128, 2), dict(dropout=0.25, recurrent_dropout=0.2, seed=9)),
]


@pytest.mark.parametrize('path,shape,drop', IDENTITY_CASES)
def test_plans_without_rounding_are_the_oracle(path, shape, drop):
    B, T, F, O, H, L = shape
    params, x, y = make_problem(B, T, F, O, H, L, seed=3, init_scale=0.4)
    mean, var = _bn(L, H, 4)
    kw = dict(num_layers=L, training=True, step=2, row0=17, bn_mean=mean, bn_var=var, **drop)
    p = bo.Plan(path, bo.identity)
    preds, fc = bo.forward(p, params, x.astype(np.float64), **kw)
    ref, rfc = orc.forward(params, x.astype(np.float64), **kw)
    assert _close(preds, ref)
    _, _, dpred, _ = orc.loss_point_estimate(y.astype(np.float64), ref, target_idx=O - 1, target_lambda=0.5,
                                             rnn_lambda=0.7)
    for g, r in zip(bo.backward(p, dpred, fc), orc.backward(dpred, rfc, num_layers=L)):
        assert g.shape == r.shape and _close(g, r)


@pytest.mark.parametrize('shape,cell,drop', [
    ((5, 4, 6, 3, 64, 1), 'gru', {}),
    ((4, 5, 7, 3, 128, 2), 'gru', dict(dropout=0.25, recurrent_dropout=0.2, seed=9)),
])
def test_general_gru_forward_without_rounding_is_the_oracle(shape, cell, drop):
    B, T, F, O, H, L = shape
    params, x, _ = make_problem(B, T, F, O, H, L, seed=3, init_scale=0.5, rnn_cell=cell)
    mean, var = _bn(L, H, 4)
    kw = dict(num_layers=L, training=True, step=2, row0=17, bn_mean=mean, bn_var=var, rnn_cell=cell, **drop)
    preds, _ = bo.forward(bo.Plan('general', bo.identity), params, x.astype(np.float64), **kw)
    ref, _ = orc.forward(params, x.astype(np.float64), **kw)
    assert _close(preds, ref)


@pytest.mark.parametrize('shape,cell', [((5, 4, 6, 3, 64, 1), 'lstm'), ((4, 5, 7, 3, 128, 2), 'gru')])
def test_general_uq_forward_without_rounding_is_the_oracle(shape, cell):
    B, T, F, O, H, L = shape
    params, x = make_uq_problem(B, T, F, O, H, L, seed=13, cell=cell)
    mean, var = _bn(L, H, 4)
    kw = dict(num_layers=L, dropout=0.2, recurrent_dropout=0.1, seed=5, step=3, row0=40, bn_mean=mean, bn_var=var,
              rnn_cell=cell)
    pred, v, _ = bo.forward(bo.Plan('general', bo.identity), params, x.astype(np.float64), uq=True, **kw)
    rp, rv, _ = orc.forward_uq(params, x.astype(np.float64), **kw)
    assert _close(pred, rp) and _close(v, rv)


def _rel(a, b):
    return float(np.max(np.abs(a - b)) / np.max(np.abs(b)))


@pytest.mark.parametrize('path,shape,drop', IDENTITY_CASES)
def test_plans_with_rounding_round(path, shape, drop):
    """Rounding on: outputs and every gradient move away from the oracle by a bf16-sized amount (not zero, not more
    than the bf16 tolerance the GPU suites hold these paths to)."""
    B, T, F, O, H, L = shape
    params, x, y = make_problem(B, T, F, O, H, L, seed=3, init_scale=0.4)
    mean, var = _bn(L, H, 4)
    kw = dict(num_layers=L, training=True, step=2, row0=17, bn_mean=mean, bn_var=var, **drop)
    p = bo.Plan(path)
    preds, fc = bo.forward(p, params, x.astype(np.float64), **kw)
    ref, rfc = orc.forward(params, x.astype(np.float64), **kw)
    assert 1e-4 < _rel(preds, ref) < 3e-2
    _, _, dpred, _ = orc.loss_point_estimate(y.astype(np.float64), ref, target_idx=O - 1, target_lambda=0.5,
                                             rnn_lambda=0.7)
    grads, ref_grads = bo.backward(p, dpred, fc), orc.backward(dpred, rfc, num_layers=L)
    # Given the same dLoss/dpred, nothing rounds dbo (column sums of the fp32 dLoss/dpred on both paths) nor, on the
    # cluster path, dbeta (Wo times those sums, or the fp32 dLoss/dy of the Dropout head)
    exact = {len(grads) - 1} | ({4} if path == 'cluster' else set())
    for k, (g, r) in enumerate(zip(grads, ref_grads)):
        if k in exact:
            assert _close(g, r), k
        else:
            assert 1e-4 < _rel(g, r) < 3e-2, k


def test_gru_and_uq_plans_with_rounding_round():
    B, T, F, O, H, L = 4, 5, 7, 3, 128, 2
    params, x, _ = make_problem(B, T, F, O, H, L, seed=3, init_scale=0.5, rnn_cell='gru')
    preds, _ = bo.forward(bo.Plan('general'), params, x.astype(np.float64), num_layers=L, rnn_cell='gru')
    ref, _ = orc.forward(params, x.astype(np.float64), num_layers=L, rnn_cell='gru')
    assert 1e-4 < _rel(preds, ref) < 3e-2
    params, x = make_uq_problem(B, T, F, O, H, L, seed=13, cell='lstm')
    kw = dict(num_layers=L, dropout=0.2, recurrent_dropout=0.1, seed=5, step=3, row0=40)
    pred, v, _ = bo.forward(bo.Plan('general'), params, x.astype(np.float64), uq=True, **kw)
    rp, rv, _ = orc.forward_uq(params, x.astype(np.float64), **kw)
    assert 1e-4 < _rel(pred, rp) < 3e-2 and 1e-4 < _rel(v, rv) < 3e-2
