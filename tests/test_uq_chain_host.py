"""RNNUqRangeEstimate with forecast_steps > 1 (reference models/uq_range_estimate/rnn_uq_range_estimate.py:114-157,
model_utils/losses.py:137-178) on the CPU: the oracle's multi-step uq graph against fp64 finite differences, its
forecast_steps = 1 case against forward_uq / backward_uq, the checkpoint naming of the graph and the assertions of
Losses.weight_adjusted_uq_loss."""
import types

import numpy as np
import pytest

import lfm_oracle as orc
import uq_chain_oracle as uco

KW = dict(target_idx=1, target_lambda=0.5, rnn_lambda=0.7)


def _problem(B, T, F, O, H, L, S, seed, cell):
    rng = np.random.RandomState(seed)
    P = uco.init_params(L, F, O, H, S, init_scale=0.5, seed=seed + 1, dtype=np.float64, rnn_cell=cell)
    P = [p + rng.normal(size=p.shape) * 0.1 for p in P]
    x = rng.normal(size=(B, T, F))
    ys = [rng.normal(size=(B, T, O)) for _ in range(S)]
    return P, x, ys


@pytest.mark.parametrize('cell,L,S', [('lstm', 1, 3), ('gru', 2, 2)])
def test_uq_chain_gradients_match_finite_differences(cell, L, S):
    """Every trainable tensor, with dropout and recurrent dropout on and the feedback of stage s's input gradient into
    the earlier target predictions."""
    B, T, F, O, H = 3, 4, 5, 2, 4
    P, x, ys = _problem(B, T, F, O, H, L, S, seed=7, cell=cell)
    w = [1.0, 0.5, 0.25][:S]
    fkw = dict(num_layers=L, forecast_steps=S, dropout=0.3, recurrent_dropout=0.25, seed=13, step=4, row0=9,
               rnn_cell=cell)

    def loss_of(params):
        preds, vars_, _ = uco.forward(params, x, **fkw)
        return uco.loss(ys, preds, vars_, w, **KW)[0]

    preds, vars_, fc = uco.forward(P, x, **fkw)
    _, _, _, dpreds, dvars = uco.loss(ys, preds, vars_, w, **KW)
    grads = uco.backward(dpreds, dvars, fc, rnn_cell=cell)
    names = uco.param_names(L, S, cell)
    assert len(grads) == len(P) == len(names)
    rng = np.random.RandomState(1)
    eps = 1e-6
    for name, p, g in zip(names, P, grads):
        assert g.shape == p.shape, name
        for idx in {tuple(rng.randint(0, n) for n in p.shape) for _ in range(4)}:
            old = p[idx]
            p[idx] = old + eps
            up = loss_of(P)
            p[idx] = old - eps
            dn = loss_of(P)
            p[idx] = old
            fd = (up - dn) / (2 * eps)
            assert g[idx] == pytest.approx(fd, rel=1e-5, abs=1e-8), (name, idx)
    # the later stages' losses reach the trunk through the fed-back target predictions
    g1 = orc.backward_uq(dpreds[0], dvars[0], fc[0][0], num_layers=L, rnn_cell=cell)
    assert not np.allclose(grads[0], g1[0])


def test_single_step_uq_chain_is_forward_uq_and_backward_uq():
    B, T, F, O, H, L = 4, 5, 6, 3, 8, 2
    P, x, ys = _problem(B, T, F, O, H, L, 1, seed=3, cell='lstm')
    fkw = dict(num_layers=L, dropout=0.2, recurrent_dropout=0.1, seed=5, step=2, row0=30)
    preds, vars_, fc = uco.forward(P, x, forecast_steps=1, **fkw)
    p, v, fc1 = orc.forward_uq(P, x, **fkw)
    np.testing.assert_array_equal(preds[0], p)
    np.testing.assert_array_equal(vars_[0], v)
    loss, uq0, mse, dpreds, dvars = uco.loss(ys, preds, vars_, [1.0], **KW)
    ref = orc.loss_uq_estimate(ys[0], p, v, **KW)
    assert (loss, uq0, mse) == (ref[0], ref[1], ref[2])
    for a, b in zip(uco.backward(dpreds, dvars, fc), orc.backward_uq(ref[3], ref[4], fc1, num_layers=L)):
        np.testing.assert_array_equal(a, b)
    assert uco.param_names(L, 1) == orc.param_names(L, uq=True)


def test_uq_chain_checkpoint_names_round_trip(tmp_path):
    """Construction order of the multi-step uq graph (rnn_uq_range_estimate.py:76-157): trunk, OUTPUT_TARGET_1,
    OUTPUT_VARIANCE_1, lstm_2, its BatchNormalization, OUTPUT_TARGET_2, OUTPUT_VARIANCE_2."""
    from lfm_quant_b200 import tf_checkpoint as tfc
    tr = uco.param_names(1, 2)
    assert tr[5:9] == ['OUTPUT_TARGET_1/kernel', 'OUTPUT_TARGET_1/bias', 'OUTPUT_VARIANCE_1/kernel',
                       'OUTPUT_VARIANCE_1/bias']
    assert tr[9:] == ['lstm_2/kernel', 'lstm_2/recurrent_kernel', 'lstm_2/bias', 'batch_normalization_1/gamma',
                      'batch_normalization_1/beta', 'OUTPUT_TARGET_2/kernel', 'OUTPUT_TARGET_2/bias',
                      'OUTPUT_VARIANCE_2/kernel', 'OUTPUT_VARIANCE_2/bias']
    # the order ForecastChainEngine.specs lists them in: stage by stage, each stage's moving statistics last
    names = (tr[:9] + ['batch_normalization/moving_mean', 'batch_normalization/moving_variance'] + tr[9:] +
             ['batch_normalization_1/moving_mean', 'batch_normalization_1/moving_variance'])
    keys = tfc.keras_keys(names, construction_order=True)
    expect = {'lstm_1/kernel': 0, 'batch_normalization/moving_mean': 1, 'OUTPUT_TARGET_1/bias': 2,
              'OUTPUT_VARIANCE_1/kernel': 3, 'lstm_2/recurrent_kernel': 4, 'batch_normalization_1/gamma': 5,
              'OUTPUT_TARGET_2/kernel': 6, 'OUTPUT_VARIANCE_2/bias': 7}
    for n, k in expect.items():
        assert keys[n].startswith('layer_with_weights-%d/' % k), (n, keys[n])
    rng = np.random.RandomState(0)
    arrs = {n: rng.normal(size=(3, 4) if n.endswith('kernel') else (4,)).astype(np.float32) for n in names}
    prefix = str(tmp_path / 'chkpt')
    tfc.write_keras_checkpoint(prefix, arrs, construction_order=True)
    back = tfc.read_keras_checkpoint(prefix, names, {n: a.shape for n, a in arrs.items()}, construction_order=True)
    for n in names:
        np.testing.assert_array_equal(back[n], arrs[n])


def test_weight_adjusted_uq_loss_asserts_as_the_reference():
    """losses.py:148-166: UQ must be set, forecast_steps positive, the arguments lists, one weight per step."""
    from lfm_quant_b200.scripts.model_utils.losses import Losses
    a = [np.zeros((2, 3, 4), np.float32)] * 2

    def cfg(**kw):
        base = dict(UQ=True, forecast_steps=2, nn_type='RNNUqRangeEstimate', forecast_steps_weights=[1.0, 0.5])
        base.update(kw)
        return types.SimpleNamespace(**base)

    with pytest.raises(AssertionError):
        Losses(cfg(UQ=False), 0).weight_adjusted_uq_loss(a, a, a)
    with pytest.raises(AssertionError):
        Losses(cfg(forecast_steps=0), 0).weight_adjusted_uq_loss(a, a, a)
    for bad in range(3):
        args = [a, a, a]
        args[bad] = a[0]
        with pytest.raises(AssertionError):
            Losses(cfg(), 0).weight_adjusted_uq_loss(*args)
    with pytest.raises(AssertionError):
        Losses(cfg(forecast_steps_weights=[1.0]), 0).weight_adjusted_uq_loss(a, a, a)
    with pytest.raises(AssertionError):
        Losses(cfg(forecast_steps=3, forecast_steps_weights=[1.0, 0.5, 0.2]), 0).weight_adjusted_uq_loss(a, a, a)
