"""forecast_steps > 1 on the GPU (SURVEY 8f-1; reference scripts/models/point_estimate/rnn_point_estimate.py:109-150,
models/model_base_class.py:18-51, model_utils/losses.py:19-53) through lfmq_chain_* against the oracle's chain."""
import sys

import numpy as np
import pytest
import torch

import lfm_oracle as orc
from util import rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-4


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()


def _problem(B, T, F, O, H, L, S, seed, cell='lstm'):
    rng = np.random.RandomState(seed)
    P = orc.init_forecast_params(L, F, O, H, S, init_scale=0.5, seed=seed + 1, dtype=np.float64, rnn_cell=cell)
    P = [(p + rng.normal(size=p.shape) * 0.05).astype(np.float32).astype(np.float64) for p in P]
    x = rng.normal(size=(B, T, F)).astype(np.float32)
    ys = [rng.normal(size=(B, T, O)).astype(np.float32) for _ in range(S)]
    for y in ys:
        y[0, :2, :] = 0.0                     # zero-padded steps: loss mask 0 (losses.py:72)
    return P, x, ys


def _engine(B, T, F, O, H, L, S, weights, cell='lstm', **kw):
    from lfm_quant_b200.engine import ForecastChainEngine
    return ForecastChainEngine(forecast_steps=S, weights=weights, max_batch=B, seq_len=T, n_inputs=F, n_outputs=O,
                               num_hidden=H, num_layers=L, rnn_cell=cell, **kw)


@pytest.mark.parametrize('shape,cell', [((6, 7, 9, 4, 8, 2, 3), 'lstm'), ((33, 12, 16, 8, 32, 1, 2), 'lstm'),
                                        ((5, 6, 7, 3, 8, 1, 3), 'gru')])
def test_chain_forward_loss_and_gradients_match_oracle(shape, cell):
    B, T, F, O, H, L, S = shape
    P, x, ys = _problem(B, T, F, O, H, L, S, seed=11, cell=cell)
    w = [1.0, 0.6, 0.3][:S]
    eng = _engine(B, T, F, O, H, L, S, w, cell=cell, target_idx=1, train=True)
    eng.set_weights(P)
    assert [n for _, n, _, _, tr in eng.specs if tr] == orc.forecast_param_names(L, S, cell)
    preds = eng.forward(_cuda(x))
    rp, fc = orc.forward_forecast(P, x.astype(np.float64), num_layers=L, forecast_steps=S, rnn_cell=cell)
    for s in range(S):
        assert rel_err(preds[s].cpu().numpy(), rp[s]) < TOL, s
    kw = dict(target_idx=1, target_lambda=0.5, rnn_lambda=0.7)
    loss, mse, dpreds = orc.loss_forecast([y.astype(np.float64) for y in ys], rp, w, **kw)
    out = eng.loss(preds, [_cuda(y) for y in ys]).cpu().numpy()
    assert out[0] == pytest.approx(loss, rel=TOL) and out[1] == pytest.approx(mse, rel=TOL)
    out = eng.backward(_cuda(x), [_cuda(y) for y in ys]).cpu().numpy()
    assert out[0] == pytest.approx(loss, rel=TOL) and out[1] == pytest.approx(mse, rel=TOL)
    ref = orc.backward_forecast(dpreds, fc, rnn_cell=cell)
    names = orc.forecast_param_names(L, S, cell)
    assert len(ref) == len(names)
    for name, g, r in zip(names, eng.grads_list(), ref):
        assert g.shape == r.shape, name
        assert rel_err(g, r) < 2 * TOL, name
    # the chain really feeds predictions back: the trunk's gradient differs from a forecast_steps = 1 backward
    g1 = orc.backward(dpreds[0] * 0 + orc.loss_point_estimate(ys[0].astype(np.float64), rp[0], **kw)[2] * w[0],
                      fc[0][0], num_layers=L, rnn_cell=cell)
    assert rel_err(ref[0], g1[0]) > 1e-3
    eng.close()


def test_chain_dropout_streams_continue_the_layer_numbering():
    B, T, F, O, H, L, S = 9, 6, 8, 3, 16, 2, 3
    P, x, ys = _problem(B, T, F, O, H, L, S, seed=3)
    eng = _engine(B, T, F, O, H, L, S, [1.0, 1.0, 1.0], target_idx=0, train=True, dropout=0.3, recurrent_dropout=0.2,
                  seed=77)
    eng.set_weights(P)
    preds = eng.forward(_cuda(x), step=5, row0=40)
    rp, _ = orc.forward_forecast(P, x.astype(np.float64), num_layers=L, forecast_steps=S, dropout=0.3,
                                 recurrent_dropout=0.2, training=True, seed=77, step=5, row0=40)
    for s in range(S):
        assert rel_err(preds[s].cpu().numpy(), rp[s]) < TOL, s
    eng.close()


def test_chain_train_steps_match_oracle():
    """Joint clip_by_global_norm over all stages' variables (train.py:196), Adadelta, MaxNorm on every recurrent kernel."""
    B, T, F, O, H, L, S = 12, 6, 8, 4, 16, 1, 2
    P, x, ys = _problem(B, T, F, O, H, L, S, seed=21)
    w = [1.0, 0.5]
    eng = _engine(B, T, F, O, H, L, S, w, target_idx=1, train=True, optimizer='Adadelta', max_grad_norm=0.05,
                  max_norm=0.8)
    eng.set_weights(P)
    p = [q.copy() for q in P]
    slots = orc.zero_slots('Adadelta', p)
    kw = dict(target_idx=1, target_lambda=0.5, rnn_lambda=0.7)
    kernel_ids = [5 * l for l in range(L)] + [5 * L + 2 + 7 * (s - 1) for s in range(1, S)]
    for it in range(3):
        out = eng.train_step(_cuda(x), [_cuda(y) for y in ys], it, 0.6).cpu().numpy()
        rp, fc = orc.forward_forecast(p, x.astype(np.float64), num_layers=L, forecast_steps=S)
        loss, mse, dpreds = orc.loss_forecast([y.astype(np.float64) for y in ys], rp, w, **kw)
        grads = orc.backward_forecast(dpreds, fc)
        grads, gn = orc.clip_by_global_norm(grads, 0.05)
        p = orc.optimizer_update('Adadelta', p, grads, slots, 0.6, it)
        for k in kernel_ids:
            p[k] = orc.max_norm_constraint(p[k], 0.8)
        assert out[0] == pytest.approx(loss, rel=TOL) and out[1] == pytest.approx(mse, rel=TOL), it
        for e in eng.stages:
            assert float(e.grads[e.n_trainable + 2]) == pytest.approx(gn, rel=TOL)
    for name, wgt, r in zip(orc.forecast_param_names(L, S), eng.get_weights(), p):
        assert rel_err(wgt, r) < 5 * TOL, name
    eng.close()


def _cfg(train, precision='fp32'):
    from lfm_quant_b200.scripts import base_config
    return base_config.get_configs(['--train=%s' % train, '--forecast_steps', '2', '--forecast_steps_weights', '1.0-0.5',
                                    '--num_hidden', '64', '--num_layers', '1', '--batch_size', '16', '--precision',
                                    precision, '--nn_type', 'RNNPointEstimate'])


def test_native_forecaster_chain_predict_checkpoint_and_refusals(tmp_path):
    """The two-step NativeForecaster (a ForecastChainEngine of two stages) through the reference's model interface: list
    outputs, save/load round trip (native and TF-format container), a bf16 forward-only graph within bf16 tolerance of
    the fp32 one, training graphs refused off the fp32 kernels; Losses.weight_adjusted_mse over the lists."""
    import os
    from lfm_quant_b200.scripts.models.point_estimate.rnn_point_estimate import NativeForecaster
    from lfm_quant_b200.scripts.model_utils.losses import Losses
    T, F, O = 5, 12, 6
    cfg = _cfg(True)
    assert cfg.forecast_steps_weights == [1.0, 0.5]
    m = NativeForecaster(cfg, T, F, O, 0)
    x = np.random.RandomState(0).normal(size=(16, T, F)).astype(np.float32)
    out = m.predict(x)
    assert isinstance(out, list) and len(out) == 2 and out[0].shape == (16, T, O)
    ys = [np.random.RandomState(s).normal(size=(16, T, O)).astype(np.float32) for s in (1, 2)]
    loss, mse = Losses(cfg, 0, engine=m.engine).weight_adjusted_mse(ys, out)
    l0 = orc.loss_point_estimate(ys[0].astype(np.float64), out[0].astype(np.float64), target_idx=0,
                                 target_lambda=cfg.target_lambda, rnn_lambda=cfg.rnn_lambda)
    l1 = orc.loss_point_estimate(ys[1].astype(np.float64), out[1].astype(np.float64), target_idx=0,
                                 target_lambda=cfg.target_lambda, rnn_lambda=cfg.rnn_lambda)
    assert loss.numpy() == pytest.approx(l0[0] + 0.5 * l1[0], rel=TOL)
    assert mse.numpy() == pytest.approx(l0[1] + 0.5 * l1[1], rel=TOL)
    r = m.train_step(x, ys, 0.6, 0).cpu().numpy()
    assert np.isfinite(r).all()
    prefix = str(tmp_path / 'chkpt')
    m.save_weights(prefix)
    m2 = NativeForecaster(_cfg(False), T, F, O, 0)
    m2.load_weights(prefix)
    a = m2.predict(x)
    os.remove(prefix + '.lfmq.npz')          # the TF-format container alone restores the same weights
    m3 = NativeForecaster(_cfg(False), T, F, O, 0)
    m3.load_weights(prefix)
    b = m3.predict(x)
    for s in range(2):
        np.testing.assert_array_equal(a[s], b[s])
    m4 = NativeForecaster(_cfg(False, 'bf16'), T, F, O, 0)
    m4.load_weights(prefix)
    c = m4.predict(x)
    for s in range(2):
        assert rel_err(c[s], a[s]) < 5e-2, s
    with pytest.raises(NotImplementedError):
        NativeForecaster(_cfg(True, 'bf16'), T, F, O, 0)
