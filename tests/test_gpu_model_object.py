"""The model object of every trained model kind -- NativeForecaster over a ForecastChainEngine of S >= 1 stages -- against
the handle-level engines it is built on (ForecasterEngine, DenseEngine, or the S = 2 ForecastChainEngine): the Keras
return types, the same training steps with the same kernel launches, the same checkpoint bytes, and the one-rank
data-parallel step."""
import os

import numpy as np
import pandas as pd
import pytest
import torch

from util import rel_err

pytestmark = pytest.mark.gpu

B, T, F, O, TIDX, LR = 300, 8, 32, 16, 3, 0.6
# kind: CLI arguments.  bf16 point models on the cluster path (H = 256, L = 1) and on the general path (H = 128, L = 2,
# dropout); the uq model at bf16x3 is forward-only.
KINDS = {
    'point-fp32': ['--num_hidden', '64', '--num_layers', '2', '--dropout', '0.1', '--recurrent_dropout', '0.1'],
    'point-bf16-cluster': ['--precision', 'bf16', '--num_hidden', '256', '--num_layers', '1'],
    'point-bf16-general': ['--precision', 'bf16', '--num_hidden', '128', '--num_layers', '2', '--dropout', '0.2',
                           '--recurrent_dropout', '0.1'],
    'gru-fp32': ['--rnn_cell', 'gru', '--num_hidden', '64', '--num_layers', '2', '--dropout', '0.1'],
    'uq-fp32': ['--nn_type', 'RNNUqRangeEstimate', '--UQ=True', '--num_hidden', '64', '--num_layers', '1',
                '--dropout', '0.1'],
    'uq-bf16x3-forward': ['--nn_type', 'RNNUqRangeEstimate', '--UQ=True', '--precision', 'bf16x3', '--train=False',
                          '--num_hidden', '64', '--num_layers', '1', '--dropout', '0.1'],
    'point-s2-fp32': ['--forecast_steps', '2', '--forecast_steps_weights', '1.0-0.5', '--num_hidden', '64',
                      '--num_layers', '1', '--dropout', '0.1'],
    'uq-s2-fp32': ['--nn_type', 'RNNUqRangeEstimate', '--UQ=True', '--forecast_steps', '2', '--forecast_steps_weights',
                   '1.0-0.5', '--num_hidden', '64', '--num_layers', '1', '--dropout', '0.1'],
    'mlp-linear': ['--nn_type', 'MLPLinearPointEstimate', '--init_scale', '0.02'],
}
TRAINS = [k for k in KINDS if k != 'uq-bf16x3-forward']
# bf16 training is not bit-reproducible between two runs (the heads sum with shared-memory atomics): the two-run bound of
# test_gpu_ensemble.py on losses and weights, and HEAD_TOL of test_gpu_bf16_rounding.py on the gradients
TWO_RUN = dict(rtol=1e-6, atol=1e-9)
HEAD_TOL = 1e-5


def _model(kind):
    from lfm_quant_b200.scripts import base_config, configs
    from lfm_quant_b200.scripts.models.point_estimate.mlp_linear_point_estimate import NativeDenseForecaster
    from lfm_quant_b200.scripts.models.point_estimate.rnn_point_estimate import NativeForecaster
    configs.reset()
    cfg = base_config.get_configs(['--train=True', '--batch_size', str(B)] + KINDS[kind])
    if 'MLP' in cfg.nn_type:
        return cfg, NativeDenseForecaster(cfg, T, F, O, TIDX)
    return cfg, NativeForecaster(cfg, T, F, O, TIDX, uq=cfg.UQ)


def _handle(cfg, model):
    """The handle-level engine the model object runs on, built on its own, with the model's weights; and its stages."""
    from lfm_quant_b200.engine import DenseEngine, ForecastChainEngine, ForecasterEngine
    kw = dict(max_batch=cfg.batch_size, seq_len=T, n_inputs=F, n_outputs=O, target_idx=TIDX, precision=cfg.precision,
              optimizer=cfg.optimizer, target_lambda=cfg.target_lambda, max_grad_norm=cfg.max_grad_norm,
              sgd_momentum=cfg.sgd_momentum, forward_only=not cfg.train)
    if 'MLP' in cfg.nn_type:
        h = DenseEngine(huber_loss=bool(cfg.huber_loss), huber_delta=cfg.huber_delta, **kw)
    else:
        kw.update(num_hidden=cfg.num_hidden, num_layers=cfg.num_layers, train=bool(cfg.train), dropout=cfg.dropout,
                  recurrent_dropout=cfg.recurrent_dropout, rnn_lambda=cfg.rnn_lambda, max_norm=float(cfg.max_norm),
                  seed=cfg.seed, rnn_cell=cfg.rnn_cell, uq=bool(cfg.UQ))
        h = ForecasterEngine(**kw) if cfg.forecast_steps == 1 else \
            ForecastChainEngine(forecast_steps=cfg.forecast_steps, weights=cfg.forecast_steps_weights, **kw)
    stages = getattr(h, 'stages', [h])
    assert len(stages) == len(model.engine.stages)
    for e, m in zip(stages, model.engine.stages):
        e.set_flat(m.get_flat())
    return h, stages


def _data(cfg, n, seed=0):
    rng = np.random.RandomState(seed)
    mlp = 'MLP' in cfg.nn_type
    x = rng.normal(size=(n, T * F) if mlp else (n, T, F)).astype(np.float32)
    ys = [rng.normal(size=(n, O) if mlp else (n, T, O)).astype(np.float32) for _ in range(cfg.forecast_steps)]
    if not mlp and not cfg.UQ:
        for y in ys:
            y[0, :2, :] = 0.0          # zero-padded steps: loss mask 0
    to = lambda a: torch.from_numpy(a).cuda()
    return to(x), [to(y) for y in ys]


def _handle_forward(h, cfg, x, step, row0):
    out = h.forward(x, step=step, row0=row0)
    return list(out) if isinstance(out, (list, tuple)) else [out]


def _same(got, ref, exact, what):
    got, ref = np.asarray(got), np.asarray(ref)
    if exact:
        np.testing.assert_array_equal(got, ref, err_msg=what)
    else:
        np.testing.assert_allclose(got, ref, err_msg=what, **TWO_RUN)


@pytest.mark.parametrize('kind', list(KINDS))
def test_outputs_follow_the_keras_rule_and_the_handle_forward(kind):
    """model(inp) and model.predict(inp) return the output list unwrapped when it holds one output; predict_device always
    returns the list.  Each call advances the dropout step once, and predict over more rows than max_batch keys each
    chunk by its global row: the handle's forward with the same step and row0 computes the same values."""
    cfg, m = _model(kind)
    h, _ = _handle(cfg, m)
    x, _ = _data(cfg, 2 * B + 7)
    n_out = cfg.forecast_steps * (2 if cfg.UQ else 1)
    shape = (lambda n: (n, O)) if 'MLP' in cfg.nn_type else (lambda n: (n, T, O))
    c0 = m._calls
    out = m(x[:B])
    dev = m.predict_device(x)
    host = m.predict(x.cpu().numpy())
    assert m._calls == c0 + 3
    assert isinstance(dev, list) and len(dev) == n_out
    assert all(isinstance(t, torch.Tensor) and t.is_cuda and tuple(t.shape) == shape(len(x)) for t in dev)
    if n_out == 1:
        assert isinstance(out, torch.Tensor) and tuple(out.shape) == shape(B)
        assert isinstance(host, np.ndarray) and host.shape == shape(len(x))
        out, host = [out], [host]
    else:
        assert isinstance(out, list) and len(out) == n_out
        assert all(isinstance(t, torch.Tensor) and tuple(t.shape) == shape(B) for t in out)
        assert isinstance(host, list) and len(host) == n_out
        assert all(isinstance(a, np.ndarray) and a.shape == shape(len(x)) for a in host)
    exact = cfg.precision == 'fp32'
    for k, t in enumerate(_handle_forward(h, cfg, x[:B].contiguous(), c0 + 1, 0)):
        _same(out[k].cpu().numpy(), t.cpu().numpy(), exact, 'model(inp)[%d]' % k)
    for outs, step in ((dev, c0 + 2), (host, c0 + 3)):
        for s in range(0, len(x), B):
            for k, t in enumerate(_handle_forward(h, cfg, x[s:s + B].contiguous(), step, s)):
                got = outs[k][s:s + B]
                _same(got.cpu().numpy() if isinstance(got, torch.Tensor) else got, t.cpu().numpy(), exact,
                      'step %d rows %d: output %d' % (step, s, k))
    h.close()
    m.engine.close()


@pytest.mark.parametrize('kind', TRAINS)
def test_train_steps_equal_the_handle_engines(kind):
    """Three model.train_step calls equal the same three train_step calls of the handle-level engine: the returned
    {loss, mse} / {uq_loss_last_tar, mse}, every stage's gradient and loss tail, and the weights -- bit for bit at fp32
    and on the dense handle -- with the same number of kernel launches per step."""
    cfg, m = _model(kind)
    h, stages = _handle(cfg, m)
    x, ys = _data(cfg, B, seed=1)
    exact = cfg.precision == 'fp32'
    for it in range(3):
        torch.cuda.synchronize()
        n0 = h.launch_count
        got = m.train_step(x, ys, LR, it).cpu().numpy()
        n1 = h.launch_count
        ref = h.train_step(x, ys if cfg.forecast_steps > 1 else ys[0], it, LR).cpu().numpy()
        n2 = h.launch_count
        assert n1 - n0 == n2 - n1 > 0, (it, n1 - n0, n2 - n1)
        _same(got, ref, exact, 'step %d output' % it)
        for s, (a, b) in enumerate(zip(m.engine.stages, stages)):
            ga, gb = (e.grads[:e.n_trainable + 2].cpu().numpy() for e in (a, b))
            if exact:
                np.testing.assert_array_equal(ga, gb, err_msg='step %d stage %d gradient' % (it, s))
            else:
                assert rel_err(ga[:-2], gb[:-2]) <= HEAD_TOL, (it, s, rel_err(ga[:-2], gb[:-2]))
                np.testing.assert_allclose(ga[-2:], gb[-2:], rtol=HEAD_TOL)
            _same(a.params.cpu().numpy(), b.params.cpu().numpy(), exact, 'step %d stage %d weights' % (it, s))
    assert rel_err(m.get_weights()[0], _model(kind)[1].get_weights()[0]) > 0      # the steps moved the weights
    h.close()
    m.engine.close()


@pytest.mark.parametrize('kind', list(KINDS))
def test_checkpoint_round_trip_and_the_handle_level_bytes(kind, tmp_path):
    """save_weights writes the TF-format container byte for byte as it was written from the handle-level names: a
    handle's own names in keras_keys' sorted layer order for one stage, the chain's in construction order; the .npz holds
    the same arrays.  Both containers restore the weights.  set_weights takes the trainable arrays, optionally followed
    by the BatchNormalization statistics."""
    from lfm_quant_b200 import tf_checkpoint
    cfg, m = _model(kind)
    rng = np.random.RandomState(5)
    full = [(w + 0.01 * rng.normal(size=w.shape)).astype(np.float32) for w in m.get_weights()]
    m.set_weights(full)
    for a, b in zip(m.get_weights(), full):
        np.testing.assert_array_equal(a, b)
    trainable = [spec[4] for spec in m.engine.specs]          # get_weights' order: every stage's specs in turn
    m.set_weights([w + 1 for w, tr in zip(full, trainable) if tr])
    for a, b, tr in zip(m.get_weights(), full, trainable):
        np.testing.assert_array_equal(a, b + 1 if tr else b)
    prefix = str(tmp_path / 'model' / 'chkpt')
    m.save_weights(prefix)
    h, stages = _handle(cfg, m)
    if cfg.forecast_steps == 1:
        flat = h.get_flat()
        arrs = {n: flat[off:off + int(np.prod(s))].reshape(s) for n, s, off, _ in h.specs}
        tf_checkpoint.write_keras_checkpoint(str(tmp_path / 'chkpt'), arrs)
    else:
        arrs = h.named_arrays()
        tf_checkpoint.write_keras_checkpoint(str(tmp_path / 'chkpt'), arrs, construction_order=True)
    for suffix in ('.index', '.data-00000-of-00001'):
        with open(prefix + suffix, 'rb') as a, open(str(tmp_path / 'chkpt') + suffix, 'rb') as b:
            assert a.read() == b.read(), suffix
    npz = np.load(prefix + '.lfmq.npz')
    assert list(npz.files) == list(arrs)
    for n in arrs:
        np.testing.assert_array_equal(npz[n], arrs[n])
    want = m.get_weights()
    for drop_npz in (False, True):
        if drop_npz:
            os.remove(prefix + '.lfmq.npz')       # the TF-format container alone restores the same weights
        _, m2 = _model(kind)
        m2.load_weights(prefix)
        for a, b in zip(m2.get_weights(), want):
            np.testing.assert_array_equal(a, b)
        m2.engine.close()
    h.close()
    m.engine.close()


@pytest.mark.parametrize('kind', TRAINS)
def test_one_rank_gloo_train_step_dp_equals_train_step(kind, tmp_path):
    """model.train_step_dp in a one-rank gloo group, with the denominators the driver all-reduces, equals
    model.train_step."""
    import torch.distributed as dist
    from lfm_quant_b200 import dp
    cfg, a = _model(kind)
    _, b = _model(kind)
    for ea, eb in zip(a.engine.stages, b.engine.stages):
        assert torch.equal(ea.params, eb.params)
    x, ys = _data(cfg, B, seed=2)
    exact = cfg.precision == 'fp32'
    dist.init_process_group('gloo', init_method='file://' + str(tmp_path / 'pg'), rank=0, world_size=1)
    try:
        for it in range(2):
            denom = dp.global_denominators(a.engine.loss_counts(ys), dist)
            got = a.train_step_dp(x, ys, it, LR, 0, denom).cpu().numpy()
            ref = b.train_step(x, ys, LR, it).cpu().numpy()
            if exact:
                assert got == pytest.approx(ref, rel=1e-6), (it, got, ref)
            else:
                np.testing.assert_allclose(got, ref, rtol=HEAD_TOL)
            for s, (ea, eb) in enumerate(zip(a.engine.stages, b.engine.stages)):
                wa, wb = ea.params.cpu().numpy(), eb.params.cpu().numpy()
                if exact:
                    np.testing.assert_array_equal(wa, wb, err_msg='step %d stage %d' % (it, s))
                else:
                    assert rel_err(wa, wb) <= HEAD_TOL, (it, s, rel_err(wa, wb))
    finally:
        dist.destroy_process_group()
        a.engine.close()
        b.engine.close()


def test_cli_trains_and_predicts_the_multi_step_point_model(tmp_path):
    """RNNPointEstimate with --forecast_steps 2 through the CLI: training, then prediction writes every step's columns."""
    from lfm_quant_b200.scripts import configs
    from lfm_quant_b200.scripts import lfm_quant as cli
    from lfm_quant_b200.scripts.synthetic import write_open_dataset, write_system_test_conf
    os.environ.setdefault('LFM_QUANT_ROOT', str(tmp_path))
    write_open_dataset(str(tmp_path / 'datasets' / 'open-dataset.dat'), n_keys=30, n_months=420, seed=9)
    conf = str(tmp_path / 'config' / 'system-test.conf')
    write_system_test_conf(conf, str(tmp_path / 'datasets'), str(tmp_path / 'experiments'))
    extra = ['--forecast_steps', '2', '--forecast_steps_weights', '1.0-0.5', '--model_dir', 'point-s2']
    configs.reset()
    try:
        assert np.isfinite(cli.main(['--config=' + conf, '--train=True'] + extra))
        configs.reset()
        df = cli.main(['--config=' + conf, '--train=False'] + extra)
    finally:
        configs.reset()
    out = pd.read_csv(tmp_path / 'experiments' / 'point-s2' / 'pred' / 'preds.dat', sep=' ', dtype={'gvkey': str})
    assert len(out) == len(df) > 100
    for s in (1, 2):
        assert np.isfinite(out['norm_preds_%d' % s]).all() and np.isfinite(out['preds_%d' % s]).all()
        assert (out['norm_variance_%d' % s] == 0).all()
    assert not np.array_equal(out['norm_preds_1'].values, out['norm_preds_2'].values)
