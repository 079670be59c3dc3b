"""RNNUqRangeEstimate with forecast_steps > 1 on the GPU (reference models/uq_range_estimate/rnn_uq_range_estimate.py:
114-157, model_utils/losses.py:137-178, train.py:201-225,338-418, predict.py:135-146) through lfmq_chain_forward_uq /
lfmq_chain_loss_uq / lfmq_chain_backward / lfmq_chain_apply against the oracle's multi-step uq graph."""
import os

import numpy as np
import pandas as pd
import pytest
import torch

import lfm_oracle as orc
import uq_chain_oracle as uco
from util import rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-4
KW = dict(target_idx=1, target_lambda=0.5, rnn_lambda=0.7)
DROP = dict(dropout=0.2, recurrent_dropout=0.15, seed=31)


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()


def _problem(B, T, F, O, H, L, S, seed, cell='lstm'):
    rng = np.random.RandomState(seed)
    P = uco.init_params(L, F, O, H, S, init_scale=0.5, seed=seed + 1, dtype=np.float64, rnn_cell=cell)
    P = [(p + rng.normal(size=p.shape) * 0.05).astype(np.float32).astype(np.float64) for p in P]
    x = rng.normal(size=(B, T, F)).astype(np.float32)
    ys = [rng.normal(size=(B, T, O)).astype(np.float32) for _ in range(S)]
    return P, x, ys


def _engine(B, T, F, O, H, L, S, weights, cell='lstm', **kw):
    from lfm_quant_b200.engine import ForecastChainEngine
    return ForecastChainEngine(forecast_steps=S, weights=weights, max_batch=B, seq_len=T, n_inputs=F, n_outputs=O,
                               num_hidden=H, num_layers=L, rnn_cell=cell, uq=True, **kw)


def _split(out):
    out = [o.cpu().numpy() for o in out]
    return out[0::2], out[1::2]


@pytest.mark.parametrize('shape,cell', [((9, 6, 8, 4, 16, 2, 2), 'lstm'), ((7, 5, 7, 3, 8, 1, 3), 'gru'),
                                        ((33, 8, 12, 6, 32, 1, 3), 'lstm')])
def test_uq_chain_forward_loss_and_gradients_match_oracle(shape, cell):
    B, T, F, O, H, L, S = shape
    P, x, ys = _problem(B, T, F, O, H, L, S, seed=5, cell=cell)
    w = [1.0, 0.5, 0.25][:S]
    eng = _engine(B, T, F, O, H, L, S, w, cell=cell, train=True, **KW, **DROP)
    eng.set_weights(P)
    assert [n for _, n, _, _, tr in eng.specs if tr] == uco.param_names(L, S, cell)
    fkw = dict(num_layers=L, forecast_steps=S, rnn_cell=cell, step=3, row0=17, **DROP)
    rp, rv, fc = uco.forward(P, x.astype(np.float64), **fkw)
    out = eng.forward(_cuda(x), step=3, row0=17)
    assert len(out) == 2 * S
    gp, gv = _split(out)
    for s in range(S):
        assert rel_err(gp[s], rp[s]) < TOL and rel_err(gv[s], rv[s]) < TOL, s
    yd = [_cuda(y) for y in ys]
    loss, uq0, mse, dpreds, dvars = uco.loss([y.astype(np.float64) for y in ys], rp, rv, w, **KW)
    got = eng.loss_uq(out[0::2], out[1::2], yd).cpu().numpy()
    assert got == pytest.approx([loss, uq0, mse], rel=TOL)
    got = eng.backward(_cuda(x), yd, step=3, row0=17).cpu().numpy()
    assert got == pytest.approx([loss, uq0, mse], rel=TOL)
    ref = uco.backward(dpreds, dvars, fc, rnn_cell=cell)
    for name, g, r in zip(uco.param_names(L, S, cell), eng.grads_list(), ref):
        assert g.shape == r.shape, name
        assert rel_err(g, r) < TOL, name
    eng.close()


def test_later_stage_called_on_its_own_keeps_its_dropout_streams():
    """Stage 1's engine alone, on the window the chain built for it, draws the masks it drew inside the chain: the
    single-handle entry points leave the Philox stream numbering of the chain in place."""
    B, T, F, O, H, L, S = 9, 6, 8, 4, 16, 2, 2
    P, x, _ = _problem(B, T, F, O, H, L, S, seed=7)
    eng = _engine(B, T, F, O, H, L, S, [1.0, 0.5], train=True, **KW, **DROP)
    eng.set_weights(P)
    out = [o.cpu().numpy() for o in eng.forward(_cuda(x), step=3, row0=17)]
    window = eng._work[:B * T * F].view(B, T, F).clone()
    p1, v1 = eng.stages[1].forward(window, step=3, row0=17)
    assert np.array_equal(p1.cpu().numpy(), out[2]) and np.array_equal(v1.cpu().numpy(), out[3])
    eng.close()


@pytest.mark.parametrize('optimizer', ['Adadelta', 'Adam'])
def test_uq_chain_train_steps_match_oracle(optimizer):
    """Joint clip_by_global_norm over every stage (train.py:214-216), the optimizer, MaxNorm on every recurrent kernel."""
    B, T, F, O, H, L, S = 12, 6, 8, 4, 16, 1, 2
    P, x, ys = _problem(B, T, F, O, H, L, S, seed=21)
    w = [1.0, 0.5]
    eng = _engine(B, T, F, O, H, L, S, w, train=True, optimizer=optimizer, max_grad_norm=0.5, max_norm=0.8, **KW,
                  **DROP)
    eng.set_weights(P)
    p = [q.copy() for q in P]
    slots = orc.zero_slots(optimizer, p)
    cfg = dict(num_layers=L, forecast_steps=S, forecast_steps_weights=w, optimizer=optimizer, max_grad_norm=0.5,
               max_norm=0.8, **KW, **DROP)
    for it in range(3):
        out = eng.train_step(_cuda(x), [_cuda(y) for y in ys], it, 0.05).cpu().numpy()
        p, mse, loss, raw, gn, uq0 = uco.train_step(p, slots, x.astype(np.float64), [y.astype(np.float64) for y in ys],
                                                        it, cfg, lr=0.05)
        assert out == pytest.approx([uq0, mse], rel=TOL), it
        for e in eng.stages:
            assert float(e.grads[e.n_trainable + 2]) == pytest.approx(gn, rel=TOL)
    for name, wgt, r in zip(uco.param_names(L, S), eng.get_weights(), p):
        assert np.max(np.abs(wgt - r)) < 5e-4, name
    eng.close()


def test_uq_chain_padded_step_gives_nan_loss():
    B, T, F, O, H, L, S = 6, 5, 6, 3, 8, 1, 2
    P, x, ys = _problem(B, T, F, O, H, L, S, seed=2)
    ys[1][0, :2, :] = 0.0
    eng = _engine(B, T, F, O, H, L, S, [1.0, 0.5], train=True, **KW)
    eng.set_weights(P)
    out = eng.backward(_cuda(x), [_cuda(y) for y in ys]).cpu().numpy()
    assert np.isnan(out[0])
    eng.close()


@pytest.mark.parametrize('cell', ['lstm', 'gru'])
def test_forward_only_uq_chain_on_tensor_cores_matches_oracle_and_fp32(cell):
    """bf16 within 3e-2, bf16x3 within 1e-4 of the oracle at the same (step, row0); bf16x3 draws the fp32 chain's masks."""
    B, T, F, O, H, L, S = 40, 8, 12, 6, 64, 2, 3
    P, x, _ = _problem(B, T, F, O, H, L, S, seed=9, cell=cell)
    w = [1.0, 0.5, 0.25]
    rp, rv, _ = uco.forward(P, x.astype(np.float64), num_layers=L, forecast_steps=S, rnn_cell=cell, step=4,
                                        row0=300, **DROP)
    res = {}
    for prec, tol in (('fp32', TOL), ('bf16x3', TOL), ('bf16', 3e-2)):
        eng = _engine(B, T, F, O, H, L, S, w, cell=cell, precision=prec, train=False, forward_only=True, **KW,
                      **DROP)
        eng.set_weights(P)
        gp, gv = _split(eng.forward(_cuda(x), step=4, row0=300))
        for s in range(S):
            assert rel_err(gp[s], rp[s]) < tol and rel_err(gv[s], rv[s]) < tol, (prec, s)
        res[prec] = gp + gv
        eng.close()
    for a, b in zip(res['bf16x3'], res['fp32']):
        assert rel_err(a, b) < TOL


@pytest.mark.parametrize('prec', ['bf16', 'bf16x3'])
def test_tensor_core_uq_chain_rows_are_invariant(prec):
    """A permuted batch (dropout rate 0: no row-keyed masks) and a slice passed with its global row0 (MC dropout on)
    reproduce the full batch's rows bit for bit."""
    T, F, O, H, L, S = 6, 8, 4, 64, 1, 2
    Bmax = 4096
    P, x, _ = _problem(Bmax, T, F, O, H, L, S, seed=13)
    xd_all = _cuda(x)
    plain = _engine(Bmax, T, F, O, H, L, S, [1.0, 0.5], precision=prec, train=False, forward_only=True, **KW)
    mc = _engine(Bmax, T, F, O, H, L, S, [1.0, 0.5], precision=prec, train=False, forward_only=True, **KW, **DROP)
    for e in (plain, mc):
        e.set_weights(P)
    R = 1000
    for B in (1, 1921, 4096):
        xd = xd_all[:B]
        perm = np.roll(np.arange(B)[::-1], 65).copy()
        full = [o.cpu().numpy() for o in plain.forward(xd, step=2, row0=R)]
        got = [o.cpu().numpy() for o in plain.forward(xd[torch.from_numpy(perm).cuda()].contiguous(), step=2, row0=R)]
        for g, f in zip(got, full):
            assert np.isfinite(f).all() and np.array_equal(g, f[perm]), (B, 'permutation')
        full = [o.cpu().numpy() for o in mc.forward(xd, step=2, row0=R)]
        for a, b in {(0, B), (B // 3, B), (max(0, B - 129), B - 1 if B > 1 else B)}:
            got = [o.cpu().numpy() for o in mc.forward(xd[a:b].contiguous(), step=2, row0=R + a)]
            for g, f in zip(got, full):
                assert np.array_equal(g, f[a:b]), (B, (a, b))
    plain.close()
    mc.close()


def _cfg(train, precision='fp32'):
    from lfm_quant_b200.scripts import base_config
    return base_config.get_configs(['--train=%s' % train, '--forecast_steps', '2', '--forecast_steps_weights', '1.0-0.5',
                                    '--num_hidden', '64', '--num_layers', '1', '--batch_size', '16', '--precision',
                                    precision, '--nn_type', 'RNNUqRangeEstimate', '--UQ=True', '--dropout', '0.1'])


def test_native_forecaster_uq_chain_and_refusals():
    """The two-step uq NativeForecaster: summary, the interleaved output list, Losses.weight_adjusted_uq_loss over the
    lists, a train step, and a bf16 training chain refused."""
    from lfm_quant_b200.scripts.models.point_estimate.rnn_point_estimate import NativeForecaster
    from lfm_quant_b200.scripts.model_utils.losses import Losses
    T, F, O = 5, 12, 6
    cfg = _cfg(True)
    m = NativeForecaster(cfg, T, F, O, 0, uq=True)
    assert 'RNNUqRangeEstimate' in m.summary() and 'OUTPUT_VARIANCE_2/kernel' in m.summary()
    x = np.random.RandomState(0).normal(size=(16, T, F)).astype(np.float32)
    out = m.predict(x)
    assert isinstance(out, list) and len(out) == 4 and all(o.shape == (16, T, O) for o in out)
    assert (out[1] > 0).all() and (out[3] > 0).all()
    ys = [np.random.RandomState(s).normal(size=(16, T, O)).astype(np.float32) for s in (1, 2)]
    uq, last, mse = Losses(cfg, 0, engine=m.engine).weight_adjusted_uq_loss(ys, out[0::2], out[1::2])
    ref = uco.loss([y.astype(np.float64) for y in ys], [o.astype(np.float64) for o in out[0::2]],
                               [o.astype(np.float64) for o in out[1::2]], [1.0, 0.5], target_idx=0,
                               target_lambda=cfg.target_lambda, rnn_lambda=cfg.rnn_lambda)
    assert [uq.numpy(), last.numpy(), mse.numpy()] == pytest.approx(list(ref[:3]), rel=TOL)
    r = m.train_step(x, ys, 0.6, 0).cpu().numpy()
    assert r.shape == (2,) and np.isfinite(r).all()
    with pytest.raises(NotImplementedError):
        NativeForecaster(_cfg(True, 'bf16'), T, F, O, 0, uq=True)


@pytest.fixture(scope='module')
def workdir(tmp_path_factory):
    from lfm_quant_b200.scripts.synthetic import write_open_dataset, write_system_test_conf
    d = tmp_path_factory.mktemp('uqchain')
    write_open_dataset(str(d / 'datasets' / 'open-dataset.dat'), n_keys=30, n_months=420, seed=9)
    write_system_test_conf(str(d / 'config' / 'system-test.conf'), str(d / 'datasets'), str(d / 'experiments'))
    os.environ.setdefault('LFM_QUANT_ROOT', str(d))
    return d


def test_cli_trains_and_predicts_the_multi_step_uq_model(workdir):
    """--nn_type RNNUqRangeEstimate --UQ=True --forecast_steps 2: training logs, prediction at fp32 and bf16x3 (every
    step's norm_preds_s / norm_variance_s), and a checkpoint restored from either container."""
    from lfm_quant_b200.scripts import configs
    from lfm_quant_b200.scripts import lfm_quant as cli
    conf = str(workdir / 'config' / 'system-test.conf')
    extra = ['--nn_type', 'RNNUqRangeEstimate', '--UQ=True', '--forecast_steps', '2', '--forecast_steps_weights',
             '1.0-0.5', '--dropout', '0.1', '--model_dir', 'system-test-uq-chain']
    configs.reset()
    valid_mse = cli.main(['--config=' + conf, '--train=True'] + extra)
    mdir = workdir / 'experiments' / 'system-test-uq-chain'
    assert np.isfinite(valid_mse)
    ep = pd.read_csv(mdir / 'train_log' / 'system-test-train-logs-epoch.csv')
    assert len(ep) == 2 and np.isfinite(ep['uq_loss']).all() and np.isfinite(ep['valid_uq_loss']).all()
    assert ep['uq_loss'].iloc[1] < ep['uq_loss'].iloc[0]
    w = np.load(mdir / 'chkpts' / 'chkpt.lfmq.npz')
    assert set(uco.param_names(1, 2)) <= set(w.files)
    outs = {}
    for prec in ('fp32', 'bf16x3'):
        configs.reset()
        cli.main(['--config=' + conf, '--train=False', '--precision', prec] + extra)
        out = pd.read_csv(mdir / 'pred' / 'preds.dat', sep=' ', dtype={'gvkey': str})
        assert len(out) > 100
        for s in (1, 2):
            assert np.isfinite(out['norm_preds_%d' % s]).all() and (out['norm_variance_%d' % s] >= 1e-6).all()
        outs[prec] = out
    for col in ('norm_preds_1', 'norm_preds_2', 'norm_variance_1', 'norm_variance_2'):
        assert rel_err(outs['bf16x3'][col].values, outs['fp32'][col].values) < TOL, col
    # the TF-format container alone restores the same weights
    os.rename(mdir / 'chkpts' / 'chkpt.lfmq.npz', mdir / 'chkpts' / 'chkpt.saved.npz')
    try:
        configs.reset()
        cli.main(['--config=' + conf, '--train=False'] + extra)
        out = pd.read_csv(mdir / 'pred' / 'preds.dat', sep=' ', dtype={'gvkey': str})
        for col in ('norm_preds_1', 'norm_preds_2', 'norm_variance_2'):
            np.testing.assert_array_equal(out[col].values, outs['fp32'][col].values)
    finally:
        os.rename(mdir / 'chkpts' / 'chkpt.saved.npz', mdir / 'chkpts' / 'chkpt.lfmq.npz')
    configs.reset()
