"""Monte-Carlo dropout samples of a uq model in one prediction (lfmq_forward_uq_mc / lfmq_chain_forward_uq_mc,
ForecastChainEngine.forward_mc, NativeForecaster.predict_mc, --mc_samples): sample s of window b is global row
row0 + s * B + b of the batch tiled `samples` times, and the four per-element moments are folded in sample order.

Checked here: sample 0 is the plain forward; the moments match float64 moments of the tiled batch run through the plain
forward; they do not depend on how the rows are cut into launches nor on the other windows; no dropout gives zero
variances; the samples are independent draws; and the CLI writes the reference ensemble's columns."""
import ctypes
import io
import os

import numpy as np
import pandas as pd
import pytest
import torch

import uq_chain_oracle as uco
from util import rel_err

pytestmark = pytest.mark.gpu
KW = dict(target_idx=1, target_lambda=0.5, rnn_lambda=0.7)
DROP = dict(dropout=0.2, recurrent_dropout=0.15, seed=31)
# float64 moments of the same samples: the fp32 Welford accumulators stay within MOMENT_TOL (max abs error over the
# array / max abs value).  Worst measured on an H100 80GB HBM3 (700 W): see DESIGN.md §5c.
MOMENT_TOL = 1e-5


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()


def _problem(B, T, F, O, H, L, S, seed, cell='lstm'):
    rng = np.random.RandomState(seed)
    P = uco.init_params(L, F, O, H, S, init_scale=0.5, seed=seed + 1, dtype=np.float64, rnn_cell=cell)
    P = [(p + rng.normal(size=p.shape) * 0.05).astype(np.float32).astype(np.float64) for p in P]
    return P, rng.normal(size=(B, T, F)).astype(np.float32)


def _engine(max_batch, T, F, O, H, L, S, prec, cell='lstm', drop=DROP):
    from lfm_quant_b200.engine import ForecastChainEngine
    return ForecastChainEngine(forecast_steps=S, weights=[1.0, 0.5, 0.25][:S], max_batch=max_batch, seq_len=T,
                               n_inputs=F, n_outputs=O, num_hidden=H, num_layers=L, rnn_cell=cell, uq=True,
                               precision=prec, train=False, forward_only=True, **KW, **drop)


def _np(moments):
    return [[t.cpu().numpy() for t in m] for m in moments]


def _tiled_samples(eng, x, samples, step, row0):
    """Every sample through the plain forward: the batch tiled `samples` times, in launches of max_batch rows at their
    own row0.  Returns per stage (preds, vars) [samples, B, T, O]."""
    B, mb = x.shape[0], eng.cfg.max_batch
    xt = x.repeat(samples, 1, 1).contiguous()
    outs = [eng.forward(xt[r:r + mb].contiguous(), step=step, row0=row0 + r) for r in range(0, samples * B, mb)]
    outs = [torch.cat([o[k] for o in outs], 0).cpu().numpy().astype(np.float64) for k in range(2 * eng.S)]
    T = x.shape[1]
    return [(outs[2 * s].reshape(samples, B, T, -1), outs[2 * s + 1].reshape(samples, B, T, -1)) for s in range(eng.S)]


def _ref_moments(p, v):
    return p.mean(0), v.mean(0), p.var(0), v.var(0)


@pytest.mark.parametrize('prec', ['fp32', 'bf16', 'bf16x3'])
@pytest.mark.parametrize('cell', ['lstm', 'gru'])
@pytest.mark.parametrize('stages', [1, 2, 3])
def test_one_sample_is_the_plain_forward(prec, cell, stages):
    """samples = 1: mean_pred and mean_var are forward's outputs at the same (step, row0) bit for bit and both variances
    are exactly 0; with more samples, sample 0 of every window is that forward too (the tiled forward's first B rows
    are the plain batch)."""
    B, T, F, O, H = 37, 6, 8, 4, 64
    L = 2 if stages == 1 else 1
    P, x = _problem(B, T, F, O, H, L, stages, seed=3, cell=cell)
    eng = _engine(B, T, F, O, H, L, stages, prec, cell)
    eng.set_weights(P)
    xd = _cuda(x)
    ref = [o.cpu().numpy() for o in eng.forward(xd, step=5, row0=211)]
    got = _np(eng.forward_mc(xd, 1, step=5, row0=211))
    assert len(got) == stages
    for s, (mp, mv, vp, vv) in enumerate(got):
        assert np.array_equal(mp, ref[2 * s]) and np.array_equal(mv, ref[2 * s + 1]), s
        assert not vp.any() and not vv.any(), s
    tiled = _tiled_samples(eng, xd, 3, 5, 211)
    for s in range(stages):
        assert np.array_equal(tiled[s][0][0], ref[2 * s]) and np.array_equal(tiled[s][1][0], ref[2 * s + 1]), s
    eng.close()


@pytest.mark.parametrize('prec', ['fp32', 'bf16'])
@pytest.mark.parametrize('B', [1, 256, 4096])
@pytest.mark.parametrize('samples', [2, 7, 64])
def test_moments_match_float64_moments_of_the_tiled_forward(prec, B, samples):
    T, F, O, H, L = 6, 8, 4, 64, 1
    P, x = _problem(B, T, F, O, H, L, 1, seed=11)
    eng = _engine(4096, T, F, O, H, L, 1, prec)
    eng.set_weights(P)
    xd = _cuda(x)
    got = _np(eng.forward_mc(xd, samples, step=2, row0=77))[0]
    p, v = _tiled_samples(eng, xd, samples, 2, 77)[0]
    errs = [rel_err(g, r) for g, r in zip(got, _ref_moments(p, v))]
    print('mc moments %s B=%d samples=%d: rel err mean_pred %.2e mean_var %.2e var_pred %.2e var_var %.2e'
          % (prec, B, samples, *errs))
    assert max(errs) < MOMENT_TOL, errs
    assert (got[2] > 0).mean() > 0.99 and (got[3] > 0).mean() > 0.99      # the samples differ
    eng.close()


@pytest.mark.parametrize('prec', ['fp32', 'bf16x3'])
def test_chain_moments_follow_each_replica_trajectory(prec):
    """A two-step chain: stage 1 of sample s reads the window built from stage 0's sample s, as the tiled chain does."""
    B, T, F, O, H, L, S, samples = 256, 6, 8, 4, 64, 1, 2, 7
    P, x = _problem(B, T, F, O, H, L, S, seed=12)
    eng = _engine(512, T, F, O, H, L, S, prec)
    eng.set_weights(P)
    xd = _cuda(x)
    got = _np(eng.forward_mc(xd, samples, step=4, row0=0))
    tiled = _tiled_samples(eng, xd, samples, 4, 0)
    for s in range(S):
        errs = [rel_err(g, r) for g, r in zip(got[s], _ref_moments(*tiled[s]))]
        print('mc chain moments %s stage %d: %s' % (prec, s, ['%.2e' % e for e in errs]))
        assert max(errs) < MOMENT_TOL, (s, errs)
    eng.close()


@pytest.mark.parametrize('prec', ['fp32', 'bf16'])
@pytest.mark.parametrize('stages', [1, 2])
def test_moments_do_not_depend_on_launch_size_or_other_windows(prec, stages):
    """max_batch = B, 3B, 50 (launches cut inside a sample) and 5B (all samples in one launch) give the same bits; so
    does a batch whose other windows hold different inputs."""
    B, T, F, O, H, samples = 37, 6, 8, 4, 64, 5
    L = 1
    P, x = _problem(B, T, F, O, H, L, stages, seed=21)
    xd = _cuda(x)
    res = []
    for mb in (B, 3 * B, 50, samples * B):
        eng = _engine(mb, T, F, O, H, L, stages, prec)
        eng.set_weights(P)
        res.append(_np(eng.forward_mc(xd, samples, step=9, row0=1000)))
        if mb == samples * B:
            x2 = np.random.RandomState(99).normal(size=x.shape).astype(np.float32)
            keep = [0, 17, 36]
            x2[keep] = x[keep]
            other = _np(eng.forward_mc(_cuda(x2), samples, step=9, row0=1000))
        eng.close()
    for r in res[1:]:
        for a, b in zip(r, res[0]):
            for u, w in zip(a, b):
                assert np.array_equal(u, w)
    for a, b in zip(other, res[0]):
        for u, w in zip(a, b):
            assert np.array_equal(u[keep], w[keep])


@pytest.mark.parametrize('prec', ['fp32', 'bf16', 'bf16x3'])
@pytest.mark.parametrize('stages', [1, 2])
def test_without_dropout_every_sample_is_the_plain_forward(prec, stages):
    B, T, F, O, H, L = 40, 6, 8, 4, 64, 1
    P, x = _problem(B, T, F, O, H, L, stages, seed=4)
    eng = _engine(64, T, F, O, H, L, stages, prec, drop=dict(dropout=0.0, recurrent_dropout=0.0, seed=31))
    eng.set_weights(P)
    xd = _cuda(x)
    ref = [o.cpu().numpy() for o in eng.forward(xd, step=1, row0=0)]
    for s, (mp, mv, vp, vv) in enumerate(_np(eng.forward_mc(xd, 9, step=1, row0=0))):
        assert np.array_equal(mp, ref[2 * s]) and np.array_equal(mv, ref[2 * s + 1]), s
        assert not vp.any() and not vv.any(), s
    eng.close()


def test_samples_are_independent_draws():
    """One layer whose BatchNormalization and target head are the identity (O = H, T = 1): the target prediction of a
    sample is h * mask, so the sample mean over 256 samples divided by the dropout-free h is the keep fraction of each
    unit times 1 / (1 - rate).  Every unit's fraction lies within 5 standard deviations of 1 - rate."""
    B, T, F, H, samples, rate = 6, 1, 8, 64, 256, 0.3
    O = H
    P, x = _problem(B, T, F, O, H, 1, 1, seed=8)
    P[5] = np.eye(H)                       # OUTPUT_TARGET_1/kernel
    P[6] = np.zeros(H)                     # OUTPUT_TARGET_1/bias
    P[3], P[4] = np.ones(H), np.zeros(H)   # gamma, beta
    bn = [(np.zeros(H), np.full(H, 1.0 - 1e-3))]
    xd = _cuda(x)
    res = {}
    for name, drop in (('plain', 0.0), ('mc', rate)):
        eng = _engine(B * samples, T, F, O, H, 1, 1, 'fp32', drop=dict(dropout=drop, recurrent_dropout=0.0, seed=5))
        eng.stages[0].set_weights(P, bn_stats=bn)
        res[name] = _np(eng.forward_mc(xd, samples if drop else 1, step=3, row0=0))[0]
        eng.close()
    h = res['plain'][0]
    assert (np.abs(h) > 1e-4).all()
    keep = res['mc'][0].astype(np.float64) / h * (1.0 - rate)
    sd = np.sqrt(rate * (1 - rate) / samples)
    print('mc keep fraction: mean %.4f, worst |dev| %.2f sd' % (keep.mean(), np.abs(keep - (1 - rate)).max() / sd))
    assert np.abs(keep - (1 - rate)).max() < 5 * sd
    assert (res['mc'][2] > 0).all()        # every unit is kept in some samples and dropped in others


def _model_cfg(argv):
    from lfm_quant_b200.scripts import base_config
    return base_config.get_configs(['--num_hidden', '64', '--num_layers', '1', '--batch_size', '16', '--dropout', '0.1']
                                   + argv)


def test_predict_mc_of_the_model_object():
    from lfm_quant_b200.scripts.models.point_estimate.rnn_point_estimate import NativeForecaster
    T, F, O = 5, 12, 6
    x = np.random.RandomState(0).normal(size=(40, T, F)).astype(np.float32)   # more windows than batch_size
    m = NativeForecaster(_model_cfg(['--train=False', '--nn_type', 'RNNUqRangeEstimate', '--UQ=True']), T, F, O, 0,
                         uq=True)
    out = m.predict_mc(x, 4)
    assert len(out) == 1 and all(t.shape == (40, T, O) for t in out[0])
    ref = m.engine.forward_mc(_cuda(x), 4, step=1, row0=0)
    for a, b in zip(out[0], ref[0]):
        assert torch.equal(a, b)
    with pytest.raises(ValueError):
        m.predict_mc(x, 0)
    p = NativeForecaster(_model_cfg(['--train=False']), T, F, O, 0)
    with pytest.raises(ValueError, match='uq model'):
        p.predict_mc(x, 4)


def test_library_refuses_point_handles_and_bad_sample_counts():
    from lfm_quant_b200 import _native as N
    from lfm_quant_b200.engine import ForecasterEngine
    kw = dict(max_batch=8, seq_len=4, n_inputs=6, n_outputs=3, num_hidden=16, train=False, forward_only=True,
              dropout=0.1)
    point = ForecasterEngine(**kw)
    x = torch.zeros(8, 4, 6, device='cuda')
    with pytest.raises(N.LfmqError, match='not a uq handle'):
        point.forward_mc(x, 4)
    uq = ForecasterEngine(uq=True, **kw)
    for bad in (0, -3):
        with pytest.raises(N.LfmqError, match='samples >= 1'):
            uq.forward_mc(x, bad)
    rc = uq.lib.lfmq_forward_uq_mc(uq.handle, x.data_ptr(), 8, 0, 0, 2, *([x.data_ptr()] * 4), x.data_ptr(), 16,
                                   None)
    assert rc == 4 and b'work needs' in uq.lib.lfmq_last_error()         # LFMQ_ERR_WORKSPACE
    n = ctypes.c_uint64(0)
    N.check(uq.lib.lfmq_forward_uq_mc_work_bytes(uq.handle, 8, 2, ctypes.byref(n)))
    assert n.value >= 8 * 4 * (6 + 2 * 3) * 4          # one launch of 8 rows: x, preds and vars, T = 4
    point.close()
    uq.close()


@pytest.fixture(scope='module')
def workdir(tmp_path_factory):
    from lfm_quant_b200.scripts.synthetic import write_open_dataset, write_system_test_conf
    d = tmp_path_factory.mktemp('mc')
    write_open_dataset(str(d / 'datasets' / 'open-dataset.dat'), n_keys=30, n_months=420, seed=9)
    write_system_test_conf(str(d / 'config' / 'system-test.conf'), str(d / 'datasets'), str(d / 'experiments'))
    os.environ.setdefault('LFM_QUANT_ROOT', str(d))
    return d


@pytest.mark.parametrize('steps', [1, 2])
def test_cli_mc_samples(workdir, steps):
    """--mc_samples 1 writes today's preds.dat byte for byte; --mc_samples 16 writes the sample mean, mean_var + var_var
    and the added norm_preds_var_s column, equal to float64 moments of 16 single-sample forwards at the same keys."""
    from lfm_quant_b200.scripts import configs
    from lfm_quant_b200.scripts import lfm_quant as cli
    from lfm_quant_b200.scripts.data_processing import Dataset
    from lfm_quant_b200.scripts.predict import Predict
    conf = str(workdir / 'config' / 'system-test.conf')
    extra = ['--nn_type', 'RNNUqRangeEstimate', '--UQ=True', '--dropout', '0.1', '--recurrent_dropout', '0.1',
             '--model_dir', 'mc-%d' % steps, '--forecast_steps', str(steps), '--forecast_steps_weights',
             '-'.join(['1.0', '0.5'][:steps])]
    mdir = workdir / 'experiments' / ('mc-%d' % steps)
    configs.reset()
    cli.main(['--config=' + conf, '--train=True'] + extra)
    files = {}
    for flag in ([], ['--mc_samples', '1'], ['--mc_samples', '16']):
        configs.reset()
        cli.main(['--config=' + conf, '--train=False'] + extra + flag)
        files[tuple(flag)] = (mdir / 'pred' / 'preds.dat').read_bytes()
    assert files[()] == files[('--mc_samples', '1')]
    base = pd.read_csv(mdir / 'pred' / 'preds.dat', sep=' ', dtype={'gvkey': str})
    old = pd.read_csv(io.BytesIO(files[()]), sep=' ', dtype={'gvkey': str})
    new_cols = ['norm_preds_var_%d' % (s + 1) for s in range(steps)]
    assert [c for c in base.columns if c not in old.columns] == new_cols
    assert [c for c in base.columns if c in old.columns] == list(old.columns)
    for c in ('date', 'gvkey', 'seq_norm', 'targets_1'):
        pd.testing.assert_series_equal(base[c], old[c])

    # the same keys through the plain forward: batch k (step k + 1), sample s at row0 = s * B
    configs.reset()
    c = cli.get_configs(['--config=' + conf, '--train=False', '--mc_samples', '16'] + extra)
    p = Predict(c, Dataset(c))
    p.model.load_weights(os.path.join(p.chkpts_dir, 'chkpt'))
    eng, ti = p.model.engine, p.target_index
    cols = {k: [] for k in ('m', 'v', 'pv')}
    for k, (inp, _, _) in enumerate(p._batches):
        B = inp.shape[0]
        outs = [[o[:, -1, ti].cpu().numpy().astype(np.float64) for o in eng.forward(inp, step=k + 1, row0=s * B)]
                for s in range(16)]
        pr = np.stack([o[0::2] for o in outs])       # [16, steps, B]
        vr = np.stack([o[1::2] for o in outs])
        cols['m'].append(pr.mean(0))
        cols['v'].append(vr.mean(0) + vr.var(0))
        cols['pv'].append(pr.var(0))
    for s in range(steps):
        for col, key in (('norm_preds_%d', 'm'), ('norm_variance_%d', 'v'), ('norm_preds_var_%d', 'pv')):
            ref = np.concatenate([a[s] for a in cols[key]])
            err = rel_err(base[col % (s + 1)].values, ref)
            print('mc cli %s: rel err %.2e' % (col % (s + 1), err))
            assert err < MOMENT_TOL, (col % (s + 1), err)
    assert (base['norm_preds_var_1'] > 0).mean() > 0.99
    configs.reset()
