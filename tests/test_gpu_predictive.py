"""Predictive quantiles and proper scores on the GPU (lfmq_chain_forward_uq_dist, ForecastChainEngine.forward_dist,
NativeForecaster.predict_dist, --pred_quantiles): each window's Monte-Carlo dropout samples as a Gaussian mixture.

Checked here: the moments against lfmq_chain_forward_uq_mc bit for bit at every precision; quantiles, CRPS, log score
and PIT against the fp64 reference (tests/predictive_oracle.py) on the samples lfmq_chain_forward_uq gives for the
same rows, multimodal mixtures included; the same bits at any launch size, on a subset of the windows and on a
repeated call; NaN and absent targets; the refusals; and the CLI files."""
import ctypes as C

import numpy as np
import pandas as pd
import pytest
import torch

import predictive_oracle as pdo
import uq_chain_oracle as uco

pytestmark = pytest.mark.gpu
KW = dict(target_idx=1, target_lambda=0.5, rnn_lambda=0.7)
DROP = dict(dropout=0.25, recurrent_dropout=0.15, seed=31)
STEP = 5
LEVELS = [0.05, 0.3, 0.6, 0.95]       # away from the gaps k / M of a multimodal mixture of M = 2 or 7 samples
ERR_ARG = 1                           # include/lfmq.h


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()


def _chain(S, T, F, O, H, L, *, max_batch=256, precision='fp32', cell='lstm', uq=True, **kw):
    from lfm_quant_b200.engine import ForecastChainEngine
    args = dict(KW, train=False, forward_only=True)
    args.update(DROP)
    args.update(kw)
    return ForecastChainEngine(forecast_steps=S, weights=[1.0, 0.5][:S], max_batch=max_batch, seq_len=T, n_inputs=F,
                               n_outputs=O, num_hidden=H, num_layers=L, rnn_cell=cell, precision=precision, uq=uq,
                               **args)


def _model(S, T, F, O, H, L, N, cell='lstm', seed=0, head_scale=1.0, **kw):
    """A uq chain with perturbed weights, the target heads' kernels scaled by head_scale (a large scale spreads the
    dropout samples far apart relative to their variances: a multimodal mixture), and inputs x [N,T,F]."""
    rng = np.random.RandomState(seed)
    P = uco.init_params(L, F, O, H, S, init_scale=0.5, seed=seed + 1, dtype=np.float64, rnn_cell=cell)
    P = [(p + rng.normal(size=p.shape) * 0.05).astype(np.float32) for p in P]
    eng = _chain(S, T, F, O, H, L, cell=cell, **kw)
    names = [n for (_, n, _, _, tr) in eng.specs if tr]
    P = [p * head_scale if ('OUTPUT_TARGET' in n and 'kernel' in n) else p for p, n in zip(P, names)]
    eng.set_weights(P)
    return eng, rng.normal(size=(N, T, F)).astype(np.float32)


def _targets(S, N, T, O, seed, nan_rows=()):
    y = np.random.RandomState(seed).normal(size=(N, T, O)).astype(np.float32)
    y[list(nan_rows)] = np.nan
    return [_cuda(y)] * S, y


def _np(t):
    return t.cpu().numpy()


# (name, S, cell, precision, H, L)
CASES = [('fp32-lstm-L2', 1, 'lstm', 'fp32', 64, 2), ('fp32-gru-S2', 2, 'gru', 'fp32', 64, 1),
         ('tf32-lstm-S2', 2, 'lstm', 'tf32', 64, 1), ('bf16-lstm', 1, 'lstm', 'bf16', 256, 1),
         ('bf16-lstm-S2', 2, 'lstm', 'bf16', 256, 1), ('bf16-gru', 1, 'gru', 'bf16', 128, 1),
         ('bf16x3-lstm', 1, 'lstm', 'bf16x3', 256, 1)]


@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_moments_are_forward_mc_bit_for_bit(case):
    _, S, cell, prec, H, L = case
    T, F, O, N, M = 8, 32, 16, 300, 5
    eng, x = _model(S, T, F, O, H, L, N, cell=cell, seed=3, precision=prec)
    ys, _ = _targets(S, N, T, O, 4)
    xd = _cuda(x)
    mc = eng.forward_mc(xd, M, step=STEP, row0=7)
    moments, q, sc = eng.forward_dist(xd, M, LEVELS, ys=ys, step=STEP, row0=7)
    for s in range(S):
        for a, b in zip(mc[s], moments[s]):
            assert torch.equal(a, b)
    assert q.shape == (S, N, len(LEVELS)) and sc.shape == (S, N, 3)
    assert torch.isfinite(q).all() and torch.isfinite(sc).all()
    assert (q[:, :, 1:] >= q[:, :, :-1]).all()
    eng.close()


def _samples(eng, x, M, step):
    """Every stage's (mu, v) [N, M] at [T-1, target_idx] from lfmq_chain_forward_uq on the batch tiled M times, in
    launches of max_batch rows keyed by their global row: the rows lfmq_chain_forward_uq_dist draws."""
    N = x.shape[0]
    xt = _cuda(np.tile(x, (M, 1, 1)))
    mb = eng.cfg.max_batch
    outs = [eng.forward(xt[a:a + mb].contiguous(), step=step, row0=a) for a in range(0, M * N, mb)]
    S = len(outs[0]) // 2
    tidx = KW['target_idx']
    res = []
    for s in range(S):
        mu = torch.cat([o[2 * s] for o in outs])[:, -1, tidx].reshape(M, N).T
        v = torch.cat([o[2 * s + 1] for o in outs])[:, -1, tidx].reshape(M, N).T
        res.append((_np(mu).astype(np.float64), _np(v).astype(np.float64)))
    return res


# (name, M, S, head_scale)
ORACLE = [('M1', 1, 1, 1.0), ('M2-bimodal', 2, 1, 300.0), ('M7', 7, 2, 1.0), ('M7-multimodal', 7, 1, 300.0),
          ('M64', 64, 1, 1.0), ('M64-spread', 64, 2, 30.0)]


@pytest.mark.parametrize('case', ORACLE, ids=[c[0] for c in ORACLE])
def test_quantiles_and_scores_match_the_fp64_oracle(case):
    _, M, S, scale = case
    T, F, O, H, L, N = 6, 12, 4, 64, 1, 40
    eng, x = _model(S, T, F, O, H, L, N, seed=M, head_scale=scale)
    ys, y = _targets(S, N, T, O, 9)
    y[3, -1, KW['target_idx']] += 50.0                    # a target far out in the tail
    ys = [_cuda(y)] * S
    _, q, sc = eng.forward_dist(_cuda(x), M, LEVELS, ys=ys, step=STEP)
    q, sc = _np(q), _np(sc)
    worst = dict(q=0.0, crps=0.0, nll=0.0, pit=0.0, sep=0.0)
    for s, (mu, v) in enumerate(_samples(eng, x, M, STEP)):
        for b in range(N):
            yb = float(y[b, -1, KW['target_idx']])
            wq, ws = pdo.window(mu[b], v[b], yb, LEVELS)
            sd = pdo.std(mu[b], v[b])
            worst['q'] = max(worst['q'], np.abs(q[s, b] - wq).max() / sd)
            worst['crps'] = max(worst['crps'], abs(sc[s, b, 0] - ws[0]) / abs(ws[0]))
            # the output is fp32: beyond 1e-5 absolute, allow the rounding of the value itself (a target far in
            # the tail has a log score of ~1e3, whose fp32 spacing is 6e-5)
            worst['nll'] = max(worst['nll'], max(0.0, abs(sc[s, b, 1] - ws[1]) - 2.0 ** -23 * abs(ws[1])))
            worst['pit'] = max(worst['pit'], abs(sc[s, b, 2] - ws[2]))
            if M > 1:
                worst['sep'] = max(worst['sep'], np.ptp(mu[b]) / np.sqrt(v[b].max()))
    print('dist %s: %s' % (case[0], {k: '%.2e' % w for k, w in worst.items()}))
    if scale > 100:
        assert worst['sep'] > 20          # components far apart: the mixture has several modes
    assert worst['q'] <= 1e-5 and worst['crps'] <= 1e-5 and worst['nll'] <= 1e-5 and worst['pit'] <= 1e-6, worst
    eng.close()


def test_launch_size_subsets_and_repeats_give_the_same_bits():
    T, F, O, H, L, N, M = 6, 12, 4, 64, 2, 300, 9
    outs = []
    for mb in (256, 8192):
        eng, x = _model(2, T, F, O, H, L, N, seed=21, max_batch=mb)
        ys, _ = _targets(2, N, T, O, 22, nan_rows=(5,))
        xd = _cuda(x)
        run = [[_np(t) for t in eng.forward_dist(xd, M, LEVELS, ys=ys, step=STEP)[1:]] for _ in range(2)]
        for a, b in zip(*run):
            assert np.array_equal(a, b, equal_nan=True)
        # one sample: window b is row b whatever the batch, so a subset of the windows gives their bits
        _, q1, s1 = eng.forward_dist(xd, 1, LEVELS, ys=ys, step=STEP)
        _, qk, sk = eng.forward_dist(xd[:77].contiguous(), 1, LEVELS, ys=[t[:77].contiguous() for t in ys], step=STEP)
        assert np.array_equal(_np(q1[:, :77]), _np(qk)) and np.array_equal(_np(s1[:, :77]), _np(sk), equal_nan=True)
        outs.append(run[0])
        eng.close()
    for a, b in zip(*outs):
        assert np.array_equal(a, b, equal_nan=True)


def _raw(eng, xd, n, m, lvls, ys, q, sc, work, **over):
    """lfmq_chain_forward_uq_dist with every argument overridable by name (None: a null pointer)."""
    S = eng.S
    mom = [[torch.empty(n, eng.T, eng.O, device='cuda') for _ in range(S)] for _ in range(4)]
    lv = np.ascontiguousarray(lvls, dtype=np.float32)
    a = dict(x=C.c_void_p(xd.data_ptr()), y=eng._ptrs(ys) if ys is not None else None,
             levels=lv.ctypes.data_as(C.c_void_p), n_levels=len(lvls), mean_pred=eng._ptrs(mom[0]),
             quantiles=eng._ptrs(q) if q is not None else None, scores=eng._ptrs(sc) if sc is not None else None,
             samples=m, B=n)
    a.update(over)
    return eng.lib.lfmq_chain_forward_uq_dist(
        eng._handles, S, a['x'], a['y'], a['B'], 0, STEP, a['samples'], a['levels'], a['n_levels'], a['mean_pred'],
        eng._ptrs(mom[1]), eng._ptrs(mom[2]), eng._ptrs(mom[3]), a['quantiles'], a['scores'],
        C.c_void_p(work.data_ptr()), work.numel(), C.c_void_p(torch.cuda.current_stream().cuda_stream))


def test_nan_and_absent_targets():
    T, F, O, H, L, N, M = 6, 12, 4, 64, 1, 50, 8
    eng, x = _model(1, T, F, O, H, L, N, seed=30)
    xd = _cuda(x)
    ys, _ = _targets(1, N, T, O, 31, nan_rows=(0, 17))
    _, q, sc = eng.forward_dist(xd, M, LEVELS, ys=ys, step=STEP)
    sc = _np(sc)
    assert np.isnan(sc[0, [0, 17]]).all() and np.isfinite(np.delete(sc[0], [0, 17], axis=0)).all()
    assert torch.isfinite(q).all()
    _, q0, none = eng.forward_dist(xd, M, LEVELS, step=STEP)
    assert none is None and torch.equal(q, q0)
    n = C.c_uint64(0)
    assert eng.lib.lfmq_chain_forward_uq_dist_work_bytes(eng._handles, 1, N, M, len(LEVELS), C.byref(n)) == 0
    work = torch.empty(n.value, dtype=torch.uint8, device='cuda')
    qq = [torch.empty(N, len(LEVELS), device='cuda')]
    sentinel = [torch.full((N, 3), 1234.5, device='cuda')]
    assert _raw(eng, xd, N, M, LEVELS, None, qq, sentinel, work) == 0
    torch.cuda.synchronize()
    assert (sentinel[0] == 1234.5).all() and torch.equal(qq[0], q[0])
    assert _raw(eng, xd, N, M, LEVELS, None, qq, None, work) == 0
    eng.close()


def test_refusals():
    from lfm_quant_b200.engine import DenseEngine, ForecastChainEngine
    T, F, O, H, N, M = 6, 12, 4, 64, 20, 3
    eng, x = _model(1, T, F, O, H, 1, N, seed=40)
    xd = _cuda(x)
    ys, _ = _targets(1, N, T, O, 41)
    n = C.c_uint64(0)
    lib = eng.lib
    assert lib.lfmq_chain_forward_uq_dist_work_bytes(eng._handles, 1, N, M, 4, C.byref(n)) == 0
    work = torch.empty(n.value, dtype=torch.uint8, device='cuda')
    q, sc = [torch.empty(N, 32, device='cuda')], [torch.empty(N, 3, device='cuda')]
    assert _raw(eng, xd, N, M, LEVELS, ys, q, sc, work) == 0
    for levels in ([], [0.0, 0.5], [0.5, 1.0], [0.6, 0.4], [0.3, 0.3], [float('nan')], [0.01 * (k + 1) for k in range(33)]):
        assert _raw(eng, xd, N, M, levels or [0.5], ys, q, sc, work, n_levels=len(levels)) == ERR_ARG, levels
    for over in (dict(x=None), dict(levels=None), dict(quantiles=None), dict(scores=None), dict(mean_pred=None),
                 dict(samples=0), dict(B=0)):
        assert _raw(eng, xd, N, M, LEVELS, ys, q, sc, work, **over) == ERR_ARG, over
    for nl in (0, 33):
        assert lib.lfmq_chain_forward_uq_dist_work_bytes(eng._handles, 1, N, M, nl, C.byref(n)) == ERR_ARG
    assert lib.lfmq_chain_forward_uq_dist_work_bytes(eng._handles, 1, N, M, 4, None) == ERR_ARG
    point = _chain(1, T, F, O, H, 1, uq=False)
    dense = ForecastChainEngine(stages=[DenseEngine(max_batch=256, seq_len=T, n_inputs=F, n_outputs=O,
                                                    target_idx=KW['target_idx'], target_lambda=0.5, forward_only=True)])
    for other in (point, dense):
        assert lib.lfmq_chain_forward_uq_dist_work_bytes(other._handles, 1, N, M, 4, C.byref(n)) == ERR_ARG
        assert _raw(other, xd, N, M, LEVELS, ys, q, sc, work) == ERR_ARG
        other.close()
    with pytest.raises(ValueError, match='needs a uq model'):
        from lfm_quant_b200.scripts.models.point_estimate.rnn_point_estimate import NativeForecaster
        NativeForecaster.predict_dist(type('P', (), {'uq': False})(), x, M, LEVELS)
    torch.cuda.synchronize()
    eng.close()


# ---- the CLI on the synthetic dataset ----------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def workdir(tmp_path_factory):
    from lfm_quant_b200.scripts.synthetic import write_open_dataset, write_system_test_conf
    d = tmp_path_factory.mktemp('predictive')
    write_open_dataset(str(d / 'datasets' / 'open-dataset.dat'), n_keys=30, n_months=420, seed=9)
    write_system_test_conf(str(d / 'config' / 'system-test.conf'), str(d / 'datasets'), str(d / 'experiments'))
    (d / 'experiments').mkdir()
    return d


@pytest.fixture()
def cli(workdir, monkeypatch):
    from lfm_quant_b200.scripts import configs
    from lfm_quant_b200.scripts import lfm_quant
    monkeypatch.setenv('LFM_QUANT_ROOT', str(workdir))
    conf = str(workdir / 'config' / 'system-test.conf')

    def main(*argv):
        configs.reset()
        try:
            return lfm_quant.main(['--config=' + conf] + list(argv))
        finally:
            configs.reset()
    return main


UQ = ['--nn_type', 'RNNUqRangeEstimate', '--UQ=True', '--dropout', '0.1', '--recurrent_dropout', '0.1']
SPEC = '0.05-0.25-0.5-0.75-0.95'


def _check_files(m, steps):
    preds = pd.read_csv(m / 'pred' / 'preds.dat', sep=' ', dtype={'gvkey': str})
    qd = pd.read_csv(m / 'pred' / 'quantiles.dat', sep=' ', dtype={'gvkey': str})
    assert qd['date'].tolist() == preds['date'].tolist() and qd['gvkey'].tolist() == preds['gvkey'].tolist()
    names = ['q5', 'q25', 'q50', 'q75', 'q95']
    for s in range(1, steps + 1):
        nq = qd[['norm_%s_%d' % (n, s) for n in names]].to_numpy()
        assert np.isfinite(nq).all() and (np.diff(nq, axis=1) >= 0).all()
        known = np.isfinite(preds['norm_targets_%d' % s].to_numpy())
        assert np.isfinite(qd.loc[known, ['crps_%d' % s, 'nll_%d' % s, 'pit_%d' % s]].to_numpy()).all()
        assert qd.loc[~known, ['crps_%d' % s, 'nll_%d' % s, 'pit_%d' % s]].isna().all().all()
        pit = qd.loc[known, 'pit_%d' % s].to_numpy()
        assert ((pit >= 0) & (pit <= 1)).all()
        pos = preds['seq_norm'].to_numpy() > 0
        assert (np.diff(qd.loc[pos, ['%s_%d' % (n, s) for n in names]].to_numpy(), axis=1) >= 0).all()
    cal = pd.read_csv(m / 'pred' / 'calibration.dat', sep=' ')
    assert len(cal) == 5 * steps and cal['step'].tolist() == sorted(cal['step'].tolist())
    return qd


@pytest.mark.parametrize('steps', [1, 2])
def test_cli_writes_quantiles_and_leaves_preds_alone(workdir, cli, steps):
    name = 'dist-%d' % steps
    m = workdir / 'experiments' / name
    args = ['--model_dir', name, '--forecast_steps', str(steps), '--forecast_steps_weights',
            '-'.join(['1.0', '0.5'][:steps])] + UQ
    cli(*args, '--train=True')
    for prec in ('fp32', 'bf16'):
        for mc in ('1', '8'):
            run = list(args) + ['--train=False', '--precision', prec, '--mc_samples', mc]
            cli(*run)
            plain = (m / 'pred' / 'preds.dat').read_bytes()
            ens = (m / 'ensemble_preds.dat').read_bytes() if mc != '1' else None
            (m / 'pred' / 'preds.dat').unlink()
            cli(*run, '--pred_quantiles', SPEC)
            assert (m / 'pred' / 'preds.dat').read_bytes() == plain, (prec, mc)
            if ens is not None:
                assert (m / 'ensemble_preds.dat').read_bytes() == ens, (prec, mc)
            qd = _check_files(m, steps)
            print('%s %s mc=%s: mean crps_1 %.4f, pit in [%.3f, %.3f]' % (name, prec, mc, qd['crps_1'].mean(),
                                                                          qd['pit_1'].min(), qd['pit_1'].max()))
            (m / 'pred' / 'quantiles.dat').unlink()


def test_cli_walk_forward_stacks_the_origins_quantiles(workdir, cli):
    origins = [199612, 199712]
    args = ['--training_type', 'iterative', '--split_date', '199612', '--end_date', '199812', '--model_dir', 'dist-wf',
            '--NPE', '2'] + UQ
    cli(*args, '--train=True')
    cli(*args, '--train=False', '--mc_samples', '4', '--pred_quantiles', SPEC)
    wf = workdir / 'experiments' / 'dist-wf'
    got = pd.read_csv(wf / 'walk_forward_quantiles.dat', sep=' ', dtype={'gvkey': str}, float_precision='round_trip')
    own = [pd.read_csv(wf / ('system-test-wf-%d' % o) / 'pred' / 'quantiles.dat', sep=' ', dtype={'gvkey': str},
                       float_precision='round_trip').assign(origin=o) for o in origins]
    pd.testing.assert_frame_equal(got, pd.concat(own, ignore_index=True))
    assert sorted(set(got['origin'])) == origins
