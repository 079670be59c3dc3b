"""Accumulated local effects on the GPU (lfmq_chain_ale, ForecastChainEngine.ale, NativeForecaster.ale, --ale_bins):
per feature the quantile edges of one input column, each bin's local effects f(upper edge) - f(lower edge) and their
centred accumulation.

Checked here: the fp64 oracle (tests/ale_oracle.py) for every model kind at fp32; at tf32, bf16 and bf16x3 every
window's local effect against the model's own forward on host-built copies; the linear model in closed form; exactly
zero for a column the model does not read; the same bits at any launch size and on a repeated call, and the same
effects under a permutation of the windows; the binning rules; the refusals; and the CLI file."""
import ctypes as C

import numpy as np
import pandas as pd
import pytest
import torch

import ale_oracle as alo
import shapley_oracle as sho
from test_gpu_shapley import DROP, KW, _chain, _cuda, _dense, _params

pytestmark = pytest.mark.gpu
STEP, N, K = 7, 300, 8
ERR_ARG, ERR_WORKSPACE = 1, 4     # include/lfmq.h
OUT = ('n_bins', 'edges', 'counts', 'ale', 'local_mean', 'local_sd')


def _run(eng, x, cols, bins=K, step=STEP):
    return dict(zip(OUT, [t.cpu().numpy() for t in eng.ale(_cuda(x), np.asarray(cols), bins, step)]))


def _cols(T, F):
    """the latest quarter of every field, then two older columns"""
    return [(T - 1) * F + f for f in range(F)] + [0, F + 2]


def _with_ties(x):
    """x with the latest value of field 1 rounded to a few levels, so that bins hold ties and quantiles repeat"""
    x = x.copy()
    x.reshape(x.shape[0], -1)[:, -x.shape[-1] + 1] = np.round(x.reshape(x.shape[0], -1)[:, -x.shape[-1] + 1] * 2) / 2
    return x


def _assert_matches(got, ref, scale, tol):
    for k in ('n_bins', 'counts'):
        assert np.array_equal(got[k], ref[k]), k
    assert np.array_equal(got['edges'], ref['edges'].astype(np.float32), equal_nan=True)
    err = 0.0
    for k in ('ale', 'local_mean', 'local_sd'):
        assert np.array_equal(np.isnan(got[k]), np.isnan(ref[k])), k
        d = np.where(np.isnan(ref[k]), 0.0, np.abs(got[k] - ref[k])) / scale
        err = max(err, float(np.nanmax(d)))
    assert err < tol, err
    return err


# (name, S, L, cell, uq)
MODELS = [('lstm-point-L2', 1, 2, 'lstm', False), ('gru-point', 1, 1, 'gru', False), ('lstm-uq', 1, 1, 'lstm', True),
          ('point-chain-S2', 2, 1, 'lstm', False), ('gru-uq-chain-S2', 2, 1, 'gru', True)]


def _outputs(P, S, L, cell, uq):
    if uq:
        return sho.uq_outputs(P, num_layers=L, rnn_cell=cell, forecast_steps=S, dropout=DROP['dropout'],
                              recurrent_dropout=DROP['recurrent_dropout'], seed=DROP['seed'], step=STEP,
                              target_idx=KW['target_idx'])
    return sho.point_outputs(P, num_layers=L, rnn_cell=cell, forecast_steps=S, target_idx=KW['target_idx'])


@pytest.mark.parametrize('model', MODELS, ids=[m[0] for m in MODELS])
def test_effects_match_the_fp64_oracle(model):
    _, S, L, cell, uq = model
    T, F, O, H = 5, 6, 3, 16
    P, x = _params(T, F, O, H, L, S, cell, uq, seed=3 + S + L)
    x = _with_ties(x)
    eng = _chain(S, T, F, O, H, L, uq=uq, cell=cell, **(DROP if uq else {}))
    eng.set_weights(P)
    f = _outputs(P, S, L, cell, uq)
    cols = _cols(T, F)
    got = _run(eng, x, cols)
    ref = alo.ale(x.astype(np.float64), cols, K, f)
    J = 2 * S if uq else S
    assert got['ale'].shape == (len(cols), K + 1, J) and got['local_mean'].shape == (len(cols), K, J)
    assert got['n_bins'][1] < K                                            # the ties collapsed some quantiles
    err = _assert_matches(got, ref, np.abs(f(x.astype(np.float64), 0)).max(axis=0), 1e-4)
    print('ale %s: rel err %.2e, max |ale| %s' % (model[0], err, np.nanmax(np.abs(ref['ale']), axis=(0, 1))))
    eng.close()


def test_linear_model_matches_the_oracle_and_the_closed_form():
    T, F, O = 5, 6, 3
    rng = np.random.RandomState(4)
    W = (rng.normal(size=(T * F, O)) * 0.2).astype(np.float32).astype(np.float64)
    b = (rng.normal(size=O) * 0.1).astype(np.float32).astype(np.float64)
    x = rng.normal(size=(N, T * F)).astype(np.float32)
    eng = _dense(T, F, O)
    eng.set_weights([W, b])
    f = sho.dense_outputs(W, b, target_idx=KW['target_idx'])
    cols = _cols(T, F)
    got = _run(eng, x, cols)
    ref = alo.ale(x.astype(np.float64), cols, K, f)
    _assert_matches(got, ref, np.abs(f(x.astype(np.float64), 0)).max(axis=0), 1e-4)
    for g, c in enumerate(cols):
        z, n = got['edges'][g].astype(np.float64), got['counts'][g]
        cbar = (n * 0.5 * (z[:-1] + z[1:])).sum() / n.sum()
        err = np.abs(got['ale'][g, :, 0] - W[c, KW['target_idx']] * (z - cbar)).max()
        assert err < 1e-5, (g, err)
    eng.close()


def test_bins_of_ties_constant_and_non_finite_columns_match_exactly():
    T, F, O = 2, 5, 2
    rng = np.random.RandomState(6)
    x = rng.normal(size=(N, T * F)).astype(np.float32)
    x[:, 5] = 0.75                                                         # constant: no bins
    x[:, 6] = np.round(x[:, 6])                                            # a few levels
    x[::7, 7] = np.nan
    x[3::11, 7] = np.inf
    x[5::13, 7] = -np.inf
    x[:, 8] = -0.0
    x[::2, 8] = 0.0                                                        # -0 and +0 are one value
    x[:3, 9] = np.nan                                                      # column 9 all non-finite
    x[3:, 9] = np.inf
    eng = _dense(T, F, O)
    W = np.zeros((T * F, O))
    W[:, KW['target_idx']] = np.linspace(-1.0, 1.0, T * F)
    W[[5, 8, 9], :] = 0.0
    eng.set_weights([W, np.zeros(O)])
    cols = [5, 6, 7, 8, 9, 0]
    got = _run(eng, x, cols, bins=16)
    ref = alo.ale(x.astype(np.float64), cols, 16, sho.dense_outputs(W, np.zeros(O), target_idx=KW['target_idx']))
    assert got['n_bins'].tolist() == ref['n_bins'].tolist() and got['n_bins'][[0, 3, 4]].tolist() == [0, 0, 0]
    assert np.array_equal(got['counts'], ref['counts'])
    assert np.array_equal(got['edges'], ref['edges'].astype(np.float32), equal_nan=True)
    assert got['counts'][2].sum() == np.isfinite(x[:, 7]).sum()
    for g in (0, 3, 4):
        assert np.isnan(got['ale'][g]).all() and np.isnan(got['local_mean'][g]).all()
    assert np.isnan(got['edges'][4]).all() and got['edges'][0, 0] == 0.75
    eng.close()


# (name, precision, cell, H, L): bf16 on the cluster shape (LSTM H=256, L=1) and on the general path
PRECISIONS = [('tf32', 'tf32', 'lstm', 64, 2), ('bf16', 'bf16', 'lstm', 256, 1), ('bf16-gru', 'bf16', 'gru', 128, 1),
              ('bf16x3', 'bf16x3', 'lstm', 256, 1)]


def _forward(eng, x, uq):
    """the explained outputs [N,J] of lfmq_chain_forward(_uq) over x in launches of max_batch rows keyed row0 = a"""
    mb = eng.cfg.max_batch
    xd = _cuda(x)
    outs = [eng.forward(xd[a:a + mb].contiguous(), step=STEP, row0=a) for a in range(0, x.shape[0], mb)]
    return np.stack([torch.cat([o[j] for o in outs])[:, -1, KW['target_idx']].cpu().numpy()
                     for j in range(len(outs[0]))], axis=1)


@pytest.mark.parametrize('case', PRECISIONS, ids=[p[0] for p in PRECISIONS])
@pytest.mark.parametrize('uq', [False, True], ids=['point', 'uq'])
def test_effects_are_the_models_own_forward_at_every_precision(case, uq):
    _, prec, cell, H, L = case
    T, F, O = 8, 32, 16
    P, x = _params(T, F, O, H, L, 1, cell, uq, seed=11)
    eng = _chain(1, T, F, O, H, L, precision=prec, uq=uq, cell=cell, **(DROP if uq else {}))
    eng.set_weights(P)
    cols = [(T - 1) * F + f for f in (0, 5, 31)]
    bins = 1024                                 # >= N: every bin after the first holds one window
    got = _run(eng, x, cols, bins=bins)
    for g, c in enumerate(cols):
        Kg = got['n_bins'][g]
        z = got['edges'][g, :Kg + 1]
        b = np.maximum(np.searchsorted(z, x.reshape(N, -1)[:, c], side='left'), 1)
        d = _forward(eng, alo.with_column(x, c, z[b]), uq) - _forward(eng, alo.with_column(x, c, z[b - 1]), uq)
        single = [k for k in range(1, Kg + 1) if got['counts'][g, k - 1] == 1]
        assert len(single) == Kg - 1
        for k in single:
            assert np.array_equal(got['local_mean'][g, k - 1], d[b == k][0]), (g, k)   # bit for bit
            assert (got['local_sd'][g, k - 1] == 0).all()
        dd = d.astype(np.float64)
        mean = np.stack([dd[b == k].mean(axis=0) for k in range(1, Kg + 1)])
        n = got['counts'][g, :Kg]
        acc = np.vstack([np.zeros((1, d.shape[1])), np.cumsum(mean, axis=0)])
        ale = acc - (n[:, None] * 0.5 * (acc[:-1] + acc[1:])).sum(axis=0) / n.sum()
        scale = max(1.0, np.abs(ale).max())
        assert np.abs(got['local_mean'][g, :Kg] - mean).max() <= 1e-6 * max(1.0, np.abs(mean).max())
        assert np.abs(got['ale'][g, :Kg + 1] - ale).max() <= 1e-6 * scale
    print('ale %s %s: max |ale| %.3e' % (case[0], 'uq' if uq else 'point', np.nanmax(np.abs(got['ale']))))
    eng.close()


@pytest.mark.parametrize('prec', ['fp32', 'bf16', 'bf16x3', 'uq-fp32', 'uq-bf16'])
def test_a_column_the_model_does_not_read_gets_exactly_zero(prec):
    uq = prec.startswith('uq')
    T, F, O, H, L, S = 8, 32, 16, 256, 1, 2
    P, x = _params(T, F, O, H, L, S, 'lstm', uq, seed=5)
    dead = 7
    kernels = [i for i, p in enumerate(P) if p.shape == (F, 4 * H)]      # each stage's first lstm kernel
    assert len(kernels) == S
    for i in kernels:
        P[i] = P[i].copy()
        P[i][dead, :] = 0.0                                # the input-kernel row of field 7 in every stage
    eng = _chain(S, T, F, O, H, L, precision=prec.split('-')[-1], uq=uq, **(DROP if uq else {}))
    eng.set_weights(P)
    cols = [(T - 1) * F + dead, (T - 1) * F + 3]
    got = _run(eng, x, cols)
    assert got['n_bins'][0] == K
    for k in ('ale', 'local_mean', 'local_sd'):
        assert np.array_equal(got[k][0], np.zeros_like(got[k][0])), k
    assert np.abs(got['ale'][1]).max() > 0
    eng.close()


@pytest.mark.parametrize('case', ['fp32', 'bf16', 'uq-fp32', 'uq-bf16'])
def test_launch_size_and_repeats_do_not_change_the_bits(case):
    uq = case.startswith('uq')
    prec = case.split('-')[-1]
    T, F, O, H, L = 6, 10, 4, 64, 2
    P, x = _params(T, F, O, H, L, 1, 'lstm', uq, seed=21)
    cols = _cols(T, F)
    outs = []
    for mb in (256, 8192):
        eng = _chain(1, T, F, O, H, L, max_batch=mb, precision=prec, uq=uq, **(DROP if uq else {}))
        eng.set_weights(P)
        outs.append([_run(eng, x, cols), _run(eng, x, cols)])
        eng.close()
    for a in (outs[0][1], outs[1][0], outs[1][1]):
        for k in OUT:
            assert np.array_equal(a[k], outs[0][0][k], equal_nan=True), k


def test_a_permutation_of_the_windows_gives_the_same_effects():
    T, F, O, H, L = 6, 10, 4, 64, 1
    P, x = _params(T, F, O, H, L, 1, 'lstm', False, seed=22)
    eng = _chain(1, T, F, O, H, L)
    eng.set_weights(P)
    cols = _cols(T, F)
    a = _run(eng, x, cols)
    b = _run(eng, x[np.random.RandomState(1).permutation(N)], cols)
    for k in ('n_bins', 'edges', 'counts'):
        assert np.array_equal(a[k], b[k], equal_nan=True), k
    scale = np.nanmax(np.abs(a['ale']))
    for k in ('ale', 'local_mean', 'local_sd'):
        assert np.nanmax(np.abs(a[k] - b[k])) <= 1e-6 * max(1.0, scale), k
    eng.close()


def test_the_handles_state_is_left_untouched():
    from test_gpu_shapley import _slots
    T, F, O, H, L, S = 5, 6, 3, 16, 1, 2
    P, x = _params(T, F, O, H, L, S, 'lstm', True, seed=8)
    y = np.random.RandomState(9).normal(size=(N, T, O)).astype(np.float32)
    eng = _chain(S, T, F, O, H, L, uq=True, train=True, forward_only=False, max_batch=N, **DROP)
    eng.set_weights(P)
    eng.train_step(_cuda(x), [_cuda(y)] * S, 1, 0.5)
    before = [(e.params.clone(), e.grads.clone(), _slots(e)) for e in eng.stages]
    _run(eng, x, _cols(T, F))
    torch.cuda.synchronize()
    for e, (p, g, s) in zip(eng.stages, before):
        assert torch.equal(e.params, p) and torch.equal(e.grads, g) and torch.equal(_slots(e), s)
    eng.close()


def test_refusals():
    from lfm_quant_b200 import _native as Nv
    T, F, O, H = 5, 6, 3, 16
    P, x = _params(T, F, O, H, 1, 1, 'lstm', False, seed=2)
    eng = _chain(1, T, F, O, H, 1)
    eng.set_weights(P)
    lib = eng.lib
    xd = _cuda(x)
    cols = np.ascontiguousarray(_cols(T, F), dtype=np.int32)
    G = len(cols)
    n = C.c_uint64(0)
    assert lib.lfmq_chain_ale_work_bytes(eng._handles, 1, N, G, K, C.byref(n)) == 0
    work = torch.empty(n.value, dtype=torch.uint8, device='cuda')
    o = [torch.empty(G, dtype=torch.int32, device='cuda'), torch.empty(G, K + 1, device='cuda'),
         torch.empty(G, K, dtype=torch.int32, device='cuda'), torch.empty(G, K + 1, 1, device='cuda'),
         torch.empty(G, K, 1, device='cuda'), torch.empty(G, K, 1, device='cuda')]
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    ptrs = [t.data_ptr() for t in o]

    def call(N_=N, G_=G, K_=K, col=cols, x_=xd.data_ptr(), out=None, wb=None):
        p = list(ptrs) if out is None else out
        return lib.lfmq_chain_ale(eng._handles, 1, C.c_void_p(x_), N_,
                                  col.ctypes.data_as(C.c_void_p) if col is not None else None, G_, K_, STEP,
                                  *[C.c_void_p(q) for q in p], C.c_void_p(work.data_ptr()),
                                  work.numel() if wb is None else wb, s)
    assert call() == 0
    bad, neg = cols.copy(), cols.copy()
    bad[1] = T * F
    neg[0] = -1
    nulls = [dict(out=[0 if j == i else q for j, q in enumerate(ptrs)]) for i in range(6)]
    for kw in [dict(N_=0), dict(G_=0), dict(K_=0), dict(K_=1025), dict(col=bad), dict(col=neg), dict(col=None),
               dict(x_=0)] + nulls:
        assert call(**kw) == ERR_ARG, kw
    for args in ((0, G, K), (N, 0, K), (N, G, 0), (N, G, 1025)):
        assert lib.lfmq_chain_ale_work_bytes(eng._handles, 1, *args, C.byref(n)) == ERR_ARG, args
    assert lib.lfmq_chain_ale_work_bytes(eng._handles, 1, N, G, K, None) == ERR_ARG
    assert lib.lfmq_chain_ale_work_bytes(eng._handles, 0, N, G, K, C.byref(n)) == ERR_ARG
    assert call(wb=work.numel() - 1) == ERR_WORKSPACE
    assert 'work needs %d bytes' % work.numel() in Nv.load().lfmq_last_error().decode()
    torch.cuda.synchronize()
    eng.close()


# ---- the CLI on the synthetic dataset ----------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def workdir(tmp_path_factory):
    from lfm_quant_b200.scripts.synthetic import write_open_dataset, write_system_test_conf
    d = tmp_path_factory.mktemp('ale')
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


def _check_ale_dat(path, outputs, bins):
    df = pd.read_csv(path, sep=' ', dtype={'field': str}, float_precision='round_trip')
    assert list(df.columns) == ['field', 'edge_idx', 'edge', 'n'] + [
        '%s_%s' % (k, o) for o in outputs for k in ('ale', 'local', 'local_sd')]
    for _, rows in df.groupby('field', sort=False):
        kf = len(rows) - 1
        assert 1 <= kf <= bins and rows['edge_idx'].tolist() == list(range(kf + 1))
        assert (np.diff(rows['edge'].to_numpy()) > 0).all() and rows['n'].iloc[0] == 0 and (rows['n'].iloc[1:] > 0).all()
        for o in outputs:
            a = rows['ale_' + o].to_numpy()
            assert np.isfinite(a).all() and rows['local_' + o].isna().iloc[0]
            n = rows['n'].to_numpy()[1:]
            assert abs((n * 0.5 * (a[:-1] + a[1:])).sum() / n.sum()) < 1e-5 * max(1.0, np.abs(a).max())
    return df


@pytest.mark.parametrize('name,extra,outputs', [
    ('point', ['--dropout', '0.1'], ['norm_preds_1']),
    ('uq', UQ, ['norm_preds_1', 'norm_variance_1']),
])
def test_cli_writes_ale_dat_and_leaves_preds_dat_alone(workdir, cli, name, extra, outputs):
    m = workdir / 'experiments' / ('ale-' + name)
    args = ['--model_dir', 'ale-' + name] + extra
    cli(*args, '--train=True')
    for prec in ('fp32', 'bf16'):
        cli(*args, '--train=False', '--precision', prec)
        plain = (m / 'pred' / 'preds.dat').read_bytes()
        assert not (m / 'pred' / 'ale.dat').exists()
        cli(*args, '--train=False', '--precision', prec, '--ale_bins', '6')
        assert (m / 'pred' / 'preds.dat').read_bytes() == plain, prec
        df = _check_ale_dat(m / 'pred' / 'ale.dat', outputs, 6)
        print('%s %s: %d fields, %d rows' % (name, prec, df['field'].nunique(), len(df)))
        (m / 'pred' / 'ale.dat').unlink()


def test_cli_walk_forward_stacks_the_origins_ale(workdir, cli):
    origins = [199612, 199712]
    args = ['--training_type', 'iterative', '--split_date', '199612', '--end_date', '199812', '--model_dir', 'ale-wf',
            '--NPE', '2']
    cli(*args, '--train=True')
    cli(*args, '--train=False', '--ale_bins', '4')
    wf = workdir / 'experiments' / 'ale-wf'
    got = pd.read_csv(wf / 'walk_forward_ale.dat', sep=' ', dtype={'field': str}, float_precision='round_trip')
    own = [pd.read_csv(wf / ('system-test-wf-%d' % o) / 'pred' / 'ale.dat', sep=' ', dtype={'field': str},
                       float_precision='round_trip').assign(origin=o) for o in origins]
    pd.testing.assert_frame_equal(got, pd.concat(own, ignore_index=True))
    assert sorted(set(got['origin'])) == origins
