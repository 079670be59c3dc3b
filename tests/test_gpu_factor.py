"""Lookahead factor backtests on the H100 (DESIGN.md section 5k): lfmq_factor_eval against factor_oracle (integers
exactly, fp64 within 1e-12, NaN in the same places), identical bits across calls and row permutations, the refusals,
and the CLI on the synthetic dataset for every model kind and a walk-forward run, with preds.dat left byte-identical."""
import ctypes as C

import numpy as np
import pandas as pd
import pytest
import torch

import factor_oracle as fo
from lfm_quant_b200 import _native as N
from lfm_quant_b200.engine import factor_eval

pytestmark = pytest.mark.gpu
ERR_ARG = 1
KEYS = ('n', 'bucket_n', 'n_pair', 'ic', 'bucket_mean', 'spread', 'turnover')


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _run(date, company, score, measure, Q):
    out = factor_eval(_cuda(np.asarray(date, np.int32)), _cuda(np.asarray(company, np.int32)),
                      _cuda(np.atleast_2d(score)), _cuda(np.atleast_2d(measure)), Q)
    return {k: v.cpu().numpy() for k, v in out.items()}


def _check(got, want, measure):
    for k in ('n', 'bucket_n', 'n_pair'):
        assert np.array_equal(got[k], want[k]), k
    scale = np.array([np.nanmax(np.abs(np.where(np.isfinite(m), m, np.nan))) if np.isfinite(m).any() else 1.0
                      for m in np.atleast_2d(measure)])
    for k in ('ic', 'turnover', 'bucket_mean', 'spread'):
        g, w = got[k], want[k]
        assert np.array_equal(np.isnan(g), np.isnan(w)), (k, np.argwhere(np.isnan(g) != np.isnan(w))[:5])
        f = ~np.isnan(w)
        if k in ('bucket_mean', 'spread'):
            # sums of the measure in another order: within 1e-12 of the measure's scale
            s = np.broadcast_to(scale[None, :, None, None] if k == 'bucket_mean' else scale[None, :, None], w.shape)
            assert np.all(np.abs(g[f] - w[f]) <= 1e-12 * s[f]), k
        else:
            assert np.all(np.abs(g[f] - w[f]) <= 1e-12 * np.maximum(np.abs(w[f]), 1e-300)), k


def _close(g, w, scale, what):
    """NaN in the same places; elsewhere within 1e-12 relative, or of `scale` (sums of the measure in another order)."""
    assert np.array_equal(np.isnan(g), np.isnan(w)), what
    f = ~np.isnan(w)
    tol = 1e-12 * (np.maximum(np.abs(w), 1e-300) if scale is None else np.broadcast_to(scale, w.shape))
    assert np.all(np.abs(g[f] - w[f]) <= tol[f]), what


def _problem(N_, D, G, M, seed, ties=0.1, nan=0.05, companies=None):
    rng = np.random.RandomState(seed)
    companies = companies or max(N_ // D + N_ // (4 * D) + 1, 1)
    # distinct (date, company) pairs, in a shuffled row order
    pairs = rng.choice(D * companies, size=N_, replace=False)
    date, company = (pairs // companies).astype(np.int32), (pairs % companies).astype(np.int32) * 7 - 1000
    score = rng.normal(size=(G, N_))
    t = rng.uniform(size=(G, N_)) < ties
    score[t] = np.float64(np.float32(np.round(score[t], 1)))           # heavy ties
    score[:, ::17] = 0.0
    score[:, 1::17] = -0.0                                             # -0 ties +0
    score[rng.uniform(size=(G, N_)) < nan] = np.nan
    score[:, 5::97] = np.inf
    measure = rng.standard_t(4, size=(M, N_)) + 0.1 * score[:1].clip(-3, 3)
    measure[rng.uniform(size=(M, N_)) < nan] = np.nan
    measure[:, ::13] = np.round(measure[:, ::13])
    return date, company, score, measure


CASES = [
    # N, D, G, M, Q
    (200, 5, 1, 1, 2),
    (1000, 20, 3, 2, 10),
    (1000, 1, 8, 4, 100),          # a single date, every cap
    (300, 100, 2, 2, 5),           # dates of 0 to 4 rows: n < 3 and empty top buckets
    (50, 10, 2, 1, 100),           # Q > n: empty buckets everywhere
    (200_000, 4096, 2, 2, 10),
]


@pytest.mark.parametrize('N_,D,G,M,Q', CASES)
def test_matches_oracle(N_, D, G, M, Q):
    date, company, score, measure = _problem(N_, D, G, M, seed=N_ + D + Q)
    got = _run(date, company, score, measure, Q)
    _check(got, fo.evaluate(date, company, score, measure, Q, D=int(date.max()) + 1), measure)


def test_one_company_and_all_tied_dates():
    date = np.array([0, 1, 1, 1, 2, 2, 2, 2], np.int32)
    company = np.array([5, 1, 2, 3, 1, 2, 3, 4], np.int32)
    score = np.array([[1.0, 2.0, 2.0, 2.0, 0.0, -0.0, 1.0, np.nan]])
    measure = np.array([[1.0, 2.0, 3.0, 4.0, 1.0, 1.0, 1.0, 1.0]])
    got = _run(date, company, score, measure, 3)
    want = fo.evaluate(date, company, score, measure, 3)
    _check(got, want, measure)
    assert np.isnan(got['ic']).all()          # n < 3, a tied score, a constant measure
    assert got['bucket_n'][0, 1].tolist() == [0, 3, 0]


def test_large_matches_oracle_and_bits_are_stable():
    N_, D, G, M, Q = 2 ** 20, 600, 2, 2, 10
    date, company, score, measure = _problem(N_, D, G, M, seed=11)
    a = _run(date, company, score, measure, Q)
    _check(a, fo.evaluate(date, company, score, measure, Q, D=D), measure)
    b = _run(date, company, score, measure, Q)
    p = np.random.RandomState(1).permutation(N_)
    c = _run(date[p], company[p], score[:, p], measure[:, p], Q)
    for k in KEYS:
        assert a[k].tobytes() == b[k].tobytes() == c[k].tobytes(), k


def test_call_captures_in_a_cuda_graph():
    # the call does not synchronise with the host: it captures into a CUDA graph, here with more dates (600) than the
    # per-segment sorts of CUB's DeviceSegmentedSort handle without a host round trip, and the replay gives its bits
    N_, D, G, M, Q = 50_000, 600, 2, 2, 10
    date, company, score, measure = _problem(N_, D, G, M, seed=5)
    want = _run(date, company, score, measure, Q)
    lib = N.load()
    n = C.c_uint64(0)
    N.check(lib.lfmq_factor_eval_work_bytes(N_, D, G, M, Q, C.byref(n)))
    work = torch.empty(n.value, dtype=torch.uint8, device='cuda')
    ins = [_cuda(date), _cuda(company), _cuda(score), _cuda(measure)]
    i32, f64 = dict(dtype=torch.int32, device='cuda'), dict(dtype=torch.float64, device='cuda')
    outs = dict(n=torch.empty(G, D, **i32), bucket_n=torch.empty(G, D, Q, **i32), n_pair=torch.empty(G, M, D, **i32),
                ic=torch.empty(G, M, D, **f64), bucket_mean=torch.empty(G, M, D, Q, **f64),
                spread=torch.empty(G, M, D, **f64), turnover=torch.empty(G, D, **f64))
    p = lambda t: C.c_void_p(t.data_ptr())       # noqa: E731
    graph, side = torch.cuda.CUDAGraph(), torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        with torch.cuda.graph(graph, stream=side):
            rc = lib.lfmq_factor_eval(p(ins[0]), p(ins[1]), N_, D, p(ins[2]), G, p(ins[3]), M, Q,
                                      *[p(outs[k]) for k in KEYS], p(work), n.value,
                                      C.c_void_p(side.cuda_stream))
    assert rc == 0, lib.lfmq_last_error()
    graph.replay()
    torch.cuda.synchronize()
    for k in KEYS:
        assert outs[k].cpu().numpy().tobytes() == want[k].tobytes(), k


def test_refusals():
    lib = N.load()
    n = C.c_uint64(0)
    for args in ((0, 5, 1, 1, 10), (10, 0, 1, 1, 10), (10, 5, 0, 1, 10), (10, 5, 9, 1, 10), (10, 5, 1, 0, 10),
                 (10, 5, 1, 5, 10), (10, 5, 1, 1, 1), (10, 5, 1, 1, 101)):
        assert lib.lfmq_factor_eval_work_bytes(*args, C.byref(n)) == ERR_ARG, args
    N.check(lib.lfmq_factor_eval_work_bytes(10, 2, 1, 1, 5, C.byref(n)))
    work = torch.empty(n.value, dtype=torch.uint8, device='cuda')
    i32 = torch.zeros(10, dtype=torch.int32, device='cuda')
    comp = torch.arange(10, dtype=torch.int32, device='cuda')
    f64 = torch.zeros(10 * 2 * 5, dtype=torch.float64, device='cuda')
    ptrs = [C.c_void_p(t.data_ptr()) for t in (i32, comp)]
    o32 = [torch.zeros(10, dtype=torch.int32, device='cuda') for _ in range(3)]
    out = [C.c_void_p(t.data_ptr()) for t in o32 + [f64] * 4]
    nul = C.c_void_p(0)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def call(p, o, G=1, Q=5, wb=n.value):
        return lib.lfmq_factor_eval(p[0], p[1], 10, 2, C.c_void_p(f64.data_ptr()), G, C.c_void_p(f64.data_ptr()), 1,
                                    Q, *o, C.c_void_p(work.data_ptr()), wb, stream)
    for k in range(2):
        assert call([nul if j == k else v for j, v in enumerate(ptrs)], out) == ERR_ARG
    for k in range(7):
        assert call(ptrs, [nul if j == k else v for j, v in enumerate(out)]) == ERR_ARG
    assert call(ptrs, out, G=9) == ERR_ARG and call(ptrs, out, Q=1) == ERR_ARG
    assert call(ptrs, out, wb=n.value - 1) != 0            # too little work
    assert call(ptrs, out) == 0
    torch.cuda.synchronize()


# ---- the CLI on the synthetic dataset ----------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def workdir(tmp_path_factory):
    from lfm_quant_b200.scripts.synthetic import write_open_dataset, write_system_test_conf
    d = tmp_path_factory.mktemp('factor')
    path = d / 'datasets' / 'open-dataset.dat'
    write_open_dataset(str(path), n_keys=30, n_months=420, seed=9)
    # this copy's own return column: each row's change in market cap over the month that ends at it
    data = pd.read_csv(path, sep=' ', dtype={'gvkey': str})
    data['ret'] = data.groupby('gvkey')['mrkcap'].pct_change()
    data.to_csv(path, sep=' ', index=False)
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


Q = 5
RET = ['--factor_return_field', 'ret', '--factor_horizon', '3']


def _oracle_files(workdir, preds, steps, uq, ret, forecast_n=12):
    """(per-date frame, summary dict) the oracle gives for a preds.dat frame."""
    sc = fo.scores(preds, steps, uq)
    names = ['lfm_%d' % s for s in range(1, steps + 1)] + ['qfm'] + (
        ['lfm_risk_%d' % s for s in range(1, steps + 1)] if uq else [])
    date = preds['date'].astype(np.int64).to_numpy()
    gvkey = preds['gvkey'].astype(str).to_numpy()
    meas = [preds['targets_1'].to_numpy(np.float64) / preds['seq_norm'].to_numpy(np.float64)]
    horizons = [forecast_n]
    if ret:
        data = pd.read_csv(workdir / 'datasets' / 'open-dataset.dat', sep=' ', dtype={'gvkey': str})
        rows = {(g, int(m)): r for g, m, r in zip(data['gvkey'], fo.months(data['date']), data['ret'])}
        meas.append(fo.forward_returns(rows, date, gvkey, 3))
        horizons.append(3)
    dates, date_idx = np.unique(date, return_inverse=True)
    company = np.unique(gvkey, return_inverse=True)[1]
    out = fo.evaluate(date_idx, company, np.stack([sc[k] for k in names]), np.stack(meas), Q, D=len(dates))
    return names, dates, out, fo.summary(dates, out, Q, horizons), np.stack(meas)


def _check_files(workdir, per_date_path, summary_path, preds, steps, uq, ret):
    names, dates, out, summ, meas = _oracle_files(workdir, preds, steps, uq, ret)
    got = pd.read_csv(per_date_path, sep=' ', float_precision='round_trip')
    M = 2 if ret else 1
    assert list(got.columns) == (['date', 'factor', 'measure', 'n', 'n_pair', 'ic'] + ['q%d' % q for q in
                                 range(1, Q + 1)] + ['spread', 'turnover'])
    assert len(got) == len(dates) * len(names) * M
    measures = ['yield', 'ret'][:M]
    g_of = {n: i for i, n in enumerate(names)}
    m_of = {n: i for i, n in enumerate(measures)}
    d_of = {int(d): i for i, d in enumerate(dates)}
    gi, mi, di = (got['factor'].map(g_of).to_numpy(), got['measure'].map(m_of).to_numpy(),
                  got['date'].map(d_of).to_numpy())
    assert (got['n'].to_numpy() == out['n'][gi, di]).all()
    assert (got['n_pair'].to_numpy() == out['n_pair'][gi, mi, di]).all()
    scale = np.array([np.max(np.abs(m[np.isfinite(m)])) for m in meas])[mi]
    for col, want, tol in (('ic', out['ic'][gi, mi, di], None), ('turnover', out['turnover'][gi, di], None),
                           ('spread', out['spread'][gi, mi, di], scale)):
        _close(got[col].to_numpy(), want, tol, col)
    for q in range(Q):
        _close(got['q%d' % (q + 1)].to_numpy(), out['bucket_mean'][gi, mi, di, q], scale, q)
    s = pd.read_csv(summary_path, sep=' ', float_precision='round_trip')
    assert len(s) == len(names) * M
    for _, row in s.iterrows():
        want = summ[(g_of[row['factor']], m_of[row['measure']])]
        for col, v in want.items():
            assert (np.isnan(v) and np.isnan(row[col])) or abs(row[col] - v) <= 1e-9 * max(1.0, abs(v)), (
                row['factor'], row['measure'], col, row[col], v)
    return got, s


UQ = ['--nn_type', 'RNNUqRangeEstimate', '--UQ=True', '--dropout', '0.1', '--recurrent_dropout', '0.1']
MODELS = [('lstm', [], 1, False, False), ('lstm', [], 1, False, True), ('gru-uq', ['--rnn_cell', 'gru'] + UQ, 1, True, True),
          ('chain', ['--forecast_steps', '2', '--forecast_steps_weights', '1.0-0.5'], 2, False, True),
          ('linear', ['--nn_type', 'MLPLinearPointEstimate'], 1, False, True)]


@pytest.mark.parametrize('name,extra,steps,uq,ret', MODELS)
def test_cli_writes_factor_files_and_leaves_preds_dat_alone(workdir, cli, name, extra, steps, uq, ret):
    model_dir = 'factor-%s' % name
    m = workdir / 'experiments' / model_dir
    args = ['--model_dir', model_dir] + extra
    if not (m / 'chkpts').exists():
        cli(*args, '--train=True')
    cli(*args, '--train=False')
    plain = (m / 'pred' / 'preds.dat').read_bytes()
    cli(*args, '--train=False', '--factor_quantiles', str(Q), *(RET if ret else []))
    assert (m / 'pred' / 'preds.dat').read_bytes() == plain
    preds = pd.read_csv(m / 'pred' / 'preds.dat', sep=' ', dtype={'gvkey': str}, float_precision='round_trip')
    got, s = _check_files(workdir, m / 'pred' / 'factor_dates.dat', m / 'pred' / 'factor.dat', preds, steps, uq, ret)
    if uq:
        assert 'lfm_risk_1' in set(got['factor'])
    if not ret:           # the current value need not be written for qfm
        cli(*args, '--train=False', '--factor_quantiles', str(Q), '--write_inp_to_out_file=False')
        again = pd.read_csv(m / 'pred' / 'factor_dates.dat', sep=' ', float_precision='round_trip')
        assert again.equals(got)


def test_cli_naive_model_lfm_equals_qfm(workdir, cli):
    import shutil
    scales = workdir / 'experiments' / 'naive-scales.dat'
    src = workdir / 'experiments' / 'factor-linear' / 'scales.dat'
    if not src.exists():
        cli('--model_dir', 'factor-linear', '--nn_type', 'MLPLinearPointEstimate', '--train=True')
    shutil.copy(src, scales)
    args = ['--nn_type', 'NaivePointEstimate', '--model_dir', 'factor-naive', '--scalesfile', str(scales),
            '--train=False']
    cli(*args)
    m = workdir / 'experiments' / 'factor-naive'
    plain = (m / 'pred' / 'preds.dat').read_bytes()
    cli(*args, '--factor_quantiles', str(Q), *RET)
    assert (m / 'pred' / 'preds.dat').read_bytes() == plain
    preds = pd.read_csv(m / 'pred' / 'preds.dat', sep=' ', dtype={'gvkey': str}, float_precision='round_trip')
    got, s = _check_files(workdir, m / 'pred' / 'factor_dates.dat', m / 'pred' / 'factor.dat', preds, 1, False, True)
    a = got[got.factor == 'lfm_1'].drop(columns='factor').reset_index(drop=True)
    b = got[got.factor == 'qfm'].drop(columns='factor').reset_index(drop=True)
    assert a.equals(b)


def test_cli_walk_forward_backtest(workdir, cli):
    args = ['--training_type', 'iterative', '--split_date', '199612', '--end_date', '199812', '--model_dir',
            'factor-wf', '--NPE', '2']
    cli(*args, '--train=True')
    cli(*args, '--train=False', '--factor_quantiles', str(Q), *RET)
    wf = workdir / 'experiments' / 'factor-wf'
    preds = pd.read_csv(wf / 'walk_forward_preds.dat', sep=' ', dtype={'gvkey': str}, float_precision='round_trip')
    _, s = _check_files(workdir, wf / 'walk_forward_factor_dates.dat', wf / 'walk_forward_factor.dat', preds, 1, False,
                        True)
    for origin in (199612, 199712):       # the origins run no backtest of their own
        assert not (wf / ('system-test-wf-%d' % origin) / 'pred' / 'factor.dat').exists()
    print(s[['factor', 'measure', 'n_dates', 'mean_ic', 't_ic', 'mean_spread', 'nw_lag']].to_string())
