"""Lookahead factor backtests without a GPU (DESIGN.md section 5k): the oracle's IC, bucket rule, turnover and
Newey-West t-statistics, forward_returns and the factor builders, the flags and their refusals, the file layouts, the
C ABI's symbols and refusals, and a no-spill compile of csrc/factor.cu."""
import ctypes as C
import math
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pandas as pd
import pytest
import scipy.stats

import factor_oracle as fo
from lfm_quant_b200 import _native as N
from lfm_quant_b200.scripts.predict import (factor_codes, factor_dates_table, factor_measures, factor_scores,
                                            factor_summary, forward_returns, newey_west_lag, newey_west_t)
from lfm_quant_b200.scripts.runtime.model_execution import ModelExecution, check_factor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ties(n, seed):
    rng = np.random.RandomState(seed)
    return np.round(rng.normal(size=n), 1), np.round(rng.normal(size=n) + 0.3 * np.arange(n) / n, 1)


@pytest.mark.parametrize('n,seed', [(5, 0), (40, 1), (500, 2)])
def test_oracle_ic_is_spearmanr_on_heavy_ties(n, seed):
    x, y = _ties(n, seed)
    x[::3] = 0.0
    assert abs(fo.spearman(x, y) - scipy.stats.spearmanr(x, y)[0]) < 1e-13
    assert np.isnan(fo.spearman(np.ones(10), np.arange(10.0))) and np.isnan(fo.spearman(x[:2], y[:2]))


@pytest.mark.parametrize('Q', [2, 3, 10, 100])
def test_bucket_rule_properties(Q):
    rng = np.random.RandomState(Q)
    n = 997
    s = np.round(rng.normal(size=n), 1)
    out = fo.evaluate(np.zeros(n, np.int32), np.arange(n, dtype=np.int32), s, s, Q)
    r = scipy.stats.rankdata(s)
    b = np.floor((r - 0.5) * Q / n).astype(int) + 1
    assert b.min() >= 1 and b.max() <= Q
    for v in np.unique(s):
        assert len(set(b[s == v].tolist())) == 1
    sizes = out['bucket_n'][0, 0]
    assert sizes.sum() == n and sizes.tolist() == np.bincount(b - 1, minlength=Q).tolist()
    # each boundary moves by at most half a tie group, so a bucket's size differs from n / Q by at most the largest
    # tie group + 1; without ties the sizes differ by at most 1
    largest_tie = np.unique(s, return_counts=True)[1].max()
    assert np.all(np.abs(sizes - n / Q) <= largest_tie + 1)
    untied = fo.evaluate(np.zeros(n, np.int32), np.arange(n, dtype=np.int32), np.arange(n) * 1.0, s, Q)['bucket_n']
    assert untied.max() - untied.min() <= 1


def test_turnover_by_hand():
    # three dates, Q = 2; the top half by score: d0 {0, 1}, d1 {1, 2}, d2 {2} (d2 has three rows, two of them tied at
    # rank 1.5, so that company 2 is alone on top)
    company = np.array([0, 1, 2, 3, 0, 1, 2, 3, 0, 2, 3], np.int32)
    date = np.array([0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2], np.int32)
    score = np.array([4, 3, 2, 1, 1, 4, 3, 2, 1, 3, 1], np.float64)
    out = fo.evaluate(date, company, score, score, 2)
    assert np.isnan(out['turnover'][0, 0])
    assert out['turnover'][0, 1] == 0.5 and out['turnover'][0, 2] == 0.0
    assert out['bucket_n'][0].tolist() == [[2, 2], [2, 2], [2, 1]]


@pytest.mark.parametrize('lag', [0, 11])
def test_newey_west_against_direct(lag):
    rng = np.random.RandomState(lag)
    x = np.cumsum(rng.normal(size=60)) * 0.1 + 0.2
    x[[5, 17]] = np.nan
    f = x[np.isfinite(x)]
    n = len(f)
    e = f - f.mean()
    gam = [np.dot(e[k:], e[:n - k]) / n for k in range(lag + 1)]
    var = gam[0] + 2 * sum((1 - k / (lag + 1)) * gam[k] for k in range(1, lag + 1))
    want = f.mean() / math.sqrt(var / n)
    assert abs(newey_west_t(x, lag) - want) <= 1e-12 * abs(want)
    assert abs(fo.nw_t(x, lag) - want) <= 1e-12 * abs(want)
    if lag == 0:
        assert abs(want - f.mean() / (f.std(ddof=0) / math.sqrt(n))) <= 1e-12 * abs(want)
    assert np.isnan(newey_west_t([1.0], lag)) and np.isnan(newey_west_t([2.0, 2.0, 2.0], lag))


def test_newey_west_lag_rule():
    monthly = [19990131, 19990228, 19990331]
    assert newey_west_lag(monthly, 12) == 11 == fo.nw_lag(monthly, 12)
    assert newey_west_lag([199901, 199904, 199907], 12) == 3 == fo.nw_lag([199901, 199904, 199907], 12)
    assert newey_west_lag(monthly, 1) == 0 and newey_west_lag([19990131], 12) == 0


def test_forward_returns_with_gaps_and_nans():
    data = pd.DataFrame({'date': [20000131, 20000229, 20000331, 20000430, 20000531, 20000131, 20000331, 20000430],
                         'gvkey': ['a'] * 5 + ['b'] * 3,
                         'r': [0.5, 0.1, 0.2, np.nan, 0.3, 9.0, 0.1, 0.2]})
    date = np.array([20000131, 20000229, 20000331, 20000131, 20000229, 20000331, 20000531])
    gvkey = np.array(['a', 'a', 'a', 'b', 'b', 'b', 'a'])
    got = forward_returns(data, 'r', date, gvkey, 2)
    want = [1.1 * 1.2 - 1, np.nan, np.nan, np.nan, 1.1 * 1.2 - 1, np.nan, np.nan]
    assert np.allclose(got, want, equal_nan=True, rtol=0, atol=1e-15)
    rows = {(g, int(m)): r for g, m, r in zip(data['gvkey'], fo.months(data['date']), data['r'])}
    assert np.allclose(fo.forward_returns(rows, date, gvkey, 2), got, equal_nan=True, rtol=0, atol=1e-15)
    assert np.allclose(forward_returns(data, 'r', date, gvkey, 1), [0.1, 0.2, np.nan, np.nan, 0.1, 0.2, np.nan],
                       equal_nan=True)
    with pytest.raises(ValueError, match='two rows'):
        forward_returns(pd.concat([data, data.iloc[:1]]), 'r', date, gvkey, 1)


def _frame(uq=False, steps=1):
    rng = np.random.RandomState(3)
    n = 12
    df = pd.DataFrame({'date': pd.to_datetime(['19990131'] * 6 + ['19990228'] * 6), 'gvkey': list('abcdef') * 2,
                       'seq_norm': rng.uniform(0.5, 3, n), 'inp_t0': rng.normal(size=n)})
    for s in range(1, steps + 1):
        df['targets_%d' % s] = rng.normal(size=n)
        df['preds_%d' % s] = rng.normal(size=n)
        if uq:
            df['variance_%d' % s] = rng.uniform(0.1, 1, n)
    return df


def test_factor_scores_and_naive_identity():
    df = _frame()
    df['preds_1'] = df['inp_t0']            # the naive forecast: the current value
    names, score = factor_scores(df, 1, False)
    assert names == ['lfm_1', 'qfm'] and np.array_equal(score[0], score[1])
    ref = fo.scores(df, 1, False)
    assert np.array_equal(score[1], ref['qfm'])
    df = _frame(uq=True, steps=2)
    df.loc[3, 'variance_2'] = 0.0
    df.loc[4, 'variance_2'] = np.nan
    names, score = factor_scores(df, 2, True)
    assert names == ['lfm_1', 'lfm_2', 'qfm', 'lfm_risk_1', 'lfm_risk_2']
    ref = fo.scores(df, 2, True)
    for k, name in enumerate(names):
        assert np.array_equal(score[k], ref[name], equal_nan=True), name
    assert np.isnan(score[4, 3]) and np.isnan(score[4, 4]) and np.isfinite(score[4]).sum() == 10
    m_names, measure, horizons = factor_measures(df, 12, np.arange(12.0), 3)
    assert m_names == ['yield', 'ret'] and horizons == [12, 3]
    assert np.array_equal(measure[0], df['targets_1'].to_numpy() / df['seq_norm'].to_numpy())


def test_codes_refuse_duplicate_rows():
    dates, idx, comp = factor_codes([19990228, 19990131, 19990228], ['b', 'a', 'a'])
    assert dates.tolist() == [19990131, 19990228] and idx.tolist() == [1, 0, 1] and comp.tolist() == [1, 0, 0]
    with pytest.raises(ValueError, match='two rows for one'):
        factor_codes([19990131, 19990131], ['a', 'a'])


def test_file_layouts_from_a_stub():
    dates = [19990131, 19990228, 19990331]
    rng = np.random.RandomState(0)
    n = 60
    date, comp = np.repeat(np.arange(3), 20).astype(np.int32), np.tile(np.arange(20), 3).astype(np.int32)
    score, measure = rng.normal(size=(2, n)), rng.normal(size=(1, n))
    Q = 4
    out = fo.evaluate(date, comp, score, measure, Q)
    t = factor_dates_table(dates, ['lfm_1', 'qfm'], ['yield'], out, Q)
    assert list(t.columns) == ['date', 'factor', 'measure', 'n', 'n_pair', 'ic', 'q1', 'q2', 'q3', 'q4', 'spread',
                               'turnover']
    assert len(t) == 3 * 2 and t['date'].tolist() == [19990131] * 2 + [19990228] * 2 + [19990331] * 2
    assert t['factor'].tolist()[:2] == ['lfm_1', 'qfm'] and (t['n'] == 20).all()
    row = t.iloc[3]
    assert row['ic'] == out['ic'][1, 0, 1] and row['q4'] == out['bucket_mean'][1, 0, 1, 3]
    s = factor_summary(dates, ['lfm_1', 'qfm'], ['yield'], out, Q, [12])
    assert list(s.columns) == (['factor', 'measure', 'n_dates', 'mean_ic', 'sd_ic', 'ir', 'hit', 't_ic']
                               + ['mean_q%d' % q for q in range(1, 5)]
                               + ['mean_spread', 'sd_spread', 't_spread', 'mean_turnover', 'nw_lag'])
    ref = fo.summary(dates, out, Q, [12])
    for g in range(2):
        for col, v in ref[(g, 0)].items():
            got = s.iloc[g][col]
            assert (np.isnan(v) and np.isnan(got)) or abs(got - v) <= 1e-12 * max(1.0, abs(v)), (g, col, got, v)
    assert (s['nw_lag'] == 11).all() and (s['n_dates'] == 3).all()


# ---- flags -------------------------------------------------------------------------------------------------------
class _C(object):
    def __init__(self, **kw):
        self.__dict__.update(dict(factor_quantiles=10, factor_return_field=None, factor_horizon=1, train=False,
                                  num_procs=1, UQ=False, forecast_steps=1, training_type='fixed_dates',
                                  write_inp_to_out_file=True, data_dir='.', datafile='x.dat'))
        self.__dict__.update(kw)


@pytest.fixture()
def datafile(tmp_path):
    pd.DataFrame({'date': [200001, 200002], 'gvkey': ['a', 'a'], 'ret': [0.1, np.nan], 'name': ['x', 'y']}).to_csv(
        tmp_path / 'd.dat', sep=' ', index=False)
    return dict(data_dir=str(tmp_path), datafile='d.dat')


@pytest.mark.parametrize('kw,msg', [
    (dict(factor_quantiles=1), r'\[2, 100\]'),
    (dict(factor_quantiles=101), r'\[2, 100\]'),
    (dict(factor_quantiles=-2), r'\[2, 100\]'),
    (dict(train=True), 'train=False'),
    (dict(num_procs=2), 'num_procs'),
    (dict(forecast_steps=4, UQ=True), 'more than 8'),
    (dict(training_type='iterative', write_inp_to_out_file=False), 'write_inp_to_out_file'),
    (dict(factor_quantiles=0, factor_return_field='ret'), 'set --factor_quantiles'),
    (dict(factor_quantiles=0, factor_horizon=3), 'set --factor_quantiles'),
    (dict(factor_horizon=0), '--factor_horizon 0'),
    (dict(factor_return_field='nope'), '--factor_return_field nope: not a numeric column'),
    (dict(factor_return_field='name'), '--factor_return_field name: not a numeric column'),
    (dict(factor_return_field='gvkey'), '--factor_return_field gvkey: not a numeric column'),
    (dict(factor_return_field='date'), '--factor_return_field date: not a numeric column'),
])
def test_refusals(kw, msg, datafile):
    with pytest.raises(ValueError, match=msg):
        check_factor(_C(**dict(datafile, **kw)))


def test_accepted_configs(datafile):
    check_factor(_C(**datafile))
    check_factor(_C(factor_quantiles=0))
    check_factor(_C(factor_return_field='ret', factor_horizon=12, **datafile))
    check_factor(_C(UQ=True, forecast_steps=3))
    check_factor(_C(training_type='iterative'))


def test_model_execution_refuses_before_any_work():
    class Cfg(_C):
        pass
    c = Cfg(train=True, mc_samples=1, ig_steps=0, perm_importance=0, shapley_samples=0, ale_bins=0,
            influence_top_k=0, pred_quantiles=None, conformal_levels=None, conformal_knn=0, validation_size=0.3,
            nn_type='RNNPointEstimate')
    with pytest.raises(ValueError, match='--factor_quantiles'):
        ModelExecution(c)()


def test_flags_parse():
    from lfm_quant_b200.scripts import base_config, configs
    configs.reset()
    try:
        c = base_config.get_configs(['--factor_quantiles', '5', '--factor_return_field', 'ret', '--factor_horizon',
                                     '3'])
        assert (c.factor_quantiles, c.factor_return_field, c.factor_horizon) == (5, 'ret', 3)
        configs.reset()
        c = base_config.get_configs([])
        assert (c.factor_quantiles, c.factor_return_field, c.factor_horizon) == (0, None, 1)
    finally:
        configs.reset()


# ---- the C ABI ---------------------------------------------------------------------------------------------------
def test_symbols_declared_and_exported():
    src = re.sub(r'/\*.*?\*/', '', open(os.path.join(ROOT, 'include', 'lfmq.h')).read(), flags=re.S)
    lib = N.load()
    for name in ('lfmq_factor_eval_work_bytes', 'lfmq_factor_eval'):
        assert re.search(r'\b%s\s*\(' % name, src), name
        assert name in N.SYMBOLS and hasattr(lib, name)


@pytest.mark.parametrize('args', [(0, 5, 1, 1, 10), (-1, 5, 1, 1, 10), (10, 0, 1, 1, 10), (10, 5, 0, 1, 10),
                                  (10, 5, 9, 1, 10), (10, 5, 1, 0, 10), (10, 5, 1, 5, 10), (10, 5, 1, 1, 1),
                                  (10, 5, 1, 1, 101)])
def test_work_bytes_refuses_without_gpu(args):
    lib = N.load()
    n = C.c_uint64(0)
    assert lib.lfmq_factor_eval_work_bytes(*args, C.byref(n)) == 1
    assert b'lfmq_factor_eval_work_bytes' in lib.lfmq_last_error()


def test_eval_refuses_null_pointers_without_gpu():
    lib = N.load()
    nul = C.c_void_p(0)
    assert lib.lfmq_factor_eval(nul, nul, 10, 2, nul, 1, nul, 1, 5, nul, nul, nul, nul, nul, nul, nul, nul, 0,
                                nul) == 1
    assert lib.lfmq_factor_eval_work_bytes(10, 2, 1, 1, 5, None) == 1


# ---- compile -----------------------------------------------------------------------------------------------------
def test_factor_kernels_compile_without_spills():
    nvcc = shutil.which('nvcc') or ('/usr/local/cuda/bin/nvcc' if os.path.exists('/usr/local/cuda/bin/nvcc') else None)
    if nvcc is None:
        pytest.skip('nvcc not found')
    with tempfile.TemporaryDirectory() as d:
        r = subprocess.run([nvcc, '-O3', '-Xptxas', '-v', '-std=c++17', '-gencode', 'arch=compute_90a,code=sm_90a',
                            '--expt-relaxed-constexpr', '-c', os.path.join(ROOT, 'lfm_quant_b200', 'csrc', 'factor.cu'),
                            '-o', os.path.join(d, 'factor.o')], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        # the report of each entry function: its name line, then its stack / spill line
        entries = re.findall(r"Compiling entry function '(\w+)'.*?\n(?:.*\n)*?\s*(\d+) bytes stack frame, (\d+) bytes "
                             r"spill stores, (\d+) bytes spill loads", r.stderr)
        ours = {name: frame for name, *frame in entries if 'factor_' in name}
        for k in ('factor_row_keys_kernel', 'factor_segments_kernel', 'factor_pred_kernel', 'factor_value_keys_kernel',
                  'factor_date_keys_kernel', 'factor_gather_kernel', 'factor_bucket_kernel',
                  'factor_pair_flags_kernel', 'factor_pair_rank_kernel', 'factor_segment_kernel'):
            hits = [frame for name, frame in ours.items() if k in name]
            assert hits, k
            assert all(f == ['0', '0', '0'] for f in hits), (k, hits)


def test_walk_forward_origins_run_no_backtest(tmp_path):
    from lfm_quant_b200.scripts import base_config, configs
    from lfm_quant_b200.scripts.runtime.model_execution import origin_configs
    configs.reset()
    try:
        c = base_config.get_configs(['--training_type', 'iterative', '--start_date', '197501', '--split_date', '199612',
                                     '--end_date', '199812', '--experiments_dir', str(tmp_path), '--factor_quantiles',
                                     '5', '--factor_return_field', 'ret', '--factor_horizon', '3'])
    finally:
        configs.reset()
    _, origins = origin_configs(c)
    assert len(origins) == 2
    for _, _, pred in origins:       # an origin's conf, run alone, passes check_factor
        assert (pred.factor_quantiles, pred.factor_return_field, pred.factor_horizon) == (0, None, 1)
        check_factor(pred)
    assert (c.factor_quantiles, c.factor_return_field, c.factor_horizon) == (5, 'ret', 3)
