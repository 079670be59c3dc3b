"""Split-conformal intervals without a GPU (DESIGN.md section 5j): the oracle's rank rule and its coverage on
exchangeable residuals, the flags and their refusals, the intervals.dat / coverage.dat layouts and a no-spill compile of
csrc/conformal.cu."""
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pandas as pd
import pytest

import conformal_oracle as co
from lfm_quant_b200.scripts import base_config
from lfm_quant_b200.scripts.predict import (conformal_level_name, conformal_subsets, coverage_table,
                                            interval_table)
from lfm_quant_b200.scripts.runtime.model_execution import ModelExecution, check_conformal

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_rank_rule_and_infinity():
    y = np.array([[0.0, 1.0, 2.0, 3.0, np.nan]], dtype=np.float32)
    pred = np.zeros_like(y)
    n, srt, q = co.calibrate(pred, y, [0.5, 0.8, 0.9])
    assert n.tolist() == [4]
    # ceil(5 * 0.5) = 3 -> 2.0; ceil(5 * 0.8) = 4 -> 3.0; ceil(5 * 0.9) = 5 > 4 -> inf
    assert q.tolist() == [[2.0, 3.0, np.inf]]
    assert np.isnan(srt[0, -1])
    lo, hi, p = co.apply(np.array([[1.0]], dtype=np.float32), n, srt, q, y=np.array([[3.5]], dtype=np.float32))
    assert lo[0, 0].tolist() == [-1.0, -2.0, -np.inf] and hi[0, 0].tolist() == [3.0, 4.0, np.inf]
    # r = 2.5: scores >= 2.5 are {3.0}: p = (1 + 1) / 5
    assert p[0, 0] == np.float32(2) / np.float32(5)


def test_pvalue_unknown_target_and_empty_calibration():
    n, srt, q = co.calibrate(np.zeros((1, 3), np.float32), np.full((1, 3), np.nan, np.float32), [0.1])
    assert n.tolist() == [0] and np.isinf(q).all()
    _, _, p = co.apply(np.zeros((1, 2), np.float32), n, srt, q, y=np.array([[np.nan, 1.0]], np.float32))
    assert np.isnan(p[0, 0]) and p[0, 1] == 1.0


def test_scores_are_float32_arithmetic():
    rng = np.random.RandomState(0)
    pred, y = rng.normal(size=(2, 100)).astype(np.float32), rng.normal(size=(2, 100)).astype(np.float32)
    sc = rng.uniform(0.1, 2, size=(2, 100)).astype(np.float32)
    r = co.scores(pred, y, sc)
    assert r.dtype == np.float32 and np.array_equal(r, np.abs(y - pred) / sc)


@pytest.mark.parametrize('level', [0.5, 0.8, 0.9])
def test_coverage_on_exchangeable_residuals(level):
    """Split-conformal validity: with n exchangeable calibration scores and one more test score, the coverage over many
    seeded draws lies in [l, l + 1/(n + 1)] within binomial error."""
    n, draws = 19, 2000
    rng = np.random.RandomState(7)
    covered = np.zeros(draws)
    for d in range(draws):
        e = rng.standard_t(3, size=n + 1).astype(np.float32)
        _, srt, q = co.calibrate(np.zeros((1, n), np.float32), e[None, :n], [level])
        covered[d] = abs(e[n]) <= q[0, 0]
    lo, hi = level, level + 1.0 / (n + 1)
    se = np.sqrt(hi * (1 - lo) / draws)
    assert lo - 4 * se <= covered.mean() <= hi + 4 * se, covered.mean()


def test_knn_oracle_ties_to_lower_index():
    b = np.array([[0.0, 0.0], [1.0, 0.0], [0.0, 0.0], [5.0, 5.0]])
    idx, d2, mean = co.knn(np.array([[0.0, 0.0]]), b, 3, value=np.array([1.0, 2.0, 3.0, 4.0]))
    assert idx.tolist() == [[0, 2, 1]] and d2[0].tolist() == [0.0, 0.0, 1.0] and mean[0] == 2.0
    idx, d2, _ = co.knn(np.array([[0.0, 0.0]]), b[:1], 3)
    assert idx.tolist() == [[0, -1, -1]] and np.isinf(d2[0, 1:]).all()


# ---- flags -------------------------------------------------------------------------------------------------------
def test_level_parsing():
    assert base_config.conformal_levels(None) is None
    assert base_config.conformal_levels('0.5-0.9') == [0.5, 0.9]
    for bad in ('0.9-0.5', '0-0.5', '0.5-1', 'a', '-'.join(['0.%02d' % i for i in range(1, 35)])):
        with pytest.raises(ValueError, match='--conformal_levels'):
            base_config.conformal_levels(bad)
    assert conformal_level_name(0.9) == '90' and conformal_level_name(0.125) == '12.5'


class _C(object):
    def __init__(self, **kw):
        self.__dict__.update(dict(conformal_levels='0.9', conformal_knn=0, train=False, num_procs=1,
                                  validation_size=0.3, UQ=False, nn_type='RNNPointEstimate', forecast_steps=1))
        self.__dict__.update(kw)


@pytest.mark.parametrize('kw,msg', [
    (dict(train=True), 'train=False'),
    (dict(num_procs=2), 'num_procs'),
    (dict(validation_size=0.0), 'validation_size'),
    (dict(conformal_levels='0.9-0.1'), 'strictly increasing'),
    (dict(conformal_knn=65), r'\[1, 64\]'),
    (dict(conformal_knn=-1), r'\[1, 64\]'),
    (dict(conformal_knn=8, UQ=True, nn_type='RNNUqRangeEstimate'), 'sigma'),
    (dict(conformal_knn=8, nn_type='NaivePointEstimate'), 'NaivePointEstimate'),
    (dict(conformal_knn=8, forecast_steps=2), 'forecast_steps'),
    (dict(conformal_knn=8, conformal_levels=None), 'set --conformal_levels'),
])
def test_refusals(kw, msg):
    with pytest.raises(ValueError, match=msg):
        check_conformal(_C(**kw))


def test_accepted_configs():
    check_conformal(_C())
    check_conformal(_C(conformal_levels=None))
    check_conformal(_C(conformal_knn=16, nn_type='MLPLinearPointEstimate'))
    check_conformal(_C(UQ=True, nn_type='RNNUqRangeEstimate', forecast_steps=2))


def test_model_execution_refuses_before_any_work():
    class Cfg(_C):
        pass
    c = Cfg(train=True, mc_samples=1, ig_steps=0, perm_importance=0, shapley_samples=0, ale_bins=0,
            influence_top_k=0, pred_quantiles=None)
    with pytest.raises(ValueError, match='--conformal_levels'):
        ModelExecution(c)()


# ---- the output files --------------------------------------------------------------------------------------------
def _tables():
    keys = pd.DataFrame({'date': pd.to_datetime(['20000131', '20000131', '20000430']), 'gvkey': ['a', 'b', 'c']})
    levels = [0.5, 0.9]
    S, N, Q = 2, 3, 2
    pred = np.array([[0.0, 1.0, 2.0], [0.5, 0.5, 0.5]], np.float32)
    scale = np.ones((S, N), np.float32)
    qhat = np.array([[0.5, 1.0], [0.25, np.inf]], np.float32)
    lower = pred[:, :, None] - qhat[:, None, :] * scale[:, :, None]
    upper = pred[:, :, None] + qhat[:, None, :] * scale[:, :, None]
    pvalue = np.array([[0.5, np.nan, 1.0], [0.2, np.nan, 0.4]], np.float32)
    seq_norm = np.array([1.0, -2.0, 1.0])
    unscale = lambda v: np.asarray(v, dtype=np.float64) * 10.0 * seq_norm       # noqa: E731
    return keys, levels, pred, scale, qhat, lower, upper, pvalue, seq_norm, unscale


def test_interval_table_layout_and_swap():
    keys, levels, pred, scale, qhat, lower, upper, pvalue, seq_norm, unscale = _tables()
    df = interval_table(keys, levels, lower, upper, scale, pvalue, seq_norm, unscale)
    want = ['date', 'gvkey']
    for s in (1, 2):
        for n in ('50', '90'):
            want += ['norm_lo%s_%d' % (n, s), 'norm_hi%s_%d' % (n, s), 'lo%s_%d' % (n, s), 'hi%s_%d' % (n, s)]
        want += ['scale_%d' % s, 'pvalue_%d' % s]
    assert list(df.columns) == want
    assert df['norm_lo50_1'].tolist() == [-0.5, 0.5, 1.5]
    # row 1 has seq_norm < 0: unscale reverses the order, so the bounds swap
    assert df['lo50_1'].tolist() == [-5.0, -30.0, 15.0] and df['hi50_1'].tolist() == [5.0, -10.0, 25.0]
    assert np.all(df['lo90_2'] <= df['hi90_2'])


def test_subsets_and_coverage_table():
    keys, levels, pred, scale, qhat, lower, upper, pvalue, seq_norm, unscale = _tables()
    date = np.array([20000131, 20000131, 20000430])
    subset = conformal_subsets(date, ['a', 'b', 'c'], [20000131], ['a'], {'b', 'c'}, 200003)
    assert subset.tolist() == ['calibration', 'training', 'out_of_sample']
    targets = np.array([[0.25, 3.0, np.nan], [0.5, 0.5, 0.5]], np.float32)
    df = coverage_table(levels, subset, np.array([10, 12]), qhat, pred, targets, scale, lower, upper, seq_norm,
                        unscale)
    assert list(df.columns) == ['step', 'level', 'subset', 'n_cal', 'qhat', 'n', 'coverage', 'mean_norm_width',
                                'mean_width']
    assert len(df) == 2 * 2 * 4
    row = df[(df.step == 1) & (df.level == 0.5) & (df.subset == 'all')].iloc[0]
    assert row.n == 2 and row.n_cal == 10 and row.coverage == 0.5 and row.mean_norm_width == 1.0
    assert df[(df.step == 1) & (df.subset == 'out_of_sample')]['n'].tolist() == [0, 0]
    row = df[(df.step == 2) & (df.level == 0.9) & (df.subset == 'all')].iloc[0]
    assert row.n == 3 and row.coverage == 1.0 and np.isinf(row.qhat)


# ---- compile -----------------------------------------------------------------------------------------------------
def test_conformal_kernels_compile_without_spills():
    if shutil.which('nvcc') is None:
        pytest.skip('nvcc not found')
    with tempfile.TemporaryDirectory() as d:
        r = subprocess.run(['nvcc', '-O3', '-Xptxas', '-v', '-std=c++17', '-gencode', 'arch=compute_90a,code=sm_90a',
                            '--expt-relaxed-constexpr', '-c', os.path.join(ROOT, 'lfm_quant_b200', 'csrc', 'conformal.cu'),
                            '-o', os.path.join(d, 'conformal.o')], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        names = re.findall(r"Compiling entry function '(\w+)'", r.stderr)
        for k in ('conformal_score_kernel', 'conformal_keys_kernel', 'conformal_select_kernel',
                  'conformal_bounds_kernel', 'conformal_pvalue_kernel'):
            assert any(k in n for n in names), k
        frames = re.findall(r'(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads', r.stderr)
        assert frames and all(f == ('0', '0', '0') for f in frames), frames
