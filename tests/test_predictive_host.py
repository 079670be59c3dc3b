"""Predictive quantiles and proper scores on the host: the fp64 reference of tests/predictive_oracle.py against closed
forms and numerical integration, the --pred_quantiles flag and the runs it is refused for, quantiles.dat and
calibration.dat from stubbed outputs, the walk-forward stacking, and what ptxas reports for predictive.cu (skipped
without nvcc).  The library's outputs are checked on the GPU (tests/test_gpu_predictive.py)."""
import os
import re
import shlex
import shutil
import subprocess
import tempfile

import numpy as np
import pandas as pd
import pytest
from scipy import integrate, special

import predictive_oracle as pdo
from lfm_quant_b200.scripts import base_config, configs
from lfm_quant_b200.scripts.predict import Predict, calibration_table, pit_ks, quantile_name, quantile_table
from lfm_quant_b200.scripts.runtime import model_execution as me

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LEVELS = [0.05, 0.25, 0.5, 0.75, 0.95]


# ---- the oracle ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('m,s,y', [(0.0, 1.0, 0.3), (-2.5, 0.2, -2.0), (4.0, 3.0, -7.0)])
def test_one_component_is_one_gaussian(m, s, y):
    q = pdo.quantiles([m], [s * s], LEVELS)
    np.testing.assert_allclose(q, m + s * special.ndtri(LEVELS), rtol=0, atol=1e-12)
    assert abs(pdo.crps([m], [s * s], y) - pdo.crps_gaussian(m, s, y)) < 1e-12
    want_nll = 0.5 * ((y - m) / s) ** 2 + np.log(s) + 0.5 * np.log(2 * np.pi)
    assert abs(pdo.nll([m], [s * s], y) - want_nll) < 1e-12
    assert abs(pdo.pit([m], [s * s], y) - special.ndtr((y - m) / s)) < 1e-15


def _mixture(M, seed, spread=1.0):
    rng = np.random.RandomState(seed)
    return rng.normal(size=M) * spread, rng.uniform(0.05, 1.5, size=M) ** 2


@pytest.mark.parametrize('M,spread,y', [(2, 1.0, 0.4), (7, 0.5, -1.3), (5, 8.0, 2.0), (16, 1.0, 10.0)])
def test_closed_form_crps_is_the_integral_of_the_squared_cdf_gap(M, spread, y):
    mu, v = _mixture(M, M, spread)
    sd = np.sqrt(v)
    lo, hi = (mu - 12 * sd).min(), (mu + 12 * sd).max()
    f = lambda z: pdo.cdf(z, mu, v) ** 2            # noqa: E731
    g = lambda z: (1.0 - pdo.cdf(z, mu, v)) ** 2    # noqa: E731
    pts = sorted(set(np.clip(np.concatenate([mu, [y]]), lo, hi)))
    want = (integrate.quad(f, lo, y, limit=400, epsabs=1e-13, points=[p for p in pts if lo < p < y] or None)[0]
            + integrate.quad(g, y, hi, limit=400, epsabs=1e-13, points=[p for p in pts if y < p < hi] or None)[0])
    assert abs(pdo.crps(mu, v, y) - want) < 1e-8


@pytest.mark.parametrize('M,spread', [(3, 1.0), (7, 6.0), (64, 2.0)])
def test_quantiles_increase_and_invert_the_cdf(M, spread):
    mu, v = _mixture(M, 10 + M, spread)
    levels = [0.01, 0.05, 0.2, 0.5, 0.8, 0.95, 0.99]
    q = pdo.quantiles(mu, v, levels)
    assert np.all(np.diff(q) > 0)
    for qk, tau in zip(q, levels):
        assert abs(pdo.cdf(qk, mu, v) - tau) < 1e-12


# ---- the flag --------------------------------------------------------------------------------------------------------
@pytest.fixture()
def fresh_flags():
    configs.reset()
    yield
    configs.reset()


def test_pred_quantiles_flag_defaults_to_off_and_parses(fresh_flags):
    assert base_config.get_configs([]).pred_quantiles is None
    c = base_config.get_configs(['--pred_quantiles', '0.05-0.25-0.5-0.75-0.95'])
    assert base_config.pred_quantile_levels(c.pred_quantiles) == LEVELS
    assert base_config.pred_quantile_levels(None) is None
    assert base_config.pred_quantile_levels('0.5') == [0.5]
    assert [quantile_name(t) for t in LEVELS + [0.125]] == ['q5', 'q25', 'q50', 'q75', 'q95', 'q12.5']


@pytest.mark.parametrize('spec', ['0.5-0.25', '0.25-0.25', '0-0.5', '0.5-1', '1.5', 'a-b', '0.1--0.2', '',
                                  '-'.join(['%.3f' % (0.01 * (k + 1)) for k in range(33)])])
def test_malformed_levels_are_refused(spec):
    if spec == '':
        assert base_config.pred_quantile_levels(spec) is None
        return
    with pytest.raises(ValueError, match='--pred_quantiles'):
        base_config.pred_quantile_levels(spec)


_UQ = ['--nn_type', 'RNNUqRangeEstimate', '--UQ=True']


@pytest.mark.parametrize('argv', [
    ['--pred_quantiles', '0.1-0.9', '--train=False'],                         # a point estimate
    ['--pred_quantiles', '0.1-0.9', '--train=True'] + _UQ,                    # training
    ['--pred_quantiles', '0.9-0.1', '--train=False'] + _UQ,                   # not increasing
    ['--pred_quantiles', '0.1-1.0', '--train=False'] + _UQ,                   # outside (0, 1)
    ['--pred_quantiles', '0.1-x', '--train=False'] + _UQ,                     # malformed
    ['--pred_quantiles', '0.1-0.9', '--train=False', '--training_type', 'iterative', '--split_date', '199501'],
])
def test_pred_quantiles_is_refused_before_any_work(fresh_flags, monkeypatch, argv):
    ran = []
    monkeypatch.setattr(me.ModelExecution, 'single_execution', staticmethod(lambda cfg: ran.append(cfg) or 'ran'))
    monkeypatch.setattr(me.ModelExecution, 'fixed_dates_execution', lambda self: ran.append(self) or 'ran')
    monkeypatch.setattr(me.ModelExecution, 'walk_forward_execution', lambda self: ran.append(self) or 'ran')
    with pytest.raises(ValueError, match='--pred_quantiles'):
        me.ModelExecution(base_config.get_configs(argv))()
    assert ran == []


@pytest.mark.parametrize('argv', [
    ['--pred_quantiles', '0.05-0.5-0.95', '--train=False'] + _UQ,
    ['--pred_quantiles', '0.5', '--train=False', '--mc_samples', '8'] + _UQ,
    ['--pred_quantiles', '0.1-0.9', '--train=False', '--forecast_steps', '2', '--forecast_steps_weights',
     '1.0-0.5'] + _UQ,
])
def test_pred_quantiles_runs_at_uq_prediction(fresh_flags, monkeypatch, argv):
    seen = []
    monkeypatch.setattr(me.ModelExecution, 'single_execution', staticmethod(lambda cfg: seen.append(cfg) or 'ran'))
    monkeypatch.setattr(me.ModelExecution, 'write_uq_ensemble', classmethod(lambda cls, cfg: None))
    assert me.ModelExecution(base_config.get_configs(argv))() == 'ran'
    assert len(seen) == 1


# ---- the files -------------------------------------------------------------------------------------------------------
def _stub(S, N_, Q, seed):
    rng = np.random.RandomState(seed)
    q = np.sort(rng.normal(size=(S, N_, Q)), axis=2).astype(np.float32)
    scores = np.stack([rng.uniform(0.1, 1, size=(S, N_)), rng.normal(size=(S, N_)), rng.uniform(size=(S, N_))],
                      axis=2).astype(np.float32)
    return q, scores


def test_quantile_table_columns_and_unscaling():
    S, N_, levels = 2, 6, [0.1, 0.5, 0.9]
    q, scores = _stub(S, N_, 3, 1)
    keys = pd.DataFrame({'date': pd.to_datetime(['2001-03-31'] * N_), 'gvkey': ['%06d' % i for i in range(N_)]})
    seq_norm = np.array([1.0, 2.0, -1.0, 0.5, 3.0, 1.0])
    unscale = lambda col: (np.asarray(col, dtype=np.float64) * 2.0 + 1.0) * seq_norm   # noqa: E731
    df = quantile_table(keys, levels, q, scores, unscale)
    names = ['date', 'gvkey']
    for s in (1, 2):
        names += ['norm_q10_%d' % s, 'norm_q50_%d' % s, 'norm_q90_%d' % s, 'q10_%d' % s, 'q50_%d' % s, 'q90_%d' % s,
                  'crps_%d' % s, 'nll_%d' % s, 'pit_%d' % s]
    assert list(df.columns) == names
    for s in range(S):
        for k, name in enumerate(('q10', 'q50', 'q90')):
            assert np.array_equal(df['norm_%s_%d' % (name, s + 1)].to_numpy(), q[s][:, k])
            np.testing.assert_allclose(df['%s_%d' % (name, s + 1)], unscale(q[s][:, k]), rtol=1e-15)
        for j, name in enumerate(('crps', 'nll', 'pit')):
            assert np.array_equal(df['%s_%d' % (name, s + 1)].to_numpy(), scores[s][:, j])
    # increasing in the fundamentals' units where seq_norm > 0, reversed where it is negative
    up = df[['q10_1', 'q50_1', 'q90_1']].to_numpy()
    assert np.all(np.diff(up[seq_norm > 0], axis=1) > 0) and np.all(np.diff(up[seq_norm < 0], axis=1) < 0)


def test_calibration_table_counts_known_targets_only():
    levels = [0.25, 0.5]
    q = np.array([[[0.0, 1.0], [0.0, 1.0], [0.0, 1.0], [0.0, 1.0], [0.0, 1.0]]], dtype=np.float32)
    y = np.array([[-1.0, 0.5, 2.0, np.nan, 0.7]])
    scores = np.array([[[1.0, 2.0, 0.1], [3.0, 4.0, 0.6], [5.0, 6.0, 0.95], [np.nan] * 3, [7.0, 8.0, 0.7]]])
    df = calibration_table(levels, q, scores, y)
    assert list(df.columns) == ['step', 'level', 'frac_below', 'n_known', 'mean_crps', 'mean_nll', 'pit_ks']
    assert df['step'].tolist() == [1, 1] and df['level'].tolist() == levels
    assert df['n_known'].tolist() == [4, 4]
    assert df['frac_below'].tolist() == [0.25, 0.75]             # below 0: -1; below 1: -1, 0.5, 0.7
    assert df['mean_crps'].tolist() == [4.0, 4.0] and df['mean_nll'].tolist() == [5.0, 5.0]
    p = np.sort([0.1, 0.6, 0.95, 0.7])
    want = max(np.max(np.arange(1, 5) / 4 - p), np.max(p - np.arange(0, 4) / 4))
    assert abs(df['pit_ks'][0] - want) < 1e-15 and abs(want - 0.35) < 1e-12
    assert abs(pit_ks(np.linspace(0.05, 0.95, 10)) - 0.05) < 1e-12
    assert np.isnan(pit_ks([]))
    none = calibration_table(levels, q, scores, np.full((1, 5), np.nan))
    assert none['n_known'].tolist() == [0, 0] and none[['frac_below', 'mean_crps', 'pit_ks']].isna().all().all()


def test_write_quantiles_from_stubbed_outputs(tmp_path):
    S, N_ = 2, 5
    q, scores = _stub(S, N_, len(LEVELS), 3)
    p = object.__new__(Predict)
    p.pred_dir = str(tmp_path)
    df = pd.DataFrame({'date': pd.to_datetime(['1999-12-31', '1999-12-31', '2000-01-31', '2000-01-31', '2000-02-29']),
                       'gvkey': ['001', '002', '001', '002', '003'], 'seq_norm': np.ones(N_)})
    y = np.random.RandomState(4).normal(size=(S, N_))
    y[1, 2] = np.nan
    for s in range(S):
        df['norm_targets_%d' % (s + 1)] = y[s]
    p._write_quantiles(df, LEVELS, q, scores, lambda col: np.asarray(col, dtype=np.float64) * 10.0)
    got = pd.read_csv(tmp_path / 'quantiles.dat', sep=' ', dtype={'gvkey': str})
    assert got['date'].tolist() == [19991231, 19991231, 20000131, 20000131, 20000229]
    assert got['gvkey'].tolist() == df['gvkey'].tolist()
    np.testing.assert_allclose(got['q50_2'], q[1][:, 2].astype(np.float64) * 10.0, rtol=1e-12)
    cal = pd.read_csv(tmp_path / 'calibration.dat', sep=' ')
    assert len(cal) == S * len(LEVELS) and cal['n_known'].tolist() == [5] * 5 + [4] * 5


def test_walk_forward_stacks_the_origins_quantiles(tmp_path, monkeypatch, fresh_flags):
    cfg = base_config.get_configs(['--training_type', 'iterative', '--split_date', '199506', '--end_date', '199612',
                                   '--stride', '12', '--train=False', '--pred_quantiles', '0.1-0.9', '--experiments_dir',
                                   str(tmp_path), '--model_dir', 'wf'] + _UQ)

    def run_members(cls, preds, npe):
        for p in preds:
            os.makedirs(os.path.join(p.model_dir, 'pred'), exist_ok=True)
            pd.DataFrame({'date': [p.start_date * 100 + 28], 'gvkey': ['007'], 'norm_preds_1': [0.5]}).to_csv(
                os.path.join(p.model_dir, 'pred', cfg.preds_fname), sep=' ', index=False)
            pd.DataFrame({'date': [p.start_date * 100 + 28], 'gvkey': ['007'], 'norm_q10_1': [p.member_id - 0.5],
                          'norm_q90_1': [p.member_id + 0.5]}).to_csv(
                os.path.join(p.model_dir, 'pred', 'quantiles.dat'), sep=' ', index=False)
    monkeypatch.setattr(me.ModelExecution, 'run_members', classmethod(run_members))
    monkeypatch.setattr(me, '_print_scaled_mse', lambda df, steps: None)
    _, origins = me.origin_configs(cfg)
    for _, _, pred in origins:
        os.makedirs(pred.model_dir, exist_ok=True)
    me.ModelExecution(cfg).walk_forward_execution()
    got = pd.read_csv(tmp_path / 'wf' / 'walk_forward_quantiles.dat', sep=' ', dtype={'gvkey': str})
    assert got['origin'].tolist() == [o for o, _, _ in origins] and len(origins) == 2
    assert got['norm_q10_1'].tolist() == [-0.5, 0.5] and got['gvkey'].tolist() == ['007', '007']


# ---- the kernels -----------------------------------------------------------------------------------------------------
def test_predictive_kernels_do_not_spill():
    nvcc = shutil.which('nvcc') or ('/usr/local/cuda/bin/nvcc' if os.path.exists('/usr/local/cuda/bin/nvcc') else None)
    if nvcc is None or shutil.which('make') is None:
        pytest.skip('nvcc or make not found')
    r = subprocess.run(['make', '-n', '-B', '-C', ROOT, 'NVCC=' + nvcc, 'all'], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    cmd = [line for line in r.stdout.splitlines() if line.startswith(nvcc + ' ') and 'predictive.cu' in line]
    assert len(cmd) == 1, r.stdout
    cmd = shlex.split(cmd[0])
    assert 'arch=compute_90a,code=sm_90a' in cmd and '-v' in ' '.join(cmd)
    with tempfile.TemporaryDirectory() as tmp:
        cmd[cmd.index('-o') + 1] = os.path.join(tmp, 'predictive.o')
        r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
    log = r.stdout + r.stderr
    kernels = re.findall(r"Compiling entry function '(\w+)' for 'sm_90a'", log)
    assert any('dist_kernel' in k for k in kernels) and any('dist_gather_kernel' in k for k in kernels), kernels
    spills = re.findall(r'(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads', log)
    assert len(spills) == len(kernels) and all(s == ('0', '0', '0') for s in spills), log
