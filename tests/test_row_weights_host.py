"""CPU checks of the row-weighted training loss (DESIGN.md section 6d): the weighted fp64 oracle that the GPU tests
compare against, and the library's new entry point."""
import os
import re

import numpy as np
import pytest

import row_weights_oracle as rwo
from lfm_quant_b200 import _native as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KW = dict(target_idx=1, target_lambda=0.4, rnn_lambda=0.7)


def _problem(B=9, T=5, O=4, seed=0):
    rng = np.random.RandomState(seed)
    y = rng.normal(size=(B, T, O))
    y[2, :2] = 0.0           # masked steps
    y[6, :] = 0.0            # a fully masked window
    return y, rng.normal(size=(B, T, O))


def test_none_is_the_unweighted_loss_and_ones_equal_it():
    y, p = _problem()
    a = rwo.loss_point(y, p, None, **KW)
    b = rwo.loss_point(y, p, np.ones(len(y)), **KW)
    np.testing.assert_allclose(a[0], b[0], rtol=1e-14)
    np.testing.assert_allclose(a[1], b[1], rtol=1e-14)
    np.testing.assert_allclose(a[2], b[2], rtol=1e-14, atol=1e-300)


@pytest.mark.parametrize('seed', [0, 1, 2])
def test_integer_weights_are_row_duplication_and_zero_is_removal(seed):
    y, p = _problem(seed=seed)
    w = np.random.RandomState(seed + 10).randint(0, 4, size=len(y))
    w[0] = 0
    w[1] = 3
    rows = np.repeat(np.arange(len(y)), w)
    lw, mw, dw = rwo.loss_point(y, p, w.astype(np.float64), **KW)
    ld, md, dd = rwo.loss_point(y[rows], p[rows], None, **KW)
    np.testing.assert_allclose(lw, ld, rtol=1e-12)
    np.testing.assert_allclose(mw, md, rtol=1e-12)
    # the gradient of a window is the sum of its copies' gradients; a removed window has none
    folded = np.zeros_like(dw)
    np.add.at(folded, rows, dd)
    np.testing.assert_allclose(dw, folded, rtol=1e-12, atol=1e-15)
    assert not np.any(dw[0])


def test_dense_integer_weights_are_row_duplication():
    rng = np.random.RandomState(3)
    y, p = rng.normal(size=(11, 4)), rng.normal(size=(11, 4))
    y[5] = 0.0
    w = rng.randint(0, 3, size=11)
    rows = np.repeat(np.arange(11), w)
    lw, mw, dw = rwo.loss_dense(y, p, w.astype(np.float64), target_idx=2, target_lambda=0.3)
    ld, md, dd = rwo.loss_dense(y[rows], p[rows], None, target_idx=2, target_lambda=0.3)
    np.testing.assert_allclose([lw, mw], [ld, md], rtol=1e-12)
    folded = np.zeros_like(dw)
    np.add.at(folded, rows, dd)
    np.testing.assert_allclose(dw, folded, rtol=1e-12, atol=1e-15)


def test_weighted_gradient_matches_finite_differences():
    y, p = _problem(seed=4)
    w = np.random.RandomState(5).uniform(0, 2, size=len(y))
    w[3] = 0.0
    _, _, d = rwo.loss_point(y, p, w, **KW)
    eps = 1e-6
    rng = np.random.RandomState(6)
    for _ in range(25):
        i = tuple(rng.randint(s) for s in p.shape)
        pp, pm = p.copy(), p.copy()
        pp[i] += eps
        pm[i] -= eps
        fd = (rwo.loss_point(y, pp, w, **KW)[0] - rwo.loss_point(y, pm, w, **KW)[0]) / (2 * eps)
        assert abs(fd - d[i]) <= 1e-7 + 1e-6 * abs(d[i]), (i, fd, d[i])


def test_zero_weight_sum_gives_zero_loss_and_gradient():
    y, p = _problem()
    loss, mse, d = rwo.loss_point(y, p, np.zeros(len(y)), **KW)
    assert loss == 0.0 and mse == 0.0 and not np.any(d)


def test_set_row_weights_is_declared_and_exported():
    src = open(os.path.join(ROOT, 'include', 'lfmq.h')).read()
    assert re.search(r'int32_t\s+lfmq_set_row_weights\s*\(\s*lfmq_handle h,\s*const float\* w_dev\s*\)', src)
    assert 'lfmq_set_row_weights' in N.SYMBOLS
    lib = N.load()
    assert hasattr(lib, 'lfmq_set_row_weights')
    assert lib.lfmq_set_row_weights(None, None) == 1          # LFMQ_ERR_ARG


# ---- the weight vector of the synthetic dataset (Dataset.row_weights_host, the NumPy form of lfmq_row_weights) ------
import pandas as pd  # noqa: E402

from lfm_quant_b200.scripts import base_config, configs  # noqa: E402
from lfm_quant_b200.scripts.runtime import model_execution as me  # noqa: E402


@pytest.fixture()
def fresh_flags():
    configs.reset()
    yield
    configs.reset()


@pytest.fixture(scope='module')
def synthetic(tmp_path_factory):
    from lfm_quant_b200.scripts.synthetic import write_open_dataset, write_system_test_conf
    d = tmp_path_factory.mktemp('rw')
    path = d / 'datasets' / 'open-dataset.dat'
    write_open_dataset(str(path), n_keys=16, n_months=360, seed=7)
    df = pd.read_csv(path, sep=' ', dtype={'gvkey': str})
    df.loc[df.index[5::97], 'mrkcap'] = np.nan                    # NaN weighs 0
    df.to_csv(path, sep=' ', index=False, na_rep='NaN')
    write_system_test_conf(str(d / 'config' / 'system-test.conf'), str(d / 'datasets'), str(d / 'experiments'))
    (d / 'experiments').mkdir()
    return d


def _cfg(synthetic, *extra):
    return base_config.get_configs(['--config=' + str(synthetic / 'config' / 'system-test.conf')] + list(extra))


def _loaded(cfg):
    from lfm_quant_b200.scripts.data_processing import Dataset
    ds = Dataset(cfg)
    ds.generate_dataset()
    return ds


def _months(ds, rows):
    d = pd.DatetimeIndex(ds._dates[rows])
    return d.year.values * 12 + d.month.values


def test_field_and_halflife_weights(fresh_flags, synthetic, monkeypatch):
    monkeypatch.setenv('LFMQ_HOST_INDEX', '1')
    ds = _loaded(_cfg(synthetic, '--sample_weight_field', 'mrkcap', '--recency_halflife', '5', '--model_dir', 'a'))
    inp = ds._dataset['train_X']
    rows = inp[:, 1]
    raw = ds.data['mrkcap'].values[rows].astype(np.float64)        # the raw column: no scaling, no log-squash
    assert np.isnan(raw).any()
    months = _months(ds, rows)
    assert ds.ref_month == months.max()
    want = np.where(np.isnan(raw), 0.0, raw) * 2.0 ** (-(months.max() - months) / 60.0)
    w = ds.row_weights_host(inp)
    assert w.dtype == np.float32 and np.array_equal(w, want.astype(np.float32))
    assert np.all(w[np.isnan(raw)] == 0) and np.all(w >= 0)


def test_halflife_alone_and_off(fresh_flags, synthetic, monkeypatch):
    monkeypatch.setenv('LFMQ_HOST_INDEX', '1')
    ds = _loaded(_cfg(synthetic, '--recency_halflife', '2', '--model_dir', 'b'))
    inp = ds._dataset['train_X']
    w = ds.row_weights_host(inp)
    assert w.max() == 1.0 and np.all(w > 0)
    configs.reset()
    assert not _loaded(_cfg(synthetic, '--model_dir', 'c')).row_weighted
    configs.reset()        # ignored at prediction
    from lfm_quant_b200.scripts.data_processing import Dataset
    assert not Dataset(_cfg(synthetic, '--train=False', '--sample_weight_field', 'nope',
                            '--recency_halflife', '3')).row_weighted


@pytest.mark.parametrize('value,what', [(-1.0, 'negative'), (np.inf, 'infinite')])
def test_bad_field_values_are_refused_at_load(fresh_flags, synthetic, tmp_path, monkeypatch, value, what):
    monkeypatch.setenv('LFMQ_HOST_INDEX', '1')
    src = synthetic / 'datasets' / 'open-dataset.dat'
    df = pd.read_csv(src, sep=' ', dtype={'gvkey': str})
    r = len(df) // 2
    df.loc[df.index[r], 'mrkcap'] = value
    (tmp_path / 'datasets').mkdir()
    df.to_csv(tmp_path / 'datasets' / 'open-dataset.dat', sep=' ', index=False, na_rep='NaN')
    c = _cfg(synthetic, '--sample_weight_field', 'mrkcap', '--data_dir', str(tmp_path / 'datasets'))
    from lfm_quant_b200.scripts.data_processing import Dataset
    with pytest.raises(ValueError, match=r'mrkcap.*gvkey %s' % df['gvkey'].iloc[r]):
        Dataset(c)


def test_unknown_field_and_negative_halflife_are_refused(fresh_flags, synthetic, monkeypatch):
    from lfm_quant_b200.scripts.data_processing import Dataset
    with pytest.raises(ValueError, match='no_such_column'):
        Dataset(_cfg(synthetic, '--sample_weight_field', 'no_such_column'))
    configs.reset()
    c = _cfg(synthetic, '--recency_halflife', '-1')
    with pytest.raises(ValueError, match='recency_halflife'):
        me.check_row_weights(c)
    with pytest.raises(ValueError, match='recency_halflife'):
        Dataset(c)


def test_naive_refuses_a_weight_flag_before_any_work(fresh_flags, synthetic, monkeypatch):
    c = _cfg(synthetic, '--nn_type', 'NaivePointEstimate', '--sample_weight_field', 'mrkcap')
    monkeypatch.setattr(me.ModelExecution, 'fixed_dates_execution', lambda self: pytest.fail('ran'))
    with pytest.raises(ValueError, match='nothing to train'):
        me.ModelExecution(c)()


def test_each_walk_forward_origin_uses_its_own_reference_date(fresh_flags, synthetic, monkeypatch):
    monkeypatch.setenv('LFMQ_HOST_INDEX', '1')
    c = _cfg(synthetic, '--training_type', 'iterative', '--split_date', '199512', '--recency_halflife', '4',
             '--model_dir', 'wf')
    _, runs = me.origin_configs(c)
    assert len(runs) >= 2
    refs = []
    for origin, train, _ in runs[:3]:
        ds = _loaded(train)
        rows = ds._dataset['train_X'][:, 1]
        m = _months(ds, rows)
        assert ds.ref_month == m.max() <= (origin // 100) * 12 + origin % 100
        w = ds.row_weights_host(ds._dataset['train_X'])
        assert np.array_equal(w, (2.0 ** (-(m.max() - m) / 48.0)).astype(np.float32))
        refs.append(ds.ref_month)
    assert refs == sorted(refs) and len(set(refs)) == len(refs)
