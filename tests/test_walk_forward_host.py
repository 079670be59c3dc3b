"""CPU tests of walk-forward backtests (training_type iterative, DESIGN.md section 6c): the origin list, the refusals,
no look-ahead in the windows and scaling parameters of every origin (the NumPy window index on the synthetic dataset),
and the run over stubbed origins: the phases, the files, the stitched walk_forward_preds.dat and read_results."""
import os
import pickle

import numpy as np
import pandas as pd
import pytest

from lfm_quant_b200.scripts import base_config, configs
from lfm_quant_b200.scripts.runtime import model_execution as me


@pytest.fixture()
def fresh_flags():
    configs.reset()
    yield
    configs.reset()


def _month(yyyymm):
    return pd.Timestamp(year=yyyymm // 100, month=yyyymm % 100, day=1)


def test_add_months():
    assert me.add_months(200112, 1) == 200201 and me.add_months(200101, -1) == 200012
    assert me.add_months(199912, 12) == 200012 and me.add_months(200006, 30) == 200212
    assert me.add_months(200011, 0) == 200011


@pytest.mark.parametrize('split,end,stride,origins,last_pred', [
    (200012, 200412, 12, [200012, 200112, 200212, 200312], (200401, 200412)),
    (200006, 200412, 12, [200006, 200106, 200206, 200306, 200406], (200407, 200412)),       # the last one clipped
    (199912, 200412, 24, [199912, 200112, 200312], (200401, 200412)),                        # clipped
    (200011, 200103, 1, [200011, 200012, 200101, 200102], (200103, 200103)),
    (200312, 200401, 12, [200312], (200401, 200401)),
])
def test_origins_and_their_date_ranges(fresh_flags, tmp_path, split, end, stride, origins, last_pred):
    assert me.walk_forward_origins(split, end, stride) == origins
    c = base_config.get_configs(['--experiments_dir', str(tmp_path), '--model_dir', 'wf', '--name', 'bt',
                                 '--training_type', 'iterative', '--start_date', '197501', '--split_date', str(split),
                                 '--end_date', str(end), '--stride', str(stride), '--forecast_n', str(stride),
                                 '--num_gpu', '2', '--seed', '33'])
    experiment_dir, runs = me.origin_configs(c)
    assert experiment_dir == os.path.join(str(tmp_path), 'wf')
    assert [o for o, _, _ in runs] == origins
    for k, (o, train, pred) in enumerate(runs):
        for r in (train, pred):
            assert r.model_dir == os.path.join(experiment_dir, 'bt-wf-%d' % o)
            assert r.training_type == 'fixed_dates' and r.member_id == k and r.default_gpu == '/gpu:%d' % (k % 2)
            assert r.num_procs == 1 and r.NPE == 1 and r.seed == 33
        assert train.train and (train.start_date, train.end_date) == (197501, o)
        assert not pred.train and pred.start_date == me.add_months(o, 1)
        assert pred.end_date == (origins[k + 1] if k + 1 < len(origins) else last_pred[1])
    assert (runs[-1][2].start_date, runs[-1][2].end_date) == last_pred
    assert c.training_type == 'iterative' and c.model_dir == 'wf' and c.train      # the backtest's config is left alone


def _iterative(tmp_path, *extra):
    (tmp_path / 'exp').mkdir(exist_ok=True)
    return base_config.get_configs(['--experiments_dir', str(tmp_path / 'exp'), '--model_dir', 'wf', '--name', 'bt',
                                    '--training_type', 'iterative', '--start_date', '197501', '--end_date', '200412',
                                    '--split_date', '200112'] + list(extra))


@pytest.mark.parametrize('extra,flag', [
    (['--split_date', '0'], '--split_date'),
    (['--split_date', '197501'], '--split_date'),
    (['--split_date', '200412'], '--split_date'),
    (['--split_date', '200612'], '--split_date'),
    (['--split_date', '200113'], '--split_date'),
    (['--num_procs', '2'], '--num_procs'),
    (['--cdrs_inference=True'], '--cdrs_inference'),
    (['--forecast_n', '24'], '--forecast_n'),
    (['--stride', '0'], '--stride'),
    (['--scalesfile', 'scales.dat'], '--scalesfile'),
    (['--train=False', '--num_procs', '3'], '--num_procs'),
])
def test_refusals_come_before_any_work(fresh_flags, tmp_path, monkeypatch, extra, flag):
    ran = []
    for name in ('single_execution', 'member_execution'):
        monkeypatch.setattr(me.ModelExecution, name, staticmethod(lambda *a: ran.append(a) or 'ran'))
    monkeypatch.setattr(me.ModelExecution, 'fixed_dates_execution', lambda self: ran.append(self) or 'ran')
    with pytest.raises(ValueError, match=flag):
        me.ModelExecution(_iterative(tmp_path, *extra))()
    assert ran == [] and not (tmp_path / 'exp' / 'wf').exists()


def test_a_missing_split_date_and_torchrun_are_refused(fresh_flags, tmp_path, monkeypatch):
    ran = []
    monkeypatch.setattr(me.ModelExecution, 'member_execution', staticmethod(lambda *a: ran.append(a)))
    c = _iterative(tmp_path)
    c.split_date = None
    with pytest.raises(ValueError, match='--split_date None'):
        me.ModelExecution(c)()
    monkeypatch.setenv('WORLD_SIZE', '2')
    with pytest.raises(ValueError, match='torchrun'):
        me.ModelExecution(_iterative(tmp_path))()
    assert ran == []


def test_search_candidates_still_refuse_iterative(fresh_flags, tmp_path):
    conf = tmp_path / 'model.conf'
    conf.write_text('--training_type iterative\n--split_date 200112\n')
    errors = me.run_candidates([str(conf)], 1)
    assert isinstance(errors[0], NotImplementedError)


def _frame(rows, seed, steps=1):
    """A preds.dat frame (predict.py's columns) of `rows` rows."""
    rng = np.random.RandomState(seed)
    d = {'date': np.full(rows, 20000101 + seed), 'gvkey': ['%06d' % (1000 + i) for i in range(rows)],
         'seq_norm': rng.uniform(10, 500, rows).astype(np.float32)}
    for s in range(1, steps + 1):
        ns = str(s)
        d['targets_' + ns] = rng.normal(size=rows) * 100
        d['targets_' + ns][1] = np.nan                                  # a window whose target does not exist yet
        d['norm_preds_' + ns] = rng.normal(size=rows).astype(np.float32)
        d['norm_targets_' + ns] = rng.normal(size=rows)
        d['norm_squared_diff_' + ns] = np.square(d['norm_targets_' + ns] - d['norm_preds_' + ns])
        d['preds_' + ns] = d['norm_preds_' + ns] * 100
    return pd.DataFrame(d)


def test_stitching_keeps_origin_order_and_adds_the_origin():
    frames = [_frame(5, 1), _frame(3, 2), _frame(7, 3)]
    df = me.stitch_walk_forward(frames, [200112, 200212, 200312])
    assert len(df) == 15 and list(df.columns) == list(frames[0].columns) + ['origin']
    assert df['origin'].tolist() == [200112] * 5 + [200212] * 3 + [200312] * 7
    pd.testing.assert_frame_equal(df.drop(columns='origin'), pd.concat(frames, ignore_index=True))
    assert 'origin' not in frames[0].columns


@pytest.mark.parametrize('num_gpu,npe,shares', [(1, 3, [3, 3, 3]), (1, 1, [1, 1, 1]), (2, 3, [2, 1, 2])])
def test_origins_train_then_predict_and_the_stitched_file_is_written(fresh_flags, tmp_path, monkeypatch, num_gpu, npe,
                                                                     shares):
    calls = []
    frames = {200112: _frame(4, 1, 2), 200212: _frame(6, 2, 2), 200312: _frame(5, 3, 2)}

    def fake_member(cfg, share_den):
        calls.append((cfg.train, cfg.member_id, cfg.default_gpu, share_den, cfg.start_date, cfg.end_date))
        if not cfg.train:
            os.makedirs(os.path.join(cfg.model_dir, 'pred'), exist_ok=True)
            origin = me.add_months(cfg.start_date, -1)
            frames[origin].to_csv(os.path.join(cfg.model_dir, 'pred', cfg.preds_fname), sep=' ', index=False)

    monkeypatch.setattr(me.ModelExecution, 'member_execution', staticmethod(fake_member))
    c = _iterative(tmp_path, '--num_gpu', str(num_gpu), '--NPE', str(npe), '--forecast_steps', '2',
                   '--forecast_steps_weights', '0.75-0.25')
    df = me.ModelExecution(c)()
    origins = [200112, 200212, 200312]
    ends = [200212, 200312, 200412]
    gpus = ['/gpu:%d' % (k % num_gpu) for k in range(3)]
    assert [x[0] for x in calls] == [True] * 3 + [False] * 3          # every origin trains before any predicts
    assert sorted(calls[:3]) == [(True, k, gpus[k], shares[k], 197501, origins[k]) for k in range(3)]
    assert sorted(calls[3:]) == [(False, k, gpus[k], shares[k], me.add_months(origins[k], 1), ends[k])
                                 for k in range(3)]
    wf = tmp_path / 'exp' / 'wf'
    for k, o in enumerate(origins):
        for name, train in (('model-%d.conf' % k, 'True'), ('predict-%d.conf' % k, 'False')):
            lines = open(wf / ('bt-wf-%d' % o) / name).read().splitlines()
            assert '--train       %s ' % train in lines and '--training_type       fixed_dates ' in lines
    # the stitched rows are the origins' preds.dat rows as written, each with its origin
    lines = (wf / 'walk_forward_preds.dat').read_text().splitlines()
    header, rows = [], []
    for o in origins:
        own = (wf / ('bt-wf-%d' % o) / 'pred' / 'preds.dat').read_text().splitlines()
        header = own[0] + ' origin'
        rows += [r + ' %d' % o for r in own[1:]]
    assert lines == [header] + rows and len(rows) == 15
    written = pd.read_csv(wf / 'walk_forward_preds.dat', sep=' ', dtype={'gvkey': str}, float_precision='round_trip')
    pd.testing.assert_frame_equal(df, written)
    want = pd.concat([frames[o].astype({c: np.float64 for c in frames[o].columns if frames[o][c].dtype == np.float32})
                      .assign(origin=o) for o in origins], ignore_index=True)
    pd.testing.assert_frame_equal(written, want, check_exact=False, rtol=1e-7)
    loss, _, back = me.ModelExecution.read_results(c)
    by_hand = 0.75 * np.mean(want['norm_squared_diff_1']) + 0.25 * np.mean(want['norm_squared_diff_2'])
    assert loss == pytest.approx(by_hand, rel=1e-12) and len(back) == 15

    # --train=False predicts from the origin directories, which the training phase would have made: here the
    # prediction phase above made them
    calls.clear()
    c.train = False
    again = me.ModelExecution(c)()
    assert [x[0] for x in calls] == [False] * 3
    pd.testing.assert_frame_equal(again, written)


def test_predicting_without_trained_origins_names_the_missing_origin(fresh_flags, tmp_path, monkeypatch):
    ran = []
    monkeypatch.setattr(me.ModelExecution, 'member_execution', staticmethod(lambda *a: ran.append(a)))
    c = _iterative(tmp_path, '--train=False')
    (tmp_path / 'exp' / 'wf' / 'bt-wf-200112').mkdir(parents=True)
    with pytest.raises(FileNotFoundError, match='origin 200212'):
        me.ModelExecution(c)()
    assert ran == []
    # the naive forecast has no checkpoint: it predicts with --scalesfile into origin directories it makes
    c = _iterative(tmp_path, '--train=False', '--nn_type', 'NaivePointEstimate', '--scalesfile', 'x.dat',
                   '--model_dir', 'naive')
    with pytest.raises(RuntimeError, match='origin 200112 wrote no .*bt-wf-200112/pred/preds.dat'):
        me.ModelExecution(c)()
    assert len(ran) == 3 and all(not r[0].train for r in ran)


def test_a_failing_origin_stops_the_origins_that_have_not_started(fresh_flags, tmp_path, monkeypatch):
    import time
    ran = []

    def fake_member(cfg, share_den):
        ran.append(cfg.member_id)
        if cfg.member_id == 0:
            raise RuntimeError('origin 0 failed')
        time.sleep(0.2)

    monkeypatch.setattr(me.ModelExecution, 'member_execution', staticmethod(fake_member))
    c = _iterative(tmp_path, '--split_date', '199712', '--NPE', '1')
    with pytest.raises(RuntimeError, match='origin 0 failed'):
        me.ModelExecution(c)()
    assert ran[0] == 0 and set(ran) <= {0, 1}


# ---- no look-ahead, from the NumPy window index on the synthetic dataset -----------------------------------------

@pytest.fixture(scope='module')
def synthetic(tmp_path_factory):
    from lfm_quant_b200.scripts.synthetic import write_open_dataset, write_system_test_conf
    d = tmp_path_factory.mktemp('wf')
    write_open_dataset(str(d / 'datasets' / 'open-dataset.dat'), n_keys=24, n_months=420, seed=5)
    write_system_test_conf(str(d / 'config' / 'system-test.conf'), str(d / 'datasets'), str(d / 'experiments'))
    (d / 'experiments').mkdir()
    return d


def _dataset(cfg):
    from lfm_quant_b200.scripts.data_processing import Dataset
    ds = Dataset(cfg)
    ds._create_index()
    return ds


def _window_dates(ds, split):
    """The dates of the windows' last input rows and of their target rows."""
    inp, tar = ds._dataset[split + '_X'], ds._dataset[split + '_Y']
    return pd.DatetimeIndex(ds._dates[inp[:, 1]]), pd.DatetimeIndex(ds._dates[tar[:, 1]])


def _keys(ds, split):
    return set(zip(ds._meta[split][:, 0].tolist(), ds._meta[split][:, 1].tolist()))


def test_no_window_of_an_origin_looks_past_it(fresh_flags, synthetic, monkeypatch):
    monkeypatch.setenv('LFMQ_HOST_INDEX', '1')
    conf = str(synthetic / 'config' / 'system-test.conf')
    c = base_config.get_configs(['--config=' + conf, '--training_type', 'iterative', '--split_date', '200012',
                                 '--model_dir', 'wf-index'])
    _, runs = me.origin_configs(c)
    assert [o for o, _, _ in runs] == [200012, 200112, 200212, 200312]
    predicted = []
    for origin, train, pred in runs:
        d = _month(origin)
        ds = _dataset(train)
        for split in ('train', 'valid'):
            inp_dates, tar_dates = _window_dates(ds, split)
            assert len(inp_dates) > 0, (origin, split)
            assert (tar_dates <= d).all() and (inp_dates <= d).all(), (origin, split)
        ds = _dataset(pred)
        inp_dates, _ = _window_dates(ds, 'test')
        assert len(inp_dates) > 0 and (inp_dates > d).all(), origin
        assert (inp_dates <= _month(me.add_months(origin, c.stride))).all(), origin
        predicted.append(_keys(ds, 'test'))
    # the origins' prediction ranges do not overlap and together cover (split_date, end_date]
    for a, b in zip(runs, runs[1:]):
        assert me.add_months(a[2].end_date, 1) == b[2].start_date
    assert runs[0][2].start_date == me.add_months(200012, 1) and runs[-1][2].end_date == c.end_date
    for i in range(len(predicted)):
        for j in range(i):
            assert not predicted[i] & predicted[j]
    configs.reset()
    whole = base_config.get_configs(['--config=' + conf, '--train=False', '--start_date', '200101', '--model_dir',
                                     'wf-whole'])
    assert set().union(*predicted) == _keys(_dataset(whole), 'test')


def test_each_origin_fits_its_scaling_on_its_own_data(fresh_flags, synthetic, monkeypatch):
    monkeypatch.setenv('LFMQ_HOST_INDEX', '1')
    from lfm_quant_b200.scripts.data_processing import Dataset
    conf = str(synthetic / 'config' / 'system-test.conf')
    c = base_config.get_configs(['--config=' + conf, '--training_type', 'iterative', '--split_date', '200112',
                                 '--model_dir', 'wf-scales'])
    _, runs = me.origin_configs(c)
    fitted = {}
    for origin, train, _ in runs:
        ds = Dataset(train)
        ds.generate_dataset()
        on_disk = pickle.load(open(os.path.join(train.model_dir, 'scales.dat'), 'rb'))
        fitted[origin] = ds.scaling_params
        for key in ('center', 'scale'):
            np.testing.assert_array_equal(on_disk[key], ds.scaling_params[key])
    for origin in fitted:
        configs.reset()
        plain = base_config.get_configs(['--config=' + conf, '--end_date', str(origin), '--model_dir',
                                         'plain-%d' % origin])
        ds = Dataset(plain)
        ds.generate_dataset()
        for key in ('center', 'scale'):
            np.testing.assert_array_equal(fitted[origin][key], ds.scaling_params[key])
    configs.reset()
    final = Dataset(base_config.get_configs(['--config=' + conf, '--model_dir', 'plain-final']))
    final.generate_dataset()
    for origin in fitted:
        assert not np.array_equal(fitted[origin]['center'], final.scaling_params['center']), origin
    assert not np.array_equal(fitted[200112]['center'], fitted[200212]['center'])
