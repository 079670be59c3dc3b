"""End-to-end test of the drop-in boundary on the GPU: the reference's CLI flow
(`lfm_quant.py --config=config/system-test.conf --train=True`, then `--train=False`; README.md:33-59) on a
synthetic open-dataset.dat -- BASELINE configs[0]: 1-layer RNN, H=64, batch=32, T=20."""
import os

import numpy as np
import pandas as pd
import pytest

import lfm_oracle as orc
from lfm_quant_b200.scripts import configs
from lfm_quant_b200.scripts import lfm_quant as cli
from lfm_quant_b200.scripts.synthetic import write_open_dataset, write_system_test_conf

pytestmark = pytest.mark.gpu

PRED_COLS_HEAD = ['date', 'gvkey', 'seq_norm']
PRED_COLS_TAIL = ['targets_1', 'norm_preds_1', 'norm_variance_1', 'norm_targets_1', 'norm_squared_diff_1', 'preds_1',
                  'variance_1', 'fcst_err_1', 'abs_err_1', 'unscaled_squared_err_1']


@pytest.fixture(scope='module')
def workdir(tmp_path_factory):
    d = tmp_path_factory.mktemp('sys')
    write_open_dataset(str(d / 'datasets' / 'open-dataset.dat'), n_keys=30, n_months=420, seed=9)
    write_system_test_conf(str(d / 'config' / 'system-test.conf'), str(d / 'datasets'), str(d / 'experiments'))
    os.environ.setdefault('LFM_QUANT_ROOT', str(d))
    return d


def test_cli_train_then_predict(workdir):
    conf = str(workdir / 'config' / 'system-test.conf')
    configs.reset()
    valid_mse = cli.main(['--config=' + conf, '--train=True'])
    mdir = workdir / 'experiments' / 'system-test-model'
    assert np.isfinite(valid_mse)
    assert (mdir / 'scales.dat').is_file() and (mdir / 'chkpts' / 'chkpt.lfmq.npz').is_file()
    ep = pd.read_csv(mdir / 'train_log' / 'system-test-train-logs-epoch.csv')
    assert list(ep.columns) == ['epoch', 'time', 'mse', 'uq_loss', 'valid_mse', 'valid_uq_loss', 'valid_mse_fcst']
    assert len(ep) == 2 and ep['mse'].iloc[1] < ep['mse'].iloc[0]            # it learns
    bt = pd.read_csv(mdir / 'train_log' / 'system-test-train-logs-batch.csv')
    assert list(bt.columns) == ['batch_n', 'time', 'mse', 'uq_loss', 'valid_mse', 'valid_uq_loss']
    w = np.load(mdir / 'chkpts' / 'chkpt.lfmq.npz')
    assert set(orc.param_names(1)) <= set(w.files) and w['lstm_1/kernel'].shape == (32, 256)
    assert np.linalg.norm(w['lstm_1/kernel'], axis=0).max() <= 3.0 * (1 + 1e-5)   # MaxNorm held

    configs.reset()
    df = cli.main(['--config=' + conf, '--train=False'])
    out = pd.read_csv(mdir / 'pred' / 'preds.dat', sep=' ', dtype={'gvkey': str})
    cols = list(out.columns)
    assert cols[:3] == PRED_COLS_HEAD and cols[-10:] == PRED_COLS_TAIL
    assert cols[3:-10] == ['inp_t%d' % t for t in range(-19, 1)]
    assert len(out) == len(df) > 100
    assert np.isfinite(out['norm_preds_1']).all() and np.isfinite(out['preds_1']).all()
    known = out['targets_1'].notna()
    assert known.any() and (~known).any()            # windows at the end of the file have no target yet
    assert (out.loc[known, 'norm_squared_diff_1'] >= 0).all()
    configs.reset()


def test_dataset_get_batch_matches_oracle(workdir):
    from lfm_quant_b200.scripts import base_config
    from lfm_quant_b200.scripts.data_processing import Dataset
    conf = str(workdir / 'config' / 'system-test.conf')
    for extra, train in ((['--model_dir', 'gb-train'], True), (['--model_dir', 'gb-train', '--train=False'], False)):
        configs.reset()
        c = base_config.get_configs(['--config=' + conf, '--aux_masking'] + extra)
        ds = Dataset(c)
        ds.generate_dataset()
        s = ds.train_set if train else ds.test_set
        inp_idx, tar_idx, meta = next(iter(s.batch(97)))
        x, y, md = ds.get_batch(inp_idx, tar_idx, meta)
        valid = np.array([m[1] == m[2] for m in meta])
        ref = orc.gather_batch(ds.table, inp_idx, tar_idx, valid, seq_len=ds.seq_len, stride=c.stride,
                               inp_cols=ds.inp_col_ids, fin_cols=ds.fin_col_ids, seq_norm_col=ds._seq_norm_idx,
                               center=np.asarray(ds.scaling_params['center']), scale=np.asarray(ds.scaling_params['scale']),
                               scale_inp_ids=ds.scale_inp_col_ids, aux_inp_ids=ds._aux_col_ids_seq, log_squash=True,
                               aux_masking=True, train=train)
        np.testing.assert_array_max_ulp(x.cpu().numpy(), ref[0], maxulp=1)
        np.testing.assert_array_equal(np.isnan(y.cpu().numpy()), np.isnan(ref[1]))
        np.testing.assert_array_max_ulp(np.nan_to_num(y.cpu().numpy()), np.nan_to_num(ref[1]), maxulp=1)
        np.testing.assert_array_equal(md[:, 2].astype(np.float64), ref[2])
        assert (x.cpu().numpy()[:, :-1, 16:] == 0).all()          # aux masking
    configs.reset()


def test_predict_serves_a_tf_format_checkpoint(workdir):
    """SURVEY 8f-3: train writes the TF-format checkpoint the reference uses (chkpt.index + chkpt.data-00000-of-00001,
    Keras object-graph keys) beside the native .npz; with the .npz gone -- the situation of a model directory trained
    by the reference -- predict.py:93's load_weights restores from the TF files and writes the same preds.dat."""
    from lfm_quant_b200 import tf_checkpoint
    conf = str(workdir / 'config' / 'system-test.conf')
    extra = ['--model_dir', 'system-test-tfck']
    configs.reset()
    cli.main(['--config=' + conf, '--train=True'] + extra)
    mdir = workdir / 'experiments' / 'system-test-tfck'
    prefix = str(mdir / 'chkpts' / 'chkpt')
    assert os.path.isfile(prefix + '.index') and os.path.isfile(prefix + '.data-00000-of-00001')
    bundle = tf_checkpoint.read_bundle(prefix)
    native = np.load(prefix + '.lfmq.npz')
    assert bundle['layer_with_weights-0/cell/kernel/.ATTRIBUTES/VARIABLE_VALUE'].shape == (32, 256)
    np.testing.assert_array_equal(bundle['layer_with_weights-2/kernel/.ATTRIBUTES/VARIABLE_VALUE'], native['OUTPUT_1/kernel'])
    configs.reset()
    cli.main(['--config=' + conf, '--train=False'] + extra)
    a = pd.read_csv(mdir / 'pred' / 'preds.dat', sep=' ', dtype={'gvkey': str})
    os.rename(prefix + '.lfmq.npz', prefix + '.lfmq.npz.away')
    configs.reset()
    cli.main(['--config=' + conf, '--train=False'] + extra)
    b = pd.read_csv(mdir / 'pred' / 'preds.dat', sep=' ', dtype={'gvkey': str})
    np.testing.assert_array_equal(a['norm_preds_1'].values, b['norm_preds_1'].values)
    configs.reset()


def test_device_validation_pass_matches_host_recomputation(workdir):
    """SURVEY 8f-4: Train._validation_metrics_point_estimate runs on the device (resident validation batches,
    predict_device, lfmq_unscale, lfmq_loss; two scalars come back).  Recomputed here on the host the way the reference
    does it (train.py:284-336): model.predict per batch -> vstack -> _unscale_preds (NumPy fp64) -> the weighted MSE of
    the oracle."""
    from lfm_quant_b200.scripts import base_config
    from lfm_quant_b200.scripts.data_processing import Dataset
    from lfm_quant_b200.scripts.train import Train
    conf = str(workdir / 'config' / 'system-test.conf')
    configs.reset()
    c = base_config.get_configs(['--config=' + conf, '--train=True', '--model_dir', 'valid-dev'])
    tr = Train(c, Dataset(c))
    assert len(tr._valid_batches) > 1
    _, v_mse, v_fcst = tr._validation_metrics_point_estimate()
    preds = np.vstack([tr.model.predict(b[0]) for b in tr._valid_batches])
    targets = np.vstack([b[1].cpu().numpy() for b in tr._valid_batches])
    kw = dict(target_idx=tr.target_index, target_lambda=c.target_lambda, rnn_lambda=c.rnn_lambda)
    _, mse_ref, _, _ = orc.loss_point_estimate(targets.astype(np.float64), preds.astype(np.float64), **kw)
    pu, tu = tr._unscale_preds(preds.copy()), tr._unscale_preds(targets.copy())
    _, fcst_ref, _, _ = orc.loss_point_estimate(tu.astype(np.float32).astype(np.float64),
                                                pu.astype(np.float32).astype(np.float64), **kw)
    assert v_mse == pytest.approx(mse_ref, rel=1e-4)
    assert v_fcst == pytest.approx(fcst_ref, rel=1e-4)
    configs.reset()


def test_cli_trains_and_predicts_with_the_gru_cell(workdir):
    """config.rnn_cell = 'gru' (lfm_quant.py:39, rnn_point_estimate.py:89-98) through the same CLI flow."""
    conf = str(workdir / 'config' / 'system-test.conf')
    extra = ['--rnn_cell', 'gru', '--model_dir', 'system-test-gru']
    configs.reset()
    valid_mse = cli.main(['--config=' + conf, '--train=True'] + extra)
    mdir = workdir / 'experiments' / 'system-test-gru'
    assert np.isfinite(valid_mse)
    ep = pd.read_csv(mdir / 'train_log' / 'system-test-train-logs-epoch.csv')
    assert len(ep) == 2 and ep['mse'].iloc[1] < ep['mse'].iloc[0]
    w = np.load(mdir / 'chkpts' / 'chkpt.lfmq.npz')
    assert set(orc.param_names(1, 'gru')) <= set(w.files)
    assert w['gru_1/kernel'].shape == (32, 192) and w['gru_1/bias'].shape == (2, 192)
    assert np.linalg.norm(w['gru_1/kernel'], axis=0).max() <= 3.0 * (1 + 1e-5)
    configs.reset()
    df = cli.main(['--config=' + conf, '--train=False'] + extra)
    out = pd.read_csv(mdir / 'pred' / 'preds.dat', sep=' ', dtype={'gvkey': str})
    assert len(out) == len(df) > 100 and np.isfinite(out['norm_preds_1']).all()
    configs.reset()


def test_cli_trains_and_predicts_the_uq_range_estimate_model(workdir):
    """nn_type=RNNUqRangeEstimate, UQ=True (model_utils/model.py:25-33; train.py:201-225,338-416; predict.py:135-138)."""
    conf = str(workdir / 'config' / 'system-test.conf')
    extra = ['--nn_type', 'RNNUqRangeEstimate', '--UQ=True', '--dropout', '0.1', '--model_dir', 'system-test-uq']
    configs.reset()
    valid_mse = cli.main(['--config=' + conf, '--train=True'] + extra)
    mdir = workdir / 'experiments' / 'system-test-uq'
    assert np.isfinite(valid_mse)
    ep = pd.read_csv(mdir / 'train_log' / 'system-test-train-logs-epoch.csv')
    assert len(ep) == 2 and np.isfinite(ep['uq_loss']).all() and np.isfinite(ep['valid_uq_loss']).all()
    assert ep['uq_loss'].iloc[1] < ep['uq_loss'].iloc[0]                     # the NLL goes down
    bt = pd.read_csv(mdir / 'train_log' / 'system-test-train-logs-batch.csv')
    assert np.isfinite(bt['uq_loss']).all()
    w = np.load(mdir / 'chkpts' / 'chkpt.lfmq.npz')
    assert set(orc.param_names(1, uq=True)) <= set(w.files) and w['OUTPUT_VARIANCE_1/kernel'].shape == (64, 16)
    configs.reset()
    df = cli.main(['--config=' + conf, '--train=False'] + extra)
    out = pd.read_csv(mdir / 'pred' / 'preds.dat', sep=' ', dtype={'gvkey': str})
    assert len(out) == len(df) > 100
    assert np.isfinite(out['norm_preds_1']).all() and (out['norm_variance_1'] >= 1e-6).all()
    assert np.isfinite(out['variance_1']).all()
    configs.reset()


def test_predict_driver_and_preds_file_match_the_reference_golden(tmp_path, monkeypatch):
    """tests/golden/reference_preds.dat was written by the UNMODIFIED reference scripts/predict.py (with its Dataset) run
    in the build container with a stub model whose predict(inp) is the fixed function below (generator:
    tests/golden/make_reference_preds.py).  This package's Predict, given the same stub and the reference's scaler
    parameters, must produce the same file: batching through the CUDA batcher, extraction of the last step / target
    field, un-scaling, reverse log-squash, seq-norm, the error columns and the column order (SURVEY 8b "Files")."""
    import pickle
    from lfm_quant_b200.scripts import base_config, predict as predict_mod
    from lfm_quant_b200.scripts.data_processing import Dataset
    gold_dir = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')

    class _StubModel(object):
        def predict(self, inp, batch_size=None):
            x = (inp.detach().cpu().numpy() if hasattr(inp, 'detach') else np.asarray(inp)).astype(np.float64)
            base = np.tanh(x.mean(axis=2, keepdims=True))
            return (base + 0.1 * np.arange(16)[None, None, :] * x[:, :, :1]).astype(np.float32)

        def load_weights(self, path):
            return None

        def summary(self):
            return 'stub'

    class _StubFactory(object):
        def __init__(self, config, dataset):
            pass

        def get_model(self):
            return _StubModel()

    monkeypatch.setattr(predict_mod, 'Model', _StubFactory)
    d = tmp_path / 'datasets'
    write_open_dataset(str(d / 'open-dataset.dat'), n_keys=8, n_months=120, seed=11)
    mdir = tmp_path / 'experiments' / 'm'
    os.makedirs(str(mdir / 'chkpts'))
    g = np.load(os.path.join(gold_dir, 'reference_batcher_train.npz'))
    pickle.dump({'center': g['center'], 'scale': g['scale']}, open(str(mdir / 'scales.dat'), 'wb'))
    configs.reset()
    c = base_config.get_configs(['--datafile', 'open-dataset.dat', '--data_dir', str(d), '--experiments_dir',
                                 str(tmp_path / 'experiments'), '--model_dir', 'm', '--financial_fields',
                                 'saleq_ttm-ltq_mrq', '--aux_fields', 'rel_mom1m-rel_mom9m', '--target_field',
                                 'oiadpq_ttm', '--scale_field', 'mrkcap', '--stride', '12', '--forecast_n', '12',
                                 '--min_unrollings', '3', '--max_unrollings', '5', '--start_date', '197001', '--end_date',
                                 '209912', '--validation_size', '0.3', '--seed', '521', '--batch_size', '64',
                                 '--train=False'])
    predict_mod.Predict(c, Dataset(c)).predict()
    got = pd.read_csv(str(mdir / 'pred' / c.preds_fname), sep=' ', dtype={'gvkey': str})
    ref = pd.read_csv(os.path.join(gold_dir, 'reference_preds.dat'), sep=' ', dtype={'gvkey': str})
    assert list(got.columns) == list(ref.columns)
    assert len(got) == len(ref) == 429
    assert (got['date'].astype(str) == ref['date'].astype(str)).all() and (got['gvkey'] == ref['gvkey']).all()
    for col in ref.columns[2:]:
        a, b = got[col].to_numpy(dtype=np.float64), ref[col].to_numpy(dtype=np.float64)
        np.testing.assert_array_equal(np.isnan(a), np.isnan(b), err_msg=col)
        ok = ~np.isnan(b)
        # un-scaled columns are multiplied by the row's seq_norm: an exact zero (padded step) comes back as fp32 rounding
        # residue ~1e-6 * seq_norm on either side, so the absolute tolerance follows the row scale
        atol = 1e-5 * np.maximum(1.0, ref['seq_norm'].to_numpy(dtype=np.float64))
        bad = np.abs(a - b) > (atol + 5e-4 * np.abs(b))
        assert not (bad & ok).any(), (col, int((bad & ok).sum()), float(np.abs(a - b)[bad & ok].max()))
    configs.reset()


def test_predict_writes_every_step_of_a_multi_step_point_model(tmp_path, monkeypatch):
    """predict.py:128-133: a point model with forecast_steps > 1 returns the list of its steps from model.predict, which
    Predict uses as it is (it wraps only a single step's array): preds_1 and preds_2 are the two outputs' last step."""
    import pickle
    from lfm_quant_b200.scripts import base_config, predict as predict_mod
    from lfm_quant_b200.scripts.data_processing import Dataset
    gold_dir = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')

    def step(x, s):
        return (np.tanh(x.mean(axis=2, keepdims=True)) * s + 0.1 * np.arange(16)[None, None, :]).astype(np.float32)

    class _StubModel(object):
        def predict(self, inp, batch_size=None):
            x = inp.detach().cpu().numpy().astype(np.float64)
            return [step(x, 1.0), step(x, 2.0)]

        def load_weights(self, path):
            return None

    class _StubFactory(object):
        def __init__(self, config, dataset):
            pass

        def get_model(self):
            return _StubModel()

    monkeypatch.setattr(predict_mod, 'Model', _StubFactory)
    d = tmp_path / 'datasets'
    write_open_dataset(str(d / 'open-dataset.dat'), n_keys=8, n_months=120, seed=11)
    mdir = tmp_path / 'experiments' / 'm'
    os.makedirs(str(mdir / 'chkpts'))
    g = np.load(os.path.join(gold_dir, 'reference_batcher_train.npz'))
    pickle.dump({'center': g['center'], 'scale': g['scale']}, open(str(mdir / 'scales.dat'), 'wb'))
    configs.reset()
    c = base_config.get_configs(['--datafile', 'open-dataset.dat', '--data_dir', str(d), '--experiments_dir',
                                 str(tmp_path / 'experiments'), '--model_dir', 'm', '--financial_fields',
                                 'saleq_ttm-ltq_mrq', '--aux_fields', 'rel_mom1m-rel_mom9m', '--target_field',
                                 'oiadpq_ttm', '--scale_field', 'mrkcap', '--stride', '12', '--forecast_n', '12',
                                 '--min_unrollings', '3', '--max_unrollings', '5', '--start_date', '197001', '--end_date',
                                 '209912', '--validation_size', '0.3', '--seed', '521', '--batch_size', '64',
                                 '--forecast_steps', '2', '--forecast_steps_weights', '1.0-0.5', '--train=False'])
    try:
        p = predict_mod.Predict(c, Dataset(c))
        df = p.predict()
        x = np.vstack([b[0].cpu().numpy() for b in p._batches]).astype(np.float64)
    finally:
        configs.reset()
    got = pd.read_csv(str(mdir / 'pred' / c.preds_fname), sep=' ', dtype={'gvkey': str})
    assert len(got) == len(df) == len(x) > 0
    for s in (1, 2):
        for col in ('targets_%d', 'norm_preds_%d', 'norm_variance_%d', 'preds_%d', 'variance_%d'):
            assert col % s in got.columns
        np.testing.assert_allclose(got['norm_preds_%d' % s].values, step(x, float(s))[:, -1, p.target_index],
                                   rtol=1e-6)
        assert (got['norm_variance_%d' % s] == 0).all()
    np.testing.assert_array_equal(got['targets_1'].values, got['targets_2'].values)
