"""Walk-forward backtests on the GPU (training_type iterative, DESIGN.md section 6c), end to end through lfm_quant.py on
the synthetic dataset: every origin's files, the stitched walk_forward_preds.dat, each origin's predictions bit for bit
what a plain fixed_dates train and predict with its dates writes (with the origins side by side and one after another),
a re-prediction from the trained origins, and UQ, MLPLinearPointEstimate and NaivePointEstimate backtests."""
import pickle

import numpy as np
import pandas as pd
import pytest

pytestmark = pytest.mark.gpu

# split_date 199612, end_date 199912, stride 12: years in which the synthetic dataset still has many companies
ORIGINS = [199612, 199712, 199812]
PRED_DATES = [(199701, 199712), (199801, 199812), (199901, 199912)]


@pytest.fixture(scope='module')
def workdir(tmp_path_factory):
    from lfm_quant_b200.scripts.synthetic import write_open_dataset, write_system_test_conf
    d = tmp_path_factory.mktemp('wf')
    write_open_dataset(str(d / 'datasets' / 'open-dataset.dat'), n_keys=30, n_months=420, seed=9)
    write_system_test_conf(str(d / 'config' / 'system-test.conf'), str(d / 'datasets'), str(d / 'experiments'))
    (d / 'experiments').mkdir()
    return d


@pytest.fixture()
def cli(workdir, monkeypatch):
    from lfm_quant_b200.scripts import configs
    from lfm_quant_b200.scripts import lfm_quant
    monkeypatch.setenv('LFM_QUANT_ROOT', str(workdir))
    monkeypatch.setenv('LFMQ_SEEDED_SHUFFLE', '1')        # the batch order follows the seed: training is repeatable
    conf = str(workdir / 'config' / 'system-test.conf')

    def main(*argv):
        configs.reset()
        try:
            return lfm_quant.main(['--config=' + conf] + list(argv))
        finally:
            configs.reset()
    return main


def _backtest(model_dir, npe, *extra):
    return ['--training_type', 'iterative', '--split_date', str(ORIGINS[0]), '--end_date', str(PRED_DATES[-1][1]),
            '--model_dir', model_dir, '--NPE', str(npe)] + list(extra)


def _origin_dir(workdir, model_dir, origin):
    return workdir / 'experiments' / model_dir / ('system-test-wf-%d' % origin)


def _stitched_rows(workdir, model_dir, fname='preds.dat'):
    """walk_forward_preds.dat as lines, and the lines it must hold: every origin's rows, with its origin."""
    got = (workdir / 'experiments' / model_dir / 'walk_forward_preds.dat').read_text().splitlines()
    header, rows = None, []
    for o in ORIGINS:
        own = (_origin_dir(workdir, model_dir, o) / 'pred' / fname).read_text().splitlines()
        header = own[0] + ' origin'
        rows += [r + ' %d' % o for r in own[1:]]
    return got, [header] + rows


def test_cli_backtest_matches_plain_fixed_dates_runs(workdir, cli):
    df = cli(*_backtest('wf3', 3), '--train=True')
    for k, o in enumerate(ORIGINS):
        m = _origin_dir(workdir, 'wf3', o)
        for f in ('model-%d.conf' % k, 'predict-%d.conf' % k, 'scales.dat', 'chkpts/chkpt.lfmq.npz',
                  'chkpts/chkpt.index', 'train_log/system-test-train-logs-epoch.csv',
                  'train_log/system-test-train-logs-batch.csv', 'pred/preds.dat'):
            assert (m / f).is_file(), (o, f)
    got, want = _stitched_rows(workdir, 'wf3')
    assert got == want and len(got) > 300
    assert len(df) == len(got) - 1 and df['origin'].tolist() == sorted(df['origin'].tolist())
    dates = pd.to_datetime(df['date'].astype(str), format='%Y%m%d')
    for o, (first, last) in zip(ORIGINS, PRED_DATES):
        mine = dates[df['origin'] == o]
        assert len(mine) > 0 and mine.min() >= pd.Timestamp(str(first) + '01') and mine.max() <= pd.Timestamp(
            str(last) + '01'), o
    w = [np.load(_origin_dir(workdir, 'wf3', o) / 'chkpts' / 'chkpt.lfmq.npz') for o in ORIGINS]
    assert not np.array_equal(w[0]['lstm_1/kernel'], w[1]['lstm_1/kernel'])      # each origin trained its own model

    # one after another (NPE = 1): the same bits
    cli(*_backtest('wf1', 1), '--train=True')
    for o in ORIGINS:
        a, b = ((_origin_dir(workdir, d, o) / 'pred' / 'preds.dat').read_bytes() for d in ('wf3', 'wf1'))
        assert a == b, o

    # each origin is a plain fixed_dates train through its origin and prediction of the months after it
    for o, (first, last) in zip(ORIGINS, PRED_DATES):
        alone = str(workdir / 'experiments' / ('alone-%d' % o))
        cli('--train=True', '--end_date', str(o), '--model_dir', alone)
        cli('--train=False', '--start_date', str(first), '--end_date', str(last), '--model_dir', alone)
        m = _origin_dir(workdir, 'wf3', o)
        sa, sb = (pickle.load(open(str(d), 'rb')) for d in (m / 'scales.dat', workdir / 'experiments' /
                                                             ('alone-%d' % o) / 'scales.dat'))
        for key in ('center', 'scale'):
            np.testing.assert_array_equal(sa[key], sb[key])
        assert (m / 'pred' / 'preds.dat').read_bytes() == (workdir / 'experiments' / ('alone-%d' % o) / 'pred' /
                                                           'preds.dat').read_bytes(), o

    # --train=False predicts again from the trained origins: the same stitched file
    before = (workdir / 'experiments' / 'wf3' / 'walk_forward_preds.dat').read_bytes()
    again = cli(*_backtest('wf3', 3), '--train=False')
    assert (workdir / 'experiments' / 'wf3' / 'walk_forward_preds.dat').read_bytes() == before
    pd.testing.assert_frame_equal(again, df)


def test_cli_uq_backtest_with_monte_carlo_samples(workdir, cli):
    uq = ['--nn_type', 'RNNUqRangeEstimate', '--UQ=True', '--dropout', '0.1', '--recurrent_dropout', '0.1']
    cli(*_backtest('wf-uq', 3), *uq, '--train=True')
    df = cli(*_backtest('wf-uq', 3), *uq, '--train=False', '--mc_samples', '4')
    got, want = _stitched_rows(workdir, 'wf-uq')
    assert got == want and len(df) == len(got) - 1 > 300
    assert np.isfinite(df['norm_preds_var_1']).all() and np.isfinite(df['norm_variance_1']).all()
    for o in ORIGINS:
        assert (_origin_dir(workdir, 'wf-uq', o) / 'ensemble_preds.dat').is_file(), o


def test_cli_mlp_linear_backtest(workdir, cli):
    mlp = ['--nn_type', 'MLPLinearPointEstimate', '--init_scale', '0.02', '--max_epoch', '2']
    df = cli(*_backtest('wf-mlp', 3), *mlp, '--train=True')
    got, want = _stitched_rows(workdir, 'wf-mlp')
    assert got == want and len(df) > 300 and np.isfinite(df['preds_1']).all()
    for o in ORIGINS:
        w = np.load(_origin_dir(workdir, 'wf-mlp', o) / 'chkpts' / 'chkpt.lfmq.npz')
        assert sorted(w.files) == ['OUTPUT_1/bias', 'OUTPUT_1/kernel']

    # the naive forecast predicts every origin without training, with the scaling of --scalesfile
    scales = str(_origin_dir(workdir, 'wf-mlp', ORIGINS[0]) / 'scales.dat')
    df = cli(*_backtest('wf-naive', 3), '--nn_type', 'NaivePointEstimate', '--scalesfile', scales, '--train=False')
    got, want = _stitched_rows(workdir, 'wf-naive')
    assert got == want and len(df) > 300
    np.testing.assert_array_equal(df['preds_1'].values, df['inp_t0'].values)
