"""Hyper-parameter search on the GPU: the candidates of a generation train side by side in one process, and each one
scores what ``lfm_quant.py --config <its model.conf>`` logs when it trains alone -- bit for bit at fp32, within the
bound of tests/test_gpu_ensemble.py at bf16.  A candidate the library refuses (GRU on the bf16 training path) scores
inf and the search completes.  At fp32 a search with NPE 4 and the same search with NPE 1 write the same
opt_hist.csv."""
import os

import numpy as np
import pandas as pd
import pytest

pytestmark = pytest.mark.gpu

SHAPE = ['--datafile', 'open-dataset.dat', '--num_layers', '1', '--batch_size', '64', '--max_epoch', '1',
         '--end_date', '200412', '--logging_interval', '1000']


@pytest.fixture(scope='module')
def workdir(tmp_path_factory):
    from lfm_quant_b200.scripts.synthetic import write_open_dataset
    d = tmp_path_factory.mktemp('hpo')
    write_open_dataset(str(d / 'datasets' / 'open-dataset.dat'), n_keys=30, n_months=420, seed=9)
    (d / 'experiments').mkdir()
    return d


@pytest.fixture
def env(workdir, monkeypatch):
    monkeypatch.setenv('LFM_QUANT_ROOT', str(workdir))
    monkeypatch.setenv('LFMQ_SEEDED_SHUFFLE', '1')       # the batch order follows the seed: training is repeatable
    monkeypatch.delenv('WORLD_SIZE', raising=False)
    return workdir


def search(workdir, argv):
    from lfm_quant_b200.scripts import configs, hyper_param_opt
    hyper_param_opt.main(['--experiments_dir', str(workdir / 'experiments')] + SHAPE + argv)
    configs.reset()


def alone(conf, out_dir):
    """Best epoch (by validation MSE) of the candidate trained alone from its model.conf, in out_dir."""
    from lfm_quant_b200.scripts import configs
    from lfm_quant_b200.scripts import lfm_quant as cli
    configs.reset()
    cli.main(['--config=' + str(conf), '--model_dir', str(out_dir)])
    configs.reset()
    log = pd.read_csv(out_dir / 'train_log' / (conf.parent.parent.parent.name + '-train-logs-epoch.csv'))
    best = log.sort_values(by='valid_mse').reset_index().iloc[0]
    return best['valid_mse'], best['valid_mse_fcst']


def check_against_alone(workdir, name, hist, mse_col, fcst_col):
    for _, row in hist.iterrows():
        conf = workdir / 'experiments' / name / 'opt_run' / ('%s-%d' % (name, row['id'])) / 'model.conf'
        mse, fcst = alone(conf, workdir / 'experiments' / 'alone' / ('%s-%d' % (name, row['id'])))
        assert np.isfinite(mse)
        if row['precision'] == 'fp32':
            assert (row[mse_col], row[fcst_col]) == (mse, fcst), row['id']
        else:       # the bound of test_gpu_ensemble.py for the bf16 paths
            np.testing.assert_allclose([row[mse_col], row[fcst_col]], [mse, fcst], rtol=1e-6, atol=1e-9)


def test_genetic_search_scores_what_each_candidate_logs_alone(env):
    search(env, ['--name', 'ga', '--search_algorithm', 'genetic', '--pop_size', '4', '--generations', '2',
                 '--NPE', '4', '--num_hidden', '64', '128', '--learning_rate', '0.3', '0.6',
                 '--precision', 'fp32', 'bf16'])
    hist = pd.read_csv(env / 'experiments' / 'ga' / 'opt_run' / 'opt_hist.csv')
    assert list(hist['id']) == list(range(1, 9)) and list(hist['gen']) == [1] * 4 + [2] * 4
    assert np.isfinite(hist['objective']).all()
    assert (hist['objective'] == hist['valid_mse']).all()
    check_against_alone(env, 'ga', hist, 'valid_mse', 'valid_mse_fcst')


def test_grid_search_scores_a_refused_candidate_inf_and_completes(env):
    search(env, ['--name', 'grid', '--search_algorithm', 'grid_search', '--NPE', '4', '--num_hidden', '64',
                 '--rnn_cell', 'lstm', 'gru', '--precision', 'fp32', 'bf16'])
    hist = pd.read_csv(env / 'experiments' / 'grid' / 'opt_run' / 'opt_hist.csv')
    assert list(zip(hist['rnn_cell'], hist['precision'])) == [('lstm', 'fp32'), ('lstm', 'bf16'), ('gru', 'fp32'),
                                                               ('gru', 'bf16')]
    refused = (hist['rnn_cell'] == 'gru') & (hist['precision'] == 'bf16')
    assert np.isinf(hist.loc[refused, ['objective', 'valid_mse', 'valid_mse_fcst']].values).all()
    assert np.isfinite(hist.loc[~refused, 'objective']).all()
    # grid search records (forecast-space MSE, validation MSE) the other way round from the genetic algorithm
    check_against_alone(env, 'grid', hist[~refused], 'valid_mse_fcst', 'objective')


def test_fp32_search_writes_the_same_history_with_one_candidate_at_a_time(env):
    argv = ['--search_algorithm', 'genetic', '--pop_size', '4', '--generations', '2', '--num_hidden', '64', '128',
            '--learning_rate', '0.1', '0.3', '0.6', '--num_layers', '1', '2']
    search(env, argv + ['--name', 'side', '--NPE', '4'])
    search(env, argv + ['--name', 'serial', '--NPE', '1'])
    side, serial = (open(os.path.join(str(env), 'experiments', n, 'opt_run', 'opt_hist.csv')).read()
                    for n in ('side', 'serial'))
    assert np.isfinite(pd.read_csv(os.path.join(str(env), 'experiments', 'side', 'opt_run',
                                                'opt_hist.csv'))['objective']).all()
    assert side == serial
