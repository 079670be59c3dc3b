"""Hyper-parameter search on the CPU, with candidate training replaced by tests/hpo_stub.py: the genetic algorithm,
grid search and DOE draw the candidates the reference draws, in the same order, and write the same model.conf and
opt_hist.csv files (tests/golden/reference_hpo.json, made by running the reference's own search classes with the same
stub: tests/golden/make_reference_hpo.py).  The project's one extra flag, ``precision``, is taken out before the
comparison.  Also: the population pickle round trip, the refusals, and a failing candidate."""
import io
import json
import os
import pickle
import subprocess
import sys

import numpy as np
import pandas as pd
import pytest

import hpo_stub

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = json.load(open(os.path.join(HERE, 'golden', 'reference_hpo.json')))
CASES = ['genetic', 'genetic_doe', 'grid_search', 'doe']


def stub_execute(conf_paths, npe):
    for path in conf_paths:
        hpo_stub.train_candidate(path)
    return [None] * len(conf_paths)


def as_json(config):
    """A config as the generator records it, without the project's `precision` flag."""
    items = json.loads(json.dumps(list(config.as_dict().items()), default=str))
    return [[k, v] for k, v in items if k != 'precision']


def without_precision(name, text):
    if name.endswith('model.conf'):
        return ''.join(l for l in text.splitlines(True) if not l.startswith('--precision '))
    rows = [l.split(',') for l in text.splitlines()]
    k = rows[0].index('precision')
    return ''.join(','.join(r[:k] + r[k + 1:]) + '\n' for r in rows)


def outputs(directory):
    found = {}
    for d, _, names in os.walk(directory):
        for n in names:
            if n in ('model.conf', 'opt_hist.csv'):
                p = os.path.join(d, n)
                found[os.path.relpath(p, directory)] = open(p).read()
    return found


@pytest.fixture
def search(tmp_path, monkeypatch):
    """search(argv, files={}, execute=stub_execute) -> (generations, search object), run in tmp_path."""
    from lfm_quant_b200.scripts import hyper_param_opt
    from lfm_quant_b200.scripts.param_search.opt_base_class import OptimizerBaseClass
    from lfm_quant_b200.scripts.param_search.optimization import HPOptimization
    monkeypatch.chdir(tmp_path)
    monkeypatch.setenv('LFM_QUANT_ROOT', GOLDEN['data_root'])
    monkeypatch.delenv('WORLD_SIZE', raising=False)
    generations = []
    train = OptimizerBaseClass._train_population

    def recorded(self, gen):
        generations.append([as_json(m) for m in self._cur_pop])
        return train(self, gen)
    monkeypatch.setattr(OptimizerBaseClass, '_train_population', recorded)

    def run(argv, files=None, execute=stub_execute):
        for name, text in (files or {}).items():
            (tmp_path / name).write_text(text)
        del generations[:]
        found = HPOptimization(hyper_param_opt.get_configs(argv), execute)()
        return list(generations), found
    return run


@pytest.mark.parametrize('case', CASES)
def test_search_draws_the_reference_candidates_and_writes_its_files(case, search, tmp_path):
    ref = GOLDEN[case]
    generations, _ = search(ref['argv'], ref['files'])
    assert len(generations) == len(ref['generations'])
    for g, (ours, theirs) in enumerate(zip(generations, ref['generations'])):
        assert ours == theirs, 'generation %d' % (g + 1)
    ours = outputs(str(tmp_path))
    assert sorted(ours) == sorted(ref['outputs'])
    for name, text in ref['outputs'].items():
        assert without_precision(name, ours[name]) == text, name


def test_the_fixture_covers_what_it_names():
    ga = GOLDEN['genetic']
    assert [len(g) for g in ga['generations']] == [6, 6, 6]
    hist = pd.read_csv(io.StringIO(ga['outputs']['ga/opt_run/opt_hist.csv']))
    assert list(hist['id']) == list(range(1, 19))            # member ids keep increasing across generations
    assert np.isinf(hist.loc[hist['id'] == hpo_stub.FAIL_ID, 'objective']).all()
    assert sorted(set(dict(m)['default_gpu'] for m in ga['generations'][0])) == ['/gpu:0', '/gpu:1']
    assert [len(g) for g in GOLDEN['grid_search']['generations']] == [5, 5]     # 12 combinations, 2 dropped
    assert [len(g) for g in GOLDEN['doe']['generations']] == [2, 2, 1]
    assert [len(g) for g in GOLDEN['genetic_doe']['generations']] == [4, 4]


def test_model_conf_parses_to_the_candidate(search, tmp_path):
    from lfm_quant_b200.scripts.runtime.model_execution import candidate_config
    search(['--name', 'one', '--search_algorithm', 'grid_search', '--NPE', '2', '--num_hidden', '32', '64',
            '--precision', 'bf16', '--batch_size', '128'])
    conf = tmp_path / 'one' / 'opt_run' / 'one-2' / 'model.conf'
    lines = conf.read_text().splitlines(True)
    assert '--num_hidden       64 \n' in lines and '--precision       bf16 \n' in lines
    assert '--forecast_steps_weights       1.0\n' in lines
    assert lines == sorted(lines)
    c = candidate_config(str(conf))
    assert (c.num_hidden, c.batch_size, c.precision, c.member_id, c.train, c.num_procs) == (64, 128, 'bf16', 2, True, 1)
    assert c.model_dir == os.path.join('one', 'opt_run', 'one-2') and c.forecast_steps_weights == [1.0]
    assert c.data_dir == os.path.join(GOLDEN['data_root'], 'datasets')


def test_latest_pop_round_trip(search, tmp_path):
    argv = ['--name', 'pop', '--generations', '2', '--pop_size', '4', '--num_hidden', '32', '64',
            '--learning_rate', '0.1', '0.3', '0.6', '--save_latest_pop']
    first, _ = search(argv)
    pkl = tmp_path / 'pop' / '_latest_pop' / 'latest_pop.pkl'
    with open(str(pkl), 'rb') as fh:
        saved = pickle.load(fh)
    assert [as_json(m) for m in saved] == first[1]      # the generation about to train when it was saved
    second, _ = search(argv + ['--name', 'pop2', '--init_pop', str(pkl)])
    assert second[0] == first[1]


def test_unknown_algorithm_is_refused(search):
    with pytest.raises(NotImplementedError):
        search(['--search_algorithm', 'bayesian'])


@pytest.mark.parametrize('algorithm', ['genetic', 'grid_search'])
def test_genetic_and_grid_refuse_uq(algorithm, search, tmp_path):
    with pytest.raises(NotImplementedError):
        search(['--search_algorithm', algorithm, '--UQ', '--num_hidden', '32', '64'])
    assert not list(tmp_path.rglob('model.conf'))            # refused before any candidate


def test_doe_scores_uq_models_by_their_uq_loss(search, tmp_path):
    search(['--name', 'uq', '--search_algorithm', 'doe', '--NPE', '2', '--UQ', '--doe_file', 'd.csv'],
           {'d.csv': 'num_hidden\n32\n64\n'})
    hist = pd.read_csv(tmp_path / 'uq' / 'opt_hist.csv')
    assert list(hist.columns[:5]) == ['id', 'gen', 'objective', 'valid_mse', 'valid_uq_loss']
    for _, row in hist.iterrows():
        conf = tmp_path / 'uq' / 'opt_run' / ('uq-%d' % row['id']) / 'model.conf'
        m = hpo_stub.objective(hpo_stub.read_conf(str(conf)))
        # the epoch with the lower UQ loss is the first one, whose MSE is the higher
        assert (row['objective'], row['valid_mse'], row['valid_uq_loss']) == (m + 0.5, m + 0.5, 3 * m)


def test_a_failing_candidate_scores_inf_and_the_search_goes_on(search, tmp_path):
    def execute(conf_paths, npe):
        stub_execute(conf_paths, npe)       # it wrote a log before it failed: the failure still scores inf
        return [RuntimeError('refused') if hpo_stub.read_conf(p)['num_hidden'] == '64' else None for p in conf_paths]
    generations, _ = search(['--name', 'f', '--search_algorithm', 'grid_search', '--NPE', '2',
                             '--num_hidden', '32', '64', '--learning_rate', '0.1', '0.3'], execute=execute)
    assert len(generations) == 2
    hist = pd.read_csv(tmp_path / 'f' / 'opt_run' / 'opt_hist.csv')
    assert list(np.isinf(hist['objective'])) == list(hist['num_hidden'] == 64)
    assert np.isinf(hist.loc[hist['num_hidden'] == 64, ['valid_mse', 'valid_mse_fcst']].values).all()


def test_search_refuses_torchrun(search, monkeypatch):
    monkeypatch.setenv('WORLD_SIZE', '2')
    with pytest.raises(NotImplementedError, match='torchrun'):
        search(['--search_algorithm', 'grid_search', '--num_hidden', '32', '64'])


def test_cli_script_needs_lfm_quant_root_and_refuses_unknown_algorithms(tmp_path):
    script = os.path.join(ROOT, 'lfm_quant_b200', 'scripts', 'hyper_param_opt.py')
    env = dict(os.environ)
    env.pop('LFM_QUANT_ROOT', None)
    r = subprocess.run([sys.executable, script], cwd=str(tmp_path), env=env, capture_output=True, text=True)
    assert r.returncode != 0 and 'LFM_QUANT_ROOT' in r.stderr
    env['LFM_QUANT_ROOT'] = str(tmp_path)
    r = subprocess.run([sys.executable, script, '--search_algorithm', 'bayesian'], cwd=str(tmp_path), env=env,
                       capture_output=True, text=True)
    assert r.returncode != 0 and 'NotImplementedError' in r.stderr
