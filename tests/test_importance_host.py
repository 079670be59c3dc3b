"""Permutation importance on the host: the bijection (lfmq_permutation_index against the NumPy oracle), the
--perm_importance flag and the runs it is refused for, and the importance.dat table with its walk-forward stacking from
stubbed outputs.  The importance itself is checked on the GPU (tests/test_gpu_importance.py)."""
import ctypes as C
import os

import numpy as np
import pandas as pd
import pytest

import importance_oracle as imo
from lfm_quant_b200 import _native as N
from lfm_quant_b200.scripts import base_config, configs
from lfm_quant_b200.scripts.predict import importance_table
from lfm_quant_b200.scripts.runtime import model_execution as me

ERR_ARG = 1             # LFMQ_ERR_ARG (include/lfmq.h)


def _native_permutation(N_, seed, g, r):
    lib, out = N.load(), C.c_int32(0)
    pi = np.empty(N_, dtype=np.int64)
    for i in range(N_):
        assert lib.lfmq_permutation_index(N_, seed, g, r, i, C.byref(out)) == 0
        pi[i] = out.value
    return pi


@pytest.mark.parametrize('n', [1, 2, 3, 4, 5, 255, 256, 257, 65537])
def test_library_bijection_is_the_oracles_and_a_permutation(n):
    for seed, g, r in ((521, 0, 0), (2 ** 40 + 7, 31, 1)):
        want = imo.permutation(n, seed, g, r)
        assert np.array_equal(np.sort(want), np.arange(n))
        assert np.array_equal(_native_permutation(n, seed, g, r), want)


def test_every_seed_group_and_repeat_gives_its_own_permutation():
    n = 1000
    keys = [(s, g, r) for s in (1, 2, 2 ** 33 + 1) for g in (0, 1, 47) for r in (0, 1)]
    perms = {k: imo.permutation(n, *k) for k in keys}
    for k in keys:
        assert not np.array_equal(perms[k], np.arange(n)), k
    for a in keys:
        for b in keys:
            if a < b:
                assert not np.array_equal(perms[a], perms[b]), (a, b)
    assert np.array_equal(imo.permutation(n, 1, 0, 0), perms[(1, 0, 0)])       # a pure function of its key


def test_bad_arguments_of_the_bijection_are_refused():
    lib, out = N.load(), C.c_int32(0)
    for args in ((0, 1, 0, 0, 0), (5, 1, 0, 0, 5), (5, 1, 0, 0, -1), (5, 1, -1, 0, 0), (5, 1, 0, -1, 0)):
        assert lib.lfmq_permutation_index(*args, C.byref(out)) == ERR_ARG, args
    assert lib.lfmq_permutation_index(5, 1, 0, 0, 0, None) == ERR_ARG


def test_permuted_copy_moves_one_group_with_its_zero_padding():
    x = np.arange(5 * 3 * 2, dtype=np.float64).reshape(5, 3, 2)
    x[2, 0, :] = 0.0                                           # a padded quarter of window 2
    pi = imo.permutation(5, 9, 1, 0)
    cg, G = imo.field_groups(3, 2)
    got = imo.permuted_copy(x, cg, 1, pi)
    assert np.array_equal(got[:, :, 0], x[:, :, 0]) and np.array_equal(got[:, :, 1], x[pi][:, :, 1])
    cg, G = imo.quarter_groups(3, 2)
    got = imo.permuted_copy(x.reshape(5, 6), cg, 0, pi).reshape(5, 3, 2)   # the flattened layout numbers c alike
    assert np.array_equal(got[:, 0], x[pi][:, 0]) and np.array_equal(got[:, 1:], x[:, 1:])


@pytest.fixture()
def fresh_flags():
    configs.reset()
    yield
    configs.reset()


def test_perm_importance_flag_defaults_to_off(fresh_flags):
    assert base_config.get_configs([]).perm_importance == 0
    assert base_config.get_configs(['--perm_importance', '2']).perm_importance == 2


@pytest.mark.parametrize('argv', [
    ['--perm_importance', '2', '--train=True'],
    ['--perm_importance', '-1', '--train=False'],
    ['--perm_importance', '2', '--train=False', '--nn_type', 'NaivePointEstimate'],
])
def test_perm_importance_is_refused_before_any_work(fresh_flags, monkeypatch, argv):
    ran = []
    monkeypatch.setattr(me.ModelExecution, 'single_execution', staticmethod(lambda cfg: ran.append(cfg) or 'ran'))
    monkeypatch.setattr(me.ModelExecution, 'fixed_dates_execution', lambda self: ran.append(self) or 'ran')
    with pytest.raises(ValueError, match='--perm_importance'):
        me.ModelExecution(base_config.get_configs(argv))()
    assert ran == []


@pytest.mark.parametrize('argv', [
    ['--perm_importance', '2', '--train=False'],
    ['--perm_importance', '1', '--train=False', '--nn_type', 'RNNUqRangeEstimate', '--UQ=True', '--mc_samples', '4'],
    ['--perm_importance', '3', '--train=False', '--nn_type', 'MLPLinearPointEstimate'],
    ['--perm_importance', '2', '--train=False', '--forecast_steps', '2', '--forecast_steps_weights', '1.0-0.5'],
    ['--perm_importance', '0', '--train=True'],
])
def test_perm_importance_runs_every_trained_model_at_prediction(fresh_flags, monkeypatch, argv):
    seen = []
    monkeypatch.setattr(me.ModelExecution, 'single_execution', staticmethod(lambda cfg: seen.append(cfg) or 'ran'))
    monkeypatch.setattr(me.ModelExecution, 'write_uq_ensemble', classmethod(lambda cls, cfg: None))
    assert me.ModelExecution(base_config.get_configs(argv))() == 'ran'
    assert len(seen) == 1


def _out(G, R, seed, uq=False):
    rng = np.random.RandomState(seed)
    out = rng.uniform(0.5, 2.0, size=(1 + G * R, 3)).astype(np.float32)
    if not uq:
        out[:, 2] = 0.0
    return out


@pytest.mark.parametrize('uq', [False, True])
def test_importance_table_from_stubbed_outputs(uq):
    T, F, R = 4, 3, 2
    names = ['f_a', 'f_b', 'f_c']
    fields, quarters = _out(F, R, 1, uq), _out(T, R, 2, uq)
    quarters[0] = fields[0]                                     # one baseline, as the model computes it
    df = importance_table(fields, quarters, R, names, uq)
    assert list(df.columns) == ['kind', 'group', 'base_loss', 'perm_loss', 'perm_loss_std', 'delta_loss', 'base_mse',
                                'perm_mse', 'delta_mse']
    assert df['kind'].tolist() == ['field'] * F + ['quarter'] * T
    assert df['group'].tolist() == names + [-3, -2, -1, 0]
    m = 2 if uq else 1
    for k, (kind, out, g) in enumerate([('field', fields, g) for g in range(F)] + [('quarter', quarters, g)
                                                                                  for g in range(T)]):
        rows = out[1 + g * R:1 + (g + 1) * R].astype(np.float64)
        row = df.iloc[k]
        assert row['base_loss'] == out[0, 0] and row['base_mse'] == out[0, m]
        assert row['perm_loss'] == pytest.approx(rows[:, 0].mean(), rel=1e-15)
        assert row['perm_loss_std'] == pytest.approx(np.sqrt(np.mean((rows[:, 0] - rows[:, 0].mean()) ** 2)),
                                                     rel=1e-12)
        assert row['delta_loss'] == pytest.approx(rows[:, 0].mean() - out[0, 0], rel=1e-12, abs=1e-15)
        assert row['perm_mse'] == pytest.approx(rows[:, m].mean(), rel=1e-15)
        assert row['delta_mse'] == pytest.approx(rows[:, m].mean() - out[0, m], rel=1e-12, abs=1e-15)


def test_walk_forward_stacks_the_origins_importance_files(fresh_flags, tmp_path, monkeypatch):
    (tmp_path / 'exp').mkdir()
    tables = {}

    def fake_member(cfg, share_den):
        assert not cfg.train and cfg.perm_importance == 2
        d = os.path.join(cfg.model_dir, 'pred')
        os.makedirs(d, exist_ok=True)
        origin = me.add_months(cfg.start_date, -1)
        pd.DataFrame({'date': [20000101], 'gvkey': ['001000'], 'norm_squared_diff_1': [0.5]}).to_csv(
            os.path.join(d, cfg.preds_fname), sep=' ', index=False)
        tables[origin] = importance_table(_out(2, 2, origin % 97), _out(3, 2, origin % 89), 2, ['x', 'y'], False)
        tables[origin].to_csv(os.path.join(d, 'importance.dat'), sep=' ', index=False)

    monkeypatch.setattr(me.ModelExecution, 'member_execution', staticmethod(fake_member))
    c = base_config.get_configs(['--experiments_dir', str(tmp_path / 'exp'), '--model_dir', 'wf', '--name', 'bt',
                                 '--training_type', 'iterative', '--start_date', '197501', '--end_date', '200412',
                                 '--split_date', '200112', '--train=False', '--perm_importance', '2'])
    for o in (200112, 200212, 200312):
        (tmp_path / 'exp' / 'wf' / ('bt-wf-%d' % o)).mkdir(parents=True)
    me.ModelExecution(c)()
    origins = [200112, 200212, 200312]
    got = pd.read_csv(tmp_path / 'exp' / 'wf' / 'walk_forward_importance.dat', sep=' ', dtype={'group': str},
                      float_precision='round_trip')
    want = pd.concat([tables[o].astype({'group': str}).assign(origin=o) for o in origins], ignore_index=True)
    assert got['origin'].tolist() == [o for o in origins for _ in range(5)]
    pd.testing.assert_frame_equal(got, want)
