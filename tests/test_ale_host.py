"""Accumulated local effects on the host: the fp64 oracle of tests/ale_oracle.py (the components of an additive
function, the closed form of a linear one, the binning rules), the --ale_bins flag and the runs it is refused for,
ale.dat from stubbed outputs, the walk-forward stacking and a no-spill compile of the kernels.  The library's effects
are checked on the GPU (tests/test_gpu_ale.py)."""
import os
import re
import shlex
import shutil
import subprocess
import tempfile
import types

import numpy as np
import pandas as pd
import pytest

import ale_oracle as alo
from lfm_quant_b200.scripts import base_config, configs
from lfm_quant_b200.scripts.predict import Predict, ale_table, shapley_output_names
from lfm_quant_b200.scripts.runtime import model_execution as me

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _centred(hz, n):
    """h at the edges minus h(z_0), centred so that the count-weighted mean over the bins is 0"""
    acc = hz - hz[0]
    return acc - (n * 0.5 * (acc[:-1] + acc[1:])).sum() / n.sum()


@pytest.mark.parametrize('K', [1, 4, 10, 1000])
def test_each_component_of_an_additive_function_is_recovered(K):
    T, F, N_ = 3, 4, 211
    rng = np.random.RandomState(1)
    x = rng.normal(size=(N_, T, F)).astype(np.float32).astype(np.float64)
    cols = [(T - 1) * F + f for f in range(F)] + [2]
    hs = [np.sin, np.tanh, np.square, np.exp, np.cos]

    def f(z, m):
        flat = z.reshape(z.shape[0], -1)
        return np.stack([sum(h(flat[:, c]) for h, c in zip(hs, cols)), flat[:, 0] * 3.0], axis=1)
    r = alo.ale(x, cols, K, f)
    for g, (h, c) in enumerate(zip(hs, cols)):
        Kg = r['n_bins'][g]
        z = r['edges'][g, :Kg + 1]
        n = r['counts'][g, :Kg]
        assert Kg == min(K, N_ - 1) and n.sum() == N_ and (n > 0).all()
        np.testing.assert_allclose(r['ale'][g, :Kg + 1, 0], _centred(h(z), n), rtol=0, atol=1e-12)
        np.testing.assert_allclose(r['local_sd'][g, :Kg, 0], 0.0, atol=1e-12)  # every window of a bin moves alike
        want1 = np.zeros(Kg + 1) if c != 0 else _centred(3.0 * z, n)
        np.testing.assert_allclose(r['ale'][g, :Kg + 1, 1], want1, rtol=0, atol=1e-12)


def test_a_linear_function_gives_its_slope_times_the_centred_edges():
    N_, K, w = 500, 16, -1.75
    x = np.random.RandomState(2).normal(size=(N_, 6)).astype(np.float32).astype(np.float64)
    r = alo.ale(x, [3], K, lambda z, m: (w * z[:, 3] + np.sin(z[:, 0]))[:, None])
    z, n = r['edges'][0, :K + 1], r['counts'][0]
    cbar = (n * 0.5 * (z[:-1] + z[1:])).sum() / N_
    np.testing.assert_allclose(r['ale'][0, :, 0], w * (z - cbar), rtol=0, atol=1e-12)
    assert np.isclose((n * 0.5 * (r['ale'][0, :-1, 0] + r['ale'][0, 1:, 0])).sum(), 0.0, atol=1e-12)


def test_edges_are_type_1_quantiles_and_bins_are_right_closed():
    v = np.array([5.0, 1.0, 3.0, 2.0, 4.0, 6.0, 7.0, 8.0])
    z, b = alo.bins(v, 4)                             # q = v_(1), v_(2), v_(4), v_(6), v_(8)
    assert z.tolist() == [1.0, 2.0, 4.0, 6.0, 8.0]
    assert b.tolist() == [3, 1, 2, 1, 2, 3, 4, 4]      # 1 = z_0 joins bin 1


def test_ties_and_repeated_quantiles_collapse():
    v = np.array([1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 2.0, 3.0])
    z, b = alo.bins(v, 4)                             # q = 1, 1, 1, 1, 3: z = 1, 3
    assert z.tolist() == [1.0, 3.0] and b.tolist() == [1] * 8
    z, b = alo.bins(v, 8)                             # q = 1, 1, 1, 1, 1, 1, 1, 2, 3
    assert z.tolist() == [1.0, 2.0, 3.0] and b.tolist() == [1] * 7 + [2]


def test_a_constant_column_has_no_bins_and_non_finite_values_are_left_out():
    z, b = alo.bins(np.full(9, 0.25), 3)
    assert z.tolist() == [0.25] and b.tolist() == [0] * 9
    z, b = alo.bins(np.array([np.nan, np.inf, -np.inf]), 3)
    assert z.size == 0 and b.tolist() == [0, 0, 0]
    v = np.array([np.nan, 2.0, -np.inf, 1.0, 3.0, np.inf, 4.0])
    z, b = alo.bins(v, 2)                             # the four finite values: q = 1, 2, 4
    assert z.tolist() == [1.0, 2.0, 4.0] and b.tolist() == [0, 1, 0, 1, 2, 0, 2]
    x = np.stack([v, np.full(7, 2.0)], axis=1)
    r = alo.ale(x, [0, 1], 2, lambda z_, m: (z_[:, 0] * 2.0)[:, None])
    assert r['n_bins'].tolist() == [2, 0] and r['counts'].tolist() == [[2, 2], [0, 0]]
    assert np.isnan(r['d'][0][[0, 2, 5]]).all() and np.isfinite(r['d'][0][[1, 3, 4, 6]]).all()
    assert r['edges'][1, 0] == 2.0 and np.isnan(r['edges'][1, 1:]).all() and np.isnan(r['ale'][1]).all()


# ---- the flag ----------------------------------------------------------------------------------------------------------
@pytest.fixture()
def fresh_flags():
    configs.reset()
    yield
    configs.reset()


def test_ale_bins_flag_defaults_to_off(fresh_flags):
    assert base_config.get_configs([]).ale_bins == 0
    assert base_config.get_configs(['--ale_bins', '16']).ale_bins == 16


@pytest.mark.parametrize('argv', [
    ['--ale_bins', '8', '--train=True'],
    ['--ale_bins', '-1', '--train=False'],
    ['--ale_bins', '8', '--train=False', '--nn_type', 'NaivePointEstimate'],
])
def test_ale_bins_is_refused_before_any_work(fresh_flags, monkeypatch, argv):
    ran = []
    monkeypatch.setattr(me.ModelExecution, 'single_execution', staticmethod(lambda cfg: ran.append(cfg) or 'ran'))
    monkeypatch.setattr(me.ModelExecution, 'fixed_dates_execution', lambda self: ran.append(self) or 'ran')
    with pytest.raises(ValueError, match='--ale_bins'):
        me.ModelExecution(base_config.get_configs(argv))()
    assert ran == []


@pytest.mark.parametrize('argv', [
    ['--ale_bins', '8', '--train=False'],
    ['--ale_bins', '1', '--train=False', '--nn_type', 'RNNUqRangeEstimate', '--UQ=True', '--mc_samples', '4'],
    ['--ale_bins', '5', '--train=False', '--nn_type', 'MLPLinearPointEstimate'],
    ['--ale_bins', '8', '--train=False', '--forecast_steps', '2', '--forecast_steps_weights', '1.0-0.5'],
    ['--ale_bins', '0', '--train=True'],
])
def test_ale_bins_runs_every_trained_model_at_prediction(fresh_flags, monkeypatch, argv):
    seen = []
    monkeypatch.setattr(me.ModelExecution, 'single_execution', staticmethod(lambda cfg: seen.append(cfg) or 'ran'))
    monkeypatch.setattr(me.ModelExecution, 'write_uq_ensemble', classmethod(lambda cls, cfg: None))
    assert me.ModelExecution(base_config.get_configs(argv))() == 'ran'
    assert len(seen) == 1


# ---- ale.dat -----------------------------------------------------------------------------------------------------------
def _stub_outputs(F, K, J, kf, seed):
    rng = np.random.RandomState(seed)
    edges = np.full((F, K + 1), np.nan, dtype=np.float32)
    counts = np.zeros((F, K), dtype=np.int32)
    ale = np.full((F, K + 1, J), np.nan, dtype=np.float32)
    lm, ls = np.full((F, K, J), np.nan, dtype=np.float32), np.full((F, K, J), np.nan, dtype=np.float32)
    for f, k in enumerate(kf):
        edges[f, :k + 1] = np.sort(rng.normal(size=k + 1))
        counts[f, :k] = rng.randint(1, 9, size=k)
        ale[f, :k + 1] = rng.normal(size=(k + 1, J))
        lm[f, :k], ls[f, :k] = rng.normal(size=(k, J)), rng.uniform(size=(k, J))
    if kf[-1] == 0:
        edges[-1, 0] = 0.5
    return np.array(kf, dtype=np.int32), edges, counts, ale, lm, ls


@pytest.mark.parametrize('steps,uq', [(1, False), (2, True)])
def test_ale_dat_from_stubbed_outputs(tmp_path, steps, uq):
    T, F, K, J = 4, 3, 5, 2 * steps if uq else steps
    out = _stub_outputs(F, K, J, [5, 2, 0], seed=6)
    calls = []

    class Model(object):
        def ale(self, inp, bins):
            calls.append((np.asarray(inp).copy(), bins))
            return tuple(types.SimpleNamespace(cpu=lambda a=a: types.SimpleNamespace(numpy=lambda: a)) for a in out)

    import torch
    sizes = [5, 2]
    windows = [torch.arange(n * T * F, dtype=torch.float32).reshape(n, T, F) + 1000 * b for b, n in enumerate(sizes)]
    p = object.__new__(Predict)
    p.model, p.pred_dir = Model(), str(tmp_path)
    p.config = types.SimpleNamespace(ale_bins=K, forecast_steps=steps, UQ=uq)
    p.dataset = types.SimpleNamespace(fin_col_names=['f_a', 'f_b'], aux_col_names=['aux'])
    p._write_ale(windows)
    assert len(calls) == 1 and calls[0][1] == K
    assert np.array_equal(calls[0][0], torch.cat(windows).numpy())       # every window at once, in preds.dat order
    df = pd.read_csv(tmp_path / 'ale.dat', sep=' ', dtype={'field': str}, float_precision='round_trip')
    names = shapley_output_names(steps, uq)
    assert list(df.columns) == ['field', 'edge_idx', 'edge', 'n'] + [
        '%s_%s' % (k, o) for o in names for k in ('ale', 'local', 'local_sd')]
    assert df['field'].tolist() == ['f_a'] * 6 + ['f_b'] * 3                # aux has K_f = 0: no rows
    assert df['edge_idx'].tolist() == list(range(6)) + list(range(3))
    n_bins, edges, counts, ale, lm, ls = out
    assert df['n'].tolist() == [0] + counts[0, :5].tolist() + [0] + counts[1, :2].tolist()
    np.testing.assert_array_equal(df['edge'], np.concatenate([edges[0, :6], edges[1, :3]]).astype(np.float64))
    for j, o in enumerate(names):
        np.testing.assert_array_equal(df['ale_' + o], np.concatenate([ale[0, :, j], ale[1, :3, j]]).astype(np.float64))
        for col, a in (('local_', lm), ('local_sd_', ls)):
            got = df[col + o].to_numpy()
            assert np.isnan(got[[0, 6]]).all()
            np.testing.assert_array_equal(got[[1, 2, 3, 4, 5, 7, 8]],
                                          np.concatenate([a[0, :5, j], a[1, :2, j]]).astype(np.float64))


def test_ale_table_of_no_field_with_bins_is_empty_with_its_columns():
    out = _stub_outputs(2, 3, 1, [0, 0], seed=7)
    df = ale_table(['a', 'b'], ['norm_preds_1'], *out)
    assert len(df) == 0 and list(df.columns)[:4] == ['field', 'edge_idx', 'edge', 'n']


def test_walk_forward_stacks_the_origins_ale(tmp_path, monkeypatch, fresh_flags):
    cfg = base_config.get_configs(['--training_type', 'iterative', '--split_date', '199506', '--end_date', '199612',
                                   '--stride', '12', '--train=False', '--ale_bins', '4', '--experiments_dir',
                                   str(tmp_path), '--model_dir', 'wf'])

    def run_members(cls, preds, npe):
        for p in preds:
            os.makedirs(os.path.join(p.model_dir, 'pred'), exist_ok=True)
            pd.DataFrame({'date': [p.start_date * 100 + 28], 'gvkey': ['007'], 'norm_preds_1': [0.5]}).to_csv(
                os.path.join(p.model_dir, 'pred', cfg.preds_fname), sep=' ', index=False)
            pd.DataFrame({'field': ['0101', '0101'], 'edge_idx': [0, 1], 'edge': [-1.0, 1.0], 'n': [0, 3],
                          'ale_norm_preds_1': [p.member_id - 0.5, p.member_id + 0.5]}).to_csv(
                os.path.join(p.model_dir, 'pred', 'ale.dat'), sep=' ', index=False)
    monkeypatch.setattr(me.ModelExecution, 'run_members', classmethod(run_members))
    monkeypatch.setattr(me, '_print_scaled_mse', lambda df, steps: None)
    _, origins = me.origin_configs(cfg)
    for _, _, pred in origins:
        os.makedirs(pred.model_dir, exist_ok=True)
    me.ModelExecution(cfg).walk_forward_execution()
    got = pd.read_csv(tmp_path / 'wf' / 'walk_forward_ale.dat', sep=' ', dtype={'field': str})
    assert len(origins) == 2
    assert got['origin'].tolist() == [o for o, _, _ in origins for _ in range(2)]
    assert got['field'].tolist() == ['0101'] * 4 and got['edge_idx'].tolist() == [0, 1, 0, 1]
    ids = [pred.member_id for _, _, pred in origins]
    assert got['ale_norm_preds_1'].tolist() == [ids[0] - 0.5, ids[0] + 0.5, ids[1] - 0.5, ids[1] + 0.5]


# ---- the kernels -----------------------------------------------------------------------------------------------------
def test_ale_kernels_do_not_spill():
    nvcc = shutil.which('nvcc') or ('/usr/local/cuda/bin/nvcc' if os.path.exists('/usr/local/cuda/bin/nvcc') else None)
    if nvcc is None or shutil.which('make') is None:
        pytest.skip('nvcc or make not found')
    r = subprocess.run(['make', '-n', '-B', '-C', ROOT, 'NVCC=' + nvcc, 'all'], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    cmd = [line for line in r.stdout.splitlines() if line.startswith(nvcc + ' ') and 'ale.cu' in line]
    assert len(cmd) == 1, r.stdout
    cmd = shlex.split(cmd[0])
    assert 'arch=compute_90a,code=sm_90a' in cmd and '-v' in ' '.join(cmd)
    with tempfile.TemporaryDirectory() as tmp:
        cmd[cmd.index('-o') + 1] = os.path.join(tmp, 'ale.o')
        r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
    log = r.stdout + r.stderr
    # the project's kernels; the toolkit's segmented radix sort kernels are CUB's own
    per = re.findall(r"Compiling entry function '(\w+)' for 'sm_90a'\s*\n[^\n]*Function properties for \1\s*\n\s*"
                     r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log)
    ours = {re.search(r'\d(ale_[a-z]+_kernel)', name).group(1): s for name, *s in per
            if re.search(r'\dale_[a-z]+_kernel', name)}
    names = sorted(ours)
    assert names == ['ale_edges_kernel', 'ale_fold_kernel', 'ale_gather_kernel', 'ale_keys_kernel',
                     'ale_pick_kernel'], names
    assert all(s == ['0', '0', '0'] for s in ours.values()), ours
