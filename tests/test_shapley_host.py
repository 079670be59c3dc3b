"""Shapley attributions on the host: the fp64 estimator of tests/shapley_oracle.py (efficiency, exactness where the
Shapley value is known in closed form, zero for an unread group), its draws against lfmq_permutation_index, the
--shapley_samples flag and the runs it is refused for, and shapley.npz from stubbed outputs.  The library's
attributions are checked on the GPU (tests/test_gpu_shapley.py)."""
import ctypes as C
import types

import numpy as np
import pytest

import importance_oracle as imo
import shapley_oracle as sho
from lfm_quant_b200 import _native as N
from lfm_quant_b200.scripts import base_config, configs
from lfm_quant_b200.scripts.predict import Predict, shapley_output_names
from lfm_quant_b200.scripts.runtime import model_execution as me


def _nonlinear(x, m):
    """Two outputs with interactions between fields and quarters; sample m shifts them, as dropout would."""
    x = np.asarray(x, dtype=np.float64).reshape(x.shape[0], -1)
    a = np.tanh(x @ np.linspace(-1.0, 1.0, x.shape[1])) * (1.0 + 0.1 * m)
    b = x[:, 0] * x[:, -1] + np.sin(x[:, 1] * x[:, 2])
    return np.stack([a, b], axis=1)


@pytest.mark.parametrize('M', [1, 2, 5])
def test_attributions_add_up_to_f_x_minus_f_bg(M):
    x = np.random.RandomState(1).normal(size=(37, 4, 3))
    for cg, G in (imo.field_groups(4, 3), imo.quarter_groups(4, 3)):
        phi, f_x, f_bg = sho.shapley(x, cg, G, M, 99, _nonlinear)
        assert phi.shape == (37, 2, G) and f_x.shape == f_bg.shape == (37, 2)
        np.testing.assert_allclose(phi.sum(axis=2), f_x - f_bg, rtol=0, atol=1e-12)
        want_x = np.mean([_nonlinear(x, m) for m in range(M)], axis=0)
        np.testing.assert_allclose(f_x, want_x, rtol=0, atol=1e-12)


@pytest.mark.parametrize('M', [1, 2, 3, 8])
def test_a_group_additive_function_is_attributed_exactly(M):
    T, F, N_ = 3, 4, 29
    rng = np.random.RandomState(2)
    x = rng.normal(size=(N_, T, F))
    w = rng.normal(size=(T, F))
    cg, G = imo.field_groups(T, F)

    def f(z, m):                          # sum over fields of h_f(column f of every quarter)
        return (np.cos(z) * w).sum(axis=(1, 2))[:, None]
    phi, f_x, f_bg = sho.shapley(x, cg, G, M, 5, f)
    donors, _ = sho.draws(N_, G, M, 5)
    h = (np.cos(x) * w).sum(axis=1)                                        # [N, F]
    want = np.mean([h - h[donors[m // 2]] for m in range(M)], axis=0)
    np.testing.assert_allclose(phi[:, 0, :], want, rtol=0, atol=1e-12)


def test_two_players_and_one_antithetic_pair_give_the_exact_shapley_values():
    N_ = 17
    x = np.random.RandomState(3).normal(size=(N_, 2))
    cg = np.array([0, 1], dtype=np.int32)

    def f(z, m):
        return (z[:, 0] * z[:, 1] + 2.0 * z[:, 0] ** 2 - z[:, 1])[:, None]
    phi, f_x, f_bg = sho.shapley(x, cg, 2, 2, 11, f)
    d = x[sho.draws(N_, 2, 2, 11)[0][0]]

    def v(s):                             # the game of window i against its donor: players in s take their own values
        z = d.copy()
        z[:, list(s)] = x[:, list(s)]
        return f(z, 0)[:, 0]
    for g, o in ((0, 1), (1, 0)):
        want = 0.5 * ((v([g]) - v([])) + (v([0, 1]) - v([o])))
        np.testing.assert_allclose(phi[:, 0, g], want, rtol=0, atol=1e-12)


def test_a_group_the_function_does_not_read_gets_exactly_zero():
    x = np.random.RandomState(4).normal(size=(23, 3, 4))
    cg, G = imo.field_groups(3, 4)

    def f(z, m):
        z = np.array(z, copy=True)
        z[:, :, 2] = 0.0                                                   # field 2 is never read
        return _nonlinear(z, m)
    phi, _, _ = sho.shapley(x, cg, G, 4, 8, f)
    assert np.array_equal(phi[:, :, 2], np.zeros((23, 2)))
    assert (np.abs(phi[:, :, [0, 1, 3]]).max(axis=(0, 1)) > 0).all()


def _lib_index(n, key, p, seed):
    lib, out = N.load(), C.c_int32(0)
    got = np.empty(n, dtype=np.int64)
    for i in range(n):
        assert lib.lfmq_permutation_index(n, seed, key, p, i, C.byref(out)) == 0
        got[i] = out.value
    return got


@pytest.mark.parametrize('N_,G,M', [(1, 1, 1), (300, 6, 4), (1001, 48, 3)])
def test_the_draws_are_the_librarys_bijection(N_, G, M):
    seed = 2 ** 35 + 17
    donors, orders = sho.draws(N_, G, M, seed)
    assert len(donors) == (M + 1) // 2 and len(orders) == M
    for p, d in enumerate(donors):
        assert np.array_equal(d, _lib_index(N_, 0x40000000, p, seed))
    for m, o in enumerate(orders):
        assert np.array_equal(np.sort(o), np.arange(G))
        want = _lib_index(G, 0x40000001, m // 2, seed)
        assert np.array_equal(o, want if m % 2 == 0 else want[::-1])


def test_the_coalition_copies_run_from_the_donor_to_x():
    x = np.arange(5 * 2 * 3, dtype=np.float64).reshape(5, 2, 3)
    cg, G = imo.field_groups(2, 3)
    donor = np.array([4, 0, 3, 1, 2])
    rank = np.array([2, 0, 1])                                             # ordering (1, 2, 0)
    assert np.array_equal(sho.coalition_copy(x, cg, rank, 0, donor), x[donor])
    assert np.array_equal(sho.coalition_copy(x, cg, rank, G, donor), x)
    got = sho.coalition_copy(x, cg, rank, 2, donor)                        # fields 1 and 2 own, field 0 the donor's
    assert np.array_equal(got[:, :, 0], x[donor][:, :, 0]) and np.array_equal(got[:, :, 1:], x[:, :, 1:])


@pytest.fixture()
def fresh_flags():
    configs.reset()
    yield
    configs.reset()


def test_shapley_samples_flag_defaults_to_off(fresh_flags):
    assert base_config.get_configs([]).shapley_samples == 0
    assert base_config.get_configs(['--shapley_samples', '8']).shapley_samples == 8


@pytest.mark.parametrize('argv', [
    ['--shapley_samples', '4', '--train=True'],
    ['--shapley_samples', '-1', '--train=False'],
    ['--shapley_samples', '4', '--train=False', '--nn_type', 'NaivePointEstimate'],
])
def test_shapley_samples_is_refused_before_any_work(fresh_flags, monkeypatch, argv):
    ran = []
    monkeypatch.setattr(me.ModelExecution, 'single_execution', staticmethod(lambda cfg: ran.append(cfg) or 'ran'))
    monkeypatch.setattr(me.ModelExecution, 'fixed_dates_execution', lambda self: ran.append(self) or 'ran')
    with pytest.raises(ValueError, match='--shapley_samples'):
        me.ModelExecution(base_config.get_configs(argv))()
    assert ran == []


@pytest.mark.parametrize('argv', [
    ['--shapley_samples', '2', '--train=False'],
    ['--shapley_samples', '1', '--train=False', '--nn_type', 'RNNUqRangeEstimate', '--UQ=True', '--mc_samples', '4'],
    ['--shapley_samples', '3', '--train=False', '--nn_type', 'MLPLinearPointEstimate'],
    ['--shapley_samples', '2', '--train=False', '--forecast_steps', '2', '--forecast_steps_weights', '1.0-0.5'],
    ['--shapley_samples', '0', '--train=True'],
])
def test_shapley_samples_runs_every_trained_model_at_prediction(fresh_flags, monkeypatch, argv):
    seen = []
    monkeypatch.setattr(me.ModelExecution, 'single_execution', staticmethod(lambda cfg: seen.append(cfg) or 'ran'))
    monkeypatch.setattr(me.ModelExecution, 'write_uq_ensemble', classmethod(lambda cls, cfg: None))
    assert me.ModelExecution(base_config.get_configs(argv))() == 'ran'
    assert len(seen) == 1


def test_output_names_follow_the_keras_list_order():
    assert shapley_output_names(1, False) == ['norm_preds_1']
    assert shapley_output_names(3, False) == ['norm_preds_1', 'norm_preds_2', 'norm_preds_3']
    assert shapley_output_names(2, True) == ['norm_preds_1', 'norm_variance_1', 'norm_preds_2', 'norm_variance_2']


@pytest.mark.parametrize('steps,uq', [(1, False), (2, True)])
def test_shapley_npz_from_stubbed_outputs(tmp_path, steps, uq):
    T, F, K = 4, 3, 2 * steps if uq else steps
    sizes = [5, 2]                                                        # two prediction batches
    Nw = sum(sizes)
    rng = np.random.RandomState(6)
    phi_f, phi_q = rng.normal(size=(Nw, K, F)), rng.normal(size=(Nw, K, T))
    f_x, f_bg = rng.normal(size=(Nw, K)), rng.normal(size=(Nw, K))
    calls = []

    class Model(object):
        def shapley(self, inp, samples):
            calls.append((np.asarray(inp).copy(), samples))
            return tuple(types.SimpleNamespace(cpu=lambda a=a: types.SimpleNamespace(numpy=lambda: a))
                         for a in (phi_f, phi_q, f_x, f_bg))

    import torch
    windows = [torch.arange(n * T * F, dtype=torch.float32).reshape(n, T, F) + 1000 * b for b, n in enumerate(sizes)]
    p = object.__new__(Predict)
    p.model, p.pred_dir = Model(), str(tmp_path)
    p.config = types.SimpleNamespace(shapley_samples=6, forecast_steps=steps, UQ=uq)
    p.dataset = types.SimpleNamespace(fin_col_names=['f_a', 'f_b'], aux_col_names=['aux'])
    dates = [np.array([[19991231 + b]] * n, dtype=np.int32) for b, n in enumerate(sizes)]
    keys = [np.array([[('%06d' % (100 * b + i)).encode()] for i in range(n)], dtype=object)
            for b, n in enumerate(sizes)]
    p._write_shapley({'date': dates, 'gvkey': keys}, windows)
    assert len(calls) == 1 and calls[0][1] == 6
    assert np.array_equal(calls[0][0], torch.cat(windows).numpy())       # every window at once, in preds.dat order
    z = np.load(tmp_path / 'shapley.npz')
    assert sorted(z.files) == sorted(['date', 'gvkey', 'fields', 'quarters', 'outputs', 'phi_field', 'phi_quarter',
                                      'f_x', 'f_bg'])
    assert z['date'].tolist() == [19991231] * 5 + [19991232] * 2 and z['date'].dtype == np.int32
    assert z['gvkey'].tolist() == ['000000', '000001', '000002', '000003', '000004', '000100', '000101']
    assert z['fields'].tolist() == ['f_a', 'f_b', 'aux'] and z['quarters'].tolist() == [-3, -2, -1, 0]
    assert z['outputs'].tolist() == shapley_output_names(steps, uq)
    for k, a in (('phi_field', phi_f), ('phi_quarter', phi_q), ('f_x', f_x), ('f_bg', f_bg)):
        assert z[k].dtype == np.float32 and np.array_equal(z[k], a.astype(np.float32))
