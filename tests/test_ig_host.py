"""Integrated gradients on the host: the fp64 oracle the GPU is checked against (tests/ig_oracle.py), and the --ig_steps
flag with the runs it is refused for.  The attributions themselves are checked on the GPU (tests/test_gpu_ig.py)."""
import numpy as np
import pytest

import ig_oracle as igo
import lfm_oracle as orc
from lfm_quant_b200.scripts import base_config, configs
from util import make_problem, rel_err


def _problem(cell, L=2, B=3, T=4, F=3, O=2, H=8, seed=5):
    P, x, _ = make_problem(B, T, F, O, H, L, seed=seed, rnn_cell=cell)
    rng = np.random.RandomState(seed + 100)
    bn = dict(bn_mean=[rng.normal(size=H) * 0.3 for _ in range(L)],          # away from (0, 1)
              bn_var=[rng.uniform(0.4, 2.5, size=H) for _ in range(L)])
    return P, x.astype(np.float64), dict(num_layers=L, target_idx=1, rnn_cell=cell, **bn)


@pytest.mark.parametrize('cell', ['lstm', 'gru'])
def test_oracle_input_gradient_matches_central_differences(cell):
    P, x, kw = _problem(cell)
    g, f = igo.input_gradient(P, x, **kw)
    assert np.array_equal(f, orc.forward(P, x, num_layers=2, rnn_cell=cell, bn_mean=kw['bn_mean'],
                                         bn_var=kw['bn_var'])[0][:, -1, 1])
    fd = np.zeros_like(x)
    eps = 1e-5
    for idx in np.ndindex(*x.shape[1:]):
        for sgn in (1, -1):
            xp = x.copy()
            xp[(slice(None),) + idx] += sgn * eps
            fd[(slice(None),) + idx] += sgn * igo.forecast(P, xp, **kw)[0] / (2 * eps)
    err = rel_err(g, fd)
    print('ig oracle %s: input gradient vs central differences, rel err %.2e' % (cell, err))
    assert err < 1e-6, err


@pytest.mark.parametrize('cell', ['lstm', 'gru'])
def test_oracle_completeness_gap_shrinks_as_one_over_m_squared(cell):
    """The midpoint rule's error is c / M^2 + O(1 / M^4): every fourfold M divides the gap by about 16."""
    P, x, kw = _problem(cell, B=4, T=5, F=4, O=3, H=8, seed=9)
    gaps = [np.abs(igo.completeness_gap(*igo.integrated_gradients(P, x, M, **kw))) for M in (16, 64, 256)]
    r1, r2 = gaps[0] / gaps[1], gaps[1] / gaps[2]
    print('ig oracle %s: gap ratios M=16/64 %s, 64/256 %s' % (cell, np.round(r1, 2), np.round(r2, 2)))
    assert (gaps[0] > 1e-9).all()
    assert np.all(np.abs(r1 - 16) < 1.6) and np.all(np.abs(r2 - 16) < 0.4), (r1, r2)


@pytest.fixture()
def fresh_flags():
    configs.reset()
    yield
    configs.reset()


def test_ig_steps_flag_defaults_to_off(fresh_flags):
    assert base_config.get_configs([]).ig_steps == 0
    assert base_config.get_configs(['--ig_steps', '16']).ig_steps == 16


@pytest.mark.parametrize('argv', [
    ['--ig_steps', '8', '--train=True'],                                                          # training
    ['--ig_steps', '8', '--train=False', '--nn_type', 'RNNUqRangeEstimate', '--UQ=True'],         # a uq model
    ['--ig_steps', '8', '--train=False', '--UQ=True'],
    ['--ig_steps', '8', '--train=False', '--nn_type', 'MLPLinearPointEstimate'],                  # a baseline
    ['--ig_steps', '8', '--train=False', '--nn_type', 'NaivePointEstimate'],
    ['--ig_steps', '8', '--train=False', '--forecast_steps', '2', '--forecast_steps_weights', '1.0-0.5'],
    ['--ig_steps', '-1', '--train=False'],
])
def test_ig_steps_outside_point_prediction_is_refused_before_any_work(fresh_flags, monkeypatch, argv):
    from lfm_quant_b200.scripts.runtime.model_execution import ModelExecution
    ran = []
    monkeypatch.setattr(ModelExecution, 'single_execution', staticmethod(lambda cfg: ran.append(cfg) or 'ran'))
    monkeypatch.setattr(ModelExecution, 'fixed_dates_execution', lambda self: ran.append(self) or 'ran')
    with pytest.raises(ValueError, match='--ig_steps'):
        ModelExecution(base_config.get_configs(argv))()
    assert ran == []


def test_ig_steps_runs_point_prediction(fresh_flags, monkeypatch):
    from lfm_quant_b200.scripts.runtime.model_execution import ModelExecution
    seen = []
    monkeypatch.setattr(ModelExecution, 'single_execution', staticmethod(lambda cfg: seen.append(cfg.ig_steps) or 'ran'))
    for argv in (['--ig_steps', '16', '--train=False'], ['--ig_steps', '0', '--train=True']):
        assert ModelExecution(base_config.get_configs(argv))() == 'ran'
    assert seen == [16, 0]
