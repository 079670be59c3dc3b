"""CPU checks of the two baselines, NaivePointEstimate and MLPLinearPointEstimate: the factory, the oracle's MLP loss
branch against the reference's own losses.py, the dense handle's C ABI and the 2-D predict extractors."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import dense_oracle as do
from lfm_quant_b200 import _native as N
from lfm_quant_b200.scripts import base_config, configs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = np.load(os.path.join(ROOT, 'tests', 'golden', 'reference_mlp_losses.npz'))
RTOL = 2e-6          # the reference side accumulated in float32


@pytest.fixture()
def fresh_flags():
    configs.reset()
    yield
    configs.reset()


def test_factory_resolves_the_baselines_and_still_refuses_the_hidden_layer_mlps(fresh_flags):
    from lfm_quant_b200.scripts.model_utils import model as factory
    assert {'MLPLinearPointEstimate', 'NaivePointEstimate'} <= set(vars(factory))
    for name in ('MLPPointEstimate', 'MLPUqRangeEstimate'):
        c = base_config.get_configs(['--nn_type', name])
        with pytest.raises(NotImplementedError):
            factory.Model(c, None).get_model()


def test_naive_refuses_training_and_multi_step(fresh_flags):
    from lfm_quant_b200.scripts.models.point_estimate.naive_point_estimate import NaivePointEstimate

    class _DS(object):
        seq_len, n_inputs, n_outputs = 4, 6, 3
    c = base_config.get_configs(['--nn_type', 'NaivePointEstimate', '--train=True'])
    with pytest.raises(ValueError, match='no variables to train'):
        NaivePointEstimate(c, _DS())
    c.train, c.forecast_steps = False, 2
    with pytest.raises(NotImplementedError):
        NaivePointEstimate(c, _DS())
    c.forecast_steps = 1
    m = NaivePointEstimate(c, _DS()).model
    x = np.arange(2 * 4 * 6, dtype=np.float32).reshape(2, 24)
    np.testing.assert_array_equal(m.predict(x), x.reshape(2, 4, 6)[:, 3, :3])
    np.testing.assert_array_equal(m.predict(x), do.naive_forecast(x, 4, 6, 3))


@pytest.mark.parametrize('k', range(int(G['n_cases'])))
def test_oracle_mlp_loss_matches_the_reference(k):
    """losses.py:100-115 (MSE form) run by the reference's own code vs dense_oracle.mlp_loss."""
    y, p = G['mse_%d_y' % k], G['mse_%d_p' % k]
    tidx, lam, loss, mse0 = G['mse_%d' % k]
    assert (np.all(y == 0, axis=1)).sum() == 2          # masked rows are part of every case
    got = do.mlp_loss(y, p, target_idx=int(tidx), target_lambda=lam)
    np.testing.assert_allclose(got, [loss, mse0], rtol=RTOL, atol=1e-7)


@pytest.mark.parametrize('k', range(int(G['n_cases'])))
def test_oracle_mlp_huber_matches_the_restated_branch(k):
    """The Huber cases are restated, not pinned (make_reference_mlp_losses.py): the reference's branch around a Huber
    written to Keras' formula.  Validation (is_validation=True) takes the MSE form whatever huber_loss is."""
    y, p = G['mse_%d_y' % k], G['mse_%d_p' % k]
    tidx, lam, delta, loss, mse0, lv, mv = G['huber_%d' % k]
    r = np.abs(y - p * (~np.all(y == 0, axis=1))[:, None])
    assert (r > delta).any() and (r[r > 0] <= delta).any()       # both sides of delta
    got = do.mlp_loss(y, p, target_idx=int(tidx), target_lambda=lam, huber=True, huber_delta=delta)
    np.testing.assert_allclose(got, [loss, mse0], rtol=RTOL, atol=1e-7)
    np.testing.assert_allclose(do.mlp_loss(y, p, target_idx=int(tidx), target_lambda=lam), [lv, mv], rtol=RTOL,
                               atol=1e-7)


def test_oracle_gradient_is_the_derivative_of_the_loss():
    rng = np.random.RandomState(3)
    y, p = rng.normal(size=(7, 4)), rng.normal(size=(7, 4))
    y[2] = 0.0
    for huber in (False, True):
        kw = dict(target_idx=1, target_lambda=0.3, huber=huber, huber_delta=0.7)
        g = do.mlp_loss_grad(y, p, **kw)
        num = np.zeros_like(p)
        for i in range(7):
            for j in range(4):
                e = np.zeros_like(p)
                e[i, j] = 1e-6
                num[i, j] = (do.mlp_loss(y, p + e, **kw)[0] - do.mlp_loss(y, p - e, **kw)[0]) / 2e-6
        np.testing.assert_allclose(g, num, atol=1e-8)
        assert (g[2] == 0).all()


def _header():
    return open(os.path.join(ROOT, 'include', 'lfmq.h')).read()


def test_dense_symbols_are_declared_and_exported():
    lib = N.load()
    src = re.sub(r'/\*.*?\*/', '', _header(), flags=re.S)
    for name in ('lfmq_dense_workspace_bytes', 'lfmq_dense_create'):
        assert re.search(r'\b%s\s*\(' % name, src), name
        assert name in N.SYMBOLS and hasattr(lib, name)


def test_dense_config_has_the_size_the_header_states():
    m = re.search(r'typedef struct lfmq_dense_config \{\s*/\* (\d+) bytes: (\d+) int32 \+ (\d+) float \*/', _header())
    assert m, 'lfmq.h states the size of lfmq_dense_config'
    size, n_int, n_float = (int(v) for v in m.groups())
    assert C.sizeof(N.LfmqDenseConfig) == size == 4 * (n_int + n_float)
    body = _header()[m.end():_header().index('} lfmq_dense_config;')]
    assert len(re.findall(r'\bint32_t\b', body)) == n_int and len(re.findall(r'\bfloat\b', body)) == n_float


def _dcfg(**kw):
    c = N.LfmqDenseConfig()
    c.struct_size = C.sizeof(N.LfmqDenseConfig)
    c.max_batch, c.seq_len, c.n_inputs, c.n_outputs, c.target_idx = 64, 8, 5, 3, 1
    c.target_lambda, c.huber_delta, c.max_grad_norm = 0.5, 1.0, 50.0
    for k, v in kw.items():
        setattr(c, k, v)
    return c


def test_dense_workspace_and_refusals_without_gpu():
    lib = N.load()
    n = C.c_uint64(0)
    assert lib.lfmq_dense_workspace_bytes(C.byref(_dcfg()), C.byref(n)) == 0
    train = n.value
    assert train > (8 * 5 + 1) * 3 * 4
    assert lib.lfmq_dense_workspace_bytes(C.byref(_dcfg(forward_only=1)), C.byref(n)) == 0 and n.value < train
    for prec in (N.PREC_BF16, N.PREC_BF16X3):        # loud: no silent fall-back to fp32
        assert lib.lfmq_dense_workspace_bytes(C.byref(_dcfg(precision=prec)), C.byref(n)) == 3
        assert b'fp32 only' in lib.lfmq_last_error()
    assert lib.lfmq_dense_workspace_bytes(C.byref(_dcfg(seq_len=48, n_inputs=1025)), C.byref(n)) == 3
    for bad in (dict(struct_size=8), dict(n_outputs=0), dict(target_idx=3), dict(optimizer=7),
                dict(huber_loss=1, huber_delta=0.0), dict(precision=9)):
        assert lib.lfmq_dense_workspace_bytes(C.byref(_dcfg(**bad)), C.byref(n)) == 1, bad


def test_predict_extracts_the_flat_layout(fresh_flags):
    """predict.py:275-300: with MLP / Naive batches, targets and predictions are [B, O] and input step i of the target
    field is column i * F + target_index."""
    from lfm_quant_b200.scripts.predict import Predict
    p = Predict.__new__(Predict)
    p.config = base_config.get_configs(['--nn_type', 'MLPLinearPointEstimate'])
    p.target_index, p.n_inputs, p.seq_len = 2, 5, 3
    inp = np.arange(4 * 15, dtype=np.float32).reshape(4, 15)
    y = np.arange(4 * 3, dtype=np.float32).reshape(4, 3)
    for i in range(3):
        np.testing.assert_array_equal(p._extract_inputs(inp, i)[:, 0], inp.reshape(4, 3, 5)[:, i, 2])
    np.testing.assert_array_equal(p._extract_targets([y])[0][:, 0], y[:, 2])
    np.testing.assert_array_equal(p._extract_preds([y])[0][:, 0], y[:, 2])


def test_losses_take_the_mlp_branch_and_refuse_its_huber_training_form(fresh_flags):
    from lfm_quant_b200.scripts.model_utils.losses import Losses
    c = base_config.get_configs(['--nn_type', 'MLPLinearPointEstimate', '--huber_loss=True'])
    with pytest.raises(NotImplementedError, match='Huber'):
        Losses(c, 0).weight_adjusted_mse([np.zeros((2, 3))], [np.zeros((2, 3))])
    c.nn_type = 'NaivePointEstimate'                # losses.py:117-119: no branch for it in the reference either
    with pytest.raises(NotImplementedError):
        Losses(c, 0).weight_adjusted_mse([np.zeros((2, 3))], [np.zeros((2, 3))], True)
