"""Training-window attributions without a GPU: the closed form of tests/influence_oracle.py against the head-parameter
gradients of the model oracle (lfm_oracle.backward / backward_uq) and, for the linear model, central differences; the
one-window loss gradient against the oracle's loss at B = 1; masked steps; the --influence_top_k flag; the npz layout;
and a no-spill compile of csrc/influence.cu."""
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

import influence_oracle as io
import lfm_oracle as orc
from lfm_quant_b200.scripts import base_config, configs
from lfm_quant_b200.scripts.predict import write_influence
from lfm_quant_b200.scripts.runtime import model_execution as me

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KW = dict(target_idx=1, target_lambda=0.5, rnn_lambda=0.7)


def _problem(B=6, T=5, F=3, O=4, seed=0):
    rng = np.random.RandomState(seed)
    x = rng.normal(size=(B, T, F))
    y = rng.normal(size=(B, T, O))
    y[1, :2] = 0.0
    y[2, -1] = 0.0
    return x, y


def _head_grad(kind, P, x, dpred, dvar, L, cell):
    """The gradients of the head parameters (kernel then bias of each head) for the given output gradients."""
    if kind == 'point':
        _, cache = orc.forward(P, x, num_layers=L, rnn_cell=cell)
        g = orc.backward(dpred, cache, num_layers=L, rnn_cell=cell)
        return np.concatenate([g[5 * L].ravel(), g[5 * L + 1].ravel()])
    _, _, cache = orc.forward_uq(P, x, num_layers=L, rnn_cell=cell)
    g = orc.backward_uq(dpred, dvar, cache, num_layers=L, rnn_cell=cell)
    return np.concatenate([g[5 * L + i].ravel() for i in range(4)])


@pytest.mark.parametrize('kind', ['point', 'uq'])
@pytest.mark.parametrize('cell', ['lstm', 'gru'])
def test_closed_form_equals_minus_gradient_dot_product(kind, cell):
    L, T, O = 1, 5, 4
    x, y = _problem(T=T, O=O)
    P = orc.init_params(L, 3, O, 8, init_scale=0.7, seed=3, dtype=np.float64, rnn_cell=cell, uq=kind == 'uq')
    u = io.train_features(kind, P, x, y, num_layers=L, rnn_cell=cell, **KW)
    a, s = io.query_features(kind, P, x, target_idx=KW['target_idx'], num_layers=L, rnn_cell=cell)
    I = io.influence(a, u, s)
    J = I.shape[0]
    z = np.zeros((1, T, O))
    for t in range(x.shape[0]):
        xt, yt = x[t:t + 1], y[t:t + 1]
        if kind == 'point':
            pred, _ = orc.forward(P, xt, num_layers=L, rnn_cell=cell)
            _, _, dl, _ = orc.loss_point_estimate(yt, pred, **KW)
            gl = _head_grad(kind, P, xt, np.nan_to_num(dl), None, L, cell)
        else:
            pred, var, _ = orc.forward_uq(P, xt, num_layers=L, rnn_cell=cell)
            with np.errstate(divide='ignore', invalid='ignore'):
                _, _, _, dp, dv = orc.loss_uq_estimate(yt, pred, var, **KW)
            gl = _head_grad(kind, P, xt, np.nan_to_num(dp), np.nan_to_num(dv), L, cell)
        for q in range(x.shape[0]):
            for j in range(J):
                seed = z.copy()
                seed[0, -1, KW['target_idx']] = 1.0
                args = (seed, z) if j == 0 else (z, seed)
                gf = _head_grad(kind, P, x[q:q + 1], *(args if kind == 'uq' else args[:1] + (None,)), L, cell)
                ref = -gl @ gf
                assert abs(I[j, q, t] - ref) <= 1e-10 * (1 + abs(ref)), (j, q, t, I[j, q, t], ref)


@pytest.mark.parametrize('huber', [False, True])
def test_linear_closed_form_equals_central_differences(huber):
    T, F, O, ti, lam, delta = 3, 2, 3, 1, 0.4, 0.3
    rng = np.random.RandomState(1)
    x = rng.normal(size=(5, T, F))
    y = rng.normal(size=(5, O))
    y[3] = 0.0
    W, b = rng.normal(size=(T * F, O)) * 0.5, rng.normal(size=O) * 0.1
    u = io.train_features('dense', [W, b], x, y, target_idx=ti, target_lambda=lam, huber=huber, huber_delta=delta)
    a, s = io.query_features('dense', [W, b], x, target_idx=ti)
    I = io.influence(a, u, s)

    def loss(t, th):
        Wc, bc = W.copy(), b.copy()
        Wc[:, ti], bc[ti] = th[:-1], th[-1]
        m = float(np.any(y[t] != 0))
        r = y[t] - (x[t].ravel() @ Wc + bc) * m
        f = (np.where(np.abs(r) > delta, delta * (np.abs(r) - 0.5 * delta), 0.5 * r * r) if huber else r * r)
        return (1 - lam) * f.mean() + lam * f[ti]

    th0 = np.concatenate([W[:, ti], [b[ti]]])
    for t in range(5):
        g = np.array([(loss(t, th0 + e) - loss(t, th0 - e)) / 2e-6 for e in np.eye(th0.size) * 1e-6])
        for q in range(5):
            gf = np.concatenate([x[q].ravel(), [1.0]])
            assert abs(I[0, q, t] + g @ gf) <= 1e-6 * (1 + abs(g @ gf))


@pytest.mark.parametrize('kind', ['point', 'uq'])
def test_window_gradient_is_the_loss_gradient_at_one_window_and_zero_where_masked(kind):
    x, y = _problem()
    y[4] = 0.0
    P = orc.init_params(1, 3, 4, 8, init_scale=0.5, seed=2, dtype=np.float64, uq=kind == 'uq')
    _, pred, var, pre = io.head_inputs(kind, P, x)
    G = io.window_grads(kind, pred, var, pre, y, **KW)
    assert np.all(np.isfinite(G))
    assert np.all(G[:, 4] == 0.0) and np.all(G[:, 1, :2] == 0.0) and np.all(G[:, 2, -1] == 0.0)
    b = 0                         # an unmasked window: the oracle's own gradient at B = 1
    if kind == 'point':
        dl = orc.loss_point_estimate(y[b:b + 1], pred[b:b + 1], **KW)[2]
        assert np.allclose(G[0, b], dl[0, :, KW['target_idx']], rtol=0, atol=1e-15)
    else:
        _, _, _, dp, dv = orc.loss_uq_estimate(y[b:b + 1], pred[b:b + 1], var[b:b + 1], **KW)
        assert np.allclose(G[0, b], dp[0, :, KW['target_idx']], rtol=0, atol=1e-15)
        gate = np.where(orc.softplus(pre[b]) > orc.VAR_FLOOR, orc.sigmoid(pre[b]), 0.0)[:, KW['target_idx']]
        assert np.allclose(G[1, b], dv[0, :, KW['target_idx']] * gate, rtol=0, atol=1e-15)


def test_topk_reference_breaks_ties_to_the_lower_index_and_pads():
    I = np.array([[[1.0, 3.0, 3.0, -2.0, 0.0, -2.0]]])
    pi, ps, ni, ns = io.topk(I, 4)
    assert pi[0, 0].tolist() == [1, 2, 0, -1] and ps[0, 0].tolist() == [3.0, 3.0, 1.0, 0.0]
    assert ni[0, 0].tolist() == [3, 5, -1, -1] and ns[0, 0].tolist() == [-2.0, -2.0, 0.0, 0.0]


# ---- the flag ----------------------------------------------------------------------------------------------------------
@pytest.fixture()
def fresh_flags():
    configs.reset()
    yield
    configs.reset()


def test_influence_top_k_flag_defaults_to_off(fresh_flags):
    assert base_config.get_configs([]).influence_top_k == 0
    assert base_config.get_configs(['--influence_top_k', '5']).influence_top_k == 5


@pytest.mark.parametrize('argv', [
    ['--influence_top_k', '5', '--train=True'],
    ['--influence_top_k', '-1', '--train=False'],
    ['--influence_top_k', '65', '--train=False'],
    ['--influence_top_k', '5', '--train=False', '--nn_type', 'NaivePointEstimate'],
    ['--influence_top_k', '5', '--train=False', '--forecast_steps', '2', '--forecast_steps_weights', '1.0-0.5'],
    ['--influence_top_k', '5', '--train=False', '--num_procs', '2'],
])
def test_influence_top_k_is_refused_before_any_work(fresh_flags, monkeypatch, argv):
    ran = []
    monkeypatch.setattr(me.ModelExecution, 'single_execution', staticmethod(lambda cfg: ran.append(cfg) or 'ran'))
    monkeypatch.setattr(me.ModelExecution, 'fixed_dates_execution', lambda self: ran.append(self) or 'ran')
    with pytest.raises(ValueError, match='--influence_top_k'):
        me.ModelExecution(base_config.get_configs(argv))()
    assert ran == []


def test_npz_layout():
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, 'influence.npz')
        N, J, K, Nt = 3, 2, 4, 7
        idx = np.arange(N * J * K).reshape(N, J, K) % Nt
        write_influence(path, [20200331, 20200630, 20200930], ['001', '002', '003'], ['norm_preds_1', 'norm_variance_1'],
                        np.arange(Nt) + 20100101, ['%03d' % i for i in range(Nt)], np.linspace(-1, 1, Nt), idx,
                        idx * 0.5, -idx, -idx * 0.5, np.ones((N, J)))
        z = np.load(path)
        assert sorted(z.files) == sorted(['date', 'gvkey', 'outputs', 'train_date', 'train_gvkey', 'train_target',
                                          'pos_idx', 'pos_score', 'neg_idx', 'neg_score', 'total'])
        assert z['pos_idx'].shape == (N, J, K) and z['pos_idx'].dtype == np.int32
        assert z['total'].shape == (N, J) and z['train_target'].shape == (Nt,)
        assert z['gvkey'].tolist() == ['001', '002', '003'] and z['outputs'].tolist()[1] == 'norm_variance_1'


def test_influence_kernels_compile_without_spills():
    with tempfile.TemporaryDirectory() as d:
        r = subprocess.run(['nvcc', '-O3', '-Xptxas', '-v', '-std=c++17', '-gencode', 'arch=compute_90a,code=sm_90a',
                            '--expt-relaxed-constexpr', '-c', os.path.join(ROOT, 'lfm_quant_b200', 'csrc', 'influence.cu'),
                            '-o', os.path.join(d, 'influence.o')], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        frames = re.findall(r'(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads', r.stderr)
        assert len(frames) >= 6
        assert all(f == ('0', '0', '0') for f in frames), frames
