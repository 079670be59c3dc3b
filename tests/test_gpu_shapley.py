"""Shapley attributions on the GPU (lfmq_chain_shapley, ForecastChainEngine.shapley, NativeForecaster.shapley,
--shapley_samples): phi [N,K,G] splits each explained output's f_x - f_bg over the groups of input columns.

Checked here: the fp64 estimator with the same draws (tests/shapley_oracle.py) for every model kind; efficiency at
every precision; f_x against the forward and against predict_mc's mean; the same bits at any launch size and on a
repeated call; exactly zero for a field the model does not read; the linear model in closed form; the handle's state
left untouched; the refusals; and the CLI file."""
import ctypes as C

import numpy as np
import pandas as pd
import pytest
import torch

import importance_oracle as imo
import lfm_oracle as orc
import shapley_oracle as sho
import uq_chain_oracle as uco

pytestmark = pytest.mark.gpu
KW = dict(target_idx=1, target_lambda=0.5, rnn_lambda=0.7)
DROP = dict(dropout=0.2, recurrent_dropout=0.15, seed=31)
SEED, STEP, M = 2024, 7, 4
N = 300                           # not a multiple of the 256 launch rows
ERR_ARG, ERR_WORKSPACE = 1, 4     # include/lfmq.h


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()


def _chain(S, T, F, O, H, L, *, max_batch=256, precision='fp32', uq=False, cell='lstm', **kw):
    from lfm_quant_b200.engine import ForecastChainEngine
    args = dict(KW, train=False, forward_only=True)
    args.update(kw)
    return ForecastChainEngine(forecast_steps=S, weights=[1.0, 0.5][:S], max_batch=max_batch, seq_len=T, n_inputs=F,
                               n_outputs=O, num_hidden=H, num_layers=L, rnn_cell=cell, precision=precision, uq=uq,
                               **args)


def _dense(T, F, O, max_batch=256):
    from lfm_quant_b200.engine import DenseEngine, ForecastChainEngine
    return ForecastChainEngine(stages=[DenseEngine(max_batch=max_batch, seq_len=T, n_inputs=F, n_outputs=O,
                                                   target_idx=KW['target_idx'], target_lambda=KW['target_lambda'],
                                                   forward_only=True)])


def _params(T, F, O, H, L, S, cell, uq, seed):
    rng = np.random.RandomState(seed)
    init = uco.init_params if uq else orc.init_forecast_params
    P = init(L, F, O, H, S, init_scale=0.5, seed=seed + 1, dtype=np.float64, rnn_cell=cell)
    P = [(p + rng.normal(size=p.shape) * 0.05).astype(np.float32).astype(np.float64) for p in P]
    x = rng.normal(size=(N, T, F)).astype(np.float32)
    return P, x


def _run(eng, x, cg, samples=M, step=STEP):
    return [t.cpu().numpy() for t in eng.shapley(_cuda(x), cg, samples, SEED, step)]


def _partitions(T, F):
    return [imo.field_groups(T, F), imo.quarter_groups(T, F)]


def _rel(got, ref):
    """max |got - ref| over the largest |ref| of each output (axis 1); an output of zeros must be zeros"""
    axes = tuple(a for a in range(ref.ndim) if a != 1)
    scale = np.abs(ref).max(axis=axes, keepdims=True)
    return float(np.max(np.abs(got - ref) / np.where(scale > 0, scale, 1.0)))


def _efficiency(phi, f_x, f_bg):
    """max over outputs of max |sum_g phi - (f_x - f_bg)| / max(|f_x|, |f_bg|), in fp64"""
    gap = np.abs(phi.astype(np.float64).sum(axis=2) - (f_x.astype(np.float64) - f_bg))
    scale = np.maximum(np.abs(f_x), np.abs(f_bg)).max(axis=0)
    return float((gap.max(axis=0) / scale).max())


# (name, S, L, cell, uq)
MODELS = [('lstm-point-L2', 1, 2, 'lstm', False), ('gru-point', 1, 1, 'gru', False), ('lstm-uq', 1, 1, 'lstm', True),
          ('point-chain-S2', 2, 1, 'lstm', False), ('gru-uq-chain-S2', 2, 1, 'gru', True)]


@pytest.mark.parametrize('model', MODELS, ids=[m[0] for m in MODELS])
def test_attributions_match_the_fp64_oracle(model):
    _, S, L, cell, uq = model
    T, F, O, H = 5, 6, 3, 16
    P, x = _params(T, F, O, H, L, S, cell, uq, seed=3 + S + L)
    eng = _chain(S, T, F, O, H, L, uq=uq, cell=cell, **(DROP if uq else {}))
    eng.set_weights(P)
    if uq:
        f = sho.uq_outputs(P, num_layers=L, rnn_cell=cell, forecast_steps=S, dropout=DROP['dropout'],
                           recurrent_dropout=DROP['recurrent_dropout'], seed=DROP['seed'], step=STEP,
                           target_idx=KW['target_idx'])
    else:
        f = sho.point_outputs(P, num_layers=L, rnn_cell=cell, forecast_steps=S, target_idx=KW['target_idx'])
    K = 2 * S if uq else S
    for cg, G in _partitions(T, F):
        phi, f_x, f_bg = _run(eng, x, cg)
        ref = sho.shapley(x.astype(np.float64), cg, G, M, SEED, f)
        assert phi.shape == (N, K, G) and f_x.shape == f_bg.shape == (N, K)
        errs = [_rel(phi, ref[0]), _rel(f_x, ref[1]), _rel(f_bg, ref[2])]
        print('shapley %s G=%d: rel err phi %.2e, f_x %.2e, f_bg %.2e; max |phi| %s'
              % (model[0], G, *errs, np.abs(ref[0]).max(axis=(0, 2))))
        assert max(errs) < 1e-4, errs
        assert (np.abs(ref[0]).max(axis=(0, 2)) > 0).all()
    eng.close()


def test_linear_model_matches_the_oracle_and_the_closed_form():
    T, F, O = 5, 6, 3
    rng = np.random.RandomState(4)
    W = (rng.normal(size=(T * F, O)) * 0.2).astype(np.float32).astype(np.float64)
    b = (rng.normal(size=O) * 0.1).astype(np.float32).astype(np.float64)
    x = rng.normal(size=(N, T * F)).astype(np.float32)
    eng = _dense(T, F, O)
    eng.set_weights([W, b])
    w = W[:, KW['target_idx']]
    xd = x.astype(np.float64)
    for cg, G in _partitions(T, F):
        phi, f_x, f_bg = _run(eng, x, cg)
        ref = sho.shapley(xd, cg, G, M, SEED, sho.dense_outputs(W, b, target_idx=KW['target_idx']))
        assert phi.shape == (N, 1, G)
        assert max(_rel(phi, ref[0]), _rel(f_x, ref[1]), _rel(f_bg, ref[2])) < 1e-4
        donors, _ = sho.draws(N, G, M, SEED)
        onehot = np.eye(G)[cg]                                              # [T*F, G]
        want = np.mean([((xd - xd[donors[m // 2]]) * w) @ onehot for m in range(M)], axis=0)
        err = _rel(phi[:, 0, :], want)
        print('shapley linear G=%d: rel err against w . (x - donor) %.2e' % (G, err))
        assert err < 1e-4
    eng.close()


# (name, precision, cell, H, L): bf16 on the cluster shape (LSTM H=256, L=1) and on the general path
PRECISIONS = [('fp32', 'fp32', 'lstm', 64, 2), ('tf32', 'tf32', 'lstm', 64, 2), ('bf16', 'bf16', 'lstm', 256, 1),
              ('bf16-general', 'bf16', 'lstm', 128, 2), ('bf16-gru', 'bf16', 'gru', 128, 1),
              ('bf16x3', 'bf16x3', 'lstm', 256, 1)]


@pytest.mark.parametrize('case', PRECISIONS, ids=[p[0] for p in PRECISIONS])
@pytest.mark.parametrize('uq', [False, True], ids=['point', 'uq'])
def test_attributions_add_up_at_every_precision(case, uq):
    _, prec, cell, H, L = case
    T, F, O = 8, 32, 16
    P, x = _params(T, F, O, H, L, 1, cell, uq, seed=11)
    eng = _chain(1, T, F, O, H, L, precision=prec, uq=uq, cell=cell, **(DROP if uq else {}))
    eng.set_weights(P)
    for cg, G in _partitions(T, F):
        phi, f_x, f_bg = _run(eng, x, cg)
        err = _efficiency(phi, f_x, f_bg)
        print('shapley efficiency %s %s G=%d: %.2e' % (case[0], 'uq' if uq else 'point', G, err))
        assert np.isfinite(phi).all() and err < 1e-5, err
    eng.close()


@pytest.mark.parametrize('prec', ['fp32', 'bf16'])
def test_a_point_models_f_x_is_its_forward(prec):
    T, F, O, H, L, S = 8, 32, 16, 256, 1, 2
    P, x = _params(T, F, O, H, L, S, 'lstm', False, seed=12)
    eng = _chain(S, T, F, O, H, L, precision=prec)
    eng.set_weights(P)
    xd = _cuda(x)
    fwd = [torch.cat([o[s] for o in [eng.forward(xd[a:a + 256].contiguous(), step=STEP, row0=a)
                                     for a in range(0, N, 256)]]) for s in range(S)]
    want = np.stack([p[:, -1, KW['target_idx']].cpu().numpy() for p in fwd], axis=1)
    _, f_x, _ = _run(eng, x, imo.field_groups(T, F)[0])
    assert np.abs(f_x - want).max() <= 1e-6 * max(1.0, np.abs(want).max())
    eng.close()


@pytest.mark.parametrize('S', [1, 2])
def test_a_uq_models_f_x_is_the_mean_of_predict_mc(S):
    T, F, O, H, L = 8, 32, 16, 256, 1
    P, x = _params(T, F, O, H, L, S, 'lstm', True, seed=13)
    eng = _chain(S, T, F, O, H, L, uq=True, max_batch=1024, **DROP)
    eng.set_weights(P)
    mc = eng.forward_mc(_cuda(x), M, step=STEP)               # B = N, sample m of window i is row m * N + i
    want = np.stack([t[:, -1, KW['target_idx']].cpu().numpy() for s in range(S) for t in (mc[s][0], mc[s][1])],
                    axis=1)
    _, f_x, _ = _run(eng, x, imo.quarter_groups(T, F)[0])
    err = np.abs(f_x - want).max()
    print('uq S=%d: |f_x - predict_mc mean| %.2e' % (S, err))
    assert err <= 1e-6 * max(1.0, np.abs(want).max())
    eng.close()


@pytest.mark.parametrize('case', ['fp32', 'tf32', 'bf16', 'uq-fp32', 'uq-bf16'])
def test_launch_size_does_not_change_the_bits(case):
    uq = case.startswith('uq')
    prec = case.split('-')[-1]
    T, F, O, H, L = 6, 10, 4, 64, 2
    P, x = _params(T, F, O, H, L, 1, 'lstm', uq, seed=21)
    outs = []
    for mb in (256, 8192):
        eng = _chain(1, T, F, O, H, L, max_batch=mb, precision=prec, uq=uq, **(DROP if uq else {}))
        eng.set_weights(P)
        outs.append([_run(eng, x, cg) for cg, _ in _partitions(T, F)])
        outs[-1].append(_run(eng, x, _partitions(T, F)[0][0]))          # a second call: the same bits
        eng.close()
    for a, b in zip(*outs):
        for u, v in zip(a, b):
            assert np.array_equal(u, v)
    for u, v in zip(outs[0][0], outs[0][2]):
        assert np.array_equal(u, v)


@pytest.mark.parametrize('prec', ['fp32', 'tf32', 'bf16', 'bf16x3', 'uq-fp32', 'uq-bf16'])
def test_a_field_the_model_does_not_read_gets_exactly_zero(prec):
    uq = prec.startswith('uq')
    T, F, O, H, L, S = 8, 32, 16, 256, 1, 2
    P, x = _params(T, F, O, H, L, S, 'lstm', uq, seed=5)
    dead = 7
    kernels = [i for i, p in enumerate(P) if p.shape == (F, 4 * H)]      # each stage's first lstm kernel
    assert len(kernels) == S
    for i in kernels:
        P[i] = P[i].copy()
        P[i][dead, :] = 0.0                                # the input-kernel row of field 7 in every stage
    eng = _chain(S, T, F, O, H, L, precision=prec.split('-')[-1], uq=uq, **(DROP if uq else {}))
    eng.set_weights(P)
    cg, G = imo.field_groups(T, F)
    phi, f_x, f_bg = _run(eng, x, cg)
    assert np.array_equal(phi[:, :, dead], np.zeros_like(phi[:, :, dead]))
    assert (np.abs(phi).max(axis=(0, 1)) > 0).sum() == G - 1
    eng.close()


def _slots(e):
    p, n = C.c_void_p(0), C.c_int64(0)
    assert e.lib.lfmq_opt_state_ptr(e.handle, C.byref(p), C.byref(n)) == 0
    off = p.value - e.workspace.data_ptr()
    return e.workspace[off:off + 4 * n.value].clone()


@pytest.mark.parametrize('uq', [False, True])
def test_the_handles_state_is_left_untouched(uq):
    T, F, O, H, L, S = 5, 6, 3, 16, 1, 2
    P, x = _params(T, F, O, H, L, S, 'lstm', uq, seed=8)
    y = np.random.RandomState(9).normal(size=(N, T, O)).astype(np.float32)
    eng = _chain(S, T, F, O, H, L, uq=uq, train=True, forward_only=False, max_batch=N, **DROP)
    eng.set_weights(P)
    eng.train_step(_cuda(x), [_cuda(y)] * S, 1, 0.5)
    before = [(e.params.clone(), e.grads.clone(), _slots(e)) for e in eng.stages]
    _run(eng, x, imo.field_groups(T, F)[0])
    torch.cuda.synchronize()
    for e, (p, g, s) in zip(eng.stages, before):
        assert torch.equal(e.params, p) and torch.equal(e.grads, g) and torch.equal(_slots(e), s)
    eng.close()


def test_refusals():
    from lfm_quant_b200 import _native as Nv
    T, F, O, H = 5, 6, 3, 16
    P, x = _params(T, F, O, H, 1, 1, 'lstm', False, seed=2)
    eng = _chain(1, T, F, O, H, 1)
    eng.set_weights(P)
    lib = eng.lib
    xd = _cuda(x)
    cg = np.ascontiguousarray(imo.field_groups(T, F)[0])
    n = C.c_uint64(0)
    assert lib.lfmq_chain_shapley_work_bytes(eng._handles, 1, N, F, M, C.byref(n)) == 0
    work = torch.empty(n.value, dtype=torch.uint8, device='cuda')
    phi = torch.empty(N, 1, F, device='cuda')
    f_x, f_bg = torch.empty(N, 1, device='cuda'), torch.empty(N, 1, device='cuda')
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def call(N_=N, G=F, samples=M, col=cg, x_=xd.data_ptr(), phi_=phi.data_ptr(), fx=f_x.data_ptr(),
             fbg=f_bg.data_ptr(), wb=None):
        return lib.lfmq_chain_shapley(eng._handles, 1, C.c_void_p(x_), N_,
                                      col.ctypes.data_as(C.c_void_p) if col is not None else None, G, samples, SEED,
                                      STEP, C.c_void_p(phi_), C.c_void_p(fx), C.c_void_p(fbg),
                                      C.c_void_p(work.data_ptr()), work.numel() if wb is None else wb, s)
    assert call() == 0
    bad = cg.copy()
    bad[4] = F
    neg = cg.copy()
    neg[0] = -1
    for kw in (dict(samples=0), dict(N_=0), dict(G=0), dict(col=bad), dict(col=neg), dict(col=None), dict(x_=0),
               dict(phi_=0), dict(fx=0), dict(fbg=0)):
        assert call(**kw) == ERR_ARG, kw
    for args in ((0, F, M), (N, 0, M), (N, F, 0)):
        assert lib.lfmq_chain_shapley_work_bytes(eng._handles, 1, *args, C.byref(n)) == ERR_ARG, args
    assert lib.lfmq_chain_shapley_work_bytes(eng._handles, 1, N, F, M, None) == ERR_ARG
    assert lib.lfmq_chain_shapley_work_bytes(eng._handles, 0, N, F, M, C.byref(n)) == ERR_ARG
    assert call(wb=work.numel() - 1) == ERR_WORKSPACE
    assert 'work needs %d bytes' % work.numel() in Nv.load().lfmq_last_error().decode()
    torch.cuda.synchronize()
    eng.close()


# ---- the CLI on the synthetic dataset ----------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def workdir(tmp_path_factory):
    from lfm_quant_b200.scripts.synthetic import write_open_dataset, write_system_test_conf
    d = tmp_path_factory.mktemp('shapley')
    write_open_dataset(str(d / 'datasets' / 'open-dataset.dat'), n_keys=30, n_months=420, seed=9)
    write_system_test_conf(str(d / 'config' / 'system-test.conf'), str(d / 'datasets'), str(d / 'experiments'))
    (d / 'experiments').mkdir()
    return d


@pytest.fixture()
def cli(workdir, monkeypatch):
    from lfm_quant_b200.scripts import configs
    from lfm_quant_b200.scripts import lfm_quant
    monkeypatch.setenv('LFM_QUANT_ROOT', str(workdir))
    conf = str(workdir / 'config' / 'system-test.conf')

    def main(*argv):
        configs.reset()
        try:
            return lfm_quant.main(['--config=' + conf] + list(argv))
        finally:
            configs.reset()
    return main


@pytest.mark.parametrize('name,extra,K', [
    ('point', ['--dropout', '0.1'], 1),
    ('uq', ['--nn_type', 'RNNUqRangeEstimate', '--UQ=True', '--dropout', '0.1', '--recurrent_dropout', '0.1'], 2),
    ('mlp', ['--nn_type', 'MLPLinearPointEstimate', '--init_scale', '0.02'], 1),
])
def test_cli_writes_shapley_npz_and_leaves_preds_dat_alone(workdir, cli, name, extra, K):
    m = workdir / 'experiments' / ('shap-' + name)
    args = ['--model_dir', 'shap-' + name] + extra
    cli(*args, '--train=True')
    cli(*args, '--train=False')
    plain = (m / 'pred' / 'preds.dat').read_bytes()
    assert not (m / 'pred' / 'shapley.npz').exists()
    cli(*args, '--train=False', '--shapley_samples', '4')
    assert (m / 'pred' / 'preds.dat').read_bytes() == plain
    df = pd.read_csv(m / 'pred' / 'preds.dat', sep=' ', dtype={'gvkey': str})
    z = np.load(m / 'pred' / 'shapley.npz')
    n = len(df)
    F, T = len(z['fields']), len(z['quarters'])
    assert z['date'].tolist() == df['date'].tolist() and z['gvkey'].tolist() == df['gvkey'].tolist()
    assert z['outputs'].tolist() == (['norm_preds_1', 'norm_variance_1'] if K == 2 else ['norm_preds_1'])
    assert z['phi_field'].shape == (n, K, F) and z['phi_quarter'].shape == (n, K, T)
    assert z['f_x'].shape == z['f_bg'].shape == (n, K) and z['quarters'].tolist() == list(range(1 - T, 1))
    assert np.isfinite(z['phi_field']).all() and np.isfinite(z['phi_quarter']).all()
    for phi in (z['phi_field'], z['phi_quarter']):
        assert _efficiency(phi, z['f_x'], z['f_bg']) < 1e-5
    if name != 'uq':                                          # a point forecast's f_x is what preds.dat holds
        assert np.abs(z['f_x'][:, 0] - df['norm_preds_1'].to_numpy()).max() < 1e-5
    top = np.argsort(-np.abs(z['phi_field'][:, 0]).mean(axis=0))[:5]
    print('%s: mean |phi| of the top fields %s' % (name, dict(zip(z['fields'][top], np.abs(z['phi_field'][:, 0])
                                                               .mean(axis=0)[top].round(5)))))
