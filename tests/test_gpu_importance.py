"""Permutation importance on the GPU (lfmq_chain_permutation_importance, ForecastChainEngine.permutation_importance,
NativeForecaster.permutation_importance, --perm_importance): row 0 of `out` is the model's loss on the held-out set,
row 1 + g * R + r its loss with group g's columns taken from window pi_{seed,g,r}(i).

Checked here: the fp64 oracle (tests/importance_oracle.py) for every model kind; each row bit for bit the loss entry
point on the copy built from the NumPy permutation, at every precision; the same bits at any launch size; exactly zero
importance for a field the model does not read; the handle's state left untouched; the refusals; and the CLI files."""
import ctypes as C

import numpy as np
import pandas as pd
import pytest
import torch

import importance_oracle as imo
import lfm_oracle as orc
import uq_chain_oracle as uco

pytestmark = pytest.mark.gpu
KW = dict(target_idx=1, target_lambda=0.5, rnn_lambda=0.7)
DROP = dict(dropout=0.2, recurrent_dropout=0.15, seed=31)
SEED, STEP, R = 2024, 7, 2
N = 1000                          # not a multiple of 256 or of the launch rows
ERR_ARG, ERR_WORKSPACE = 1, 4     # include/lfmq.h


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()


def _chain(S, T, F, O, H, L, *, max_batch=256, precision='fp32', uq=False, cell='lstm', weights=None, **kw):
    from lfm_quant_b200.engine import ForecastChainEngine
    args = dict(KW, train=False, forward_only=True)
    args.update(kw)
    return ForecastChainEngine(forecast_steps=S, weights=weights or [1.0, 0.5, 0.25][:S], max_batch=max_batch,
                               seq_len=T, n_inputs=F, n_outputs=O, num_hidden=H, num_layers=L, rnn_cell=cell,
                               precision=precision, uq=uq, **args)


def _dense(T, F, O, max_batch=256):
    from lfm_quant_b200.engine import DenseEngine, ForecastChainEngine
    return ForecastChainEngine(stages=[DenseEngine(max_batch=max_batch, seq_len=T, n_inputs=F, n_outputs=O,
                                                   target_idx=KW['target_idx'], target_lambda=KW['target_lambda'],
                                                   forward_only=True)])


def _point_problem(T, F, O, H, L, S, cell, seed):
    rng = np.random.RandomState(seed)
    P = orc.init_forecast_params(L, F, O, H, S, init_scale=0.5, seed=seed + 1, dtype=np.float64, rnn_cell=cell)
    P = [(p + rng.normal(size=p.shape) * 0.05).astype(np.float32).astype(np.float64) for p in P]
    x = rng.normal(size=(N, T, F)).astype(np.float32)
    y = rng.normal(size=(N, T, O)).astype(np.float32)
    y[::7, :2, :] = 0.0                                           # zero-padded steps: masked in the loss
    return P, x, [y] * S


def _uq_problem(T, F, O, H, L, S, cell, seed):
    rng = np.random.RandomState(seed)
    P = uco.init_params(L, F, O, H, S, init_scale=0.5, seed=seed + 1, dtype=np.float64, rnn_cell=cell)
    P = [(p + rng.normal(size=p.shape) * 0.05).astype(np.float32).astype(np.float64) for p in P]
    x = rng.normal(size=(N, T, F)).astype(np.float32)
    y = rng.normal(size=(N, T, O)).astype(np.float32)              # no all-zero row: the uq loss of one is NaN
    return P, x, [y] * S


def _rel(got, ref):
    """max |got - ref| over the largest |ref| of each column (a column of zeros must be zeros)"""
    scale = np.abs(ref).max(axis=0)
    return float(np.max(np.abs(got - ref) / np.where(scale > 0, scale, 1.0)))


def _partitions(T, F):
    return [imo.field_groups(T, F), imo.quarter_groups(T, F)]


def _run(eng, x, ys, cg):
    return eng.permutation_importance(_cuda(x), [_cuda(y) for y in ys], cg, R, SEED, STEP).cpu().numpy()


# (name, S, L, cell, uq)
MODELS = [('lstm-point-L2', 1, 2, 'lstm', False), ('gru-point', 1, 1, 'gru', False), ('lstm-uq', 1, 1, 'lstm', True),
          ('point-chain-S2', 2, 1, 'lstm', False), ('uq-chain-S2', 2, 1, 'gru', True)]


@pytest.mark.parametrize('model', MODELS, ids=[m[0] for m in MODELS])
def test_rows_match_the_fp64_oracle(model):
    _, S, L, cell, uq = model
    T, F, O, H = 5, 6, 3, 16
    w = [1.0, 0.5][:S]
    P, x, ys = (_uq_problem if uq else _point_problem)(T, F, O, H, L, S, cell, seed=3 + S + L)
    eng = _chain(S, T, F, O, H, L, uq=uq, cell=cell, weights=w, **(DROP if uq else {}))
    eng.set_weights(P)
    if uq:
        loss = imo.uq_loss(P, ys, w, num_layers=L, rnn_cell=cell, dropout=DROP['dropout'],
                           recurrent_dropout=DROP['recurrent_dropout'], seed=DROP['seed'], step=STEP, **KW)
    else:
        loss = imo.point_loss(P, ys, w if S > 1 else [1.0], num_layers=L, rnn_cell=cell, **KW)
    for cg, G in _partitions(T, F):
        got = _run(eng, x, ys, cg)
        ref = imo.importance(x, cg, G, R, SEED, loss)
        assert got.shape == ref.shape == (1 + G * R, 3)
        err = _rel(got, ref)
        print('importance %s G=%d: max rel err %.2e, max |delta loss| %.2e'
              % (model[0], G, err, np.abs(ref[1:, 0] - ref[0, 0]).max()))
        assert err < 1e-4, err
        assert np.abs(ref[1:, 0] - ref[0, 0]).max() > 0                # the shuffles do change the loss
    eng.close()


def test_linear_model_rows_match_the_fp64_oracle():
    T, F, O = 5, 6, 3
    rng = np.random.RandomState(4)
    W = (rng.normal(size=(T * F, O)) * 0.2).astype(np.float32).astype(np.float64)
    b = (rng.normal(size=O) * 0.1).astype(np.float32).astype(np.float64)
    x = rng.normal(size=(N, T * F)).astype(np.float32)
    y = rng.normal(size=(N, O)).astype(np.float32)
    y[::9] = 0.0
    eng = _dense(T, F, O)
    eng.set_weights([W, b])
    loss = imo.dense_loss(W, b, y, **{k: KW[k] for k in ('target_idx', 'target_lambda')})
    for cg, G in _partitions(T, F):
        got = _run(eng, x, [y], cg)
        ref = imo.importance(x, cg, G, R, SEED, loss)
        err = _rel(got, ref)
        print('importance linear G=%d: max rel err %.2e' % (G, err))
        assert err < 1e-4, err
        assert np.array_equal(got[:, 2], np.zeros(1 + G * R, dtype=np.float32))
    eng.close()


def _by_hand(eng, x, ys, cg, G):
    """Every copy built from the NumPy permutation, forwarded by the same engine in launches of max_batch rows keyed
    by window index, then reduced by the model's loss entry point."""
    mb = eng.cfg.max_batch
    rows = []
    copies = [x] + [imo.permuted_copy(x, cg, g, imo.permutation(N, SEED, g, r)) for g in range(G) for r in range(R)]
    yd = [_cuda(y) for y in ys]
    for xc in copies:
        xd = _cuda(xc)
        outs = [eng.forward(xd[a:a + mb].contiguous(), step=STEP, row0=a) for a in range(0, N, mb)]
        outs = [torch.cat([o[k] for o in outs]) for k in range(len(outs[0]))]
        if eng.uq:
            o = eng.loss_uq(outs[0::2], outs[1::2], yd)
        else:
            o = torch.cat([eng.loss(outs, yd), torch.zeros(1, device=xd.device)])
        rows.append(o.cpu().numpy())
    return np.stack(rows)


@pytest.mark.parametrize('case', ['fp32', 'tf32', 'bf16', 'bf16x3', 'uq-fp32', 'uq-bf16', 'chain-bf16'])
def test_rows_are_the_loss_entry_point_on_each_copy(case):
    uq = case.startswith('uq')
    prec = case.split('-')[-1]
    S = 2 if case.startswith('chain') else 1
    T, F, O, H, L = 8, 32, 16, 256, 1
    P, x, ys = (_uq_problem if uq else _point_problem)(T, F, O, H, L, S, 'lstm', seed=11)
    eng = _chain(S, T, F, O, H, L, precision=prec, uq=uq, **(DROP if uq else {}))
    eng.set_weights(P)
    for cg, G in _partitions(T, F):
        got = _run(eng, x, ys, cg)
        want = _by_hand(eng, x, ys, cg, G)
        assert np.array_equal(got, want), (case, G, np.abs(got - want).max())
    eng.close()


@pytest.mark.parametrize('case', ['fp32', 'tf32', 'uq-fp32'])
def test_launch_size_does_not_change_the_bits(case):
    uq = case.startswith('uq')
    T, F, O, H, L = 6, 10, 4, 64, 2
    P, x, ys = (_uq_problem if uq else _point_problem)(T, F, O, H, L, 1, 'lstm', seed=21)
    outs = []
    for mb in (256, 8192):
        eng = _chain(1, T, F, O, H, L, max_batch=mb, precision=case.split('-')[-1], uq=uq, **(DROP if uq else {}))
        eng.set_weights(P)
        outs.append([_run(eng, x, ys, cg) for cg, _ in _partitions(T, F)])
        outs[-1].append(_run(eng, x, ys, _partitions(T, F)[0][0]))          # a second call: the same bits
        eng.close()
    for a, b in zip(*outs):
        assert np.array_equal(a, b)
    assert np.array_equal(outs[0][0], outs[0][2])


@pytest.mark.parametrize('prec', ['fp32', 'tf32', 'bf16'])
def test_a_field_the_model_does_not_read_has_zero_importance(prec):
    T, F, O, H, L = 8, 32, 16, 256, 1
    P, x, ys = _point_problem(T, F, O, H, L, 1, 'lstm', seed=5)
    dead = 7
    P[0] = P[0].copy()
    P[0][dead, :] = 0.0                                          # lstm_1/kernel row of field 7
    eng = _chain(1, T, F, O, H, L, precision=prec)
    eng.set_weights(P)
    cg, G = imo.field_groups(T, F)
    out = _run(eng, x, ys, cg)
    perm = out[1:].reshape(G, R, 3)
    assert np.array_equal(perm[dead], np.broadcast_to(out[0], (R, 3)))
    assert np.abs(perm[:, :, 0] - out[0, 0]).max() > 0
    eng.close()


def _slots(e):
    p, n = C.c_void_p(0), C.c_int64(0)
    assert e.lib.lfmq_opt_state_ptr(e.handle, C.byref(p), C.byref(n)) == 0
    off = p.value - e.workspace.data_ptr()
    return e.workspace[off:off + 4 * n.value].clone()


@pytest.mark.parametrize('uq', [False, True])
def test_the_handles_state_is_left_untouched(uq):
    T, F, O, H, L, S = 5, 6, 3, 16, 1, 2
    P, x, ys = (_uq_problem if uq else _point_problem)(T, F, O, H, L, S, 'lstm', seed=8)
    eng = _chain(S, T, F, O, H, L, uq=uq, train=True, forward_only=False, max_batch=N, **DROP)
    eng.set_weights(P)
    eng.train_step(_cuda(x), [_cuda(y) for y in ys], 1, 0.5)
    before = [(e.params.clone(), e.grads.clone(), _slots(e)) for e in eng.stages]
    _run(eng, x, ys, imo.field_groups(T, F)[0])
    torch.cuda.synchronize()
    for e, (p, g, s) in zip(eng.stages, before):
        assert torch.equal(e.params, p) and torch.equal(e.grads, g) and torch.equal(_slots(e), s)
    eng.close()


def test_refusals():
    from lfm_quant_b200 import _native as Nv
    T, F, O, H = 5, 6, 3, 16
    P, x, ys = _point_problem(T, F, O, H, 1, 1, 'lstm', seed=2)
    eng = _chain(1, T, F, O, H, 1)
    eng.set_weights(P)
    lib = eng.lib
    xd, yd = _cuda(x), _cuda(ys[0])
    ysp = (C.c_void_p * 1)(yd.data_ptr())
    w = (C.c_float * 1)(1.0)
    cg = np.ascontiguousarray(imo.field_groups(T, F)[0])
    n = C.c_uint64(0)
    assert lib.lfmq_chain_permutation_importance_work_bytes(eng._handles, 1, N, C.byref(n)) == 0
    work = torch.empty(n.value, dtype=torch.uint8, device='cuda')
    out = torch.empty(1 + F * R, 3, device='cuda')
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def call(N_=N, G=F, reps=R, col=cg, x_=xd.data_ptr(), y_=ysp, w_=w, out_=out.data_ptr(), wb=None):
        return lib.lfmq_chain_permutation_importance(eng._handles, 1, C.c_void_p(x_), y_, w_, N_,
                                                     col.ctypes.data_as(C.c_void_p) if col is not None else None, G,
                                                     reps, SEED, STEP, C.c_void_p(out_), C.c_void_p(work.data_ptr()),
                                                     work.numel() if wb is None else wb, s)
    assert call() == 0
    bad = cg.copy()
    bad[4] = F
    neg = cg.copy()
    neg[0] = -1
    for kw in (dict(reps=0), dict(N_=0), dict(G=0), dict(col=bad), dict(col=neg), dict(col=None), dict(x_=0),
               dict(y_=(C.c_void_p * 1)(0)), dict(y_=None), dict(w_=None), dict(out_=0)):
        assert call(**kw) == ERR_ARG, kw
    assert lib.lfmq_chain_permutation_importance_work_bytes(eng._handles, 1, 0, C.byref(n)) == ERR_ARG
    assert call(wb=work.numel() - 1) == ERR_WORKSPACE
    assert 'work needs %d bytes' % work.numel() in Nv.load().lfmq_last_error().decode()
    torch.cuda.synchronize()
    eng.close()


# ---- the CLI on the synthetic dataset ----------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def workdir(tmp_path_factory):
    from lfm_quant_b200.scripts.synthetic import write_open_dataset, write_system_test_conf
    d = tmp_path_factory.mktemp('importance')
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


def _check_table(path, fields, T):
    df = pd.read_csv(path, sep=' ', dtype={'group': str})
    assert df['kind'].tolist() == ['field'] * len(fields) + ['quarter'] * T
    assert df['group'].tolist() == list(fields) + [str(t) for t in range(1 - T, 1)]
    assert np.isfinite(df.drop(columns=['kind', 'group']).to_numpy()).all()
    return df


def _fields_and_T(workdir, cli_args):
    from lfm_quant_b200.scripts import configs, lfm_quant
    from lfm_quant_b200.scripts.data_processing import Dataset
    configs.reset()
    c = lfm_quant.get_configs(['--config=' + str(workdir / 'config' / 'system-test.conf')] + list(cli_args))
    configs.reset()
    d = Dataset(c)
    return d.fin_col_names + d.aux_col_names, d.seq_len


def test_cli_writes_importance_dat_and_leaves_preds_dat_alone(workdir, cli):
    m = workdir / 'experiments' / 'imp'
    args = ['--model_dir', 'imp', '--dropout', '0.1']
    cli(*args, '--train=True')
    cli(*args, '--train=False')
    plain = (m / 'pred' / 'preds.dat').read_bytes()
    assert not (m / 'pred' / 'importance.dat').exists()
    cli(*args, '--train=False', '--perm_importance', '2')
    assert (m / 'pred' / 'preds.dat').read_bytes() == plain
    first = (m / 'pred' / 'importance.dat').read_bytes()
    fields, T = _fields_and_T(workdir, args + ['--train=False'])
    df = _check_table(m / 'pred' / 'importance.dat', fields, T)
    assert df['base_loss'].nunique() == 1 and (df['perm_loss_std'] >= 0).all()
    print(df.sort_values('delta_loss', ascending=False).head(8).to_string())
    cli(*args, '--train=False', '--perm_importance', '2')
    assert (m / 'pred' / 'importance.dat').read_bytes() == first


@pytest.mark.parametrize('name,extra', [
    ('uq', ['--nn_type', 'RNNUqRangeEstimate', '--UQ=True', '--dropout', '0.1', '--recurrent_dropout', '0.1']),
    ('steps2', ['--forecast_steps', '2', '--forecast_steps_weights', '1.0-0.5']),
    ('mlp', ['--nn_type', 'MLPLinearPointEstimate', '--init_scale', '0.02']),
])
def test_cli_other_models(workdir, cli, name, extra):
    args = ['--model_dir', 'imp-' + name] + extra
    cli(*args, '--train=True')
    cli(*args, '--train=False', '--perm_importance', '1')
    fields, T = _fields_and_T(workdir, args + ['--train=False'])
    _check_table(workdir / 'experiments' / ('imp-' + name) / 'pred' / 'importance.dat', fields, T)


def test_cli_walk_forward_stacks_the_origins_files(workdir, cli):
    origins = [199612, 199712]
    args = ['--training_type', 'iterative', '--split_date', '199612', '--end_date', '199812', '--model_dir', 'imp-wf',
            '--NPE', '2']
    cli(*args, '--train=True')
    cli(*args, '--train=False', '--perm_importance', '1')
    wf = workdir / 'experiments' / 'imp-wf'
    got = pd.read_csv(wf / 'walk_forward_importance.dat', sep=' ', dtype={'group': str}, float_precision='round_trip')
    own = [pd.read_csv(wf / ('system-test-wf-%d' % o) / 'pred' / 'importance.dat', sep=' ', dtype={'group': str},
                       float_precision='round_trip').assign(origin=o) for o in origins]
    pd.testing.assert_frame_equal(got, pd.concat(own, ignore_index=True))
    assert got['origin'].tolist() == sorted(got['origin'].tolist())
