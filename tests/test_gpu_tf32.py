"""LFMQ_PREC_TF32 on the GPU: the fp32 step with its GEMMs on tf32 tensor cores (tf32_gemm.cu).

1. Parity: LSTM and GRU, point and UQ, one and two layers with both dropouts, and point / UQ chains, against the fp64
   oracle and against the rounding oracle (tests/tf32_oracle.py: the same oracle with every matrix product's operands
   rounded as the kernels round them).  Outputs, losses, every gradient tensor, and the weights after three Adadelta
   steps with clip_by_global_norm and MaxNorm biting.  The shapes reach B in {1, 127, 129}, H in {4, 132, 1020},
   F in {1, 33, 300}, O in {1, 17}, T in {1, 48}; B = 4096 at T = 48 is checked on row blocks of the full batch.
2. Determinism: forward rows are bit-identical under permutation, row0 slicing and launch size; two backward calls give
   the same bits; Monte-Carlo sample 0 is lfmq_forward_uq and the moments do not depend on the launch size.
3. The weights the GEMMs read follow every update: after train steps or set_weights, a forward equals a fresh handle's.
4. Data parallel: row shards with the global denominators sum to the whole batch's gradients.
5. The model object and the CLI: GRU point and two-step UQ models train at --precision tf32 and predict at fp32 from
   the tf32 checkpoint; a tf32 loss trajectory follows the fp32 one.

Bounds (relative to each tensor's largest entry) were measured on an H100 80GB HBM3 at a 700 W power limit and are set
at >= 1.5x the worst value seen; every test prints its worst values next to the bounds.
"""
import os

import numpy as np
import pytest
import torch

import lfm_oracle as orc
import tf32_oracle as t3
from test_gpu_fp32_models import (DROP, FAMILIES, ROW0, STEP, WEIGHTS, _close, _cuda, _engine, _gpu_backward,
                                  _gpu_forward, _loss_kw, _names, _oracle_forward, _oracle_loss_backward,
                                  _oracle_train_step, _problem, _scalar_err)
from util import rel_err

pytestmark = pytest.mark.gpu

# {kind: (bound against the rounding oracle, bound against the fp64 oracle)}
# worst measured (rounding, fp64): output 3.2e-4, 1.0e-3; loss 4.2e-4, 3.7e-3; gradient 1.3e-3, 6.8e-3; step loss
# 3.1e-4, 3.7e-3; weights after three steps 1.4e-4, 1.9e-3.  The rounding oracle's bounds sit 3x (outputs) to 12x
# (weights) below the fp64 ones: what it leaves is fp32 accumulation and the fp32 pointwise arithmetic.
BOUNDS = {
    'output': (5e-4, 1.5e-3),
    'loss': (7e-4, 6e-3),
    'gradient': (2e-3, 1.1e-2),
    'step loss': (5e-4, 6e-3),
    'weights': (2.5e-4, 3e-3),
}
FAMS = dict(FAMILIES, lstm=('lstm', False, 1))
LR, CLIP, N_STEPS = 0.6, 0.5, 3


class _Worst(object):
    """Records each error against both oracles; asserts after printing the worst of each kind."""

    def __init__(self, title):
        self.title, self.worst, self.fail = title, {}, []

    def check(self, kind, which, err, where):
        bound = BOUNDS[kind][which]
        key = (kind, ('rounding', 'fp64')[which])
        self.worst[key] = max(self.worst.get(key, 0.0), err)
        if not err < bound:
            self.fail.append((kind, which, where, err, bound))

    def done(self):
        print('%s: %s' % (self.title, ', '.join('%s/%s %.2e' % (k[0], k[1], w) for k, w in sorted(self.worst.items()))))
        assert not self.fail, (self.title, self.fail[:5])


def _both(fn, *a, **k):
    """fn through the fp64 oracle and through the rounding oracle."""
    with t3.rounding():
        r = t3.call(fn, *a, **k)
    return fn(*a, **k), r


SHAPES = {                       # (B, T, F, O, H, L)
    'b1-f1': (1, 48, 1, 1, 132, 2),
    'b127-h4': (127, 48, 33, 17, 4, 1),
    'b129-t1-f300-h1020': (129, 1, 300, 17, 1020, 1),
    'b129-splitk': (129, 48, 33, 1, 132, 2),       # B*T = 6192: split-K weight gradients, ragged 128-wide tiles
}
FAMILY_LIST = ['lstm', 'gru', 'uq-lstm', 'uq-gru', 'chain2', 'chain3', 'uq-chain2']


@pytest.fixture(autouse=True)
def _families(monkeypatch):
    import test_gpu_fp32_models as m
    monkeypatch.setattr(m, 'FAMILIES', FAMS)


@pytest.mark.parametrize('shape', list(SHAPES))
@pytest.mark.parametrize('family', FAMILY_LIST)
def test_tf32_training_matches_both_oracles(family, shape):
    B, T, F, O, H, L = SHAPES[shape]
    if FAMS[family][2] > T + 1:
        pytest.skip('the window of a %d-step chain holds its %d appended predictions: T >= %d'
                    % (FAMS[family][2], FAMS[family][2] - 1, FAMS[family][2] - 1))
    lkw = _loss_kw(O)
    P, x, ys = _problem(family, B, T, F, O, H, L, seed=sum(map(ord, family + shape)))
    max_norm = 0.9 * float(np.linalg.norm(P[0], axis=0).max())
    eng = _engine(family, B, T, F, O, H, L, train=True, precision='tf32', optimizer='Adadelta', max_grad_norm=CLIP,
                  max_norm=max_norm, **lkw, **DROP)
    eng.set_weights(P)
    chk = _Worst('tf32 %s %s' % (family, shape))
    xd, yd = _cuda(x), [_cuda(y) for y in ys]
    (o64, fc64), (o32, fc32) = _both(_oracle_forward, family, P, x, L, STEP, ROW0)
    for i, g in enumerate(_gpu_forward(eng, xd, STEP, ROW0)):
        chk.check('output', 0, rel_err(g, o32[i]), i)
        chk.check('output', 1, rel_err(g, o64[i]), i)
    s64, g64 = _oracle_loss_backward(family, ys, o64, fc64, L, lkw)
    with t3.rounding():
        s32, g32 = t3.call(_oracle_loss_backward, family, ys, o32, fc32, L, lkw)
    for i, g in enumerate(_gpu_backward(family, eng, xd, yd, STEP, ROW0)):
        chk.check('loss', 0, _scalar_err(g, s32[i]), i)
        chk.check('loss', 1, _scalar_err(g, s64[i]), i)
    names = _names(eng)
    for name, g, r32, r64 in zip(names, eng.grads_list(), g32, g64):
        chk.check('gradient', 0, rel_err(g, r32), name)
        chk.check('gradient', 1, rel_err(g, r64), name)
    p64 = [q.copy() for q in P]
    p32 = [q.copy() for q in P]
    sl64, sl32 = orc.zero_slots('Adadelta', p64), orc.zero_slots('Adadelta', p32)
    S = FAMS[family][2]
    for it in range(N_STEPS):
        out = eng.train_step(xd, yd[0] if S == 1 else yd, it, LR).cpu().numpy()
        p64, ref64 = _oracle_train_step(family, p64, sl64, x, ys, it, L, lkw, LR, CLIP, max_norm)
        with t3.rounding():
            p32, ref32 = t3.call(_oracle_train_step, family, p32, sl32, x, ys, it, L, lkw, LR, CLIP, max_norm)
        for i, g in enumerate(out):
            chk.check('step loss', 0, _scalar_err(g, ref32[i]), (it, i))
            chk.check('step loss', 1, _scalar_err(g, ref64[i]), (it, i))
    got = eng.get_weights()
    for name, w, r32, r64 in zip(names, got, p32, p64):
        chk.check('weights', 0, rel_err(w, r32), name)
        chk.check('weights', 1, rel_err(w, r64), name)
    assert np.linalg.norm(got[0], axis=0).max() <= max_norm * (1 + 1e-5)
    chk.done()
    _close(eng)


@pytest.mark.parametrize('family', ['gru', 'uq-lstm'])
def test_tf32_forward_rows_at_product_scale(family):
    """B = 4096, T = 48, F = 32, O = 16, H = 256, both dropouts: blocks of the full batch's forward rows against the
    rounding oracle on those rows alone (row0 offsets carry the dropout masks)."""
    B, T, F, O, H, L = 4096, 48, 32, 16, 256, 1
    P, x, _ = _problem(family, B, T, F, O, H, L, seed=11, init_scale=0.3)
    eng = _engine(family, B, T, F, O, H, L, train=True, precision='tf32', **_loss_kw(O), **DROP)
    eng.set_weights(P)
    full = _gpu_forward(eng, _cuda(x), STEP, ROW0)
    chk = _Worst('tf32 rows %s B=4096' % family)
    for a, b in [(0, 8), (127, 129), (2040, 2056), (B - 8, B)]:
        (o64, _), (o32, _) = _both(_oracle_forward, family, P, x[a:b], L, STEP, ROW0 + a)
        for i, g in enumerate(full):
            chk.check('output', 0, rel_err(g[a:b], o32[i]), (a, i))
            chk.check('output', 1, rel_err(g[a:b], o64[i]), (a, i))
    chk.done()
    _close(eng)


# ---- 2. determinism ---------------------------------------------------------------------------------------------------
def _small(family, B=300, T=12, F=33, O=17, H=132, L=2, drop=True, **kw):
    P, x, ys = _problem(family, B, T, F, O, H, L, seed=5)
    eng = _engine(family, B, T, F, O, H, L, train=True, precision='tf32', **_loss_kw(O), **(DROP if drop else {}),
                  **kw)
    eng.set_weights(P)
    return eng, P, _cuda(x), [_cuda(y) for y in ys]


@pytest.mark.parametrize('family', ['lstm', 'gru', 'uq-gru', 'chain2'])
def test_tf32_forward_rows_are_bit_identical_under_slicing_and_permutation(family):
    eng, _, xd, _ = _small(family)
    full = eng.forward(xd, step=STEP, row0=ROW0)
    full = [t.clone() for t in (full if isinstance(full, (list, tuple)) else [full])]
    for a, b in [(0, 1), (5, 134), (129, 300)]:
        part = eng.forward(xd[a:b].contiguous(), step=STEP, row0=ROW0 + a)
        for f, p in zip(full, part if isinstance(part, (list, tuple)) else [part]):
            assert torch.equal(f[a:b], p), (a, b)
    _close(eng)
    eng, _, xd, _ = _small(family, drop=False)          # no dropout: the masks do not follow the rows
    perm = torch.randperm(xd.shape[0], generator=torch.Generator().manual_seed(1)).cuda()
    a = eng.forward(xd)
    a = [t.clone() for t in (a if isinstance(a, (list, tuple)) else [a])]
    b = eng.forward(xd[perm].contiguous())
    for f, p in zip(a, b if isinstance(b, (list, tuple)) else [b]):
        assert torch.equal(f[perm], p)
    _close(eng)


@pytest.mark.parametrize('family', ['lstm', 'uq-gru', 'uq-chain2'])
def test_tf32_two_backward_calls_give_the_same_bits(family):
    eng, _, xd, yd = _small(family, B=200, T=48)       # B*T = 9600: split-K weight gradients
    s1 = _gpu_backward(family, eng, xd, yd, STEP, ROW0)
    g1 = [g.copy() for g in eng.grads_list()]
    s2 = _gpu_backward(family, eng, xd, yd, STEP, ROW0)
    g2 = eng.grads_list()
    assert [float(v) for v in s1] == [float(v) for v in s2]
    for a, b in zip(g1, g2):
        np.testing.assert_array_equal(a, b)
    _close(eng)


@pytest.mark.parametrize('family', ['uq-lstm', 'uq-chain2'])
def test_tf32_mc_sample_zero_and_launch_size_independence(family):
    B, T, F, O, H, L, SAMPLES = 40, 12, 33, 17, 132, 1, 7
    P, x, _ = _problem(family, B, T, F, O, H, L, seed=8)
    xd = _cuda(x)
    moments = []
    for mb in (B, 3 * B + 5, SAMPLES * B):
        eng = _engine(family, mb, T, F, O, H, L, train=False, forward_only=True, precision='tf32', **_loss_kw(O),
                      **DROP)
        eng.set_weights(P)
        if mb == B:
            one = [t.cpu() for t in eng.forward(xd, step=STEP, row0=ROW0)]
            m1 = eng.forward_mc(xd, 1, step=STEP, row0=ROW0)
        moments.append(eng.forward_mc(xd, SAMPLES, step=STEP, row0=ROW0))
        _close(eng)

    def flat(m):
        out = []
        for v in m:
            out += flat(v) if isinstance(v, (list, tuple)) else [v.cpu()]
        return out

    first = flat(moments[0])
    for m in moments[1:]:
        for a, b in zip(first, flat(m)):
            assert torch.equal(a, b)
    # one sample: its means are sample 0, i.e. the forward's target prediction and variance of stage 0
    m1 = flat(m1)
    assert torch.equal(m1[0], one[0]) and torch.equal(m1[1], one[1])


# ---- 3. weights the GEMMs read follow updates ---------------------------------------------------------------------------
@pytest.mark.parametrize('family', ['gru', 'uq-lstm', 'chain2'])
def test_tf32_forward_after_updates_equals_a_fresh_handle(family):
    eng, P, xd, yd = _small(family, B=130, T=10)
    S = FAMS[family][2]
    for it in range(3):
        eng.train_step(xd, yd[0] if S == 1 else yd, it, LR)
        got = eng.forward(xd, step=STEP, row0=ROW0)
        got = [t.clone() for t in (got if isinstance(got, (list, tuple)) else [got])]
        fresh, _, _, _ = _small(family, B=130, T=10)
        for e, m in zip(getattr(fresh, 'stages', [fresh]), getattr(eng, 'stages', [eng])):
            e.set_flat(m.get_flat())
        ref = fresh.forward(xd, step=STEP, row0=ROW0)
        for a, b in zip(got, ref if isinstance(ref, (list, tuple)) else [ref]):
            assert torch.equal(a, b), it
        _close(fresh)
    eng.set_weights(P)                                       # and back through set_weights
    fresh, _, _, _ = _small(family, B=130, T=10)
    a, b = eng.forward(xd, step=STEP, row0=ROW0), fresh.forward(xd, step=STEP, row0=ROW0)
    for u, v in zip(a if isinstance(a, (list, tuple)) else [a], b if isinstance(b, (list, tuple)) else [b]):
        assert torch.equal(u, v)
    _close(eng)
    _close(fresh)


# ---- 4. data parallel ---------------------------------------------------------------------------------------------------
SHARD_TOL = 1e-5         # worst measured 3.3e-6


@pytest.mark.parametrize('family', ['gru', 'uq-gru', 'uq-chain2'])
def test_tf32_row_shards_sum_to_the_whole_batch(family):
    """Shards of the batch at their global row offsets, with the whole batch's denominators, sum to the whole batch's
    gradients (fp32 sums in another order: within SHARD_TOL of the largest entry)."""
    B = 300
    eng, _, xd, yd = _small(family, B=B, T=16)
    S = FAMS[family][2]
    uq = FAMS[family][1]
    if S == 1:
        denom = eng.mask_count_uq(yd[0]) if uq else eng.mask_count(yd[0])
    else:
        denom = eng.mask_count(yd)
    _gpu_backward(family, eng, xd, yd, STEP, ROW0, denom=denom)
    whole = [g.copy() for g in eng.grads_list()]
    acc = [np.zeros_like(g, dtype=np.float64) for g in whole]
    for a, b in [(0, 129), (129, 200), (200, B)]:
        _gpu_backward(family, eng, xd[a:b].contiguous(), [y[a:b].contiguous() for y in yd], STEP, ROW0 + a,
                      denom=denom)
        for s, g in zip(acc, eng.grads_list()):
            s += g
    worst = max(rel_err(s, w) for s, w in zip(acc, whole))
    print('tf32 %s shard sums: %.2e (bound %.0e)' % (family, worst, SHARD_TOL))
    assert worst < SHARD_TOL
    _close(eng)


# ---- 5. the model object and the CLI ------------------------------------------------------------------------------------
def _cli_env(tmp_path):
    from lfm_quant_b200.scripts.synthetic import write_open_dataset, write_system_test_conf
    os.environ.setdefault('LFM_QUANT_ROOT', str(tmp_path))
    write_open_dataset(str(tmp_path / 'datasets' / 'open-dataset.dat'), n_keys=30, n_months=420, seed=9)
    conf = str(tmp_path / 'config' / 'system-test.conf')
    write_system_test_conf(conf, str(tmp_path / 'datasets'), str(tmp_path / 'experiments'))
    return conf


@pytest.mark.parametrize('extra', [['--rnn_cell', 'gru', '--model_dir', 'gru-tf32'],
                                   ['--nn_type', 'RNNUqRangeEstimate', '--UQ=True', '--forecast_steps', '2',
                                    '--forecast_steps_weights', '1.0-0.5', '--model_dir', 'uq-s2-tf32']],
                         ids=['gru', 'uq-s2'])
def test_cli_trains_at_tf32_and_predicts_at_fp32(tmp_path, extra):
    import pandas as pd
    from lfm_quant_b200.scripts import configs
    from lfm_quant_b200.scripts import lfm_quant as cli
    conf = _cli_env(tmp_path)
    configs.reset()
    try:
        assert np.isfinite(cli.main(['--config=' + conf, '--train=True', '--precision', 'tf32'] + extra))
        configs.reset()
        df = cli.main(['--config=' + conf, '--train=False', '--precision', 'fp32'] + extra)
    finally:
        configs.reset()
    mdir = tmp_path / 'experiments' / extra[-1]
    out = pd.read_csv(mdir / 'pred' / 'preds.dat', sep=' ', dtype={'gvkey': str})
    assert len(out) == len(df) > 100
    assert np.isfinite(out['norm_preds_1']).all()


TRAJ_TOL = 1e-3          # worst measured 3.5e-4


@pytest.mark.parametrize('uq', [False, True])
def test_tf32_loss_trajectory_follows_fp32(uq):
    """50 train steps of the same model at fp32 and at tf32 on the same batches: the per-step losses stay within
    TRAJ_TOL (relative) of each other."""
    from lfm_quant_b200.scripts import base_config, configs
    from lfm_quant_b200.scripts.models.point_estimate.rnn_point_estimate import NativeForecaster
    B, T, F, O = 256, 20, 32, 16
    models = []
    for prec in ('fp32', 'tf32'):
        configs.reset()
        args = ['--train=True', '--batch_size', str(B), '--precision', prec, '--num_hidden', '128', '--num_layers', '2',
                '--dropout', '0.1', '--rnn_cell', 'gru']
        if uq:
            args += ['--nn_type', 'RNNUqRangeEstimate', '--UQ=True']
        cfg = base_config.get_configs(args)
        models.append(NativeForecaster(cfg, T, F, O, 3, uq=uq))
    configs.reset()
    rng = np.random.RandomState(4)
    worst = 0.0
    for it in range(50):
        x = torch.from_numpy(rng.normal(size=(B, T, F)).astype(np.float32)).cuda()
        y = [torch.from_numpy((0.5 * rng.normal(size=(B, T, O))).astype(np.float32)).cuda()]
        a = models[0].train_step(x, y, 0.6, it).cpu().numpy()
        b = models[1].train_step(x, y, 0.6, it).cpu().numpy()
        worst = max(worst, float(np.max(np.abs(a - b) / np.maximum(np.abs(a), 1e-12))))
    print('tf32 %s loss trajectory vs fp32: %.2e (bound %.0e)' % ('uq' if uq else 'point', worst, TRAJ_TOL))
    assert worst < TRAJ_TOL
    for m in models:
        m.engine.close()
