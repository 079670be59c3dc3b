"""fp32 training of the models that train on the SIMT kernels only -- the GRU point estimate, RNNUqRangeEstimate (LSTM
and GRU cells) and multi-step forecasts (point and UQ chains) -- against the fp64 oracle at the shapes they train at.

The SIMT kernels change their code path with the shape, and these tests pick shapes that reach each branch:
- split-K in `sgemm` (K = B*T >= 2048 with few output tiles): every weight gradient, GRU's ragged 3H column tiles, the
  variance head's dWv and each chain stage's head;
- the multi-block `colsum` (B*T >= 128): GRU's two bias rows, the variance bias;
- the thread layouts of `bn_dropout_bwd` (nq = H/4 quads by RL = 256/nq rows): RL = 256 (H=4), a partial warp (H=132),
  RL = 1 with nq = 255 (H=1020) and the largest H (1024);
- the chain glue (`chain_next_input_kernel`, `chain_scatter_dx_kernel`) at the product batch size, B=4096.

1. Shape sweep: the oracle runs the whole problem: forward, loss, every gradient tensor, then three Adadelta steps with
   clip_by_global_norm and MaxNorm clipping.
2. Product scale (B=4096, T=48, F=32, O=16; H=256, L=1 and H=512, L=2, both dropouts).  Point models: one probe row
   has targets, every other row is masked, so the full-batch backward is that row's gradient with the full batch's
   denominators (losses.py:72; the oracle takes batch_global=B).  UQ models cannot mask a row (the loss turns NaN, as in
   the reference), so the backward runs on row slices with the full batch's counts as the denominators: with nothing
   masked every denominator scales by n/B, and (B/n) x a slice's gradients equals the oracle's on that slice alone.
   The slices that tile the batch sum to the full-batch gradient.
3. The variance floor var = max(softplus(a), 1e-6) and its gradient mask (tf.maximum) on every path that has it: the
   fp32 training handles and the forward-only bf16 / bf16x3 UQ handles, single-step and chains.

Bounds are the fp32 ones (1e-4 relative to the tensor's largest entry on outputs, losses and gradients, 5e-4 on weights
after steps); every test prints its worst value next to the bound.
"""
import time

import numpy as np
import pytest
import torch

import lfm_oracle as orc
import uq_chain_oracle as uco
from util import PATTERNS, probe_rows, rel_err, target_row

pytestmark = pytest.mark.gpu

TOL = 1e-4               # outputs, losses, gradients
W_TOL = 5e-4             # weights after optimizer steps
SUM_TOL = 1e-5           # full-batch gradient vs the sum of row slices (fp32 sums in another order)
BF16_TOL = 3e-2
STEP, ROW0 = 3, 5000
DROP = dict(dropout=0.2, recurrent_dropout=0.1, seed=521)
WEIGHTS = [1.0, 0.5, 0.25]

# name: (cell, uq, forecast steps)
FAMILIES = {
    'gru': ('gru', False, 1),
    'uq-lstm': ('lstm', True, 1),
    'uq-gru': ('gru', True, 1),
    'chain2': ('lstm', False, 2),
    'chain3': ('gru', False, 3),
    'uq-chain2': ('lstm', True, 2),
}


@pytest.fixture(scope='module', autouse=True)
def _wall_time():
    t0 = time.time()
    yield
    print('\ntest_gpu_fp32_models.py: %.1f s wall time' % (time.time() - t0))


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()


def _loss_kw(O):
    return dict(target_idx=O - 1, target_lambda=0.5, rnn_lambda=0.7)


class _Worst(object):
    """Asserts each measured value against its bound and keeps the worst per kind for the report."""

    def __init__(self, title):
        self.title = title
        self.worst = {}

    def check(self, kind, err, bound, where):
        w = self.worst.get(kind, (0.0, bound))
        self.worst[kind] = (max(w[0], err), bound)
        assert err < bound, (self.title, kind, where, err, bound)

    def report(self):
        print('%s: %s' % (self.title, ', '.join('%s %.2e (bound %.0e)' % (k, w, b)
                                                for k, (w, b) in self.worst.items())))


def _scalar_err(g, r):
    return abs(float(g) - float(r)) / max(abs(float(r)), 1e-30)


# ---- one interface over the four kinds of model -------------------------------------------------------------------
def _problem(family, B, T, F, O, H, L, seed, init_scale=0.5):
    cell, uq, S = FAMILIES[family]
    rng = np.random.RandomState(seed)
    if S == 1:
        P = orc.init_params(L, F, O, H, init_scale=init_scale, seed=seed + 1, dtype=np.float64, rnn_cell=cell, uq=uq)
    elif uq:
        P = uco.init_params(L, F, O, H, S, init_scale=init_scale, seed=seed + 1, dtype=np.float64, rnn_cell=cell)
    else:
        P = orc.init_forecast_params(L, F, O, H, S, init_scale=init_scale, seed=seed + 1, dtype=np.float64,
                                     rnn_cell=cell)
    P = [(p + rng.normal(size=p.shape) * 0.05).astype(np.float32).astype(np.float64) for p in P]
    x = rng.normal(size=(B, T, F)).astype(np.float32)
    ys = [rng.normal(size=(B, T, O)).astype(np.float32) for _ in range(S)]
    if not uq and B > 1 and T > 2:            # zero-padded steps: loss mask 0 (a uq loss would be NaN)
        for y in ys:
            y[0, :2, :] = 0.0
            y[B - 1, 0, :] = 0.0
    return P, x, ys


def _engine(family, B, T, F, O, H, L, **kw):
    from lfm_quant_b200.engine import ForecastChainEngine, ForecasterEngine
    cell, uq, S = FAMILIES[family]
    shape = dict(max_batch=B, seq_len=T, n_inputs=F, n_outputs=O, num_hidden=H, num_layers=L, rnn_cell=cell, uq=uq)
    if S == 1:
        return ForecasterEngine(**shape, **kw)
    return ForecastChainEngine(forecast_steps=S, weights=WEIGHTS[:S], **shape, **kw)


def _names(eng):
    if hasattr(eng, 'stages'):
        return [n for _, n, _, _, tr in eng.specs if tr]
    return [s[0] for s in eng.trainable_specs]


def _gpu_forward(eng, xd, step, row0):
    """[pred] / [pred, var] / [pred_1 .. pred_S] / [pred_1, var_1, ..]: the oracle's order."""
    out = eng.forward(xd, step=step, row0=row0)
    out = list(out) if isinstance(out, (list, tuple)) else [out]
    return [o.cpu().numpy() for o in out]


def _gpu_backward(family, eng, xd, yds, step, row0, denom=None):
    """Backward; returns {loss, mse} (point) or {uq_loss, uq_loss_last_tar, mse} (uq).  denom: the full batch's counts
    (the uq models' slices)."""
    _, uq, S = FAMILIES[family]
    if S == 1:
        eng.backward(xd, yds[0], step=step, row0=row0, denom=denom)
        t = eng.grads[eng.n_trainable:eng.n_trainable + 5].cpu().numpy()
        return [t[0], t[4], t[1]] if uq else [t[0], t[1]]
    if denom is None:
        return list(eng.backward(xd, yds, step=step, row0=row0).cpu().numpy())
    return list(eng.backward_dp(xd, yds, denom, step=step, row0=row0).cpu().numpy())


def _oracle_forward(family, P, x, L, step, row0):
    cell, uq, S = FAMILIES[family]
    x = x.astype(np.float64)
    kw = dict(num_layers=L, rnn_cell=cell, step=step, row0=row0, **DROP)
    if S == 1 and not uq:
        p, fc = orc.forward(P, x, training=True, **kw)
        return [p], fc
    if S == 1:
        p, v, fc = orc.forward_uq(P, x, **kw)
        return [p, v], fc
    if not uq:
        ps, fc = orc.forward_forecast(P, x, forecast_steps=S, training=True, **kw)
        return ps, fc
    ps, vs, fc = uco.forward(P, x, forecast_steps=S, **kw)
    return [t for pv in zip(ps, vs) for t in pv], fc


def _oracle_loss_backward(family, ys, outs, fc, L, lkw, batch_global=None):
    """The scalars _gpu_backward returns and the gradients in trainable-variable order."""
    cell, uq, S = FAMILIES[family]
    ys = [y.astype(np.float64) for y in ys]
    if S == 1 and not uq:
        loss, mse, dpred, _ = orc.loss_point_estimate(ys[0], outs[0], batch_global=batch_global, **lkw)
        return [loss, mse], orc.backward(dpred, fc, num_layers=L, rnn_cell=cell)
    if S == 1:
        loss, uq0, mse, dp, dv = orc.loss_uq_estimate(ys[0], outs[0], outs[1], **lkw)
        return [loss, uq0, mse], orc.backward_uq(dp, dv, fc, num_layers=L, rnn_cell=cell)
    if not uq:
        loss, mse, dpreds = orc.loss_forecast(ys, outs, WEIGHTS[:S], batch_global=batch_global, **lkw)
        return [loss, mse], orc.backward_forecast(dpreds, fc, rnn_cell=cell)
    loss, uq0, mse, dpreds, dvars = uco.loss(ys, outs[0::2], outs[1::2], WEIGHTS[:S], **lkw)
    return [loss, uq0, mse], uco.backward(dpreds, dvars, fc, rnn_cell=cell)


def _oracle_train_step(family, p, slots, x, ys, it, L, lkw, lr, clip, max_norm):
    """One Train step (train.py:178-225) of the family's graph at row0 = 0, step = it; returns the new weights and what
    the engine's train_step returns: {loss, mse} (point) or {uq_loss_last_tar, mse} (uq)."""
    cell, uq, S = FAMILIES[family]
    x = x.astype(np.float64)
    ys = [y.astype(np.float64) for y in ys]
    cfg = dict(num_layers=L, rnn_cell=cell, train=True, uq=uq, optimizer='Adadelta', max_grad_norm=clip,
               max_norm=max_norm, **lkw, **DROP)
    if S == 1:
        r = orc.train_step(p, slots, x, ys[0], it, cfg, lr=lr)
        return r[0], [r[5] if uq else r[2], r[1]]
    if uq:
        cfg.update(forecast_steps=S, forecast_steps_weights=WEIGHTS[:S])
        new, mse, _, _, _, uq_last = uco.train_step(p, slots, x, ys, it, cfg, lr=lr)
        return new, [uq_last, mse]
    rp, fc = orc.forward_forecast(p, x, num_layers=L, forecast_steps=S, training=True, rnn_cell=cell, step=it, **DROP)
    loss, mse, dpreds = orc.loss_forecast(ys, rp, WEIGHTS[:S], **lkw)
    grads, _ = orc.clip_by_global_norm(orc.backward_forecast(dpreds, fc, rnn_cell=cell), clip)
    new = orc.optimizer_update('Adadelta', p, grads, slots, lr, it)
    for k in [5 * l for l in range(L)] + [5 * L + 2 + 7 * (s - 1) for s in range(1, S)]:
        new[k] = orc.max_norm_constraint(new[k], max_norm)
    return new, [loss, mse]


def _close(eng):
    eng.close()
    del eng
    torch.cuda.empty_cache()


# ---- 1. shape sweep ----------------------------------------------------------------------------------------------------
# name: (B, T, F, O, H, L).  F = 33 and O in {1, 17}: ragged input and head widths, the chains' aux columns x0[:, :, O:]
# and their dx scatter with O < F.
SHAPES = {
    'splitk-h64': (64, 48, 33, 17, 64, 1),      # B*T = 3072: split-K on every weight gradient, 48-block colsum
    'splitk-h132': (43, 48, 33, 1, 132, 2),     # B*T = 2064; 3H = 396, 4H = 528: ragged 64-wide column tiles;
                                                # bn_dropout_bwd nq = 33, RL = 7 (a partial warp)
    'h4': (6, 5, 33, 1, 4, 1),                  # bn_dropout_bwd nq = 1, RL = 256
    'h1020': (3, 4, 33, 17, 1020, 1),           # nq = 255, RL = 1
    'h1024': (2, 3, 20, 17, 1024, 2),           # the largest H lfmq_config accepts: nq = 256, RL = 1
    'deep': (8, 48, 16, 4, 32, 3),              # T=48, three layers
}
LR, CLIP, N_STEPS = 0.6, 0.5, 3


@pytest.mark.parametrize('shape', list(SHAPES))
@pytest.mark.parametrize('family', list(FAMILIES))
def test_fp32_training_matches_oracle(family, shape):
    """Forward, loss, every gradient tensor and three Adadelta steps with clip_by_global_norm and MaxNorm, both
    dropouts on, against the oracle on the whole problem."""
    B, T, F, O, H, L = SHAPES[shape]
    lkw = _loss_kw(O)
    P, x, ys = _problem(family, B, T, F, O, H, L, seed=sum(map(ord, family + shape)))
    max_norm = 0.9 * float(np.linalg.norm(P[0], axis=0).max())      # binds on the first kernel at least
    eng = _engine(family, B, T, F, O, H, L, train=True, optimizer='Adadelta', max_grad_norm=CLIP, max_norm=max_norm,
                  **lkw, **DROP)
    eng.set_weights(P)
    chk = _Worst('fp32 %s %s B=%d T=%d F=%d O=%d H=%d L=%d' % (family, shape, B, T, F, O, H, L))
    xd, yd = _cuda(x), [_cuda(y) for y in ys]
    outs, fc = _oracle_forward(family, P, x, L, STEP, ROW0)
    for i, (g, r) in enumerate(zip(_gpu_forward(eng, xd, STEP, ROW0), outs)):
        chk.check('output', rel_err(g, r), TOL, i)
    ref_s, ref_g = _oracle_loss_backward(family, ys, outs, fc, L, lkw)
    for i, (g, r) in enumerate(zip(_gpu_backward(family, eng, xd, yd, STEP, ROW0), ref_s)):
        chk.check('loss', _scalar_err(g, r), TOL, i)
    names = _names(eng)
    assert len(names) == len(ref_g)
    for name, g, r in zip(names, eng.grads_list(), ref_g):
        assert g.shape == r.shape, name
        chk.check('gradient', rel_err(g, r), TOL, name)
    p = [q.copy() for q in P]
    slots = orc.zero_slots('Adadelta', p)
    for it in range(N_STEPS):
        out = eng.train_step(xd, yd[0] if FAMILIES[family][2] == 1 else yd, it, LR).cpu().numpy()
        p, ref = _oracle_train_step(family, p, slots, x, ys, it, L, lkw, LR, CLIP, max_norm)
        for i, (g, r) in enumerate(zip(out, ref)):
            chk.check('step loss', _scalar_err(g, r), TOL, (it, i))
    got = eng.get_weights()
    for name, w, r in zip(names, got, p):
        chk.check('weights', rel_err(w, r), W_TOL, name)
    assert np.linalg.norm(got[0], axis=0).max() <= max_norm * (1 + 1e-5)
    chk.report()
    _close(eng)


# ---- 2. product scale --------------------------------------------------------------------------------------------------
BIG_B, BIG_T, BIG_F, BIG_O = 4096, 48, 32, 16
BIG = [(256, 1), (512, 2)]
BLOCKS = [(0, 16), (2040, 2056), (BIG_B - 16, BIG_B)]            # full-batch forward rows checked against the oracle
# rows 0 and B-1, both sides of 64 and of every 1024th row (64-row sgemm tiles), rows past 2048
PROBES = probe_rows(BIG_B, 1024, extra=(63, 64))
# uq slices: at 0, across a 64-row boundary, across and past row 2048, a ragged end
SLICES = [(0, 24), (50, 78), (2036, 2060), (3001, 3025), (BIG_B - 21, BIG_B)]
TILES = [(0, 1000), (1000, 2100), (2100, BIG_B)]


def _check_blocks(family, eng, xd, x, P, L, chk):
    full = _gpu_forward(eng, xd, STEP, ROW0)
    for o in full:
        assert np.isfinite(o).all()
    for a, b in BLOCKS:
        outs, _ = _oracle_forward(family, P, x[a:b], L, STEP, ROW0 + a)
        for i, (g, r) in enumerate(zip(full, outs)):
            chk.check('forward block', rel_err(g[a:b], r), TOL, ((a, b), i))


@pytest.mark.parametrize('H,L', BIG)
@pytest.mark.parametrize('family', ['gru', 'chain2'])
def test_point_models_row_probes_at_product_scale(family, H, L):
    """One probe row with targets, every other row masked: the full-batch backward equals the oracle's gradients of
    that row alone with batch_global = B.  Chain: the probe row's feedback into the trunk's dLoss/dpred as well."""
    B, T, F, O = BIG_B, BIG_T, BIG_F, BIG_O
    S = FAMILIES[family][2]
    lkw = _loss_kw(O)
    P, x, _ = _problem(family, B, T, F, O, H, L, seed=7 + H + L, init_scale=0.3)
    eng = _engine(family, B, T, F, O, H, L, train=True, **lkw, **DROP)
    eng.set_weights(P)
    names = _names(eng)
    chk = _Worst('row probes %s B=%d T=%d H=%d L=%d, %d rows' % (family, B, T, H, L, len(PROBES)))
    xd = _cuda(x)
    _check_blocks(family, eng, xd, x, P, L, chk)
    yd = [torch.zeros(B, T, O, dtype=torch.float32, device='cuda') for _ in range(S)]
    rng = np.random.RandomState(H + L)
    for i, r in enumerate(PROBES):
        pattern = PATTERNS[i % len(PATTERNS)]
        y_rows = [target_row(rng, T, O, pattern) for _ in range(S)]
        for y, yr in zip(yd, y_rows):
            y[r] = _cuda(yr)
        got_s = _gpu_backward(family, eng, xd, yd, STEP, ROW0)
        grads = eng.grads_list()
        for y in yd:
            y[r] = 0.0
        outs, fc = _oracle_forward(family, P, x[r:r + 1], L, STEP, ROW0 + r)
        ref_s, ref_g = _oracle_loss_backward(family, [yr[None] for yr in y_rows], outs, fc, L, lkw, batch_global=B)
        where = (r, pattern)
        chk.check('loss', _scalar_err(got_s[0], ref_s[0]), TOL, where)
        if pattern == 't0':                     # the last step is masked
            assert got_s[1] == 0.0 and ref_s[1] == 0.0, where
        else:
            # mse of one row is sum_s w_s d_s^2 / B with d_s = pred_s - y_s at the target column of the last step; pred
            # and y may nearly cancel, so d is held to the forward tolerance: |d^2 - d'^2| <= |d - d'| (|d| + |d'|)
            mp = max(np.abs(o).max() for o in outs)
            my = max(np.abs(yr).max() for yr in y_rows)
            bound = 2 * TOL * mp * (mp + my) * sum(WEIGHTS[:S]) / B
            chk.check('mse / forward bound', abs(float(got_s[1]) - float(ref_s[1])) / bound, 1.0, where)
        for name, g, rf in zip(names, grads, ref_g):
            assert np.isfinite(g).all(), where + (name,)
            if pattern == 't0' and name.endswith('recurrent_kernel'):
                assert not np.any(g), where + (name, 'dU of a row with a target at t=0 only is exactly zero')
            if not np.any(rf):
                assert not np.any(g), where + (name,)
                continue
            chk.check('gradient', rel_err(g, rf), TOL, where + (name,))
    chk.report()
    _close(eng)


def _stage_grads(eng):
    return [e.grads[:e.n_trainable].clone() for e in getattr(eng, 'stages', [eng])]


@pytest.mark.parametrize('H,L', BIG)
@pytest.mark.parametrize('family', ['uq-lstm', 'uq-gru', 'uq-chain2'])
def test_uq_models_row_slices_at_product_scale(family, H, L):
    """Nothing masked: a slice's backward with the full batch's counts, scaled by B/n, equals the oracle's gradients of
    that slice alone; the slices that tile the batch sum to the full-batch gradient."""
    B, T, F, O = BIG_B, BIG_T, BIG_F, BIG_O
    S = FAMILIES[family][2]
    lkw = _loss_kw(O)
    P, x, ys = _problem(family, B, T, F, O, H, L, seed=11 + H + L, init_scale=0.3)
    eng = _engine(family, B, T, F, O, H, L, train=True, **lkw, **DROP)
    eng.set_weights(P)
    names = _names(eng)
    chk = _Worst('uq slices %s B=%d T=%d H=%d L=%d' % (family, B, T, H, L))
    xd, yd = _cuda(x), [_cuda(y) for y in ys]
    _check_blocks(family, eng, xd, x, P, L, chk)
    counts = eng.mask_count_uq(yd[0]) if S == 1 else eng.mask_count(yd)
    assert np.array_equal(counts.cpu().numpy().reshape(S, 3), np.tile([B, B * T, B], (S, 1)))
    for a, b in SLICES:
        n = b - a
        got_s = _gpu_backward(family, eng, xd[a:b].contiguous(), [y[a:b].contiguous() for y in yd], STEP, ROW0 + a,
                              denom=counts)
        grads = eng.grads_list()
        outs, fc = _oracle_forward(family, P, x[a:b], L, STEP, ROW0 + a)
        ref_s, ref_g = _oracle_loss_backward(family, [y[a:b] for y in ys], outs, fc, L, lkw)
        scale = B / n
        for i, (g, r) in enumerate(zip(got_s, ref_s)):
            chk.check('loss', _scalar_err(scale * g, r), TOL, ((a, b), i))
        for name, g, r in zip(names, grads, ref_g):
            chk.check('gradient', rel_err(scale * g.astype(np.float64), r), TOL, ((a, b), name))
    _gpu_backward(family, eng, xd, yd, STEP, ROW0)
    full = _stage_grads(eng)
    acc = [torch.zeros_like(g) for g in full]
    for a, b in TILES:
        _gpu_backward(family, eng, xd[a:b].contiguous(), [y[a:b].contiguous() for y in yd], STEP, ROW0 + a,
                      denom=counts)
        for s, g in enumerate(_stage_grads(eng)):
            acc[s] += g
    for s, (g, f) in enumerate(zip(acc, full)):
        assert torch.isfinite(f).all() and float(f.abs().max()) > 0
        chk.check('tile sum', rel_err(g.cpu().numpy(), f.cpu().numpy()), SUM_TOL, s)
    chk.report()
    _close(eng)


# ---- 3. the variance floor ---------------------------------------------------------------------------------------------
# Column DEEP: bv = -30, so a < -20 and var is exactly 1e-6 everywhere; its target head is zero with bias C_DEEP and its
# targets are C_DEEP, so the column's loss term is log(1e-6) and its variance gradient is blocked by the floor: dWv[:, DEEP]
# and dbv[DEEP] are exactly zero.  Column EDGE reads one hidden unit J of the last layer: Wv[:, EDGE] = e_J, bv = -14.5,
# and that unit's BatchNormalization (gamma 0.5, beta 3) keeps its output in (3.1, 4.4) after the dropout scaling unless
# dropout zeroes it.  So a = bv = -14.5 (floored: softplus < 1e-6) where dropout dropped unit J and -11.4 < a < -10.1 (not
# floored) elsewhere, both far from the threshold; its target head is zero as well, so the column contributes through
# the variance only.
DEEP, EDGE, J = 0, 1, 3
C_DEEP, C_EDGE = 0.75, -0.5
FLOOR_A = np.log(np.expm1(orc.VAR_FLOOR))        # softplus(a) > 1e-6 <=> a > FLOOR_A (-13.8155)
FLOOR_SHAPE = (130, 8, 12, 6, 128, 2)           # B, T, F, O, H, L


def _heads(family, L):
    """(Wt, bt, Wv, bv, gamma, beta of the layer below) indices of every stage's heads."""
    S = FAMILIES[family][2]
    out = [(5 * L, 5 * L + 1, 5 * L + 2, 5 * L + 3, 5 * (L - 1) + 3, 5 * (L - 1) + 4)]
    n0 = 5 * L + 4
    for s in range(1, S):
        k = n0 + 9 * (s - 1)
        out.append((k + 5, k + 6, k + 7, k + 8, k + 3, k + 4))
    return out


def _floor_problem(family):
    B, T, F, O, H, L = FLOOR_SHAPE
    P, x, ys = _problem(family, B, T, F, O, H, L, seed=23)
    for it, ib, iv, ibv, ig, ibeta in _heads(family, L):
        P[iv][:, DEEP] *= 0.1
        P[ibv][DEEP] = -30.0
        P[iv][:, EDGE] = 0.0
        P[iv][J, EDGE] = 1.0
        P[ibv][EDGE] = -14.5
        P[ig][J], P[ibeta][J] = 0.5, 3.0
        P[it][:, [DEEP, EDGE]] = 0.0
        P[ib][DEEP], P[ib][EDGE] = C_DEEP, C_EDGE
    for y in ys:
        y[..., DEEP] = C_DEEP
        y[..., EDGE] = C_EDGE
    P = [p.astype(np.float32).astype(np.float64) for p in P]
    outs, fc = _oracle_forward(family, P, x, L, STEP, ROW0)
    caches = [fc] if FAMILIES[family][2] == 1 else fc[0]
    pre = [c[4] for c in caches]                # every stage's variance pre-activation a
    for a in pre:
        assert (a[..., DEEP] < -20).all()
        edge = a[..., EDGE]
        assert (edge <= FLOOR_A).any() and (edge > FLOOR_A).any()
        assert (np.abs(edge - FLOOR_A) > 1e-3 * abs(FLOOR_A)).all()       # no flip by rounding
    return P, x, ys, outs, fc, pre


@pytest.mark.parametrize('family', ['uq-lstm', 'uq-gru', 'uq-chain2'])
def test_variance_floor_fp32_training(family):
    """Forward, loss and gradients with columns below, across and above the floor; the blocked columns' variance-head
    gradients are exactly zero."""
    B, T, F, O, H, L = FLOOR_SHAPE
    lkw = _loss_kw(O)
    P, x, ys, outs, fc, pre = _floor_problem(family)
    eng = _engine(family, B, T, F, O, H, L, train=True, **lkw, **DROP)
    eng.set_weights(P)
    chk = _Worst('variance floor fp32 %s' % family)
    xd, yd = _cuda(x), [_cuda(y) for y in ys]
    got = _gpu_forward(eng, xd, STEP, ROW0)
    for i, (g, r) in enumerate(zip(got, outs)):
        chk.check('output', rel_err(g, r), TOL, i)
    for s, a in enumerate(pre):
        var = got[2 * s + 1]
        assert (var[a < -20] == np.float32(orc.VAR_FLOOR)).all(), s
        assert (var[..., EDGE][a[..., EDGE] <= FLOOR_A] == np.float32(orc.VAR_FLOOR)).all(), s
    ref_s, ref_g = _oracle_loss_backward(family, ys, outs, fc, L, lkw)
    for i, (g, r) in enumerate(zip(_gpu_backward(family, eng, xd, yd, STEP, ROW0), ref_s)):
        chk.check('loss', _scalar_err(g, r), TOL, i)
    names = _names(eng)
    grads = dict(zip(names, eng.grads_list()))
    for name, r in zip(names, ref_g):
        chk.check('gradient', rel_err(grads[name], r), TOL, name)
    for name in names:
        if 'OUTPUT_VARIANCE' in name:
            g = grads[name]
            col = g[:, DEEP] if g.ndim == 2 else g[DEEP]
            assert not np.any(col), (name, 'the floored column passes no gradient')
            edge = g[:, EDGE] if g.ndim == 2 else g[EDGE]
            assert np.any(edge), (name, 'the straddling column has unfloored elements')
    chk.report()
    _close(eng)


@pytest.mark.parametrize('precision', ['bf16', 'bf16x3'])
@pytest.mark.parametrize('family', ['uq-lstm', 'uq-gru', 'uq-chain2'])
def test_variance_floor_forward_on_tensor_cores(family, precision):
    """Forward-only bf16 / bf16x3 handles: var is exactly 1e-6 wherever the oracle's a < -20, every output within the
    path's bound."""
    B, T, F, O, H, L = FLOOR_SHAPE
    P, x, _, outs, _, pre = _floor_problem(family)
    eng = _engine(family, B, T, F, O, H, L, precision=precision, train=False, forward_only=True, **_loss_kw(O),
                  **DROP)
    eng.set_weights(P)
    tol = BF16_TOL if precision == 'bf16' else TOL
    chk = _Worst('variance floor %s %s' % (precision, family))
    got = _gpu_forward(eng, _cuda(x), STEP, ROW0)
    for i, (g, r) in enumerate(zip(got, outs)):
        chk.check('output', rel_err(g, r), tol, i)
    for s, a in enumerate(pre):
        assert (got[2 * s + 1][a < -20] == np.float32(orc.VAR_FLOOR)).all(), s
    chk.report()
    _close(eng)
