"""The bf16 general path (rnn_tc.cu) at cfg3's batch size, on the schedules gen_run_trunk and gen_backward pick there.

cfg3 (B = 4096, T = 48, F = 32, O = 16, H = 512, L = 2, dropout 0.2) is 32 row tiles of 128 rows.  The figures below are
for 132 SMs (an H100 SXM); the tests derive them from the device's SM count.

* Forward recurrence: a layer's steps 1 .. T-1 run as one persistent launch when its nrt * 4H / 256 CTAs fit at once
  (one per SM), else as one launch per step chained by programmatic dependent launch.  At H = 512 that is 8 CTAs per tile:
  B = 4096 needs 256 and B = 2100 (17 tiles) 136, so both are stepped; H = 128, B = 4096 needs 64 and persists.
* Backward recurrence: from 16 row tiles on, the tiles are split into two chains (ceil(nrt / 2) and floor(nrt / 2)
  tiles) on two streams, each a persistent launch with its own grid-barrier counters when both fit at once (H / 128 CTAs
  per tile): B = 4096 runs chains of 16 and 16 tiles (128 CTAs at H = 512), B = 2100 chains of 9 and 8 tiles whose last
  tile has 52 rows, B <= 1920 one chain.
* The weight-gradient GEMMs sum over all T * Bp time-major rows, with their K-splits sized from that.

The other suites hold this path to the rounding oracle only at B <= 300 (at most 3 tiles: persistent forward, one
backward chain), and at T = 48 only at H = 192; at cfg3's batch nothing tighter than the fp64 bounds checks it.

1. The rounding oracle (tests/bf16_oracle.py, Plan('general')) at T = 16: B = 4096 and 2100 (H = 512, L = 2, both
   dropouts) and B = 4096 at H = 128, with BN moving statistics away from (0, 1) and a nonzero row0: predictions
   (closer to the rounding oracle than to the fp64 one by RATIO), loss, mse_0 and every gradient tensor within
   test_gpu_bf16_rounding.BOUNDS['general'] (CASE_BOUNDS below).  Each case's oracles are computed once.
2. The same cases on a handle whose device share admits no persistent launch (the schedule of ensemble members and
   hyper-parameter search), bit for bit against the default schedule.
3. cfg3 at T = 48 across launches: the state after train steps against a fresh handle, and one handle switching between
   two-chain, one-chain and two-tile batches against a fresh handle per call.
4. The cfg3 loss trajectory of the bf16 path against the fp32 path over 50 of bench.py's train steps.
"""
import time

import numpy as np
import pytest
import torch

import bf16_oracle as bo
import lfm_oracle as orc
from test_gpu_bf16_rounding import (D21, HEAD_TOL, LR, ROW0, STEP, _bn_kw, _bn_stats, _cuda, _flat_from, _kind,
                                    _loss_tail, _max_norm_that_clips, _Report)
from util import make_engine, make_problem, rel_err

pytestmark = pytest.mark.gpu

F, O = 32, 16
LKW = dict(target_idx=O - 1, target_lambda=0.5, rnn_lambda=0.7)


def _engine(B, T, H, L, **kw):
    return make_engine(B, T, F, O, H, L, target_idx=O - 1, precision='bf16', **kw)


def _names(eng):
    return [s[0] for s in eng.trainable_specs]


def _step(eng, xd, yd, step, row0):
    """(preds, gradients, loss tail, names) of a forward and a backward call on eng, and the launches of each call."""
    n0 = eng.launch_count
    preds = eng.forward(xd, step=step, row0=row0).cpu().numpy()
    n1 = eng.launch_count
    eng.backward(xd, yd, step=step, row0=row0)
    n2 = eng.launch_count
    return (preds, eng.grads_list(), _loss_tail(eng), _names(eng)), (n1 - n0, n2 - n1)


def _assert_same_step(got, want, where):
    """got / want: _step of two handles.  Predictions and every gradient but the head bias bit for bit: the recurrences'
    stores, the BN/Dropout backward and the weight-gradient GEMMs (OUTPUT_1/kernel included) run the same arithmetic in
    the same order whatever the schedule.  OUTPUT_1/bias and the loss are sums over rows through shared-memory atomics:
    within HEAD_TOL."""
    (p1, g1, t1, names), (p0, g0, t0, _) = got, want
    assert np.isfinite(p1).all(), where
    assert np.array_equal(p1, p0), where + ('pred', float(np.max(np.abs(p1 - p0))))
    for name, a, b in zip(names, g1, g0):
        assert np.isfinite(a).all(), where + (name,)
        if name == 'OUTPUT_1/bias':
            scale = max(float(np.max(np.abs(b))), 1e-30)
            assert float(np.max(np.abs(a - b))) <= HEAD_TOL * scale, where + (name, float(np.max(np.abs(a - b))) / scale)
        else:
            assert np.array_equal(a, b), where + (name, float(np.max(np.abs(a - b))))
    np.testing.assert_allclose(t1, t0, rtol=HEAD_TOL, err_msg=str(where))


# ---- 1. the rounding oracle at cfg3's batch size ----------------------------------------------------------------------
# (B, T, H, L, dropout keywords).  cfg3: stepped forward, two backward chains of 16 tiles.  b2100: 17 tiles, stepped
# forward (136 CTAs), backward chains of 9 and 8 tiles, a last tile of 52 rows.  h128-b4096: persistent forward over 32
# tiles, split backward.  T = 16: cfg3 at T = 48 would take three times the oracle time and memory (about 8.5 GB at
# T = 16); T = 48 at H = 512 is test_gpu_bf16_rounding.py's h512-l2-t48 (B = 256) and sections 3 and 4 here.
# The bounds are BOUNDS['general'] (set at B <= 300; its gradient bounds are within 1.5x of the worst values here, for
# the reason its comment gives).  The worst values over these cases, measured on an H100 80GB HBM3 (700 W power limit):
# pred 1.53e-3, loss 1.12e-5, mse_0 3.10e-5, kernel 1.17e-2, recurrent_kernel 1.45e-2, bias
# 1.46e-2 (these six at b2100), gamma 8.77e-3, beta 1.02e-2, OUTPUT_1/bias 1.03e-4 (these three at cfg3); OUTPUT_1/kernel
# 3.26e-4 (cfg3), 6.18e-5 (h128-b4096) and 1.09e-3 (b2100, CASE_BOUNDS).  The fp32 sums of the weight-gradient GEMMs over
# B T = 65536 rows do not make the gradients worse than at B <= 300 (worst there 1.54e-2, H=512 at T=48).
CASES = {
    'cfg3': (4096, 16, 512, 2, D21),
    'b2100': (2100, 16, 512, 2, D21),
    'h128-b4096': (4096, 16, 128, 1, {}),
}
# Looser than BOUNDS['general'], as test_gpu_bf16_rounding.CASE_BOUNDS is for h512-l2-t48: OUTPUT_1/kernel at H=512
# (the fp64 oracle is x1.4 further from the kernel than the emulated one).
CASE_BOUNDS = {'b2100': {'OUTPUT_1/kernel': 2e-3}}

_ORACLE = {}


def _oracle(case):
    """Inputs, BN statistics and both oracles' predictions, loss, mse_0 and gradients of a case, computed once."""
    if case not in _ORACLE:
        B, T, H, L, drop = CASES[case]
        params, x, y = make_problem(B, T, F, O, H, L, seed=21, init_scale=0.3)
        bn = _bn_stats(L, H, seed=19)
        x64, y64 = x.astype(np.float64), y.astype(np.float64)
        fkw = dict(num_layers=L, training=True, step=STEP, row0=ROW0, **_bn_kw(bn), **drop)
        t0 = time.time()
        res = dict(params=params, x=x, y=y, bn=bn)
        emu_p = bo.Plan('general')
        out, fc = bo.forward(emu_p, params, x64, **fkw)
        loss, mse, dpred, _ = orc.loss_point_estimate(y64, out, **LKW)
        res['emu'] = (out, loss, mse, bo.backward(emu_p, dpred, fc))
        del fc, dpred
        out, fc = orc.forward(params, x64, **fkw)
        loss, mse, dpred, _ = orc.loss_point_estimate(y64, out, **LKW)
        res['ref'] = (out, loss, mse, orc.backward(dpred, fc, num_layers=L))
        del fc, dpred
        print('oracles of %s (B=%d, T=%d, H=%d, L=%d): %.1f s' % (case, B, T, H, L, time.time() - t0))
        _ORACLE[case] = res
    return _ORACLE[case]


def _case_step(case, share=None):
    """_step of a fresh handle with the case's weights and inputs; `share`: its device share (num, den)."""
    B, T, H, L, drop = CASES[case]
    o = _oracle(case)
    eng = _engine(B, T, H, L, **drop)
    if share:
        eng.set_device_share(*share)
    eng.set_weights(o['params'], bn_stats=o['bn'])
    res = _step(eng, _cuda(o['x']), _cuda(o['y']), STEP, ROW0)
    eng.close()
    return res


@pytest.mark.parametrize('case', list(CASES))
def test_general_schedule_matches_emulated_oracle(case):
    o = _oracle(case)
    (preds, grads, tail, names), _ = _case_step(case)
    (ep, el, em, eg), (rp, rl, rm, rg) = o['emu'], o['ref']
    rep = _Report('general', case, CASE_BOUNDS.get(case))
    rep.check('pred', 'pred', preds, ep, rp, ratio=True)
    rep.check('loss', 'loss', tail[0], el, rl)
    rep.check('mse_0', 'mse_0', tail[1], em, rm)
    for name, g, ge, gr in zip(names, grads, eg, rg):
        rep.check(name, _kind(name), g, ge, gr)
    rep.done()


# ---- 2. persistent against stepped launches ---------------------------------------------------------------------------
def _persistent_launches_saved(B, T, H, L, sm):
    """Launches a forward and a backward call save on the whole device of `sm` SMs over one launch per step
    (gen_can_persist: a persistent launch replaces the T - 1 launches of steps 1 .. T-1, resp. T-2 .. 0, by one)."""
    nrt = (B + 127) // 128
    fwd = L * (T - 2) if nrt * (4 * H // 256) <= sm else 0
    chains = 2 if nrt >= 16 else 1
    n_a = (nrt + 1) // 2 if chains == 2 else nrt
    bwd = L * chains * (T - 2) if n_a * (H // 128) * chains <= sm else 0
    return fwd, fwd + bwd


@pytest.mark.parametrize('case', list(CASES))
def test_stepped_launches_bit_identical_to_default_schedule(case):
    """A device share of one SM's worth admits no persistent launch: every recurrence runs one launch per step.  That is
    the schedule of handles trained side by side (ensembles, hyper-parameter search)."""
    B, T, H, L, _ = CASES[case]
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    want, n_default = _case_step(case)
    got, n_stepped = _case_step(case, share=(1, sm))
    saved = _persistent_launches_saved(B, T, H, L, sm)
    print('%s: launches per forward / backward call: default %s, stepped %s' % (case, n_default, n_stepped))
    assert saved[1] > 0
    assert (n_stepped[0] - n_default[0], n_stepped[1] - n_default[1]) == saved, (n_default, n_stepped, saved)
    _assert_same_step(got, want, (case,))


# ---- 3. cfg3 at T = 48 across launches --------------------------------------------------------------------------------
@pytest.mark.parametrize('k', [1, 3])
def test_state_after_cfg3_train_steps(k):
    """After k Adadelta steps at cfg3 (clip 50, a MaxNorm that clips; each step's backward on two streams), the handle's
    forward and backward are those of a fresh handle loaded with the trained weights: the bf16 weight copies were
    repacked after the last update."""
    B, T, H, L = 4096, 48, 512, 2
    params, x, y = make_problem(B, T, F, O, H, L, seed=31, init_scale=0.3)
    bn = _bn_stats(L, H, seed=19)
    kw = dict(optimizer='Adadelta', max_grad_norm=50.0, max_norm=_max_norm_that_clips(params, L), **D21)
    eng = _engine(B, T, H, L, **kw)
    eng.set_weights(params, bn_stats=bn)
    xd, yd = _cuda(x), _cuda(y)
    for it in range(k):
        eng.train_step(xd, yd, it, LR)
    got, _ = _step(eng, xd, yd, k, ROW0)
    trained = eng.get_weights(trainable_only=False)
    assert max(rel_err(w, p) for w, p in zip(eng.get_weights(), params)) > 1e-4    # the steps moved the weights
    eng.close()
    fresh = _engine(B, T, H, L, **kw)
    fresh.set_flat(_flat_from(fresh, trained))
    want, _ = _step(fresh, xd, yd, k, ROW0)
    fresh.close()
    _assert_same_step(got, want, ('k=%d' % k,))


def test_one_handle_across_batch_sizes():
    """One handle (max_batch 4224, H = 512, L = 2, T = 16) runs B = 4096 (two backward chains), 1920 (15 tiles, one
    chain), 4096, 2100 (chains of 9 and 8) and 129 (two tiles, the second of one row) in turn; each call computes what a
    fresh handle computes making that one call.  The calls reuse the side stream and the grid-barrier counters, and the
    smaller batches zero the dz rows of the tiles they do not launch."""
    MB, T, H, L = 4224, 16, 512, 2
    params, x, y = make_problem(MB, T, F, O, H, L, seed=33, init_scale=0.3)
    bn = _bn_stats(L, H, seed=19)
    eng = _engine(MB, T, H, L, **D21)
    eng.set_weights(params, bn_stats=bn)
    for i, B in enumerate([4096, 1920, 4096, 2100, 129]):
        xd, yd = _cuda(x[:B]), _cuda(y[:B])
        got, _ = _step(eng, xd, yd, i, ROW0)
        fresh = _engine(MB, T, H, L, **D21)
        fresh.set_weights(params, bn_stats=bn)
        want, _ = _step(fresh, xd, yd, i, ROW0)
        fresh.close()
        _assert_same_step(got, want, ('call %d' % i, 'B=%d' % B))
    eng.close()


# ---- 4. the cfg3 loss trajectory against fp32 -------------------------------------------------------------------------
# bf16 against fp32 {loss, mse_0} at every one of 50 steps, relative: 1.5x the worst value measured on an H100 80GB HBM3
# (700 W power limit), rounded up to one significant digit: worst over four runs 2.44e-4 (mse_0; loss 1.48e-4), at
# step 15.  It varies from run to run (2.16e-4 in one), as the loss and head-bias sums go through fp32 atomics.
TRAJ_STEPS, TRAJ_BOUND = 50, 4e-4


def test_cfg3_bf16_loss_trajectory_tracks_fp32_on_bench_batches():
    """50 train steps of bench.py's cfg3 workload (B = 4096, T = 48, H = 512, L = 2, dropout 0.2, 4 rotating synthetic
    batches, Adadelta lr 0.6, clip 50, MaxNorm 3, seed bench.SEED) at bf16 and at fp32; both precisions draw the same
    Philox dropout masks.  bench.py checks no loss for cfg3 (it has dropout), so this is its loss check."""
    import bench
    w = bench.WORKLOADS['cfg3']
    rng = np.random.default_rng(bench.SEED)
    host = [bench.synthetic(w['B'], rng, w) for _ in range(4)]
    traj = {}
    for prec in ('fp32', 'bf16'):
        eng = make_engine(w['B'], w['T'], w['F'], w['O'], w['H'], w['L'], target_idx=bench.TARGET_IDX, precision=prec,
                          optimizer='Adadelta', dropout=w['dropout'], target_lambda=0.5, rnn_lambda=0.7,
                          max_grad_norm=50.0, max_norm=3.0, seed=bench.SEED)
        eng.set_weights(bench.initial_weights(w))
        dev = [(_cuda(a), _cuda(b)) for a, b in host]
        outs = [eng.train_step(dev[i % 4][0], dev[i % 4][1], i, 0.6) for i in range(TRAJ_STEPS)]
        traj[prec] = torch.stack(outs).cpu().numpy()
        eng.close()
        del eng, dev
        torch.cuda.empty_cache()
    d = np.abs(traj['bf16'] - traj['fp32']) / np.abs(traj['fp32'])
    print('cfg3 bf16 vs fp32 trajectory: max rel diff loss %.3e mse %.3e (step %d); fp32 loss %.4f -> %.4f'
          % (d[:, 0].max(), d[:, 1].max(), int(d.max(axis=1).argmax()), traj['fp32'][0, 0], traj['fp32'][-1, 0]))
    assert np.isfinite(traj['bf16']).all() and np.isfinite(traj['fp32']).all()
    assert d.max() < TRAJ_BOUND
    assert traj['fp32'][-1, 0] < traj['fp32'][0, 0]          # and it actually trains
