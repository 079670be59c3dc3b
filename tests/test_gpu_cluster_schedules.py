"""The bf16 cluster recurrences (lstm_tc.cu) at the batch sizes they train at, on every schedule tc_rounds picks there.

cfg2 (B = 4096, T = 48, F = 32, O = 16, H = 256, L = 1) runs both recurrences as one round of pair groups: a tile's
four CTAs as two 2-CTA clusters that exchange state through L2 under per-CTA step flags.  The flags only grow (TcImpl::seq
carries them from launch to launch) and the backward's L2 scratch is double-buffered by send parity.  The other suites
hold these kernels to the rounding oracle only at B <= 300 (64-row half tiles) and to each other only at T = 8, so a
fault of the 128-row or pair kernels that shows after step 8 reaches nothing tighter than the fp64 bounds.

1. The rounding oracle (tests/bf16_oracle.py, Plan('cluster')) at B = 4096, 4224 and 4225, with BN moving statistics
   away from (0, 1) and a nonzero row0: predictions (closer to the rounding oracle than to the fp64 one by RATIO), loss,
   mse_0 and every gradient tensor within test_gpu_bf16_rounding.BOUNDS['cluster'], on the default schedule and, at
   B = 4096, on 4-CTA clusters (LFMQ_TC_PAIR_GROUPS=0: 30 128-row tiles, then 4 half tiles).  Each case's oracles are
   computed once (cfg2 at T = 48 takes about a minute of CPU time).
2. Pair groups across launches: the state after k train steps, a handle that switches schedules with the batch size,
   bit-identity with 4-CTA clusters at T = 48 and, with pair groups forced, over four rounds of the backward.

LFMQ_TC_PAIR_GROUPS / LFMQ_TC_HALF_TILES are read when a handle is created; each handle here is created with the
schedule's variables set (or unset) and the environment is restored afterwards.
"""
import contextlib
import os
import time

import numpy as np
import pytest

import bf16_oracle as bo
import lfm_oracle as orc
from test_gpu_bf16_rounding import (HEAD_TOL, LR, ROW0, STEP, _bn_kw, _bn_stats, _cuda, _flat_from, _kind, _loss_tail,
                                    _max_norm_that_clips, _Report)
from util import make_engine, make_problem, rel_err

pytestmark = pytest.mark.gpu

F, O, H = 32, 16, 256
D2 = dict(dropout=0.2, seed=77)
LKW = dict(target_idx=O - 1, target_lambda=0.5, rnn_lambda=0.7)
SCHEDULE_VARS = ('LFMQ_TC_PAIR_GROUPS', 'LFMQ_TC_HALF_TILES')
SCHEDULES = {'default': {}, 'clusters': {'LFMQ_TC_PAIR_GROUPS': '0'}, 'pairs': {'LFMQ_TC_PAIR_GROUPS': '1'}}


@contextlib.contextmanager
def _schedule(name):
    """The environment of schedule `name` (every schedule variable it does not set is unset), restored on exit."""
    old = {k: os.environ.get(k) for k in SCHEDULE_VARS}
    for k in SCHEDULE_VARS:
        os.environ.pop(k, None)
    os.environ.update(SCHEDULES[name])
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _engine(B, T, schedule='default', **kw):
    with _schedule(schedule):
        return make_engine(B, T, F, O, H, 1, target_idx=O - 1, precision='bf16', **kw)


def _names(eng):
    return [s[0] for s in eng.trainable_specs]


def _assert_same_step(got, want, where):
    """got / want: _step of two handles.  Predictions and the LSTM W, U, b gradients
    (one weight-gradient GEMM over the same dz rows in the same split-K order) bit for bit; the head gradients and the
    loss, sums over rows through shared-memory atomics, within HEAD_TOL."""
    (p1, g1, t1, names), (p0, g0, t0, _) = got, want
    if p0 is not None:
        assert np.isfinite(p1).all(), where
        assert np.array_equal(p1, p0), where + ('pred', float(np.max(np.abs(p1 - p0))))
    for name, a, b in zip(names[:3], g1[:3], g0[:3]):
        assert np.isfinite(a).all(), where + (name,)
        assert np.array_equal(a, b), where + (name, float(np.max(np.abs(a - b))))
    for name, a, b in zip(names[3:], g1[3:], g0[3:]):
        scale = max(float(np.max(np.abs(b))), 1e-30)
        assert float(np.max(np.abs(a - b))) <= HEAD_TOL * scale, where + (name, float(np.max(np.abs(a - b))) / scale)
    np.testing.assert_allclose(t1, t0, rtol=HEAD_TOL, err_msg=str(where))


def _step(eng, xd, yd, step, row0, forward=True):
    """(preds, gradients, loss tail, names) of a forward (if asked) and a backward call on eng."""
    preds = eng.forward(xd, step=step, row0=row0).cpu().numpy() if forward else None
    eng.backward(xd, yd, step=step, row0=row0)
    return preds, eng.grads_list(), _loss_tail(eng), _names(eng)


# ---- 1. the rounding oracle at the batch sizes the cluster path trains at -------------------------------------------
# (B, T, dropout keywords, schedules).  cfg2: pair groups (the fused-head pair kernels); clusters: 30 128-row tiles on
# 4-CTA clusters, then 4 half tiles.  cfg2-drop: the dropout head (dLoss/dh read from HBM, not fused).  b4224: 33 tiles,
# every co-resident pair group busy.  b4225: one row past the pair limit, 4-CTA clusters: 30 tiles, then 7 half tiles,
# the last with one row.  The bounds are BOUNDS['cluster'] (set at B <= 300); the worst values over these cases, measured
# on an H100 80GB HBM3 (700 W power limit), stay below them: pred 7.2e-4, loss 6.3e-7, mse_0 1.5e-6, kernel 1.5e-3,
# recurrent_kernel 1.1e-3, bias 9.9e-4, gamma 2.2e-5, beta 6.9e-6, OUTPUT_1/kernel 3.5e-5, OUTPUT_1/bias 3.9e-6.  The
# longer fp32 sums of the weight-gradient GEMM at B T = 196608 rows do not make the gradients worse than at B <= 300.
CASES = {
    'cfg2': (4096, 48, {}, ('default', 'clusters')),
    'cfg2-drop': (4096, 16, D2, ('default', 'clusters')),
    'b4224': (4224, 16, {}, ('default',)),
    'b4225': (4225, 16, {}, ('default',)),
}

_ORACLE = {}


def _oracle(case):
    """Inputs, BN statistics and both oracles' predictions, loss, mse_0 and gradients of a case, computed once."""
    if case not in _ORACLE:
        B, T, drop, _ = CASES[case]
        params, x, y = make_problem(B, T, F, O, H, 1, seed=21, init_scale=0.3)
        bn = _bn_stats(1, H, seed=19)
        x64, y64 = x.astype(np.float64), y.astype(np.float64)
        fkw = dict(num_layers=1, training=True, step=STEP, row0=ROW0, **_bn_kw(bn), **drop)
        t0 = time.time()
        res = dict(params=params, x=x, y=y, bn=bn)
        emu_p = bo.Plan('cluster')
        out, fc = bo.forward(emu_p, params, x64, **fkw)
        loss, mse, dpred, _ = orc.loss_point_estimate(y64, out, **LKW)
        res['emu'] = (out, loss, mse, bo.backward(emu_p, dpred, fc))
        del fc, dpred
        out, fc = orc.forward(params, x64, **fkw)
        loss, mse, dpred, _ = orc.loss_point_estimate(y64, out, **LKW)
        res['ref'] = (out, loss, mse, orc.backward(dpred, fc, num_layers=1))
        del fc, dpred
        print('oracles of %s (B=%d, T=%d): %.1f s' % (case, B, T, time.time() - t0))
        _ORACLE[case] = res
    return _ORACLE[case]


@pytest.mark.parametrize('case,schedule', [(c, s) for c in CASES for s in CASES[c][3]])
def test_cluster_schedule_matches_emulated_oracle(case, schedule):
    B, T, drop, _ = CASES[case]
    o = _oracle(case)
    eng = _engine(B, T, schedule, **drop)
    eng.set_weights(o['params'], bn_stats=o['bn'])
    xd, yd = _cuda(o['x']), _cuda(o['y'])
    preds = eng.forward(xd, step=STEP, row0=ROW0).cpu().numpy()
    eng.backward(xd, yd, step=STEP, row0=ROW0)
    tail, grads, names = _loss_tail(eng), eng.grads_list(), _names(eng)
    eng.close()
    (ep, el, em, eg), (rp, rl, rm, rg) = o['emu'], o['ref']
    rep = _Report('cluster', '%s/%s' % (case, schedule))
    rep.check('pred', 'pred', preds, ep, rp, ratio=True)
    rep.check('loss', 'loss', tail[0], el, rl)
    rep.check('mse_0', 'mse_0', tail[1], em, rm)
    for name, g, ge, gr in zip(names, grads, eg, rg):
        rep.check(name, _kind(name), g, ge, gr)
    rep.done()


# ---- 2. pair groups across launches -----------------------------------------------------------------------------------
@pytest.mark.parametrize('k', [1, 4])
@pytest.mark.parametrize('drop', [{}, D2], ids=['nodrop', 'drop'])
def test_state_after_pair_group_train_steps(drop, k):
    """After k Adadelta steps at cfg2 on pair groups (each step two pair launches, so the flags' seq has moved on), the
    handle's forward and backward are those of a fresh handle, whose flags start at zero, loaded with the trained
    weights."""
    B, T = 4096, 48
    params, x, y = make_problem(B, T, F, O, H, 1, seed=31, init_scale=0.3)
    bn = _bn_stats(1, H, seed=19)
    max_norm = _max_norm_that_clips(params, 1)
    kw = dict(optimizer='Adadelta', max_norm=max_norm, **drop)
    eng = _engine(B, T, **kw)
    eng.set_weights(params, bn_stats=bn)
    xd, yd = _cuda(x), _cuda(y)
    for it in range(k):
        eng.train_step(xd, yd, it, LR)
    got = _step(eng, xd, yd, k, ROW0)
    trained = eng.get_weights(trainable_only=False)
    assert max(rel_err(w, p) for w, p in zip(eng.get_weights(), params)) > 1e-4    # the steps moved the weights
    eng.close()
    fresh = _engine(B, T, **kw)
    fresh.set_flat(_flat_from(fresh, trained))
    want = _step(fresh, xd, yd, k, ROW0)
    fresh.close()
    _assert_same_step(got, want, ('k=%d' % k,))


@pytest.mark.parametrize('drop', [{}, D2], ids=['nodrop', 'drop'])
def test_one_handle_switches_schedules_with_the_batch(drop):
    """One handle (max_batch 4224, T = 16) runs B = 4096 (pair groups), 3000 (one round of 24 128-row tiles on 4-CTA
    clusters), 4096, 1000 (16 half tiles, the last partial) and 4224 (33 pair groups) in turn; each call computes what a
    fresh handle computes making that one call."""
    MB, T = 4224, 16
    params, x, y = make_problem(MB, T, F, O, H, 1, seed=33, init_scale=0.3)
    bn = _bn_stats(1, H, seed=19)
    eng = _engine(MB, T, **drop)
    eng.set_weights(params, bn_stats=bn)
    for i, B in enumerate([4096, 3000, 4096, 1000, 4224]):
        xd, yd = _cuda(x[:B]), _cuda(y[:B])
        got = _step(eng, xd, yd, i, ROW0)
        fresh = _engine(MB, T, **drop)
        fresh.set_weights(params, bn_stats=bn)
        want = _step(fresh, xd, yd, i, ROW0)
        fresh.close()
        _assert_same_step(got, want, ('call %d' % i, 'B=%d' % B))
    eng.close()


def _pairs_against_clusters(B, T, drop, forward, seed):
    """One forward (if asked) and backward call on forced pair groups and on forced 4-CTA clusters."""
    params, x, y = make_problem(B, T, F, O, H, 1, seed=seed, init_scale=0.3)
    xd, yd = _cuda(x), _cuda(y)
    steps, launches = [], []
    for schedule in ('pairs', 'clusters'):
        eng = _engine(B, T, schedule, **drop)
        eng.set_weights(params)
        n0 = eng.launch_count
        steps.append(_step(eng, xd, yd, 3, 1000, forward=forward))
        launches.append(eng.launch_count - n0)
        eng.close()
    # pair groups run each recurrence in one launch, 4-CTA clusters in two (their last round as half tiles); a backward
    # call runs the forward recurrence and the backward one
    assert launches[0] == launches[1] - (3 if forward else 2), launches
    _assert_same_step(steps[0], steps[1], ('B=%d' % B, 'T=%d' % T))


@pytest.mark.parametrize('drop', [{}, D2], ids=['nodrop', 'drop'])
def test_pair_groups_bit_identical_at_t48(drop):
    """cfg2: the backward exchanges through L2 47 times per tile, the forward 47 times."""
    _pairs_against_clusters(4096, 48, drop, True, 41)


@pytest.mark.parametrize('drop', [{}, D2], ids=['nodrop', 'drop'])
def test_pair_groups_bit_identical_over_four_backward_rounds(drop):
    """B = 16384 on forced pair groups: 128 tiles in 4 rounds of at most 33 groups, so the backward's send and receive
    counts (and the scratch parity) run on across rounds within a launch."""
    _pairs_against_clusters(16384, 16, drop, False, 43)
