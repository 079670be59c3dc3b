"""The bf16 cluster recurrences on pair groups compute exactly what they compute on 4-CTA clusters.

A pair group runs a tile's four weight-slice CTAs as two 2-CTA clusters and exchanges what crosses between the two
through L2.  The receiver adds the three peers' slices in the same order and the MMAs, tiles and saved state do not
change, so predictions, the saved state and hence dz and the LSTM weight gradients must be bit-identical; only the
head's shared-memory atomics may order sums differently.  LFMQ_TC_PAIR_GROUPS=0 / 1, read when a handle is created,
forces 4-CTA clusters / pair groups; a handle with a device share below one never runs pair groups.
"""
import os
import re

import numpy as np
import pytest
import torch

from util import make_engine, make_problem
from test_ptxas_report import build, _spills  # noqa: F401  (build: the module-scoped compile fixture)

T, F, O, H = 8, 32, 16, 256
HEAD_TOL = 1e-5          # relative to the tensor's largest entry: fp32 atomics summed in another order
# 32 tiles (1 pair round, 2 cluster rounds), 31, 33 (33 groups), 8 tiles with a partial one, one partial tile
BATCHES = [4096, 3968, 4224, 1000, 64]
PAIR_KERNELS = ('lstm_fwd_pair_kernel', 'lstm_bwd_pair_kernel')


def _engine(B, pair, **kw):
    old = os.environ.get('LFMQ_TC_PAIR_GROUPS')
    os.environ['LFMQ_TC_PAIR_GROUPS'] = '1' if pair else '0'
    try:
        return make_engine(B, T, F, O, H, 1, precision='bf16', **kw)
    finally:
        if old is None:
            os.environ.pop('LFMQ_TC_PAIR_GROUPS', None)
        else:
            os.environ['LFMQ_TC_PAIR_GROUPS'] = old


def _predict(B, pair, seed, share=None):
    params, x, _ = make_problem(B, T, F, O, H, 1, seed=seed, init_scale=0.3)
    eng = _engine(B, pair, train=False, forward_only=True)
    if share:
        eng.set_device_share(*share)
    eng.set_weights(params)
    xd = torch.from_numpy(x).cuda()
    n0 = eng.launch_count
    out = eng.forward(xd).cpu().numpy()
    launches = eng.launch_count - n0
    eng.close()
    return out, launches


@pytest.mark.gpu
@pytest.mark.parametrize('B', BATCHES + [16384])    # 16384: several rounds on either schedule
def test_pair_group_predictions_bit_identical(B):
    pair, _ = _predict(B, True, 41)
    quad, _ = _predict(B, False, 41)
    assert np.isfinite(pair).all()
    assert np.array_equal(pair, quad)


@pytest.mark.gpu
@pytest.mark.parametrize('row0', [0, 1000])          # 1000: a data-parallel shard's global row offset
@pytest.mark.parametrize('dropout', [0.0, 0.2])      # fused head dLoss/dh on the backward's MMAs / read from HBM
@pytest.mark.parametrize('B', BATCHES)
def test_pair_group_gradients(B, dropout, row0):
    params, x, y = make_problem(B, T, F, O, H, 1, seed=42, init_scale=0.3)
    xd, yd = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
    grads, tails, names = [], [], None
    for pair in (True, False):
        eng = _engine(B, pair, target_idx=O - 1, dropout=dropout)
        eng.set_weights(params)
        eng.backward(xd, yd, step=3, row0=row0)
        grads.append(eng.grads_list())
        tails.append(eng.grads[eng.n_trainable:eng.n_trainable + 2].cpu().numpy())
        names = [s[0] for s in eng.trainable_specs]
        eng.close()
    # LSTM kernel W, recurrent U, bias: one weight-gradient GEMM over the same dz rows in the same split-K order
    for name, g1, g0 in zip(names[:3], grads[0][:3], grads[1][:3]):
        assert np.isfinite(g1).all(), name
        assert np.array_equal(g1, g0), (name, float(np.max(np.abs(g1 - g0))))
    # head gradients and the loss: sums over rows through shared-memory atomics
    for name, g1, g0 in zip(names[3:], grads[0][3:], grads[1][3:]):
        scale = max(float(np.max(np.abs(g0))), 1e-30)
        assert float(np.max(np.abs(g1 - g0))) <= HEAD_TOL * scale, name
    np.testing.assert_allclose(tails[0], tails[1], rtol=HEAD_TOL)


@pytest.mark.gpu
def test_device_share_below_one_keeps_clusters():
    # B = 4096: 4-CTA clusters take a round of 30 tiles and one of 4 half tiles (two forward launches), a pair group
    # round all 32 tiles (one)
    B = 4096
    _, quad = _predict(B, False, 43)
    _, pair = _predict(B, True, 43)
    assert pair == quad - 1
    _, shared = _predict(B, True, 43, share=(1, 2))
    assert shared == quad


@pytest.mark.parametrize('kernel', PAIR_KERNELS)
def test_pair_kernels_do_not_spill(build, kernel):  # noqa: F811
    log, sass = build
    spills = _spills(log)
    found = [k for k in spills if re.match(r'_ZN4lfmq%d%sILb[01]EEEv' % (len(kernel), kernel), k)]
    assert len(found) == 2, (kernel, sorted(spills))
    for k in found:
        assert spills[k] == (0, 0), '%s: %d B spill stores, %d B spill loads' % ((k,) + spills[k])
    if sass is None:
        pytest.skip('cuobjdump not found')
    funcs, cur = {}, None
    for line in sass.splitlines():
        m = re.search(r'Function : (\w+)', line)
        if m:
            cur = m.group(1)
            funcs[cur] = []
        elif cur:
            funcs[cur].append(line)
    for k in found:
        local = [l.strip() for l in funcs[k] if re.search(r'\b(LDL|STL)\b', l)]
        assert not local, '%s: %d local-memory instructions, e.g. %s' % (k, len(local), local[:3])
