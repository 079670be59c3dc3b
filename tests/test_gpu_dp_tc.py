"""Data-parallel training on the bf16 tensor-core paths, checked on one GPU.

Under torchrun every step of a bf16 model is ForecasterEngine._train_step_dp_flat: each rank runs lfmq_backward on its
row shard with its global row0 (which keys the dropout masks the backward regenerates) and the all-reduced loss
denominators {B_global, mask_count_global}, which the tensor-core heads read; one all-reduce sums
grads[:n_trainable + 2]; every rank runs the same apply.  Here one global batch, with about 10 % of its (row, step)
targets zeroed and most of those in the first shard (so a shard's {B, mask count} is not the global one over R), is
split as dp.shard_rows splits it (R = 2, 3, 8) and unevenly with an empty rank.  The shards take other schedules than
the whole batch (DESIGN 5a / 5b): 128-row tiles, 64-row half tiles or a ragged last tile on the cluster path, one
backward chain instead of two and a persistent forward instead of a stepped one on the general path.

(a) The shards' mask counts sum to the whole batch's exactly, and their gradients and {loss, mse_0}, each shard run on
    a handle of its own and again one after another on the whole batch's handle, sum to the whole batch's backward
    within DP_TOL: what separates them is only the fp32 summation order of the split-K weight gradient and the heads'
    partial sums.
(b) Two mistakes miss that bound by at least 100x in every tensor kind: local denominators (a rank that skipped the
    count all-reduce) and a shard without its row offset (dropout cases).  The second draws other masks from the same
    distribution, so it moves the summed gradients only by their sampling noise; that is still 560x or more the bound
    of every kind.
(c) One shard's loss tail, mse_0 and gradients against the oracle that rounds where the kernels round
    (tests/bf16_oracle.py), with the whole batch's counts as denominators, at test_gpu_bf16_rounding.BOUNDS.
(d) The apply on the summed vector follows the whole batch's train_step through two Adadelta steps with a MaxNorm bound
    that clips, and the next forward agrees.
(e) train_step_dp in a one-rank gloo group equals train_step; a rank without rows returns zeros and applies a zero
    gradient.
Then the point model (fp32, bf16 on both paths) and the linear baseline through the CLI with two gloo ranks on this
device against one rank.
"""
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist

import bf16_oracle as bo
import lfm_oracle as orc
from lfm_quant_b200 import dp
from test_gpu_bf16_rounding import BOUNDS, HEAD_TOL, _bn_kw, _bn_stats, _kind, _max_norm_that_clips
from test_gpu_dp_models import _cli_rank
from util import make_engine, make_problem, rel_err

pytestmark = pytest.mark.gpu

ROW0, STEP, LR = 3000, 4, 0.6
LKW = dict(target_lambda=0.5, rnn_lambda=0.7)
D2 = dict(dropout=0.2, seed=77)
D21 = dict(dropout=0.2, recurrent_dropout=0.1, seed=77)
MISS = 100               # a wrong answer misses the whole batch by at least this multiple of DP_TOL

# Max-norm relative error of the summed shards against the whole batch's backward, per path and kind: at least 1.5x the
# worst value over the path's cases of DP_CASES (both ways of running the shards, every split), measured on an H100
# 80GB HBM3 (700 W power limit), rounded up to one significant digit, and no less than 1e-6: the heads sum with
# shared-memory atomics, so those kinds differ between two runs in the last bits (DESIGN 6a).  The worst value is in
# the comment.  The LSTM weight gradients sum T * B rows split K-wise into fp32 partials, and their error grows with
# that count: the worst is at R = 8 of the largest T * B of the path.
DP_TOL = {
    'cluster': {
        'kernel': 3e-5,               # 1.63e-5 (t48-drop, R = 8)
        'recurrent_kernel': 7e-5,     # 4.14e-5 (t48-drop, R = 8)
        'bias': 5e-5,                 # 2.87e-5 (t48-drop, R = 8)
        'gamma': 1e-6,                # 1.72e-7
        'beta': 1e-6,                 # 1.59e-7
        'OUTPUT_1/kernel': 1e-6,      # 1.46e-7
        'OUTPUT_1/bias': 1e-6,        # 6.81e-8
        'loss': 1e-6,                 # 1.17e-7
        'mse_0': 1e-6,                # 6.99e-8
    },
    'general': {
        'kernel': 2e-4,               # 9.68e-5 (b4096-t48, R = 8)
        'recurrent_kernel': 2e-4,     # 9.99e-5 (b4096-t48, R = 8)
        'bias': 2e-5,                 # 9.96e-6 (b4096-t48, R = 8)
        'gamma': 1e-6,                # 1.27e-7
        'beta': 1e-6,                 # 1.07e-7
        'OUTPUT_1/kernel': 8e-6,      # 5.14e-6 (b4096-t48, R = 8)
        'OUTPUT_1/bias': 1e-6,        # 8.94e-8
        'loss': 1e-6,                 # 1.11e-7
        'mse_0': 1e-6,                # 8.60e-8
    },
}


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()


def _problem(shape, seed):
    """make_problem, then about 10 % of the (row, step) targets zeroed (masked): 70 % of them in rows [0, B/8), which
    lie in the first shard of every split, and a fifth of them at the last step, so mse_0 and mse_1 see masked rows."""
    B, T, F, O, H, L = shape
    params, x, y = make_problem(B, T, F, O, H, L, seed=seed, init_scale=0.3 * min(1.0, np.sqrt(32.0 / F)))
    rng = np.random.RandomState(seed + 1000)
    n = B * T // 8          # some (row, step) pairs are drawn twice
    n_hot = 7 * n // 10
    b = np.concatenate([rng.randint(0, max(1, B // 8), n_hot), rng.randint(0, B, n - n_hot)])
    t = rng.randint(0, T, n)
    t[::5] = T - 1
    y[b, t, :] = 0.0
    return params, x, y


def _splits(B):
    """dp.shard_rows for R = 2, 3, 8, and an uneven split whose middle rank has no rows."""
    out = {}
    for R in (2, 3, 8):
        out['R=%d' % R] = [(a, a + n) for a, n in (dp.shard_rows(B, r, R) for r in range(R))]
    cut = 1000 if B > 1000 else 100
    out['uneven'] = [(0, cut), (cut, cut), (cut, B)]
    return out


def _schedule(path, n, H):
    """The schedule DESIGN 5a / 5b gives n rows (cluster path: 30 co-resident four-CTA clusters, as on an H100 SXM)."""
    tiles = -(-n // 128)
    if path == 'cluster':
        ncl = min(tiles, 30)
        full_rounds = -(-tiles // ncl) - 1
        halves = -(-(n - full_rounds * ncl * 128) // 64)
        full, half = (full_rounds * ncl, halves) if halves <= 30 else (tiles, 0)
        parts = (['%d tiles' % full] if full else []) + (['%d half tiles' % half] if half else [])
        ragged = ', ragged last tile' if not half and n % 128 else ''
        return ' + '.join(parts) + ragged
    chains = 'backward chains of %d and %d tiles' % ((tiles + 1) // 2, tiles // 2) if tiles >= 16 else \
        'one backward chain of %d tiles' % tiles
    return '%d tiles, %s' % (tiles, chains)


def _engine(n, shape, drop, bn, params, **kw):
    B, T, F, O, H, L = shape
    e = make_engine(n, T, F, O, H, L, target_idx=O - 1, precision='bf16', optimizer='Adadelta', **LKW, **drop, **kw)
    e.set_weights(params, bn_stats=bn)
    return e


def _backward(e, xd, yd, a, b, row0, denom):
    """This shard's backward; returns grads[:n_trainable + 2] (a copy) and the launches it took."""
    n0 = e.launch_count
    e.backward(xd[a:b], yd[a:b], step=STEP, row0=row0, denom=denom)
    return e.grads[:e.n_trainable + 2].clone(), e.launch_count - n0


def _errors(e, got, ref):
    """{tensor name or 'loss' / 'mse_0': max-norm relative error} of two grads[:n_trainable + 2] vectors."""
    got, ref = got.cpu().numpy(), ref.cpu().numpy()
    out = {name: rel_err(got[off:off + int(np.prod(shp))], ref[off:off + int(np.prod(shp))])
           for name, shp, off, _ in e.trainable_specs}
    out['loss'] = rel_err(got[e.n_trainable], ref[e.n_trainable])
    out['mse_0'] = rel_err(got[e.n_trainable + 1], ref[e.n_trainable + 1])
    return out


def _kind_of(name):
    return name if name in ('loss', 'mse_0') else _kind(name)


# name: path, (B, T, F, O, H, L), dropout keywords
DP_CASES = {
    'cluster-t16': ('cluster', (4096, 16, 32, 16, 256, 1), {}),
    'cluster-t16-drop': ('cluster', (4096, 16, 32, 16, 256, 1), D2),
    'cluster-t48-drop': ('cluster', (4096, 48, 32, 16, 256, 1), D2),
    'general-b4096-t48': ('general', (4096, 48, 32, 16, 512, 2), D21),
    'general-b2100': ('general', (2100, 16, 32, 16, 512, 2), D21),
    'general-b256-h64': ('general', (256, 5, 32, 16, 64, 2), D21),
}


@pytest.mark.parametrize('case', list(DP_CASES))
def test_shards_sum_to_the_whole_batch(case):
    """(a) and (b) on every split of the case's batch."""
    path, shape, drop = DP_CASES[case]
    B, T, F, O, H, L = shape
    keyed = bool(drop)
    params, x, y = _problem(shape, seed=sum(shape))
    bn = _bn_stats(L, H, seed=19)
    xd, yd = _cuda(x), _cuda(y)
    whole = _engine(B, shape, drop, bn, params)
    glob = whole.mask_count(yd)
    assert glob.cpu().numpy().tolist() == [B, float((~np.all(y == 0, axis=-1)).sum())]
    ref, n_whole = _backward(whole, xd, yd, 0, B, ROW0, None)
    assert np.isfinite(ref.cpu().numpy()).all()
    print('\n%s %s: whole batch B=%d: %s; %d launches' % (case, path, B, _schedule(path, B, H), n_whole))
    tol = DP_TOL[path]
    worst = {}           # kind -> (error, where)
    misses = {'local denominators': np.inf, 'local row0': np.inf}
    failures = []
    for split, shards in _splits(B).items():
        counts = [whole.mask_count(yd[a:b]) for a, b in shards if b > a]
        assert torch.equal(sum(counts), glob), (split, [c.tolist() for c in counts], glob.tolist())
        local = [c.cpu().numpy().tolist() for c in counts]
        print('  %s: shards %s, their {B, mask count} %s' % (split, shards, local))
        acc = {k: torch.zeros_like(ref) for k in ('rank handles', 'one handle', 'local denominators', 'local row0')}
        for a, b in shards:
            if b == a:       # a rank without rows contributes a zero vector
                continue
            e = _engine(b - a, shape, drop, bn, params)
            g, n = _backward(e, xd, yd, a, b, ROW0 + a, glob)
            acc['rank handles'] += g
            acc['local denominators'] += _backward(e, xd, yd, a, b, ROW0 + a, None)[0]
            if keyed:
                acc['local row0'] += _backward(e, xd, yd, a, b, ROW0, glob)[0]
            e.close()
            print('    rows [%d, %d): %s; %d launches' % (a, b, _schedule(path, b - a, H), n))
        for a, b in shards:  # the same shards one after another on the whole batch's handle
            if b > a:
                acc['one handle'] += _backward(whole, xd, yd, a, b, ROW0 + a, glob)[0]
        for how in ('rank handles', 'one handle'):
            for name, err in _errors(whole, acc[how], ref).items():
                k = _kind_of(name)
                if err > worst.get(k, (-1.0,))[0]:
                    worst[k] = (err, '%s, %s, %s' % (split, how, name))
                if not err < tol[k]:
                    failures.append((split, how, name, err, tol[k]))
        for wrong in ('local denominators', 'local row0') if keyed else ('local denominators',):
            miss = {}        # kind -> largest error / DP_TOL over the tensors of that kind
            for name, err in _errors(whole, acc[wrong], ref).items():
                k = _kind_of(name)
                miss[k] = max(miss.get(k, 0.0), err / tol[k])
            k = min(miss, key=miss.get)
            print('    %s: misses DP_TOL by at least x%.0f (%s); by kind %s' % (wrong, miss[k], k, ', '.join(
                '%s x%.0f' % (q, m) for q, m in miss.items())))
            misses[wrong] = min(misses[wrong], miss[k])
    whole.close()
    print('  worst shard-sum error per kind (DP_TOL):')
    for k in tol:
        if k in worst:
            print('    %-18s %.3e  (%.0e)  at %s' % (k, worst[k][0], tol[k], worst[k][1]))
    print('  least miss of the wrong answers: %s' % ', '.join(
        '%s x%.0f' % (w, m) for w, m in misses.items() if np.isfinite(m)))
    assert not failures, failures
    for wrong, m in misses.items():
        assert not np.isfinite(m) or m >= MISS, (wrong, m)


# ---- (c) one shard against the rounding oracle ---------------------------------------------------------------------
# name: path, (B, T, F, O, H, L), dropout keywords, a split row that is not a multiple of 64 (test_gpu_bf16_rounding's
# shapes t8-f32, t8-f32-drop, h192-l2-f20)
ORACLE_CASES = {
    'cluster': ('cluster', (300, 8, 32, 16, 256, 1), {}, 137),
    'cluster-drop': ('cluster', (300, 8, 32, 16, 256, 1), D2, 137),
    'general-h192-l2': ('general', (160, 5, 20, 7, 192, 2), D21, 77),
}


@pytest.mark.parametrize('case', list(ORACLE_CASES))
def test_shard_is_its_share_of_the_global_loss(case):
    """(c) Each shard, run with the whole batch's counts and its global row0, computes its own share of the global loss
    and gradient as the rounding oracle computes it over that shard alone."""
    path, shape, drop, cut = ORACLE_CASES[case]
    B, T, F, O, H, L = shape
    params, x, y = _problem(shape, seed=21)
    bn = _bn_stats(L, H, seed=19)
    bkw = _bn_kw(bn)
    xd, yd = _cuda(x), _cuda(y)
    x64, y64 = x.astype(np.float64), y.astype(np.float64)
    eng = _engine(B, shape, drop, bn, params)
    glob = eng.mask_count(yd)
    Bg, Mg = glob.cpu().numpy().tolist()
    names = [s[0] for s in eng.trainable_specs]
    bounds = BOUNDS[path]
    rows, failures = [], []
    for a, b in ((0, cut), (cut, B)):
        vec = _backward(eng, xd, yd, a, b, ROW0 + a, glob)[0].cpu().numpy()
        grads = eng.grads_list()
        emu, fc = bo.forward(bo.Plan(path), params, x64[a:b], num_layers=L, training=True, step=STEP, row0=ROW0 + a,
                             **bkw, **drop)
        loss, mse, dpred, _ = orc.loss_point_estimate(y64[a:b], emu, target_idx=O - 1, batch_global=Bg,
                                                      mask_count_global=Mg, **LKW)
        want = [('loss', vec[eng.n_trainable], loss), ('mse_0', vec[eng.n_trainable + 1], mse)]
        want += list(zip(names, grads, bo.backward(bo.Plan(path), dpred, fc)))
        for name, got, ref in want:
            assert np.isfinite(got).all(), (case, a, name)
            err, bound = rel_err(got, ref), bounds[_kind_of(name)]
            rows.append('%s rows [%d, %d) %-32s emulated %.3e  bound %.0e' % (case, a, b, name, err, bound))
            if not err < bound:
                failures.append((a, b, name, err, bound))
    eng.close()
    print('\n' + '\n'.join(rows))
    assert not failures, failures


# ---- (d) the step on the summed vector -------------------------------------------------------------------------------
# Max-norm relative error of the data-parallel step (the apply on the summed shard gradients) against the whole batch's
# train_step: the returned {loss, mse_0} of both steps, the weights after them and the next forward.  At least 1.5x the
# worst value over both cases, measured on an H100 80GB HBM3 (700 W power limit), rounded up to one significant digit,
# the loss no less than 1e-6 (head atomics).  The forward differs more than the weights: a weight that moved by 1e-5
# relative can round to the neighbouring bf16 value in the packed copies.
STEP_TOL = {
    'loss': 1e-6,         # 4.32e-7 (general, step 1)
    'weights': 3e-5,      # 1.42e-5 (general, lstm_2/kernel)
    'pred': 2e-3,         # 8.54e-4 (general)
}

STEP_CASES = {
    'cluster': ('cluster', (4096, 16, 32, 16, 256, 1), D2),
    'general': ('general', (2100, 16, 32, 16, 512, 2), D21),
}


@pytest.mark.parametrize('case', list(STEP_CASES))
def test_apply_on_the_summed_shards_steps_like_the_whole_batch(case):
    path, shape, drop = STEP_CASES[case]
    B, T, F, O, H, L = shape
    params, x, y = _problem(shape, seed=5)
    bn = _bn_stats(L, H, seed=19)
    max_norm = _max_norm_that_clips(params, L)
    xd, yd = _cuda(x), _cuda(y)
    whole = _engine(B, shape, drop, bn, params, max_norm=max_norm)
    ranks = _engine(B, shape, drop, bn, params, max_norm=max_norm)
    n = ranks.n_trainable
    shards = _splits(B)['R=3']
    errs = {}
    for it in range(2):
        ref = whole.train_step(xd, yd, it, LR).cpu().numpy()       # train_step keys dropout by row0 = 0
        glob = ranks.mask_count(yd)
        acc = torch.zeros(n + 2, dtype=torch.float32, device='cuda')
        for a, b in shards:
            ranks.backward(xd[a:b], yd[a:b], step=it, row0=a, denom=glob)
            acc += ranks.grads[:n + 2]
        ranks.grads[:n + 2].copy_(acc)
        ranks.apply(LR, it)
        got = acc[n:].cpu().numpy()
        errs['step %d loss' % it] = ('loss', rel_err(got[0], ref[0]))
        errs['step %d mse_0' % it] = ('loss', rel_err(got[1], ref[1]))
    for (name, _, _, _), w, v in zip(whole.trainable_specs, ranks.get_weights(), whole.get_weights()):
        errs['weights ' + name] = ('weights', rel_err(w, v))
    moved = max(rel_err(v, p) for v, p in zip(whole.get_weights(), params))
    got = ranks.forward(xd, step=2, row0=ROW0).cpu().numpy()
    want = whole.forward(xd, step=2, row0=ROW0).cpu().numpy()
    errs['forward'] = ('pred', rel_err(got, want))
    whole.close()
    ranks.close()
    print()
    for what, (kind, e) in errs.items():
        print('%s step: %-34s %.3e  (%.0e)' % (case, what, e, STEP_TOL[kind]))
    print('%s step: the steps moved the weights by %.3e' % (case, moved))
    assert moved > 1e-4
    for what, (kind, e) in errs.items():
        assert e < STEP_TOL[kind], (case, what, e)


# ---- (e) train_step_dp on bf16 handles in a one-rank group ---------------------------------------------------------
@pytest.mark.parametrize('case', ['cluster-drop', 'general-h192-l2'])
def test_one_rank_gloo_train_step_dp_equals_train_step(case, tmp_path):
    path, shape, drop, _ = ORACLE_CASES[case]
    B, T, F, O, H, L = shape
    params, x, y = _problem(shape, seed=3)
    bn = _bn_stats(L, H, seed=19)
    max_norm = _max_norm_that_clips(params, L)
    a, b = (_engine(B, shape, drop, bn, params, max_norm=max_norm) for _ in range(2))
    xd, yd = _cuda(x), _cuda(y)
    dist.init_process_group('gloo', init_method='file://' + str(tmp_path / 'pg'), rank=0, world_size=1)
    try:
        for it in range(2):
            got = a.train_step_dp(xd, yd, it, LR, 0, a.loss_counts(yd)).cpu().numpy()
            ref = b.train_step(xd, yd, it, LR).cpu().numpy()
            np.testing.assert_allclose(got, ref, rtol=HEAD_TOL)
            for (name, _, _, _), w, v in zip(a.trainable_specs, a.get_weights(), b.get_weights()):
                assert rel_err(w, v) <= HEAD_TOL, (case, it, name, rel_err(w, v))
        b.set_flat(a.get_flat())          # with a zero gradient the update is MaxNorm alone, whatever the slots hold
        out = a.train_step_dp(None, None, 2, LR, B, a.loss_counts(None)).cpu().numpy()
        assert (out == 0).all()
        b.grads[:b.n_trainable].zero_()
        b.apply(LR, 2)
        assert torch.equal(a.params, b.params)
    finally:
        dist.destroy_process_group()
        a.close()
        b.close()


# ---- the point model and the linear baseline through the CLI with two ranks ----------------------------------------
# name: CLI arguments, bound on the batch and epoch logs' mse, bound on the saved weights.  fp32 and the linear model
# keep the bounds of test_gpu_dp_models.py.  bf16 runs are not bit-reproducible even on one rank (the heads' atomics):
# worst measured on an H100 80GB HBM3 (700 W power limit) 3.01e-5 on the logs and 5.58e-4 on the weights (cluster path,
# OUTPUT_1/kernel and recurrent_kernel), 1.2e-5 and 1.3e-4 on the general path; the bounds are more than 3x those, as
# the trajectories of two runs drift apart over the steps, and far below the 3e-2 tools/dp_cli_check.py allows.
CLI_CASES = {
    'fp32': (['--dropout', '0.1'], 1e-4, 1e-3),
    'bf16-general': (['--precision', 'bf16', '--dropout', '0.1'], 1e-4, 2e-3),
    'bf16-cluster': (['--precision', 'bf16', '--num_hidden', '256', '--dropout', '0.1'], 1e-4, 2e-3),
    'mlp-linear': (['--nn_type', 'MLPLinearPointEstimate', '--init_scale', '0.02'], 1e-4, 1e-3),
}


@pytest.mark.timeout(600)
@pytest.mark.parametrize('case', list(CLI_CASES))
def test_cli_two_ranks_train_the_one_rank_point_model(tmp_path, case):
    """RNNPointEstimate (the default nn_type) and MLPLinearPointEstimate through the CLI with two data-parallel gloo
    ranks on this device log the one-rank run's global losses and save its weights."""
    import pandas as pd
    import torch.multiprocessing as mp
    from lfm_quant_b200.scripts.synthetic import write_open_dataset, write_system_test_conf
    extra, log_tol, w_tol = CLI_CASES[case]
    write_open_dataset(str(tmp_path / 'datasets' / 'open-dataset.dat'), n_keys=30, n_months=420, seed=9)
    write_system_test_conf(str(tmp_path / 'config' / 'system-test.conf'), str(tmp_path / 'datasets'),
                           str(tmp_path / 'experiments'))
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    mp.spawn(_cli_rank, args=(1, 0, str(tmp_path), extra, 'one'), nprocs=1, join=True)
    mp.spawn(_cli_rank, args=(2, port, str(tmp_path), extra, 'two'), nprocs=2, join=True)
    ex = tmp_path / 'experiments'
    errs = {}
    for kind in ('batch', 'epoch'):
        one, two = (pd.read_csv(ex / m / 'train_log' / ('system-test-train-logs-%s.csv' % kind)) for m in ('one', 'two'))
        assert len(one) == len(two) > 1
        assert np.isfinite(two['mse']).all()
        errs['%s mse' % kind] = (rel_err(two['mse'].values, one['mse'].values), log_tol)
    w1, w2 = (np.load(ex / m / 'chkpts' / 'chkpt.lfmq.npz') for m in ('one', 'two'))
    assert set(w1.files) == set(w2.files)
    for k in w1.files:
        errs['weights ' + k] = (rel_err(w2[k], w1[k]), w_tol)
    print()
    for what, (e, tol) in errs.items():
        print('cli %s: two ranks vs one, %-40s %.3e  (%.0e)' % (case, what, e, tol))
    for what, (e, tol) in errs.items():
        assert e < tol, (case, what, e, tol)
