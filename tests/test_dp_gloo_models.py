"""Data parallelism of RNNUqRangeEstimate and of multi-step forecasts on CPU: world-size-2 gloo processes run the step
plumbing of lfm_quant_b200/dp.py on oracle gradients of their row shards -- the per-stage loss counts all-reduced once
per batch, the packed vector of every stage's gradients and reduced loss tail all-reduced once per step -- and must
reproduce the single-process gradients, losses and update.  A rank without rows joins every collective."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import lfm_oracle as orc
import uq_chain_oracle as uco
from lfm_quant_b200 import dp

KW = dict(target_idx=1, target_lambda=0.5, rnn_lambda=0.7)
DROP = dict(dropout=0.2, recurrent_dropout=0.15, seed=31)
SHAPE = dict(T=5, F=6, O=3, H=8)
STEP = 2


def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _counts(y):
    """{B, unmasked rows, unmasked last-step rows} of one stage's targets: what lfmq_mask_count_uq / lfmq_chain_mask_count
    return."""
    mask = ~np.all(y == 0.0, axis=-1)
    return np.array([y.shape[0], mask.sum(), mask[:, -1].sum()], dtype=np.float64)


def _uq_loss(y, p, v, counts, *, target_idx, target_lambda, rnn_lambda):
    """losses.py:180-284 as lfm_oracle.loss_uq_estimate, with the denominators given: {B, unmasked rows, unmasked
    last-step rows} of the global batch.  Returns this shard's contributions (uq_loss, uq_loss_last_tar, mse_0) and
    dLoss/dpred, dLoss/dvar."""
    Bg, ms_all, ms_last = counts
    K = y.shape[-1]
    m3 = (~np.all(y == 0.0, axis=-1)).astype(p.dtype)[..., None]
    pm, vm = p * m3, v * m3
    diff = (pm - y) ** 2
    term = diff * (1.0 / vm) + np.log(vm)
    uq0 = np.sum(term[:, -1, target_idx]) / ms_last
    uq1 = np.sum(term[:, -1, :]) / (ms_last * K)
    uq2 = np.sum(term) / (ms_all * K)
    mse_0 = np.sum(diff[:, -1, target_idx]) / Bg
    p1, p2 = target_lambda, rnn_lambda
    loss = p1 * uq0 + (1 - p1) * (p2 * uq1 + (1 - p2) * uq2)
    coef = np.full(y.shape, (1 - p1) * (1 - p2) / (ms_all * K))
    coef[:, -1, :] += (1 - p1) * p2 / (ms_last * K)
    coef[:, -1, target_idx] += p1 / ms_last
    return loss, uq0, mse_0, coef * (2.0 * (pm - y) / vm) * m3, coef * (-diff / (vm * vm) + 1.0 / vm) * m3


def test_uq_loss_with_the_whole_batch_counts_is_the_oracle_loss():
    rng = np.random.RandomState(4)
    y, p = rng.normal(size=(2, 7, 5, 3))
    v = rng.uniform(0.5, 2.0, size=(7, 5, 3))
    got = _uq_loss(y, p, v, _counts(y), **KW)
    ref = orc.loss_uq_estimate(y, p, v, **KW)
    for g, r in zip(got, ref):
        np.testing.assert_allclose(g, r, rtol=1e-12, atol=1e-15)


def _problem(kind, B, S, seed=11):
    T, F, O, H = SHAPE['T'], SHAPE['F'], SHAPE['O'], SHAPE['H']
    rng = np.random.RandomState(seed)
    if kind == 'point_chain':
        params = orc.init_forecast_params(1, F, O, H, S, init_scale=0.5, seed=seed + 1, dtype=np.float64)
    else:
        params = uco.init_params(1, F, O, H, S, init_scale=0.5, seed=seed + 1, dtype=np.float64)
    x = rng.normal(size=(B, T, F))
    ys = [rng.normal(size=(B, T, O)) for _ in range(S)]
    if kind == 'point_chain' and B > 2:      # masked rows (a uq loss would be NaN with them)
        ys[0][0, :2, :] = 0.0
        ys[-1][B - 1, 0, :] = 0.0
    return params, x, ys


def _stage_sizes(kind, S):
    T, F, O, H = SHAPE['T'], SHAPE['F'], SHAPE['O'], SHAPE['H']
    names = orc.forecast_param_names(1, S) if kind == 'point_chain' else uco.param_names(1, S)
    per = 5 + 2 if kind == 'point_chain' else 5 + 4
    return [per] * S if S > 1 else [len(names)], names


def _shard_grads(kind, params, x, ys, counts, weights, row0):
    """One shard's gradients (trainable_variables order) and each stage's loss tail, with the global counts."""
    S = len(ys)
    fkw = dict(num_layers=1, forecast_steps=S, step=STEP, row0=row0, **DROP)
    tails, dps, dvs = [], [], []
    if kind == 'point_chain':
        preds, fc = orc.forward_forecast(params, x, training=True, **fkw)
        for s in range(S):
            l, m, d, _ = orc.loss_point_estimate(ys[s], preds[s], batch_global=counts[s][0],
                                                 mask_count_global=counts[s][1], **KW)
            tails.append([l, m])
            dps.append(weights[s] * d)
        return orc.backward_forecast(dps, fc), tails
    preds, vars_, fc = uco.forward(params, x, **fkw)
    for s in range(S):
        l, u, m, d, dv = _uq_loss(ys[s], preds[s], vars_[s], counts[s], **KW)
        tails.append([l, m, u])           # {uq_loss, mse_0, uq_loss_last_tar}, the packed order
        dps.append(weights[s] * d)
        dvs.append(weights[s] * dv)
    return uco.backward(dps, dvs, fc), tails


def _pack(grads, tails, per_stage):
    """every stage's gradients followed by its reduced tail: the layout of lfmq_chain_grad_pack"""
    out, i = [], 0
    for n, tail in zip(per_stage, tails):
        out += [g.ravel() for g in grads[i:i + n]] + [np.asarray(tail, dtype=np.float64)]
        i += n
    return np.concatenate(out)


def _worker(rank, world, port, out_dir, kind, B, S):
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    calls = []
    all_reduce = dist.all_reduce

    def counted(t, *a, **k):              # every collective this rank joins, in order
        calls.append(t.numel())
        return all_reduce(t, *a, **k)

    dist.all_reduce = counted
    params, x, ys = _problem(kind, B, S)
    weights = [1.0, 0.5, 0.25][:S]
    per_stage, _ = _stage_sizes(kind, S)
    row0, n = dp.shard_rows(B, rank, world)
    xs, yss = x[row0:row0 + n], [y[row0:row0 + n] for y in ys]
    local = np.stack([_counts(y) for y in yss]) if n else np.zeros((S, 3))
    counts = dp.global_stage_counts(torch.from_numpy(local), dist).numpy()       # once per batch
    k = 2 if kind == 'point_chain' else 3
    size = sum(p.size for p in params) + k * S
    if n:
        grads, tails = _shard_grads(kind, params, xs, yss, counts, weights, row0)
        flat = torch.from_numpy(_pack(grads, tails, per_stage))
        assert flat.numel() == size
    else:                                 # no rows: zeros, the same collective
        flat = torch.zeros(size, dtype=torch.float64)
    flat = dp.allreduce_packed(flat, dist).numpy()
    np.savez(os.path.join(out_dir, 'rank%d.npz' % rank), flat=flat, counts=counts, calls=np.array(calls))
    dist.destroy_process_group()


@pytest.mark.timeout(180)
@pytest.mark.parametrize('B', [9, 1])
@pytest.mark.parametrize('kind,S', [('uq', 1), ('point_chain', 2), ('uq_chain', 2), ('uq_chain', 3)])
def test_two_rank_step_equals_single_process(tmp_path, kind, S, B):
    """B = 1: rank 1 has no rows and still joins the count all-reduce and the gradient all-reduce."""
    world = 2
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path), kind, B, S), nprocs=world, join=True)
    params, x, ys = _problem(kind, B, S)
    weights = [1.0, 0.5, 0.25][:S]
    per_stage, _ = _stage_sizes(kind, S)
    counts = np.stack([_counts(y) for y in ys])
    grads, tails = _shard_grads(kind, params, x, ys, counts, weights, 0)
    ref = _pack(grads, tails, per_stage)
    r = [np.load(tmp_path / ('rank%d.npz' % i)) for i in range(world)]
    np.testing.assert_array_equal(r[0]['counts'], counts)
    np.testing.assert_allclose(r[0]['flat'], ref, rtol=1e-10, atol=1e-12)
    np.testing.assert_array_equal(r[0]['flat'], r[1]['flat'])              # replicas agree bit for bit
    assert list(r[0]['calls']) == list(r[1]['calls']) == [3 * S, ref.size]  # two collectives per batch, on every rank
    if kind == 'uq':                  # the whole-batch oracle step: gradients, losses, and the update from the tail
        new, mse, loss, raw, gn, uq0 = orc._train_step_uq([p.copy() for p in params], orc.zero_slots('Adadelta', params),
                                                          x, ys[0], STEP, dict(num_layers=1, max_grad_norm=0.5,
                                                                               optimizer='Adadelta', max_norm=0.8,
                                                                               **KW, **DROP), lr=0.6)
        n_tr = ref.size - 3
        np.testing.assert_allclose(r[0]['flat'][n_tr:], [loss, mse, uq0], rtol=1e-10)
        np.testing.assert_allclose(r[0]['flat'][:n_tr], np.concatenate([g.ravel() for g in raw]), rtol=1e-10,
                                   atol=1e-12)


def _cli_worker(rank, world, port, out_dir, extra):
    """What scripts/train.py does under torchrun for RNNUqRangeEstimate and multi-step forecasts: the process group
    from the launcher's environment, the dataset's shuffled global batches, this rank's rows of each."""
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank), CUDA_VISIBLE_DEVICES='')
    from lfm_quant_b200.scripts import lfm_quant
    from lfm_quant_b200.scripts.data_processing import Dataset
    r, w = dp.init_from_env()
    assert (r, w) == (rank, world) and dist.is_initialized()
    conf = os.path.join(out_dir, 'config', 'system-test.conf')
    config = lfm_quant.get_configs(['--config=' + conf, '--train=True', '--model_dir', 'rank%d' % rank] + extra)
    ds = Dataset(config)
    ds.generate_dataset()
    batches = ds.train_set.shuffle(buffer_size=10000, seed=config.seed).batch(batch_size=config.batch_size)
    rows = []
    for inp, tar, meta in batches:
        a, b, m, row0 = dp.shard_batch_indices(inp, tar, meta, r, w)
        rows.append((row0, a.tolist(), b.tolist(), inp.tolist(), tar.tolist()))
    np.save(os.path.join(out_dir, 'cli%d.npy' % rank), np.array(rows, dtype=object), allow_pickle=True)
    dist.destroy_process_group()


@pytest.mark.timeout(300)
@pytest.mark.parametrize('extra', [['--nn_type', 'RNNUqRangeEstimate', '--UQ=True'],
                                   ['--forecast_steps', '2', '--forecast_steps_weights', '1.0-0.5'],
                                   ['--nn_type', 'RNNUqRangeEstimate', '--UQ=True', '--forecast_steps', '2',
                                    '--forecast_steps_weights', '1.0-0.5']])
def test_cli_sharding_covers_every_global_batch_exactly_once(tmp_path, extra):
    from lfm_quant_b200.scripts.synthetic import write_open_dataset, write_system_test_conf
    write_open_dataset(str(tmp_path / 'datasets' / 'open-dataset.dat'), n_keys=30, n_months=420, seed=9)
    write_system_test_conf(str(tmp_path / 'config' / 'system-test.conf'), str(tmp_path / 'datasets'),
                           str(tmp_path / 'experiments'))
    world = 2
    mp.spawn(_cli_worker, args=(world, _free_port(), str(tmp_path), extra), nprocs=world, join=True)
    per_rank = [np.load(str(tmp_path / ('cli%d.npy' % r)), allow_pickle=True) for r in range(world)]
    assert len(per_rank[0]) == len(per_rank[1]) > 1
    for bi in range(len(per_rank[0])):
        full_inp, full_tar = per_rank[0][bi][3], per_rank[0][bi][4]
        expect_row0, inp, tar = 0, [], []
        for r in range(world):
            row0, a, b, fi, ft = per_rank[r][bi]
            assert fi == full_inp and ft == full_tar            # every rank walks the same global batch
            assert row0 == expect_row0
            expect_row0 += len(a)
            inp += a
            tar += b
        assert inp == full_inp and tar == full_tar              # the shards tile it in order, each row once
