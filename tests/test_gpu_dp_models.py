"""Data-parallel steps of RNNUqRangeEstimate and of multi-step forecasts, checked on one GPU: one global batch is split
into R uneven row shards (R = 3 leaves one shard empty), each shard runs its backward on the same handles with the
global batch's loss denominators and its own global row0, and the packed vectors (every stage's gradients and reduced
loss tail) are summed as the all-reduce would.  The sum must equal the packed vector of the whole-batch backward, and
the apply on it must give the whole-batch step's weights."""
import numpy as np
import pytest
import torch

import lfm_oracle as orc
import uq_chain_oracle as uco
from util import rel_err

pytestmark = pytest.mark.gpu
KW = dict(target_idx=1, target_lambda=0.5, rnn_lambda=0.7)
DROP = dict(dropout=0.2, recurrent_dropout=0.15, seed=31)
STEP, ROW0, LR = 3, 17, 0.6


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()


def _shards(B, R):
    cuts = [0, B // 3, B] if R == 2 else [0, B // 4, B // 4, B]      # uneven; with R = 3 the middle shard is empty
    return list(zip(cuts[:-1], cuts[1:]))


def _engine(B, T, F, O, H, L, S, uq, cell, weights):
    from lfm_quant_b200.engine import ForecastChainEngine
    return ForecastChainEngine(forecast_steps=S, weights=weights, max_batch=B, seq_len=T, n_inputs=F, n_outputs=O,
                               num_hidden=H, num_layers=L, rnn_cell=cell, uq=uq, train=True, max_grad_norm=0.5,
                               max_norm=0.8, **KW, **DROP)


def _problem(B, T, F, O, H, L, S, uq, cell, seed):
    rng = np.random.RandomState(seed)
    if uq:
        P = uco.init_params(L, F, O, H, S, init_scale=0.5, seed=seed + 1, dtype=np.float64, rnn_cell=cell)
    else:
        P = orc.init_forecast_params(L, F, O, H, S, init_scale=0.5, seed=seed + 1, dtype=np.float64, rnn_cell=cell)
    P = [(p + rng.normal(size=p.shape) * 0.05).astype(np.float32) for p in P]
    x = rng.normal(size=(B, T, F)).astype(np.float32)
    ys = [rng.normal(size=(B, T, O)).astype(np.float32) for _ in range(S)]
    if not uq:                    # masked rows: the point loss's mask count differs from B * T (a uq loss would be NaN)
        for s, y in enumerate(ys):
            y[s, :2, :] = 0.0
            y[B - 1 - s, 0, :] = 0.0
    return P, x, ys


def _segments(eng):
    """(gradient slice, tail slice) of every stage in the packed vector."""
    k = 3 if eng.uq else 2
    out, off = [], 0
    for e in eng.stages:
        out.append((slice(off, off + e.n_trainable), slice(off + e.n_trainable, off + e.n_trainable + k)))
        off += e.n_trainable + k
    return out


def _run(B, T, F, O, H, L, S, uq, cell, R, single):
    """single: one uq handle through lfmq_backward / lfmq_mask_count_uq (a chain of one stage packs it); otherwise the
    chain through lfmq_chain_backward_dp / lfmq_chain_mask_count."""
    w = [1.0, 0.5, 0.25][:S]
    P, x, ys = _problem(B, T, F, O, H, L, S, uq, cell, seed=7 + S + R)
    eng = _engine(B, T, F, O, H, L, S, uq, cell, w)
    eng.set_weights(P)
    xd, yd = _cuda(x), [_cuda(y) for y in ys]
    e0 = eng.stages[0]
    k = 3 if uq else 2
    assert eng.n_packed == sum(e.n_trainable + k for e in eng.stages)

    def counts(a, b):
        if single:
            return e0.mask_count_uq(yd[0][a:b].contiguous())
        return eng.mask_count([y[a:b].contiguous() for y in yd])

    shards = _shards(B, R)
    glob = sum(counts(a, b) for a, b in shards if b > a)
    whole_counts = counts(0, B)
    assert torch.equal(glob, whole_counts)
    total = torch.zeros(eng.n_packed, dtype=torch.float32, device='cuda')
    for a, b in shards:
        if b == a:                # a rank without rows contributes a zero vector
            continue
        xs, yss = xd[a:b].contiguous(), [y[a:b].contiguous() for y in yd]
        if single:
            e0.backward(xs, yss[0], step=STEP, row0=ROW0 + a, denom=glob)
        else:
            eng.backward_dp(xs, yss, glob, step=STEP, row0=ROW0 + a)
        total += eng.pack()
    if single:
        e0.backward(xd, yd[0], step=STEP, row0=ROW0)
        whole_out = None
    else:
        whole_out = eng.backward(xd, yd, step=STEP, row0=ROW0).cpu().numpy()
    whole = eng.pack().clone()
    tot, ref = total.cpu().numpy(), whole.cpu().numpy()
    assert np.isfinite(ref).all()
    for s, (g, t) in enumerate(_segments(eng)):
        assert rel_err(tot[g], ref[g]) < 1e-5, s
        assert tot[t] == pytest.approx(ref[t], rel=1e-5), s

    # the same step from the reduced vector on fresh handles: unpack, then the joint clip, optimizer and MaxNorm
    eng.apply(LR, STEP)
    after = [e.params.clone() for e in eng.stages]
    for vec, exact in ((whole, True), (total, False)):
        other = _engine(B, T, F, O, H, L, S, uq, cell, w)
        other.set_weights(P)
        out = torch.empty(k, dtype=torch.float32, device='cuda')
        other.unpack(vec, out)
        other.apply(LR, STEP)
        for s, (e, a) in enumerate(zip(other.stages, after)):
            if exact:             # one unpack + lfmq_chain_apply == lfmq_chain_apply on the per-stage buffers
                assert torch.equal(e.params, a), s
            else:
                assert float((e.params - a).abs().max()) < 1e-6, s
        if whole_out is not None:
            assert out.cpu().numpy() == pytest.approx(whole_out, rel=1e-5)
        other.close()
    eng.close()


@pytest.mark.parametrize('R', [2, 3])
@pytest.mark.parametrize('cell', ['lstm', 'gru'])
def test_uq_shards_sum_to_the_whole_batch_step(cell, R):
    _run(B=29, T=6, F=8, O=4, H=16, L=2, S=1, uq=True, cell=cell, R=R, single=True)


@pytest.mark.parametrize('R', [2, 3])
@pytest.mark.parametrize('S', [2, 3])
def test_point_chain_shards_sum_to_the_whole_batch_step(S, R):
    _run(B=31, T=7, F=9, O=3, H=16, L=1, S=S, uq=False, cell='lstm', R=R, single=False)


@pytest.mark.parametrize('R', [2, 3])
@pytest.mark.parametrize('S', [2, 3])
def test_uq_chain_shards_sum_to_the_whole_batch_step(S, R):
    _run(B=26, T=6, F=8, O=4, H=16, L=1 if S == 3 else 2, S=S, uq=True, cell='gru' if S == 3 else 'lstm', R=R,
         single=False)


def test_uq_engine_train_step_dp_without_rows_and_the_packed_tail():
    """The single-step uq engine's packed vector carries {uq_loss, mse_0, uq_loss_last_tar}, not grad_norm or
    clip_scale; a rank with no rows sends zeros.  One process plays world size 1 of a gloo group."""
    import os
    import tempfile
    import torch.distributed as dist
    from lfm_quant_b200.engine import ForecasterEngine
    B, T, F, O, H, L = 12, 5, 6, 3, 8, 1
    P, x, ys = _problem(B, T, F, O, H, L, 1, True, 'lstm', seed=3)
    mk = lambda: ForecasterEngine(max_batch=B, seq_len=T, n_inputs=F, n_outputs=O, num_hidden=H, num_layers=L,
                                  uq=True, train=True, max_grad_norm=0.5, **KW, **DROP)
    a, b = mk(), mk()
    a.set_weights(P)
    b.set_weights(P)
    init = tempfile.mktemp()
    dist.init_process_group('gloo', init_method='file://' + init, rank=0, world_size=1)
    try:
        xd, yd = _cuda(x), _cuda(ys[0])
        got = a.train_step_dp(xd, yd, 0, LR, 0, a.loss_counts(yd)).cpu().numpy()
        ref = b.train_step(xd, yd, 0, LR).cpu().numpy()
        assert got == pytest.approx(ref, rel=1e-6)
        assert torch.equal(a.params, b.params)
        assert a._dp.flat.numel() == a.n_trainable + 3
        flat = a._dp.flat.cpu().numpy()
        tail = a.grads[a.n_trainable:a.n_trainable + 5].cpu().numpy()
        assert list(flat[-3:]) == [tail[0], tail[1], tail[4]]
        out = a.train_step_dp(None, None, 1, LR, B, a.loss_counts(None)).cpu().numpy()
        assert (out == 0).all()
        b.grads[:b.n_trainable].zero_()                # the same apply on a zero gradient
        b.apply(LR, 1)
        assert torch.equal(a.params, b.params)
    finally:
        dist.destroy_process_group()
        os.path.exists(init) and os.remove(init)


def _cli_rank(rank, world, port, root, extra, model_dir):
    """One rank of `lfm_quant.py --train=True` under a launcher (world > 1) or alone (world = 1).  The ranks share one
    device through a gloo group: dp.init_from_env uses the group that is already there."""
    import os
    import torch.distributed as dist
    os.environ.update(LFM_QUANT_ROOT=root, LFMQ_SEEDED_SHUFFLE='1')
    torch.cuda.set_device(0)
    if world > 1:
        os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                          LOCAL_RANK='0')
        dist.init_process_group('gloo', rank=rank, world_size=world)
    from lfm_quant_b200.scripts import lfm_quant as cli
    conf = os.path.join(root, 'config', 'system-test.conf')
    cli.main(['--config=' + conf, '--train=True', '--model_dir', model_dir] + extra)
    if world > 1:
        dist.destroy_process_group()


@pytest.mark.timeout(600)
@pytest.mark.parametrize('extra', [['--nn_type', 'RNNUqRangeEstimate', '--UQ=True', '--dropout', '0.1'],
                                   ['--forecast_steps', '2', '--forecast_steps_weights', '1.0-0.5', '--dropout', '0.1'],
                                   ['--nn_type', 'RNNUqRangeEstimate', '--UQ=True', '--forecast_steps', '2',
                                    '--forecast_steps_weights', '1.0-0.5']],
                         ids=['uq', 'forecast2', 'uq-forecast2'])
def test_cli_two_ranks_train_the_one_rank_model(tmp_path, extra):
    """The CLI with two data-parallel ranks (gloo, both on this device) logs the 1-rank run's global losses and saves
    its weights."""
    import socket
    import pandas as pd
    import torch.multiprocessing as mp
    from lfm_quant_b200.scripts.synthetic import write_open_dataset, write_system_test_conf
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
    cols = ['mse', 'uq_loss'] if '--UQ=True' in extra else ['mse']
    for kind in ('batch', 'epoch'):
        one, two = (pd.read_csv(ex / m / 'train_log' / ('system-test-train-logs-%s.csv' % kind)) for m in ('one', 'two'))
        assert len(one) == len(two) > 1
        for c in cols:
            assert np.isfinite(two[c]).all()
            assert rel_err(two[c].values, one[c].values) < 1e-4, (kind, c)
    w1, w2 = (np.load(ex / m / 'chkpts' / 'chkpt.lfmq.npz') for m in ('one', 'two'))
    assert set(w1.files) == set(w2.files)
    for k in w1.files:
        assert rel_err(w2[k], w1[k]) < 1e-3, k
