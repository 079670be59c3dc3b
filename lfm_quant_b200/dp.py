"""Data parallelism over the company-batch axis (SURVEY section 8e): host-side plumbing shared by the handle engines'
train_step_dp (ForecasterEngine, DenseEngine), ForecastChainEngine.train_step_dp -- which every model object's step
goes through, delegating to the handle's own with one stage -- bench.py and the gloo tests.  One process per GPU;
exactly ONE collective on the data path per step -- the SUM all-reduce of the flat gradient (+ its loss / mse tail)
over NCCL for a point or dense handle; for chains and uq handles, of the packed vector of every stage's gradients and
loss tail."""
from __future__ import absolute_import, division, print_function

from ._native import TAIL_MSE0


def shard_rows(batch_global, rank, world):
    """Rank r takes rows [r*B/R, (r+1)*B/R) of each global batch; returns (row0, n_rows)."""
    base, rem = divmod(batch_global, world)
    n = base + (1 if rank < rem else 0)
    row0 = rank * base + min(rank, rem)
    return row0, n


def global_denominators(local_denom, dist):
    """{B_local, mask_count_local} -> {B_global, mask_count_global}, or any engine's loss_counts -> their sums over the
    ranks: the loss denominators are global (losses.py:87,90,131-135), so each rank scales dLoss/dpred with them before
    the gradient all-reduce.
    Targets only -- done once per batch when it is built, not on the step path."""
    out = local_denom.clone()
    dist.all_reduce(out, op=dist.ReduceOp.SUM)
    return out


def allreduce_flat_gradient(flat_grads, n_trainable, dist):
    """The single data-path collective: SUM over ranks of grads[0 : n_trainable + 2] (gradient, loss, mse_0).
    clip_by_global_norm, the optimizer and MaxNorm then run redundantly on every rank on the reduced gradient."""
    dist.all_reduce(flat_grads[:n_trainable + TAIL_MSE0 + 1], op=dist.ReduceOp.SUM)
    return flat_grads


def global_stage_counts(local_counts, dist):
    """Multi-step forecasts and RNNUqRangeEstimate: every forecast stage's {B, unmasked rows, unmasked last-step rows}
    ([S, 3], or the 3 counts of one uq handle) -> their sums over the ranks, in ONE all-reduce of the small vector.
    Each stage's loss takes its own denominators (losses.py:47-51,159-177); done once per batch when it is built."""
    assert local_counts.shape[-1] == 3, tuple(local_counts.shape)
    return global_denominators(local_counts, dist)


def allreduce_packed(flat, dist):
    """The single data-path collective of a chain or uq step: SUM over ranks of the packed vector, every stage's
    gradients followed by its loss tail -- {loss, mse_0}, or {uq_loss, mse_0, uq_loss_last_tar} on uq handles
    (ForecastChainEngine.pack).  grad_norm and clip_scale are not in it: the apply computes them afterwards."""
    dist.all_reduce(flat, op=dist.ReduceOp.SUM)
    return flat


def init_from_env():
    """(rank, world) of this process.  Under ``torchrun`` (WORLD_SIZE > 1) the default process group is created on first
    use -- NCCL when CUDA is present (one process per GPU, LOCAL_RANK selects the device), gloo otherwise -- so that
    ``lfm_quant.py --config ... --train=True`` launched with ``torchrun --nproc-per-node N`` trains ONE model data-parallel
    over the company-batch axis instead of N replicas.  Without torchrun: (0, 1) and nothing is initialised."""
    import os
    world = int(os.environ.get('WORLD_SIZE', '1'))
    if world <= 1:
        return 0, 1
    import torch
    import torch.distributed as dist
    if not dist.is_initialized():
        os.environ.setdefault('MASTER_ADDR', '127.0.0.1')
        if torch.cuda.is_available():
            local = int(os.environ.get('LOCAL_RANK', '0'))
            torch.cuda.set_device(local)
            dist.init_process_group('nccl', device_id=torch.device('cuda', local))
        else:
            dist.init_process_group('gloo')
    return dist.get_rank(), dist.get_world_size()


def shard_batch_indices(inp_idx, tar_idx, meta, rank, world):
    """This rank's rows of one global batch of window indices (data_processing.py:267-281 triples), with the global row
    offset of its first row (keys the dropout streams, so masks do not depend on the GPU count)."""
    row0, n = shard_rows(len(inp_idx), rank, world)
    return inp_idx[row0:row0 + n], tar_idx[row0:row0 + n], meta[row0:row0 + n], row0
