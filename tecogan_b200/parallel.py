"""Data parallelism over clips (SURVEY 8e): one process per GPU, clips sharded over ranks, ONE all-reduce per training
step on a flat bucket [G grads | FNet grads | D grads | control + loss scalars].  Inference needs no communication.
Pure torch.distributed plumbing -- works with NCCL on GPUs and with gloo on CPU tensors (tests)."""
import torch
import torch.distributed as dist


def world():
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def shard_clips(n_clips, rank=None, world_size=None):
    """Contiguous, balanced shard [begin, end) of n_clips independent clips for this rank."""
    if rank is None:
        rank, world_size = world()
    base, rem = divmod(n_clips, world_size)
    begin = rank * base + min(rank, rem)
    return begin, begin + base + (1 if rank < rem else 0)


def gather_ranks(bucket):
    """[world, n] tensor whose row r is rank r's `bucket` (the same on every rank)."""
    _, w = world()
    out = torch.empty((w,) + tuple(bucket.shape), device=bucket.device, dtype=bucket.dtype)
    dist.all_gather(list(out.unbind(0)), bucket)
    return out


def allreduce_bucket(bucket):
    """Sum `bucket` over all ranks in place (the single collective of a training step).  Returns 1/world, the scale that
    turns the sums into means (applied inside the fused Adam kernel and to the scalars).  In deterministic mode
    (config.set_deterministic) the ranks' buckets are gathered and summed in rank order (teco_sum_ranks_f32), so every
    rank holds the same bits and a rerun at the same rank count reproduces them; otherwise NCCL sums in its own order."""
    _, w = world()
    if w > 1:
        from . import config
        if config.deterministic():
            from . import kernels as K
            K.sum_ranks(gather_ranks(bucket), out=bucket)
        else:
            dist.all_reduce(bucket, op=dist.ReduceOp.SUM)
    return 1.0 / w


def decide_with_d(tb_ema, t_balance_mean, dbalance):
    """Adaptive-D branch of reference lib/Teco.py:415-417,493-494: the predicate reads the EMA *before* this step's
    update.  Both inputs are identical on every rank (t_balance travels in the all-reduced bucket), so ranks never
    disagree on whether D is updated.  Returns (with_d, new_ema)."""
    return (tb_ema < dbalance), 0.99 * tb_ema + 0.01 * t_balance_mean
