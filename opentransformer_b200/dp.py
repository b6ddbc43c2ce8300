"""Data-parallel plumbing for the hot path (SURVEY.md 8e): utterances are independent at inference,
so a batch list is sharded over ranks with NO collective on the data path; only results (token ids,
scores) are gathered for reporting.  torch.distributed is used as plumbing (NCCL on GPUs, gloo in the
CPU tests)."""
import torch
import torch.distributed as dist


def shard_range(n_items, rank, world):
    """Contiguous, balanced [lo, hi) slice of n_items for `rank` (sizes differ by at most one)."""
    base, rem = divmod(n_items, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def gather_variable(t, group=None):
    """all_gather of per-rank tensors whose first dimension differs (ids / scores of each rank's shard);
    returns the concatenation in rank order on every rank."""
    world = dist.get_world_size(group)
    n = torch.tensor([t.shape[0]], dtype=torch.int64, device=t.device)
    sizes = [torch.zeros_like(n) for _ in range(world)]
    dist.all_gather(sizes, n, group=group)
    m = int(max(int(s) for s in sizes))
    pad = torch.zeros((m,) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
    pad[:t.shape[0]] = t
    out = [torch.zeros_like(pad) for _ in range(world)]
    dist.all_gather(out, pad, group=group)
    return torch.cat([o[:int(s)] for o, s in zip(out, sizes)], 0)


def max_over_ranks(values, device, group=None):
    """Element-wise MAX of a list of python floats over ranks (device-time reporting rule)."""
    t = torch.tensor(values, dtype=torch.float64, device=device)
    if dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX, group=group)
    return t.tolist()


def allreduce_mean_(flat, group=None):
    """In-place mean over ranks of a flat gradient buffer: the single exchange step of synchronous data-parallel
    training (the reference's DistributedDataParallel, train/trainer.py:59-61).  No-op without a process group."""
    if not (dist.is_available() and dist.is_initialized()):
        return flat
    world = dist.get_world_size(group)
    if world > 1:
        dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
        flat.mul_(1.0 / world)
    return flat


def rank_in(group=None):
    """This process's rank in `group` (0 without a process group)."""
    if not (dist.is_available() and dist.is_initialized()):
        return 0
    return dist.get_rank(group)


def broadcast_from_first_(tensors, group=None):
    """In place: every rank takes the first rank's values of `tensors` (the model's buffers, as the reference's
    DistributedDataParallel broadcasts them from rank 0 before each forward).  No-op without a process group."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) < 2:
        return
    src = dist.get_global_rank(group, 0) if group is not None else 0
    for t in tensors:
        dist.broadcast(t, src=src, group=group)
