"""Multi-GPU plumbing of the hot path: frames are independent (every KNN / gather stays inside
one batch item: NN/knn_.cxx:109-113, models/ffb6d.py:172-174), so ranks take disjoint frame
ranges and the only cross-rank traffic is the timing reduction of bench.py.  No data-path
collective exists ("replicas / weak scaling", SURVEY.md §8e).  Training is the one opt-in exception: a
model converted with ``nn.SyncBatchNorm.convert_sync_batchnorm`` gathers each BatchNorm layer's per-rank
moments and gradient sums with :func:`all_gather_rows` (ffb6d_b200.modules)."""
import torch
import torch.distributed as dist


def all_gather_rows(row, group, world):
    """``[world, n]``: the 1-D ``row`` of every rank of ``group`` in rank order.  ``all_gather_into_tensor``, or the
    list form on gloo, which lacks it (as torch's SyncBatchNorm does).  A gather rather than an all-reduce: the
    caller combines the rows in rank order, so the result does not depend on the backend's reduction order."""
    if dist.get_backend(group) == "gloo":
        parts = [torch.empty_like(row) for _ in range(world)]
        dist.all_gather(parts, row, group=group)
        return torch.stack(parts)
    out = torch.empty((world, row.numel()), dtype=row.dtype, device=row.device)
    dist.all_gather_into_tensor(out, row, group=group)
    return out


def frame_shard(frames_per_rank, rank, world):
    """Global frame ids of one rank under weak scaling: rank r owns [r*F, (r+1)*F)."""
    if not (0 <= rank < world):
        raise ValueError("rank %d outside world of %d" % (rank, world))
    return range(rank * frames_per_rank, (rank + 1) * frames_per_rank)


def split_frames(n_frames, rank, world):
    """Strong-scaling split of a fixed set of frames: contiguous, sizes differ by at most one."""
    base, rem = divmod(n_frames, world)
    lo = rank * base + min(rank, rem)
    return range(lo, lo + base + (1 if rank < rem else 0))


def max_over_ranks(values, device=None):
    """Element-wise max of a list of floats over all ranks (identity when not distributed)."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return list(values)
    t = torch.tensor(list(values), dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return t.tolist()


def sum_over_ranks(value, device=None):
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return value
    t = torch.tensor([value], dtype=torch.int64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return int(t.item())
