"""Sharding of an evaluation pass over the ranks of a process group, with the same bits as one process.

Each rank runs a contiguous block of whole batches (`shard_range`), so every batch it runs is a batch the single
process would have run, with the same size and contents.  Ranks that run batches in rank order therefore see the
sample sequence of the single process cut into consecutive pieces, and the pieces are put back together in rank
order: the support vectors before the running mean (valid.sharded_ensemble_dynamic_weights) and the detection pools
of the device evaluators before scoring (eval_pool.DetectionPool.gather).  This module holds the shard plan and the
collectives they use.
"""


def shard_range(n_items, batch_size, world, rank):
    """[start, stop) of the items rank `rank` of `world` runs: ceil(batches / world) whole batches of `batch_size` per
    rank, in order.  The partial last batch lands on the last rank that gets work; trailing ranks may get none."""
    if batch_size <= 0 or world <= 0 or not 0 <= rank < world:
        raise ValueError('bad shard: %d items, batch %d, rank %d of %d' % (n_items, batch_size, rank, world))
    n_batches = -(-n_items // batch_size)
    per = -(-n_batches // world)
    b0 = min(rank * per, n_batches)
    b1 = min(b0 + per, n_batches)
    return min(b0 * batch_size, n_items), min(b1 * batch_size, n_items)


def group_info(process_group=None):
    import torch.distributed as dist
    return dist.get_world_size(process_group), dist.get_rank(process_group)


def global_rank(process_group, r):
    import torch.distributed as dist
    return r if process_group is None else dist.get_global_rank(process_group, r)


def all_gather_padded(t, rows, process_group=None):
    """Every rank's `t` ([n_r, ...], n_r <= rows) as one [world, rows, ...] tensor, zero padded."""
    import torch
    import torch.distributed as dist
    world, _ = group_info(process_group)
    pad = torch.zeros((rows,) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
    if t.size(0):
        pad[:t.size(0)].copy_(t)
    out = torch.empty((world * rows,) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
    dist.all_gather_into_tensor(out, pad, group=process_group)
    return out.view((world, rows) + tuple(t.shape[1:]))


def gather_padded(t, rows, process_group=None, dst=0):
    """Every rank's `t` ([n_r, ...], n_r <= rows), zero padded, as one [world, rows, ...] tensor on rank `dst` (a
    rank of the group); None on the other ranks.  Only `dst` holds the world's buffers."""
    import torch
    import torch.distributed as dist
    world, rank = group_info(process_group)
    pad = torch.zeros((rows,) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
    if t.size(0):
        pad[:t.size(0)].copy_(t)
    out = [torch.empty_like(pad) for _ in range(world)] if rank == dst else None
    dist.gather(pad, out, dst=global_rank(process_group, dst), group=process_group)
    return torch.stack(out) if rank == dst else None


def rank0_first(fn, process_group=None):
    """fn() on rank 0 of the group, then on the others: for work that creates a shared file (an annotation cache)
    which the other ranks then read."""
    import torch.distributed as dist
    _, rank = group_info(process_group)
    if rank != 0:
        dist.barrier(group=process_group)
    r = fn()
    if rank == 0:
        dist.barrier(group=process_group)
    return r
