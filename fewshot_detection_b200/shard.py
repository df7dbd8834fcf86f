"""Sharding of an evaluation pass over the ranks of a process group, with the same bits as one process.

Each rank runs a contiguous block of whole batches (`shard_range`), so every batch it runs is a batch the single
process would have run, with the same size and contents.  Ranks that run batches in rank order therefore see the
sample sequence of the single process cut into consecutive pieces, and the pieces are put back together in rank
order: the support vectors before the running mean (valid.sharded_ensemble_dynamic_weights) and the detection pools
of the device evaluators before scoring (`merge_pools`, `gather_pools`: csrc/voc_eval.cu / coco_eval.cu
fsdet_*_merge).
"""
from ._lib import call, ptr, lib


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


def _pool(ev):
    """The key (rank_key or score), box and group tensors of a DeviceVocEval / DeviceCocoEval."""
    return getattr(ev, ev.POOL_KEY), ev.box, ev.groups


def _merge_stacked(dst, counters, key, box, groups, total):
    """Write the stacked pools of R sources (counters [R, 4] int64, key [R, P], box [R, P, 4], groups [R, G, 4], all
    on dst's device) into the empty evaluator `dst`; `total` = the sum of the sources' record counts."""
    import torch
    n_src, stride_p, stride_g = int(counters.size(0)), int(key.size(1)), int(groups.size(1))
    dst._reserve(total)
    ws = torch.empty(int(lib.fsdet_eval_merge_workspace_bytes(n_src, len(dst.imagenames))), dtype=torch.uint8,
                     device=dst.device)
    dkey, dbox, dgroups = _pool(dst)
    call(dst.MERGE_FN, n_src, ptr(counters), ptr(key), ptr(box), stride_p, ptr(groups), stride_g, len(dst.imagenames),
         ptr(ws), ws.numel(), ptr(dkey), ptr(dbox), dst.pool_cap, ptr(dgroups), dst.group_cap, ptr(dst.counters),
         torch.cuda.current_stream(dst.device).cuda_stream)
    return dst


def merge_pools(evaluators):
    """One evaluator holding the detections of `evaluators` (same class, image set and device), in their order."""
    import torch
    evs = list(evaluators)
    if not evs:
        raise ValueError('nothing to merge')
    counters = torch.stack([e.counters for e in evs])
    host = counters.cpu()
    P, G = max(1, int(host[:, 0].max())), max(1, int(host[:, 1].max()))
    key = torch.zeros(len(evs), P, dtype=evs[0].POOL_KEY_DTYPE, device=evs[0].device)
    box = torch.zeros(len(evs), P, 4, dtype=torch.float64, device=evs[0].device)
    groups = torch.zeros(len(evs), G, 4, dtype=torch.int32, device=evs[0].device)
    for r, e in enumerate(evs):
        n, g = int(host[r, 0]), int(host[r, 1])
        ek, eb, eg = _pool(e)
        if n:
            key[r, :n].copy_(ek[:n])
            box[r, :n].copy_(eb[:n])
        if g:
            groups[r, :g].copy_(eg[:g])
    dst = evs[0].empty_like()
    for e in evs:
        dst._added |= e._added
    return _merge_stacked(dst, counters, key, box, groups, int(host[:, 0].sum()))


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


def gather_pools(ev, process_group=None, dst=0):
    """Collective over `process_group`: every rank's pool, in rank order, merged into a new evaluator on rank `dst`
    (a rank of the group).  Returns it on `dst`, None elsewhere.  The counts are all-gathered first; the padded
    records and groups then go to `dst` alone."""
    import torch
    world, rank = group_info(process_group)
    counters = all_gather_padded(ev.counters.reshape(1, 4), 1, process_group).reshape(world, 4)
    host = counters.cpu()
    P, G = max(1, int(host[:, 0].max())), max(1, int(host[:, 1].max()))
    n, g = int(host[rank, 0]), int(host[rank, 1])
    ek, eb, eg = _pool(ev)
    empty_key = torch.zeros(0, dtype=ev.POOL_KEY_DTYPE, device=ev.device)
    key = gather_padded(ek[:n] if n else empty_key, P, process_group, dst)
    box = gather_padded(eb[:n] if n else torch.zeros(0, 4, dtype=torch.float64, device=ev.device), P, process_group,
                        dst)
    groups = gather_padded(eg[:g], G, process_group, dst)
    if rank != dst:
        return None
    return _merge_stacked(ev.empty_like(), counters, key, box, groups, int(host[:, 0].sum()))


def gather_result(ev, process_group=None, dst=0, **result_kwargs):
    """gather_pools, `result(**result_kwargs)` once on `dst`, and the small result dict broadcast to every rank.  An
    error of the scoring on `dst` (for example a pool flag) is broadcast instead and raised on every rank."""
    import torch.distributed as dist
    merged = gather_pools(ev, process_group, dst)
    box = [None]
    if merged is not None:
        try:
            box = [('ok', merged.result(**result_kwargs))]
        except Exception as e:                        # every rank raises, none waits in the broadcast
            box = [('error', '%s: %s' % (type(e).__name__, e))]
    dist.broadcast_object_list(box, src=global_rank(process_group, dst), group=process_group)
    status, value = box[0]
    if status == 'error':
        raise RuntimeError(value)
    return value
