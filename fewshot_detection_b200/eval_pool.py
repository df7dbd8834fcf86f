"""The detection pool of the device evaluators (voc_eval.DeviceVocEval, coco_eval.DeviceCocoEval).

An evaluator accumulates, on its device, one record per kept detection (`key`, `box`) and one group descriptor per
(image, class) row of every batch added (`groups`: first record, record count, image index, class), with counters
[records, groups, first group of the last batch, error flags].  The two metrics differ only in the record key (VOC: an
int32 rank key, COCO: a float64 score), in how many records a row may add, and in the kernels that gather and score;
everything else lives here: the image index, capacity growth, the argument checks of `add`, and the merging of several
pools in order, on one device (`merge`) or over the ranks of a process group (`gather`, see shard.py).

Every C call of both evaluators goes through `_call`, `_call_size` and `_stream` of this module.
"""


def _call(name, *args):
    from ._lib import call
    return call(name, *args)


def _call_size(name, *args):
    from ._lib import lib
    return int(getattr(lib, name)(*args))


def _ptr(t):
    return None if t is None else t.data_ptr()


def _stream(device=None):
    import torch
    return torch.cuda.current_stream(device).cuda_stream


def _is_merged(dets):
    from .utils import MergedDetections
    return isinstance(dets, MergedDetections)


def check_pool_flags(flags):
    """Raise on the error bits the gather / merge kernels leave in counters[3]."""
    if flags & 1:
        raise RuntimeError('detection pool overflow')
    if flags & 2:
        raise RuntimeError('merged pools: an image was evaluated on two ranks')
    if flags & 4:
        raise RuntimeError('merged pools: a group outside its pool')


class DetectionPool(object):
    """Base of the device evaluators.  A subclass sets KEY_DTYPE (torch dtype name of `key`) and MERGE_FN (its
    fsdet_*_merge entry point), builds its ground-truth tables, and implements `_gather` (one batch's C call) and
    `result`; `_row_bound` is the most records one (image, class) row may add."""
    KEY_DTYPE = MERGE_FN = None

    def __init__(self, classes, imagenames, device=None):
        import torch
        self.classes, self.imagenames = list(classes), list(imagenames)
        self.index = dict((n, k) for k, n in enumerate(self.imagenames))
        if len(self.index) != len(self.imagenames):
            raise ValueError('image names must be distinct')
        self.device = torch.device(device) if device is not None else torch.device('cuda', torch.cuda.current_device())
        self.group_cap = len(self.classes) * len(self.imagenames)
        self.groups = torch.zeros(max(self.group_cap, 1), 4, dtype=torch.int32, device=self.device)
        self.counters = torch.zeros(4, dtype=torch.int64, device=self.device)
        self.pool_cap = 0
        self.key = self.box = None
        self._known, self._pending = 0, 0          # records at the last read of counters[0], upper bound added since
        self._added = set()
        self.last = None

    def empty_like(self):
        """A new evaluator over the same classes, image set, ground truth and device, with no detections."""
        import copy
        import torch
        ev = copy.copy(self)
        ev.groups = torch.zeros_like(self.groups)
        ev.counters = torch.zeros_like(self.counters)
        ev.pool_cap, ev.key, ev.box = 0, None, None
        ev._known, ev._pending, ev._added, ev.last = 0, 0, set(), None
        return ev

    def _reserve(self, bound):
        """Room for `bound` more records.  Reads the record count (8 bytes) only when the upper bound could overflow."""
        import torch
        if self._known + self._pending + bound <= self.pool_cap:
            self._pending += bound
            return
        self._known, self._pending = int(self.counters[0]), 0
        if self._known + bound > self.pool_cap:
            cap = min(max(1 << 20, 2 * self.pool_cap, 8 * bound, self._known + bound), 2 ** 31 - 1)
            if self._known + bound > cap:
                raise RuntimeError('more than 2^31 - 1 detections')
            key = torch.empty(cap, dtype=getattr(torch, self.KEY_DTYPE), device=self.device)
            box = torch.empty(cap, 4, dtype=torch.float64, device=self.device)
            if self._known:
                key[:self._known].copy_(self.key[:self._known])
                box[:self._known].copy_(self.box[:self._known])
            self.key, self.box, self.pool_cap = key, box, cap
        self._pending = bound

    def _row_bound(self, cap):
        return cap

    def add(self, dets, image_indices, sizes):
        """dets: utils.Detections of one batch after .nms(), or utils.MergedDetections of a test-time augmentation plan
        after .nms(); image_indices[b]: position in `imagenames` (or the name) of image b; sizes[b] = (width, height)."""
        import torch
        n_cls = len(self.classes)
        if dets.keep is None:
            raise ValueError('Detections.nms() has not been run')
        if dets.nC != 1:
            raise ValueError('rows with %d class scores: only the meta detector (nC = 1) is supported' % dets.nC)
        if dets.N % n_cls:
            raise ValueError('%d rows are not images x %d classes' % (dets.N, n_cls))
        bs = dets.N // n_cls
        idx = [self.index[i] if isinstance(i, str) else int(i) for i in image_indices]
        if len(idx) != bs or len(sizes) != bs:
            raise ValueError('%d images in the batch, %d indices, %d sizes' % (bs, len(idx), len(sizes)))
        for i in idx:
            if not 0 <= i < len(self.imagenames):
                raise IndexError('image index %d outside the image set' % i)
            if i in self._added:
                raise ValueError('image %s added twice' % self.imagenames[i])
            self._added.add(i)
        if bs == 0:
            return
        cap = dets.cap if _is_merged(dets) else dets.A * dets.H * dets.W
        self._reserve(dets.N * self._row_bound(cap))
        idx_t = torch.tensor(idx, dtype=torch.int32).to(self.device)
        size_t = torch.tensor([[float(w), float(h)] for w, h in sizes], dtype=torch.float64).to(self.device)
        self._gather(dets, cap, idx_t, size_t)

    def _gather(self, dets, cap, image_index, image_size):
        """Append the batch's records and groups to the pool (one C call on the current stream; the *_merged entry
        point for MergedDetections)."""
        raise NotImplementedError

    def _merge_into(self, counters, key, box, groups, total):
        """Write the stacked pools of R sources (counters [R, 4] int64, key [R, P], box [R, P, 4], groups [R, G, 4], all
        on this evaluator's device) into this empty evaluator; `total` = the sum of the sources' record counts."""
        import torch
        n_src, stride_p, stride_g = int(counters.size(0)), int(key.size(1)), int(groups.size(1))
        self._reserve(total)
        ws = torch.empty(_call_size('fsdet_eval_merge_workspace_bytes', n_src, len(self.imagenames)),
                         dtype=torch.uint8, device=self.device)
        _call(self.MERGE_FN, n_src, _ptr(counters), _ptr(key), _ptr(box), stride_p, _ptr(groups), stride_g,
              len(self.imagenames), _ptr(ws), ws.numel(), _ptr(self.key), _ptr(self.box), self.pool_cap,
              _ptr(self.groups), self.group_cap, _ptr(self.counters), _stream(self.device))
        return self

    @classmethod
    def merge(cls, evaluators):
        """One evaluator with the detections of `evaluators` (same class, image set and device) in their order: the
        pool a single evaluator would hold had it been given their batches in that order."""
        import torch
        evs = list(evaluators)
        if not evs:
            raise ValueError('nothing to merge')
        counters = torch.stack([e.counters for e in evs])
        host = counters.cpu()
        P, G = max(1, int(host[:, 0].max())), max(1, int(host[:, 1].max()))
        key = torch.zeros(len(evs), P, dtype=getattr(torch, evs[0].KEY_DTYPE), device=evs[0].device)
        box = torch.zeros(len(evs), P, 4, dtype=torch.float64, device=evs[0].device)
        groups = torch.zeros(len(evs), G, 4, dtype=torch.int32, device=evs[0].device)
        for r, e in enumerate(evs):
            n, g = int(host[r, 0]), int(host[r, 1])
            if n:
                key[r, :n].copy_(e.key[:n])
                box[r, :n].copy_(e.box[:n])
            if g:
                groups[r, :g].copy_(e.groups[:g])
        dst = evs[0].empty_like()
        for e in evs:
            dst._added |= e._added
        return dst._merge_into(counters, key, box, groups, int(host[:, 0].sum()))

    def gather(self, process_group=None, dst=0, **result_kwargs):
        """Collective over `process_group`: every rank's pool, in rank order, merged into a new evaluator on rank `dst`
        (a rank of the group) and scored there once with result(**result_kwargs); every rank returns that dict.  The
        counts are all-gathered first; the padded records and groups then go to `dst` alone.  An error of the scoring
        on `dst` (for example a pool flag) is broadcast instead and raised on every rank."""
        import torch
        import torch.distributed as dist
        from .shard import all_gather_padded, gather_padded, global_rank, group_info
        world, rank = group_info(process_group)
        counters = all_gather_padded(self.counters.reshape(1, 4), 1, process_group).reshape(world, 4)
        host = counters.cpu()
        P, G = max(1, int(host[:, 0].max())), max(1, int(host[:, 1].max()))
        n, g = int(host[rank, 0]), int(host[rank, 1])
        empty_key = torch.zeros(0, dtype=getattr(torch, self.KEY_DTYPE), device=self.device)
        key = gather_padded(self.key[:n] if n else empty_key, P, process_group, dst)
        box = gather_padded(self.box[:n] if n else torch.zeros(0, 4, dtype=torch.float64, device=self.device), P,
                            process_group, dst)
        groups = gather_padded(self.groups[:g], G, process_group, dst)
        status = [None]
        if rank == dst:
            merged = self.empty_like()._merge_into(counters, key, box, groups, int(host[:, 0].sum()))
            try:
                status = [('ok', merged.result(**result_kwargs))]
            except Exception as e:                    # every rank raises, none waits in the broadcast
                status = [('error', '%s: %s' % (type(e).__name__, e))]
        dist.broadcast_object_list(status, src=global_rank(process_group, dst), group=process_group)
        outcome, value = status[0]
        if outcome == 'error':
            raise RuntimeError(value)
        return value
