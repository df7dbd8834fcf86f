"""CUDA-graph capture of the whole meta-training step, and of the detection pass (GraphedDetect, at the end).

The eager step issues ~3,000 kernel launches through ctypes (tens of ms of host time per step at config 2, about
as long as the GPU work).  `GraphedTrainStep` captures forward + RegionLoss(V2) + backward (+ the gradient
all-reduce) + SGD once per (input shape, warm-up regime) into a CUDA graph and replays it: the host cost drops to a
few launches and the GPU runs back to back.

Semantics kept from the eager loop (train_meta.py:201-226):
  * inputs are copied into static device buffers before each replay (the query batch, the support images/masks and
    the float64 target tensor);
  * negative-row sampling (`cfg.neg_ratio` = 1 for base training, 0 for fine-tuning; region_loss.py:15-34) stays on
    the host with the reference's `random()` draws: `RegionLoss.stage_filter` uploads the kept rows / per-image
    prefix / live-row count into fixed-capacity device buffers before the replay and the loss kernels - launched for
    all rows - skip the dead slots, so ONE graph serves every outcome of the draw;
  * multi-scale training (dataset.py:223-245 re-draws the input side every 64 samples, 320...608): one graph per
    input shape, all captured into one shared memory pool (the step's activations are dead at the end of a step, so
    the graphs can reuse each other's memory; only their static inputs / loss stay reserved);
  * the learning-rate schedule keeps working: lr / momentum / weight decay are read by the fused SGD kernel from
    device memory (`FusedSGD.sync_hyper`);
  * `region_loss.seen` only selects the warm-up branch of build_targets (seen < 12800): part of the cache key;
  * multi-GPU: the bucketed gradient all-reduce (NCCL, summed) is captured INSIDE the graph, launched from the
    backward pass on NCCL's stream as soon as a bucket's last weight gradient is enqueued (fork / join edges in the
    graph), so it overlaps the rest of the backward pass; SGD follows the join.  If the collective cannot be captured
    (old NCCL) the step falls back to backward-graph | all-reduce | SGD-graph.
Requirements: fixed shapes per cache entry, at least one eager step done before capture (lazy initialisation and the
momentum buffers must exist), the CPU label tensor when neg_ratio is numeric (the reference keeps it on the host too).
"""
import collections

import torch

from .cfg import cfg
from .distributed import GradAllReducer


class _Entry(object):
    __slots__ = ('graph_fb', 'graph_opt', 'static', 'loss', 'loss_static', 'counters')


class GraphedTrainStep(object):
    def __init__(self, model, region_loss, optimizer, reducer=None, max_graphs=12, strict=True):
        self.model, self.loss_mod, self.opt = model, region_loss, optimizer
        self.reducer = reducer if reducer is not None else GradAllReducer(model)
        self.entries = collections.OrderedDict()       # key -> _Entry (LRU)
        self.max_graphs = max_graphs
        self.pool = None                               # shared by all captures
        self.loss = None
        self.captures = 0
        self._chk = None                               # (pinned counters, event, armed): degenerate-label check, one step late
        self.in_graph_allreduce = None                 # None = try to capture the collective, False = known not to work
        # 'thread_local': other host threads (the input pipeline's background preparation, pinned-memory bookkeeping)
        # may keep calling CUDA while this thread captures - the default 'global' mode turns any such call into a
        # capture error
        self.capture_error_mode = 'thread_local'
        self.strict = strict                           # False: fall back to eager launches if a capture fails
        self.capture_failed = None
        self.stepped = False                           # has this object run a step yet (see __call__)

    # ------------------------------------------------------------------ eager (very first step)
    def _eager(self, x, metax, mask, target):
        self.reducer.begin_step()
        out = self.model(x, metax, mask)
        loss = self.loss_mod(out, target)
        loss.backward()
        self.reducer.finish()
        self.opt.step()
        # detached: a loss that still references its autograd graph keeps the parameters' AccumulateGrad nodes alive,
        # and those remember the stream they were created on - a later capture on another stream would then make the
        # autograd engine wait on uncaptured work (cudaErrorStreamCaptureIsolation)
        return loss.detach()

    # ------------------------------------------------------------------ capture
    def _key(self, x, metax, target):
        return (tuple(x.shape), tuple(metax.shape), tuple(target.shape), self.loss_mod.seen < 12800, str(cfg.neg_ratio),
                getattr(self.model, 'replicas', 1))

    def _capture(self, key, x, metax, mask, target):
        dev = x.device
        e = _Entry()
        e.static = [t.detach().clone() for t in (x, metax, mask)] + [target.to(dev).clone()]
        self.loss_mod.verbose = False
        self.opt.capturable = True
        self.opt.sync_hyper()
        self.opt.prepare()
        sampled = cfg.neg_ratio != 'full'
        if target.dim() == 3:
            self.loss_mod.warm_caches(dev, target.size(0), target.size(1))
        else:
            self.loss_mod.warm_caches(dev)
        if sampled:
            rows = target.view(-1, target.size(-1)).size(0)
            bs = target.size(0) if target.dim() == 3 else 0
            e.loss_static = self.loss_mod.make_static(rows, bs, dev)
            import random as _random
            rng = _random.getstate()     # valid buffer contents for the capture run, without consuming the step's draws
            self.loss_mod.stage_filter(e.loss_static, target if not target.is_cuda else target.cpu())
            _random.setstate(rng)
        else:
            e.loss_static = None
        self.loss_mod.static = e.loss_static            # forward() takes the fixed-capacity form while this is set
        multi = self.reducer.world > 1
        two_graphs = multi and self.in_graph_allreduce is False
        torch.cuda.synchronize()

        def body(with_opt, overlap):
            self.reducer.overlap = overlap
            self.reducer.begin_step()
            out = self.model(*e.static[:3])
            loss = self.loss_mod(out, e.static[3])
            loss.backward()
            e.loss = loss.detach()
            if overlap:
                self.reducer.finish()          # join: the capturing stream waits for the bucket all-reduces
            if with_opt:
                self.opt.step()

        e.graph_opt = None
        e.graph_fb = torch.cuda.CUDAGraph()
        pool = self.pool
        try:
            try:
                with torch.cuda.graph(e.graph_fb, pool=pool, capture_error_mode=self.capture_error_mode):
                    body(with_opt=not two_graphs, overlap=multi and not two_graphs)
                if two_graphs:
                    if self.pool is None:
                        self.pool = e.graph_fb.pool()
                    e.graph_opt = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(e.graph_opt, pool=self.pool, capture_error_mode=self.capture_error_mode):
                        self.opt.step()
            except Exception as err:      # NCCL not capturable here: one exposed all-reduce between two graphs
                if not multi or self.in_graph_allreduce is False:
                    raise
                import sys
                sys.stderr.write('GraphedTrainStep: in-graph all-reduce unavailable (%r); falling back to two graphs\n' % (err,))
                self.in_graph_allreduce = False
                torch.cuda.synchronize()
                e.graph_fb = torch.cuda.CUDAGraph()
                with torch.cuda.graph(e.graph_fb, pool=pool, capture_error_mode=self.capture_error_mode):
                    body(with_opt=False, overlap=False)
                if self.pool is None:
                    self.pool = e.graph_fb.pool()
                e.graph_opt = torch.cuda.CUDAGraph()
                with torch.cuda.graph(e.graph_opt, pool=self.pool, capture_error_mode=self.capture_error_mode):
                    self.opt.step()
        finally:
            self.loss_mod.static = None
        if self.pool is None:
            self.pool = e.graph_fb.pool()
        e.counters = self.loss_mod.last['counters'] if self.loss_mod.last else None
        self.captures += 1
        self.entries[key] = e
        while len(self.entries) > self.max_graphs:
            self.entries.popitem(last=False)
        return e

    # ------------------------------------------------------------------ degenerate labels, two steps late
    def _check_and_arm(self, counters):
        """The kernel's degenerate-label counter (the reference raises `math domain error` there) is copied to pinned
        memory behind every replay and examined two steps later - by then the copy has long completed, so the host
        never waits for the GPU and the launch of the next step is not delayed."""
        if counters is None:
            return
        if self._chk is None:
            self._chk = [[torch.zeros(4, dtype=torch.int32).pin_memory(), torch.cuda.Event(), False] for _ in range(2)]
            self._turn = 0
        slot = self._chk[self._turn]
        if slot[2]:
            slot[1].synchronize()
            slot[2] = False
            self.loss_mod._raise_if_degenerate(slot[0])
        slot[0].copy_(counters, non_blocking=True)
        slot[1].record()
        slot[2] = True
        self._turn ^= 1

    def poll(self):
        """Examine the outstanding degenerate-label checks now (blocks until those steps have finished)."""
        for slot in (self._chk or []):
            if slot[2]:
                slot[1].synchronize()
                slot[2] = False
                self.loss_mod._raise_if_degenerate(slot[0])

    # ------------------------------------------------------------------ one step
    def __call__(self, x, metax, mask, target, target_host=None):
        """One training step. Returns the (static, device) loss tensor.  `target`: the float64 label tensor, on the
        host (the reference's convention) or on the device; with a numeric cfg.neg_ratio the host copy is needed for
        the row sampling - pass it as `target_host` when `target` is a device tensor."""
        if not self.stepped:
            # the first step of this object runs eagerly: it initialises lazily (weight plans, the momentum buffers of
            # a fresh run).  After a resume the momentum is loaded already, so it is a seasoned step, bit-equal to a
            # replay; the captures follow from the next call on
            self.stepped = True
            return self._eager(x, metax, mask, target)
        if self.capture_failed is not None:
            return self._eager(x, metax, mask, target)
        key = self._key(x, metax, target)
        e = self.entries.get(key)
        if e is None:
            try:
                e = self._capture(key, x, metax, mask, target)
            except Exception as err:
                if self.strict:
                    raise
                # a failed capture must not take the training run down: report it once and launch eagerly from now on
                import sys
                import traceback
                self.capture_failed = err
                sys.stderr.write('GraphedTrainStep: CUDA-graph capture failed, continuing with eager launches:\n%s\n'
                                 % ''.join(traceback.format_exception_only(type(err), err)))
                torch.cuda.synchronize()
                return self._eager(x, metax, mask, target)
        else:
            self.entries.move_to_end(key)
        for s, t in zip(e.static, (x, metax, mask, target)):
            s.copy_(t, non_blocking=True)
        if e.loss_static is not None:
            host_t = target_host if target_host is not None else (target if not target.is_cuda else target.cpu())
            self.loss_mod.stage_filter(e.loss_static, host_t)
        self.opt.sync_hyper()
        e.graph_fb.replay()
        if e.graph_opt is not None:
            self.reducer.overlap = False
            self.reducer.finish()          # one NCCL all-reduce over the flat gradient buffer
            e.graph_opt.replay()
        self._check_and_arm(e.counters)
        self.loss = e.loss
        return e.loss


# ---------------------------------------------------------------------------------------------------------------------
class _DetectEntry(object):
    __slots__ = ('graph', 'x', 'sizes', 'out')


class GraphedDetect(object):
    """valid.detect_images replayed as one CUDA graph per (batch, side): the query forward (detect_forward), the decode
    and NMS (fsdet_region_detect, fsdet_nms) and the per-image selection (fsdet_detect_select).

    The model must be in eval mode; its parameters and buffers are only read.  The reweighting vectors are copied
    once into a static buffer, the anchors are staged on the device once, and every call copies the batch and the
    image sizes into static buffers and replays.  A batch of fewer than `batch` images is padded to `batch` with zero
    images whose results are dropped; the forward's tiling depends on the batch size, so its results are those of the
    eager pass over the padded batch, which can differ in the last bits from an eager pass over the real images
    alone.  Each (batch, side) is run once eagerly (lazy planning) and then captured; the
    capture is strict: a host synchronisation or pageable copy inside the pass fails the capture instead of falling
    back to eager launches.

    `__call__(data, sizes)` returns a utils.ImageDetections over this graph's static result buffer: it is valid until
    the next call with the same side, so read it (`.lists()`) or copy it first."""

    def __init__(self, model, dynamic_weights, batch, side, n_cls, conf=0.5, nms=0.4, max_det=100):
        if model.training:
            raise ValueError('GraphedDetect needs the model in eval mode')
        self.model, self.batch, self.side = model, int(batch), int(side)
        self.n_cls, self.conf, self.nms, self.max_det = int(n_cls), float(conf), float(nms), int(max_det)
        self.device = next(model.parameters()).device
        dw = dynamic_weights if isinstance(dynamic_weights, (list, tuple)) else [dynamic_weights]
        self.dw = [t.detach().to(self.device, torch.float32).clone() for t in dw]
        if self.dw[0].size(0) != self.n_cls:
            raise ValueError('vectors for %d classes, n_cls = %d' % (self.dw[0].size(0), self.n_cls))
        self.anchors = torch.tensor([float(a) for a in model.anchors], dtype=torch.float32).to(self.device)
        self.entries = {}                              # (batch, side) -> _DetectEntry
        self.pool = None
        self.captures = 0
        self._capture((self.batch, self.side))

    def _pass(self, e):
        from . import valid as VA
        dets = VA.detect(self.model, e.x, self.dw, self.n_cls, self.conf, self.nms, anchors_dev=self.anchors)
        dets.select(self.n_cls, e.sizes, self.max_det, out=e.out)

    def _capture(self, key):
        from .utils import ImageDetections
        B, side = key
        e = _DetectEntry()
        e.x = torch.zeros(B, 3, side, side, dtype=torch.float32, device=self.device)
        e.sizes = torch.full((B, 2), side, dtype=torch.int32, device=self.device)
        e.out = ImageDetections.empty(B, self.max_det, self.device)
        self._pass(e)                                  # eager: the forward's per-shape plans are built here
        torch.cuda.synchronize()
        e.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(e.graph, pool=self.pool, capture_error_mode='thread_local'):
            self._pass(e)
        if self.pool is None:
            self.pool = e.graph.pool()
        self.captures += 1
        self.entries[key] = e
        return e

    def __call__(self, data, sizes):
        """data: float32 [b, 3, side, side] (b <= batch, any device), sizes: b (width, height) pairs."""
        b = int(data.size(0))
        if data.dim() != 4 or data.size(1) != 3 or data.size(2) != data.size(3):
            raise ValueError('data must be [b, 3, side, side], got %s' % (tuple(data.shape),))
        if not 0 < b <= self.batch or len(sizes) != b:
            raise ValueError('%d images and %d sizes for a batch of %d' % (b, len(sizes), self.batch))
        key = (self.batch, int(data.size(2)))
        e = self.entries.get(key)
        if e is None:
            e = self._capture(key)
        e.x[:b].copy_(data, non_blocking=True)
        if b < self.batch:
            e.x[b:].zero_()
        size_rows = [[int(w), int(h)] for w, h in sizes] + [[key[1], key[1]]] * (self.batch - b)
        e.sizes.copy_(torch.tensor(size_rows, dtype=torch.int32))   # pageable: the host list is free on return
        e.graph.replay()
        return e.out.narrow(b)
