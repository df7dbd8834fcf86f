"""Data-parallel gradient exchange: ONE NCCL all-reduce (sum) over gradient
buckets, overlapped with the backward pass.

The reference's only multi-GPU path is single-process `nn.DataParallel`
(train_meta.py:137-141): replicate parameters, scatter inputs, gather outputs,
reduce gradients onto GPU 0 every step.  The H100-native equivalent is one
process per GPU with identical replicas and a single sum-all-reduce of the 66 M
fp32 gradients over NVLink / NVSwitch: no broadcast, no scatter, no gather.
Gradients are *summed* (the reference's losses are sums, region_loss.py:340-345,
and the driver divides lr by the global batch, train_meta.py:143-147).

All parameter gradients live in one flat fp32 buffer (so the collective works in
place, without packing copies); buckets are contiguous slices of it, ordered by
the time their last gradient is produced in the backward pass, and each
bucket's all-reduce is launched asynchronously as soon as it is complete.
"""
import torch
import torch.distributed as dist


class GradAllReducer(object):
    def __init__(self, model, bucket_mb=32, process_group=None):
        self.group = process_group
        self.params = [p for p in model.parameters() if p.requires_grad]
        for p in self.params:  # conv weights are stored OHWI (channels_last) by the engine
            if p.dim() == 4 and not p.is_contiguous(memory_format=torch.channels_last):
                p.data = p.data.contiguous(memory_format=torch.channels_last)
        # backward produces gradients roughly in reverse parameter order:
        # lay the flat buffer out in that order so that buckets fill front to back
        order = list(reversed(self.params))
        align = 32  # floats: every gradient view starts on a 128-byte boundary (kernels need 16-byte alignment)
        total = sum((p.numel() + align - 1) // align * align for p in order)
        dev = order[0].device
        self.flat = torch.zeros(total, dtype=torch.float32, device=dev)
        self.bucket_of = {}
        self.buckets = []  # [start, end, remaining, n_params]
        cap = int(bucket_mb * 1024 * 1024 // 4)
        off = 0
        cur_start, cur_n = 0, 0
        for p in order:
            n = p.numel()
            view = self.flat[off:off + n]
            if p.dim() == 4:
                g = view.view(p.shape[0], p.shape[2], p.shape[3], p.shape[1]).permute(0, 3, 1, 2)  # OHWI storage
            else:
                g = view.view(p.shape)
            p.grad = g
            p._fsdet_overwrite = True  # the engine may overwrite .grad in place (no accumulate)
            self.bucket_of[id(p)] = len(self.buckets)
            off += (n + align - 1) // align * align
            cur_n += 1
            if off - cur_start >= cap:
                self.buckets.append([cur_start, off, cur_n, cur_n])
                cur_start, cur_n = off, 0
        if cur_n:
            self.buckets.append([cur_start, off, cur_n, cur_n])
        self.handles = []
        self.overlap = True   # launch bucket all-reduces from inside backward (False: one call in finish())
        self.world = dist.get_world_size(self.group) if dist.is_initialized() else 1
        for r in (getattr(model, '_det', None), getattr(model, '_ler', None), getattr(model, '_net', None)):
            if r is not None:     # a single process has no collective to launch from the backward pass
                r.grad_hook = self.grad_ready if self.world > 1 else None

    def begin_step(self):
        for b in self.buckets:
            b[2] = b[3]
        self.handles = []

    def grad_ready(self, p):
        bi = self.bucket_of.get(id(p))
        if bi is None:
            return
        b = self.buckets[bi]
        b[2] -= 1
        if b[2] == 0 and self.world > 1 and self.overlap:
            self.handles.append(dist.all_reduce(self.flat[b[0]:b[1]], op=dist.ReduceOp.SUM, group=self.group,
                                                async_op=True))

    def finish(self):
        """Wait (on the compute stream) for every bucket launched during backward."""
        if self.world > 1 and not self.overlap:
            dist.all_reduce(self.flat, op=dist.ReduceOp.SUM, group=self.group)
        for h in self.handles:
            h.wait()
        self.handles = []
