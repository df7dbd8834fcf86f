"""Fused multi-tensor SGD for the hot path's optimiser step.

`FusedSGD(params, lr, momentum, dampening, weight_decay)` has torch.optim.SGD's
constructor and `param_groups` semantics as used by the reference driver
(train_meta.py:143-163: lr rewritten every batch through
`param_group['lr']`, weight decay applied to every parameter), but `step()` is
ONE kernel launch over all parameter tensors (csrc/sgd.cu) instead of ~5
pointwise passes per tensor.  State: `state[p]['momentum_buffer']`, as torch.
"""
import torch

from ._lib import call, ptr
from .engine import same_layout

_CHUNK = 65536


class FusedSGD(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, momentum=0.0, dampening=0.0, weight_decay=0.0, nesterov=False):
        if nesterov:
            raise NotImplementedError('nesterov momentum is not used by the reference driver')
        defaults = dict(lr=lr, momentum=momentum, dampening=dampening, weight_decay=weight_decay)
        super(FusedSGD, self).__init__(params, defaults)
        self._tables = {}
        self._hyper = {}       # group index -> (device float[4], pinned host float[4]) for CUDA-graph mode
        self.capturable = False

    def _table(self, gi, plist):
        """Device pointer/size/chunk tables for one param group (rebuilt when any pointer changes)."""
        key = tuple((p.data_ptr(), p.grad.data_ptr(), self.state[p]['momentum_buffer'].data_ptr(), p.numel())
                    for p in plist)
        cached = self._tables.get(gi)
        if cached is not None and cached[0] == key:
            return cached[1]
        dev = plist[0].device
        pp = [k[0] for k in key]
        gp = [k[1] for k in key]
        mp = [k[2] for k in key]
        sz = [k[3] for k in key]
        ct, co = [], []
        for t, n in enumerate(sz):
            for off in range(0, n, _CHUNK):
                ct.append(t)
                co.append(off)
        tab = dict(
            params=torch.tensor(pp, dtype=torch.int64).to(dev), grads=torch.tensor(gp, dtype=torch.int64).to(dev),
            moms=torch.tensor(mp, dtype=torch.int64).to(dev), sizes=torch.tensor(sz, dtype=torch.int64).to(dev),
            chunk_tensor=torch.tensor(ct, dtype=torch.int32).to(dev),
            chunk_offset=torch.tensor(co, dtype=torch.int64).to(dev), n_chunks=len(ct))
        self._tables[gi] = (key, tab)
        return tab

    def prepare(self):
        """Build the device pointer tables now (they are uploaded with host->device copies, which must not happen
        inside a CUDA-graph capture). Needs gradients and momentum buffers to exist already."""
        for gi, group in enumerate(self.param_groups):
            plist = [p for p in group['params'] if p.grad is not None and 'momentum_buffer' in self.state[p]]
            if plist:
                self._table((gi, False), plist)

    def sync_hyper(self):
        """Graph mode: push lr / momentum / dampening / weight decay of every group to device memory
        (call outside the captured region, before each replay; a copy is issued only when a value changed)."""
        for gi, group in enumerate(self.param_groups):
            dev = group['params'][0].device
            vals = (float(group['lr']), float(group['momentum']), float(group['dampening']), float(group['weight_decay']))
            if gi not in self._hyper:
                self._hyper[gi] = [torch.zeros(4, device=dev), torch.zeros(4).pin_memory(), None]
            d, h, last = self._hyper[gi]
            if last != vals:
                torch.cuda.current_stream().synchronize()   # the previous async copy out of `h` must have completed
                for i, v in enumerate(vals):
                    h[i] = v
                d.copy_(h, non_blocking=True)
                self._hyper[gi][2] = vals

    @torch.no_grad()
    def load_state_dict(self, state_dict):
        """torch.optim.Optimizer.load_state_dict (the `state_dict()` layout is torch's), except that momentum is COPIED
        into the buffers that exist, bits unchanged: the device pointer tables and any captured step graph address those
        tensors, so swapping them would leave a graph updating freed memory.  A missing buffer is created (like the
        first step does) and then filled, so loading works before and after a capture.  Refused: a different group or
        parameter layout, a buffer of another shape or dtype, and a state without momentum for a parameter that already
        has some (a graph cannot be made to take the first-step path again)."""
        groups = state_dict['param_groups']
        if len(groups) != len(self.param_groups) or \
                any(len(g['params']) != len(s['params']) for g, s in zip(self.param_groups, groups)):
            raise ValueError('optimizer state of %s parameters per group, this optimizer has %s'
                             % ([len(s['params']) for s in groups], [len(g['params']) for g in self.param_groups]))
        pairs = []
        for group, saved in zip(self.param_groups, groups):
            for p, idx in zip(group['params'], saved['params']):
                buf = state_dict['state'].get(idx, {}).get('momentum_buffer')
                if buf is None:
                    if 'momentum_buffer' in self.state[p]:
                        raise ValueError('optimizer state without momentum for parameter %d, which already has a buffer' % idx)
                    continue
                if tuple(buf.shape) != tuple(p.shape) or buf.dtype != p.dtype:
                    raise ValueError('momentum of parameter %d is %s %s, the parameter is %s %s'
                                     % (idx, buf.dtype, tuple(buf.shape), p.dtype, tuple(p.shape)))
                pairs.append((p, buf))
        for p, buf in pairs:
            if 'momentum_buffer' not in self.state[p]:
                self.state[p]['momentum_buffer'] = torch.empty_like(p)
            self.state[p]['momentum_buffer'].copy_(buf)
        for group, saved in zip(self.param_groups, groups):
            group.update({k: v for k, v in saved.items() if k != 'params'})

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        st = torch.cuda.current_stream().cuda_stream
        for gi, group in enumerate(self.param_groups):
            fresh, seasoned = [], []
            for p in group['params']:
                if p.grad is None:
                    continue
                if not p.is_cuda:
                    raise TypeError('FusedSGD updates CUDA parameters only (no CPU fallback)')
                if not same_layout(p.grad, p):
                    p.grad = p.grad.contiguous(
                        memory_format=torch.channels_last if p.is_contiguous(memory_format=torch.channels_last)
                        and p.dim() == 4 else torch.contiguous_format)
                (fresh if 'momentum_buffer' not in self.state[p] else seasoned).append(p)
            for p in fresh:
                self.state[p]['momentum_buffer'] = torch.empty_like(p)
            for first, plist in ((True, fresh), (False, seasoned)):
                if not plist:
                    continue
                tab = self._table((gi, first), plist)
                call('fsdet_sgd_step', ptr(tab['params']), ptr(tab['grads']), ptr(tab['moms']), ptr(tab['sizes']),
                     ptr(tab['chunk_tensor']), ptr(tab['chunk_offset']), tab['n_chunks'], _CHUNK, float(group['lr']),
                     float(group['momentum']), float(group['dampening']), float(group['weight_decay']),
                     1 if first else 0, ptr(self._hyper[gi][0]) if self.capturable else None, st)
        return loss
