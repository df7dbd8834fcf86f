"""Host -> device input staging for the training loop (the `data.cuda()` of train_meta.py:209-213, pipelined).

The reference copies each batch synchronously right before the forward pass (`data, metax, mask = data.cuda(),
metax.cuda(), mask.cuda()`), so the PCIe transfer of step i (190 MB at config 2, ~3.5 ms) is serial with its compute.
`DevicePrefetcher` issues the copy of batch i+1 on a side stream (into reused staging buffers) while step i runs; the
training stream only waits on an event.  Host tensors should be pinned (DataLoader(pin_memory=True), train_meta.py:107) for the copy to be
asynchronous.  `host_fields` stay on the host untouched (the float64 target, which RegionLoss takes as a CPU tensor,
train_meta.py:211)."""
import torch


class DevicePrefetcher(object):
    """Iterator over device copies of host batches (tuples of tensors), one batch ahead.

    Two fixed sets of device staging buffers are reused (no allocator traffic in steady state): while the training
    stream consumes slot k, the copy stream fills slot k^1; events order both directions.  A batch handed out by
    `next()` therefore stays valid until the FOLLOWING `next()` call (its slot is refilled after everything the
    training stream had queued by then)."""

    def __init__(self, batches, device, host_fields=()):
        self.it = iter(batches)
        self.device = torch.device(device)
        if self.device.type != 'cuda':
            raise TypeError('DevicePrefetcher stages batches for a CUDA device')
        self.host_fields = set(host_fields)
        self.stream = torch.cuda.Stream(self.device)
        self.h2d_bytes = 0
        self._slots = [None, None]                 # per slot: list of device buffers (None for host fields)
        self._ready = [torch.cuda.Event(), torch.cuda.Event()]   # recorded on the copy stream: slot filled
        self._free = [None, None]                  # recorded on the training stream: slot may be overwritten
        self._k = 0                                # slot holding the batch the next `next()` returns
        self._next = None
        self._preload(0)

    def _preload(self, slot):
        try:
            batch = next(self.it)
        except StopIteration:
            self._next = None
            return
        bufs = self._slots[slot]
        fresh = bufs is None or len(bufs) != len(batch)
        if fresh:
            bufs = [None] * len(batch)
        out = []
        main = torch.cuda.current_stream(self.device)
        with torch.cuda.stream(self.stream):
            if self._free[slot] is not None:
                self.stream.wait_event(self._free[slot])
            for i, t in enumerate(batch):
                if i in self.host_fields or not torch.is_tensor(t):
                    out.append(t)
                    continue
                b = bufs[i]
                if b is None or b.shape != t.shape or b.dtype != t.dtype:
                    b = torch.empty(t.shape, dtype=t.dtype, device=self.device)
                    b.record_stream(main)          # consumed on the training stream: keep the allocator informed
                    bufs[i] = b
                b.copy_(t, non_blocking=True)
                self.h2d_bytes += t.numel() * t.element_size()
                out.append(b)
            self._ready[slot].record(self.stream)
        self._slots[slot] = bufs
        self._next = tuple(out)

    def __iter__(self):
        return self

    def __next__(self):
        if self._next is None:
            raise StopIteration
        cur = torch.cuda.current_stream(self.device)
        k = self._k
        cur.wait_event(self._ready[k])
        batch = self._next
        # everything queued so far on the training stream may still read the other slot (the previous batch)
        ev = torch.cuda.Event()
        ev.record(cur)
        self._free[k ^ 1] = ev
        self._k = k ^ 1
        self._preload(k ^ 1)
        return batch

    next = __next__


class AsyncLossReader(object):
    """Device -> host read-back of per-step scalars (the loss train_meta.py:221-223 logs) without stalling the launch
    of the next step: `push(loss)` enqueues a 4-byte copy into pinned memory behind the step, `pop()` returns the
    oldest outstanding value (blocking only on ITS event).  With depth 2 the training loop reads step i-1's loss
    while step i is already running, so the GPU never idles waiting for the host."""

    def __init__(self, depth=2):
        self.depth = depth
        self.buf = [torch.zeros(1, dtype=torch.float32).pin_memory() for _ in range(depth)]
        self.ev = [torch.cuda.Event() for _ in range(depth)]
        self.head = 0      # next slot to pop
        self.count = 0     # outstanding values

    def push(self, loss):
        if self.count == self.depth:
            raise RuntimeError('AsyncLossReader: %d values outstanding, pop() first' % self.count)
        slot = (self.head + self.count) % self.depth
        self.buf[slot].copy_(loss.detach().reshape(1), non_blocking=True)
        self.ev[slot].record()
        self.count += 1

    def pop(self):
        if self.count == 0:
            raise IndexError('AsyncLossReader: nothing outstanding')
        slot = self.head
        self.ev[slot].synchronize()
        v = float(self.buf[slot][0])
        self.head = (self.head + 1) % self.depth
        self.count -= 1
        return v

    def drain(self):
        out = []
        while self.count:
            out.append(self.pop())
        return out


class BackgroundPrep(object):
    """Runs the HOST half of the input pipeline one batch ahead in a worker thread (what the reference's DataLoader
    worker processes do, train_meta.py:173-193): `thunks` is an iterable of zero-argument callables, each returning one
    prepared batch; iteration yields their results in order.  Exceptions of the worker surface at the consumer.

    The thunks draw from the global random generators, and so does the consumer (neg_filter's one `random()` per empty
    label row, made when step i is launched).  To keep a seeded run reproducible the draws must come in the serial
    order - prepare 0, step 0, prepare 1, step 1, ... - whatever the thread timing, so the worker starts thunk i+1 only
    after the consumer has called `draws_done()` for item i.  The worker therefore prepares batch i+1 while the GPU
    runs step i, and never runs further ahead."""

    def __init__(self, thunks, depth=2):
        import queue
        import threading
        self._q = queue.Queue(maxsize=depth)
        self._done = object()
        self._go = threading.Semaphore(0)     # one release per item whose consumer-side draws are finished
        self._closed = False

        self.busy_s = 0.0      # time the worker spent preparing (diagnostics)

        def work():
            import time as _t
            try:
                for i, t in enumerate(thunks):
                    if i:
                        self._go.acquire()
                        if self._closed:
                            return
                    t0 = _t.time()
                    item = t()
                    self.busy_s += _t.time() - t0
                    self._q.put((True, item))
                self._q.put((True, self._done))
            except BaseException as e:      # hand the failure to the consumer instead of dying silently
                self._q.put((False, e))
        self._thread = threading.Thread(target=work, daemon=True)
        self._thread.start()

    def draws_done(self):
        """The consumer has made every random draw that belongs to the item it last received: the worker may start
        preparing the next one."""
        self._go.release()

    def close(self):
        """Stop the worker after its current thunk (a consumer that leaves the loop early)."""
        self._closed = True
        self._go.release()

    def __iter__(self):
        return self

    def __next__(self):
        ok, item = self._q.get()
        if not ok:
            raise item
        if item is self._done:
            self._q.put((True, self._done))
            raise StopIteration
        return item
