"""The training loop of the reference's driver (train_meta.py:86-255) as a class over this package's parts.

The reference's script wires everything through module globals; `MetaTrainer` keeps its arithmetic and bookkeeping -
learning-rate factor per negative-sampling mode (train_meta.py:124-135), SGD hyper-parameters (:143-147), the
`steps/scales` schedule applied before every batch (:150-163, :204), `seen` / `processed_batches` accounting
(:93-95, :205, :220), one fresh query / support stream per epoch (:172-197) and the Darknet weight files every
`cfg.save_interval` epochs (:251-254) - and takes the pieces as arguments: the model (`darknet_meta.Darknet`), an
optimizer (`optim.FusedSGD` or `torch.optim.SGD`), factories for the epoch's `dataset.DetectionBatcher` /
`dataset.MetaBatcher`, optionally a `distributed.GradAllReducer` (one process per GPU instead of nn.DataParallel).
`tools/train_meta_b200.py` is the command-line front end with the reference's four arguments.
"""
import collections
import math
import time


def lr_factor(neg_ratio, n_classes):
    """train_meta.py:124-135: the loss sums over B*n_cls rows, so the driver divides the base rate by a factor that
    depends on how many negative rows survive neg_filter."""
    if neg_ratio == 'full':
        return 15.
    if neg_ratio == 1:
        return 3.0
    if neg_ratio == 0:
        return 1.5
    if neg_ratio == 5:
        return 8.0
    return n_classes


def learning_rate_at(batch, learning_rate, steps, scales):
    """train_meta.py:150-160 (`adjust_learning_rate` without the optimizer side effect)."""
    lr = learning_rate
    for i in range(len(steps)):
        scale = scales[i] if i < len(scales) else 1
        if batch >= steps[i]:
            lr = lr * scale
            if batch == steps[i]:
                break
        else:
            break
    return lr


def sgd_hyper_parameters(learning_rate, momentum, decay, batch_size, factor):
    """Keyword arguments of the driver's optim.SGD (train_meta.py:136, 143-147); `learning_rate` is the cfg value
    BEFORE the division by `factor`."""
    return dict(lr=learning_rate / factor / batch_size, momentum=momentum, dampening=0,
                weight_decay=decay * batch_size * factor)


def epoch_plan(model_seen, nsamples, batch_size, max_batches, tuning=False, max_epoch=None, repeat=1):
    """(processed_batches, init_epoch, max_epochs) as train_meta.py:94-101 computes them."""
    processed = 0 if tuning else model_seen // batch_size
    init_epoch = 0 if tuning else model_seen // nsamples
    max_epochs = max_batches * batch_size // nsamples + 1
    if tuning:
        max_epochs = int(math.ceil(max_epoch * 1. / repeat))
    return processed, init_epoch, max_epochs


def rng_state():
    """The states of the generators the input pipeline and neg_filter draw from - Python `random`, numpy, torch CPU -
    with numpy's key array as an int64 tensor, so resume.write_state can store it."""
    import random
    import numpy as np
    import torch
    name, keys, pos, has_gauss, cached = np.random.get_state()
    return dict(python=random.getstate(), numpy=(name, torch.from_numpy(keys.astype(np.int64)), int(pos), int(has_gauss),
                                                 float(cached)), torch=torch.get_rng_state())


def set_rng_state(state):
    import random
    import numpy as np
    import torch
    random.setstate(state['python'])
    name, keys, pos, has_gauss, cached = state['numpy']
    np.random.set_state((name, keys.numpy().astype(np.uint32), pos, has_gauss, cached))
    torch.set_rng_state(state['torch'])


class MetaTrainer(object):
    def __init__(self, model, optimizer, learning_rate, batch_size, steps, scales, make_train_batcher, make_meta_batcher,
                 backupdir=None, save_interval=10, reducer=None, world=1, processed_batches=0, log=print, use_graph=None,
                 evaluate=None, save_state=None):
        """learning_rate: the cfg rate already divided by `lr_factor` (what the driver calls `learning_rate` after
        :136); batch_size: GLOBAL batch; make_train_batcher(seen) / make_meta_batcher(): the epoch's data streams.
        use_graph: replay the step from CUDA graphs (graph.GraphedTrainStep: one graph per input shape, neg_filter
        staged from the host) - the default whenever the model's parameters live on a CUDA device.
        evaluate: optional evaluate(model, epoch), run on every rank at the end of each checkpoint epoch (every
        `save_interval` epochs), after the weight file is written where one is written (rank 0 with a backupdir) and
        whether or not one is: every rank takes part in a sharded evaluation.  What it returns is logged
        (see evaluate_checkpoint).
        save_state: optional save_state(trainer, epoch), run on every rank at the end of each checkpoint epoch, after
        the weight file and before `evaluate` (the driver writes the training-state file there, see resume.py)."""
        self.model, self.optimizer = model, optimizer
        self.region_loss = model.loss
        self.learning_rate, self.batch_size = learning_rate, batch_size
        self.steps, self.scales = list(steps), list(scales)
        self.make_train_batcher, self.make_meta_batcher = make_train_batcher, make_meta_batcher
        self.backupdir, self.save_interval = backupdir, save_interval
        self.reducer, self.world = reducer, world
        self.processed_batches = processed_batches
        self.region_loss.seen = model.seen           # train_meta.py:93
        self.log = log
        self.evaluate, self.save_state = evaluate, save_state
        self.epoch = 0                 # the next epoch to run (after train_epoch(e): e + 1)
        self.resume_epoch = None       # set by load_state_dict
        self.losses = collections.deque(maxlen=100)   # detached loss tensors of the most recent steps (no host sync)
        import os
        if use_graph is None:
            use_graph = any(p.is_cuda for p in model.parameters()) and os.environ.get('FSDET_NO_GRAPH', '0') != '1'
        self.graphed = None
        if use_graph:
            from .distributed import GradAllReducer
            from .graph import GraphedTrainStep
            if self.reducer is None:
                self.reducer = GradAllReducer(model)      # flat gradient buffer: in-place all-reduce and fused SGD
            self.graphed = GraphedTrainStep(model, self.region_loss, optimizer, self.reducer,
                                            strict=os.environ.get('FSDET_STRICT_CAPTURE', '0') == '1')

    def adjust_learning_rate(self, batch):
        lr = learning_rate_at(batch, self.learning_rate, self.steps, self.scales)
        for group in self.optimizer.param_groups:
            group['lr'] = lr / self.batch_size
        return lr

    def train_step(self, data, metax, mask, target):
        """One optimisation step (train_meta.py:214-225).  No `zero_grad()`: the engine OVERWRITES every parameter
        gradient each step (and with a GradAllReducer the gradients are views into its flat buffer, which
        `zero_grad(set_to_none=True)` would silently detach - the all-reduce would then run over stale zeros)."""
        if self.graphed is not None:
            self.region_loss.seen = self.region_loss.seen + data.size(0) * self.world
            return self.graphed(data, metax, mask, target)
        if self.reducer is not None:
            self.reducer.begin_step()
        elif not getattr(self.model, '_fsdet_overwrites_grads', False):
            self.optimizer.zero_grad()            # plain torch modules (the CPU tests' stub model) accumulate
        output = self.model(data, metax, mask)
        self.region_loss.seen = self.region_loss.seen + data.size(0) * self.world
        loss = self.region_loss(output, target)
        loss.backward()
        if self.reducer is not None:
            self.reducer.finish()
        self.optimizer.step()
        return loss

    def train_epoch(self, epoch, max_epochs=None):
        t0 = time.time()
        batcher = self.make_train_batcher(self.model.seen)     # train_meta.py:181: seen = cur_model.seen (updated at saves)
        meta = self.make_meta_batcher()
        lr = self.adjust_learning_rate(self.processed_batches)
        self.log('epoch %d/%s, processed %d samples, lr %f' % (epoch, max_epochs, epoch * len(batcher) * self.world, lr))
        self.model.train()
        n_meta = meta.batch_size
        nb = 0
        import os
        if hasattr(batcher, 'prepare') and hasattr(meta, 'prepare') and os.environ.get('FSDET_NO_BG_PREP', '0') != '1':
            # host half (draws, file decode, labels) of batch i+1 in a worker thread while the GPU runs step i
            from .prefetch import BackgroundPrep
            ranges = batcher.batch_ranges()
            prep = BackgroundPrep((lambda i=i, r=r: (batcher.prepare(r), meta.prepare(range(i * n_meta, (i + 1) * n_meta))))
                                  for i, r in enumerate(ranges))
            stream = ((batcher.finish(q), meta.finish(s)) for q, s in prep)
            self._prep = prep
        else:
            prep = None
            stream = (((data, target), meta.batch(range(i * n_meta, (i + 1) * n_meta))) for i, (data, target) in enumerate(batcher))
        prof = os.environ.get('FSDET_TRAIN_PROFILE', '0') == '1'
        t_wait = t_step = 0.0
        tp = time.time()
        try:
            for nb, ((data, target), support) in enumerate(stream, 1):
                metax, mask = support[:2]
                if prof:
                    t_wait += time.time() - tp
                    tp = time.time()
                self.adjust_learning_rate(self.processed_batches)
                self.processed_batches = self.processed_batches + 1
                loss = self.train_step(data, metax, mask, target)
                if prep is not None:
                    prep.draws_done()         # this step's neg_filter draws are made: batch i+1's may start
                # a graph replay returns its static loss buffer, overwritten by the next replay of that graph (and, being
                # in the graphs' shared pool, possibly by another graph's scratch): keep a device copy of this step's value
                self.losses.append(loss.detach().clone() if self.graphed is not None else loss.detach())
                if prof:
                    t_step += time.time() - tp
                    tp = time.time()
        except BaseException:
            if prep is not None:
                prep.close()
            raise
        if prof and nb:
            self.log('host time per step: %.1f ms waiting for / finishing the input batch, %.1f ms launching the step, '
                     'background preparation %.1f ms per batch'
                     % (1e3 * t_wait / nb, 1e3 * t_step / nb, 1e3 * getattr(getattr(self, '_prep', None), 'busy_s', 0.0) / nb))
        dt = time.time() - t0
        self.log('training with %f samples/s' % (len(batcher) * self.world / max(dt, 1e-9)))
        if self.backupdir is not None and (epoch + 1) % self.save_interval == 0:
            path = '%s/%06d.weights' % (self.backupdir, epoch + 1)
            self.log('save weights to %s' % path)
            self.model.seen = (epoch + 1) * len(batcher) * self.world
            self.model.save_weights(path)
        self.epoch = epoch + 1
        if (epoch + 1) % self.save_interval == 0:
            if self.save_state is not None:
                self.save_state(self, epoch + 1)
            self.evaluate_checkpoint(epoch + 1)
        return nb

    def evaluate_checkpoint(self, epoch):
        """Run `evaluate(model, epoch)` without changing training: the model goes to eval() (BatchNorm uses and keeps
        its running statistics) and back to its mode; the Python `random`, numpy and torch CPU generators that the
        batchers and neg_filter draw from are restored.  The step graphs stay valid: the evaluation forwards reuse the
        engine's weight plan (same weight tensors) and allocate outside the graphs' pool.  Returns and logs the
        callback's value."""
        if self.evaluate is None:
            return None
        import random
        import numpy as np
        import torch
        py_state, np_state, torch_state = random.getstate(), np.random.get_state(), torch.get_rng_state()
        was_training = self.model.training
        try:
            self.model.eval()
            r = self.evaluate(self.model, epoch)
        finally:
            self.model.train(was_training)
            random.setstate(py_state)
            np.random.set_state(np_state)
            torch.set_rng_state(torch_state)
        if r is not None:
            self.log('evaluation at epoch %d: %s' % (epoch, r))
        return r

    def state_dict(self):
        """What a resumed run needs besides the weight file: the next epoch, `processed_batches` (the schedule
        position), both `seen` counters (region_loss.seen counts every sample trained on; model.seen is only updated at
        saves and seeds the next epoch's multi-scale schedule), the optimizer's state with its momentum buffers copied
        to the host, bits unchanged, and this process's random generators (Python, numpy, torch CPU)."""
        import torch
        opt = self.optimizer.state_dict()
        opt['state'] = {k: {n: (v.detach().to('cpu', copy=True) if torch.is_tensor(v) else v) for n, v in s.items()}
                        for k, s in opt['state'].items()}
        return dict(epoch=int(self.epoch), processed_batches=int(self.processed_batches),
                    region_loss_seen=int(self.region_loss.seen), model_seen=int(self.model.seen), optimizer=opt,
                    rng=rng_state())

    def load_state_dict(self, state):
        """Continue where `state` (from state_dict) was taken: fit() then starts at its epoch, whatever init_epoch it
        is given.  Momentum is copied into the optimizer's buffers (FusedSGD keeps the tensors its pointer tables and
        step graphs address)."""
        self.optimizer.load_state_dict(state['optimizer'])
        self.epoch = self.resume_epoch = int(state['epoch'])
        self.processed_batches = int(state['processed_batches'])
        self.region_loss.seen = int(state['region_loss_seen'])
        self.model.seen = int(state['model_seen'])
        set_rng_state(state['rng'])

    def fit(self, init_epoch, max_epochs):
        if self.resume_epoch is not None:
            init_epoch = self.resume_epoch
        for epoch in range(int(init_epoch), int(max_epochs)):
            self.train_epoch(epoch, max_epochs)
