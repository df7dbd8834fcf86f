"""The training step as it ships, against the checked step: two streams, memory reuse, CUDA graphs and the optimizer.

The step checkers (test_gpu_zz_step_gemms, test_gpu_zz_step_memops) synchronise the device before every launch and run
each kernel alone, so they prove the kernels, not the step that ships.  That step differs in four ways: the weight
gradients run on a second stream (NetRunner._convbn_bwd), the caching allocator hands freed blocks to the next
allocation of the stream that owns them while the other stream may still use them, GraphedTrainStep replays the step
from graphs that share one memory pool, and fsdet_sgd_step updates all 89 parameter tensors in one launch.

  test_shipped_step_equals_checked_step   full size (configs[1]: B = 64, 20 classes, 416; configs[4]: B = 64, 80
                               classes, 608): the step under both checkers chained (bars unchanged), the same step
                               unchecked with the shipped defaults and with the weight gradients on the main stream are
                               bit-equal in the head output, every parameter gradient and every BatchNorm running
                               statistic; the loss (a sum of double atomics) to 1e-12.  The unchecked step must have
                               launched on the second stream.
  test_graph_replay_equals_checked_step   GraphedTrainStep (GradAllReducer of world 1, FusedSGD with the driver's
                               hyper-parameters) through an eager step at 416, a capture + replay at 416 and at 608 and
                               a replay at 416 after the learning rate changed, at neg = full and neg = 1: before every
                               step the state is loaded into a twin model whose checked eager step must give bit-equal
                               gradients and BatchNorm statistics.  Then every element of every parameter and momentum
                               buffer against the SGD kernel's fma chain in float64 rounded to fp32 after each
                               operation (within one ulp), with the hyper-parameter path each step took.
  test_accumulated_gradients   two backward passes without zeroing the gradients in between: every gradient bit-equal
                               to fl32(g1 + g2) of the single-pass gradients, with the second stream on and off.
  test_lifetime_audit          one backward of the plain and of the accumulating step with the second stream held back
                               and the main stream's free memory poisoned with NaN in between (LifetimeAudit): a buffer
                               the second stream reads or writes after its owner released it reads back NaN.  Both
                               results bit-equal to the unaudited ones.
  test_lifetime_audit_has_teeth   the same audit with NetRunner._keep disabled reports NaN or a mismatch.
"""
import random
import time

import numpy as np
import pytest
import torch

from test_gpu_zz_step_gemms import StepChecker, report as report_gemms
from test_gpu_zz_step_memops import MemChecker, dev, report as report_mem
from test_gpu_zz_step_scales import check_region

pytestmark = pytest.mark.gpu

SEED = 2101                    # model seed of configs[1]; its two batches are SEED + 1 and SEED + 2
N_PARAMS = 89
# torch.cuda._sleep cycles: about 10 ms at the H100's 1.755 - 1.98 GHz
SLEEP_CYCLES = 20000000


# ------------------------------------------------------------------------------------------------------------ runner
def _model(side, seed, replicas=1):
    from fewshot_detection_b200 import netcfg
    from fewshot_detection_b200.darknet_meta import Darknet
    from seeding import seeded_init
    m = Darknet(netcfg.darknet_dynamic_blocks(side, side), netcfg.reweighting_net_blocks(), replicas=replicas)
    seeded_init(m, seed)
    m = m.cuda().train()
    L = m.models[len(m.models) - 1]
    L.seen = 20000
    L.verbose = False
    return m, L


def _bn_stats(m):
    return {n: b for n, b in m.named_buffers() if n.endswith(('running_mean', 'running_var'))}


class Run(object):
    """What one run leaves: the model, the last head output, loss, label tensor and region loss module, every parameter
    gradient and BatchNorm running statistic by name (copied to the host) and the wall time."""


def run(side, bs, cs, seed, batch_seeds, wrap=None, replicas=1):
    """The seeded full model (configs side x side, `cs` classes, B = `bs`), then forward + RegionLossV2 + backward on
    each batch of `batch_seeds` without zeroing the gradients in between, while engine.call is wrap(engine.call).
    replicas = R: the R-replica step (Darknet(..., replicas=R), R support sets of `cs` images)."""
    from fewshot_detection_b200 import engine
    from test_gpu_zz_configs import _batch
    m, L = _model(side, seed, replicas)
    real = engine.call
    if wrap is not None:
        engine.call = wrap(real)
    t0 = time.time()
    try:
        for bseed in batch_seeds:
            x, metax, mask, tgt = _batch(bs, cs, side, bseed, replicas=replicas)
            out = m(x.cuda(), metax.cuda(), mask.cuda())
            loss = L(out, tgt)
            loss.backward()
        torch.cuda.synchronize()
    finally:
        engine.call = real
    r = Run()
    r.secs = time.time() - t0
    r.model, r.L, r.tgt = m, L, tgt
    r.out = out.detach()
    r.loss = loss.item()
    r.grads = {n: p.grad.detach().cpu() for n, p in m.named_parameters()}
    r.bn = {n: b.detach().cpu() for n, b in _bn_stats(m).items()}
    assert len(r.grads) == N_PARAMS, len(r.grads)
    return r


def release(r):
    """Drop the run's device state (its model and head output) and return the cached blocks to the device."""
    r.model = r.L = r.out = None
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def bit_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def differing(a, b):
    """names of the tensors of dict `a` whose bits differ from dict `b`'s, in parameter order"""
    assert list(a) == list(b)
    return [n for n in a if not bit_equal(a[n], b[n])]


class StreamCount(object):
    """Counts the engine's launches and those issued while a stream other than the main one was current."""

    def __init__(self, real):
        self.real = real
        self.main = torch.cuda.current_stream()
        self.total = self.side = 0

    def __call__(self, fn, *a):
        self.total += 1
        if torch.cuda.current_stream() != self.main:
            self.side += 1
        return self.real(fn, *a)


def checked(made):
    """wrap() that chains both step checkers, as test_gpu_zz_step_scales does"""
    from fewshot_detection_b200 import _lib

    def chain(real):
        made['gemm'] = StepChecker(real, _lib.lib)
        made['mem'] = MemChecker(made['gemm'], _lib.lib)
        return made['mem']
    return chain


def report_checked(made, secs):
    errors = []
    for rep, chk in ((report_gemms, made['gemm']), (report_mem, made['mem'])):
        try:
            rep(chk, secs)
        except AssertionError as e:
            errors.append(e)
    return errors


_SINGLE = {}


def single(bseed):
    """Single-pass gradients of the configs[1] model (SEED) on batch `bseed`, shipped defaults (cached)."""
    if bseed not in _SINGLE:
        cnt = {}
        r = run(416, 64, 20, SEED, [bseed], lambda real: cnt.setdefault('c', StreamCount(real)))
        assert cnt['c'].side > 0
        release(r)
        _SINGLE[bseed] = r
    return _SINGLE[bseed]


# ------------------------------------------------------------------------------------------------------------ part 1
@pytest.mark.parametrize('side,bs,cs,seed', [pytest.param(416, 64, 20, SEED, id='configs1'),
                                             pytest.param(608, 64, 80, 2111, id='configs4')])
def test_shipped_step_equals_checked_step(side, bs, cs, seed, monkeypatch):
    """(a) checked, (b) unchecked with the shipped defaults, (c) unchecked with every launch on the main stream: the
    same seeded model and batch give bit-equal head outputs, parameter gradients and BatchNorm running statistics."""
    from fewshot_detection_b200 import engine
    print('\n==== side %d, B = %d, %d classes' % (side, bs, cs))
    made = {}
    a = run(side, bs, cs, seed, [seed + 1], checked(made))
    errors = report_checked(made, a.secs)
    fails, row = check_region(a.out, a.L, a.tgt, 'full', None)
    print(row)
    errors += fails
    out_a = a.out.cpu()
    release(a)
    cnt = {}
    b = run(side, bs, cs, seed, [seed + 1], lambda real: cnt.setdefault('c', StreamCount(real)))
    out_b = b.out.cpu()
    release(b)
    if side == 416 and cs == 20:
        _SINGLE[seed + 1] = b
    monkeypatch.setattr(engine, 'WGRAD_STREAM', False)
    cnt1 = {}
    c = run(side, bs, cs, seed, [seed + 1], lambda real: cnt1.setdefault('c', StreamCount(real)))
    out_c = c.out.cpu()
    release(c)
    print('launches: %d, %d of them on the second stream (single-stream run: %d of %d)' % (
        cnt['c'].total, cnt['c'].side, cnt1['c'].side, cnt1['c'].total))
    print('wall time: checked %.1f s, unchecked %.2f s, single-stream %.2f s' % (a.secs, b.secs, c.secs))
    for name, r, out in (('unchecked', b, out_b), ('single-stream', c, out_c)):
        dg, db = differing(r.grads, a.grads), differing(r.bn, a.bn)
        print('%-13s vs checked: head output %s, gradients %s, BatchNorm statistics %s, loss %.17g / %.17g' % (
            name, 'bit-equal' if bit_equal(out, out_a) else 'DIFFERS', 'bit-equal' if not dg else 'first differing %s (%d of %d)'
            % (dg[0], len(dg), len(r.grads)), 'bit-equal' if not db else 'first differing %s' % db[0], r.loss, a.loss))
        if not bit_equal(out, out_a):
            errors.append((name, 'head output'))
        if dg:
            errors.append((name, 'gradient', dg[0], len(dg)))
        if db:
            errors.append((name, 'BatchNorm running statistic', db[0], len(db)))
        if not abs(r.loss - a.loss) <= 1e-12 * abs(a.loss):
            errors.append((name, 'loss', r.loss, a.loss))
    assert not errors, errors
    assert cnt['c'].side > 0, 'the shipped step launched nothing on the second stream'
    assert cnt1['c'].side == 0


# ------------------------------------------------------------------------------------------------------ parts 2 + 3
# (side, factor applied to the learning rate before the step): the eager first step, a capture + replay at 416 and at
# 608 (one shared pool), and a second replay at 416 after the schedule lowered the rate
SCHEDULE = ((416, 1.0), (416, 1.0), (608, 1.0), (416, 0.1))


def ordered(t):
    """fp32 bit patterns as integers whose difference counts ulps (+0 and -0 both 0)"""
    i = t.contiguous().view(torch.int32).long()
    return torch.where(i < 0, -(i & 0x7fffffff), i)


def sgd_chain(p, g, m, hyper, first):
    """csrc/sgd.cu in float64, rounded to fp32 after every operation: d = fma(wd, p, g); m' = d on the first step, else
    fma(mu, m, (1 - damp) * d); p' = fma(-lr, m', p).  The products of two fp32 values are exact in float64, so each
    fma is rounded twice (to float64, then to fp32), which can differ from the kernel's single rounding by one ulp."""
    lr, mu, damp, wd = (float(np.float32(v)) for v in hyper)
    one = float(np.float32(1.0) - np.float32(damp))
    f = lambda t: t.float().double()
    P = p.double()
    d = f(wd * P + g.double())
    M = d if first else f(mu * m.double() + f(one * d))
    return f(-lr * M + P).float(), M.float()


def sgd_check(before, grads, after, hyper, first):
    """(worst ulp, elements not bit-equal, elements) of every parameter and momentum buffer after the step against
    sgd_chain of the state before it"""
    worst, off, n = 0, 0, 0
    for p0, m0, g, p1, m1 in zip(before[0], before[1], grads, after[0], after[1]):
        rp, rm = sgd_chain(p0, g, m0, hyper, first)
        for got, ref in ((p1, rp), (m1, rm)):
            u = (ordered(got) - ordered(ref)).abs()
            worst = max(worst, u.max().item())
            off += int((u != 0).sum())
            n += u.numel()
    return worst, off, n


def _state(m, opt):
    params = [p.detach().clone() for p in m.parameters()]
    moms = [opt.state[p]['momentum_buffer'].detach().clone() if 'momentum_buffer' in opt.state[p] else None
            for p in m.parameters()]
    bufs = {n: b.detach().clone() for n, b in m.named_buffers()}
    return params, moms, bufs


@pytest.mark.parametrize('neg', ['full', 1], ids=['neg-full', 'neg1'])
def test_graph_replay_equals_checked_step(neg, monkeypatch):
    """configs[1] (B = 64, 20 classes) through GraphedTrainStep: every step's gradients and BatchNorm statistics
    bit-equal to a checked eager step of a twin model loaded with the state before it, and the fused SGD update within
    one ulp of its float64 chain on every element."""
    from fewshot_detection_b200 import engine, optim
    from fewshot_detection_b200.cfg import cfg
    from fewshot_detection_b200.distributed import GradAllReducer
    from fewshot_detection_b200.graph import GraphedTrainStep
    from fewshot_detection_b200.optim import FusedSGD
    from fewshot_detection_b200.trainer import lr_factor, sgd_hyper_parameters
    from test_gpu_zz_configs import _batch
    bs, cs = 64, 20
    monkeypatch.setattr(cfg, 'neg_ratio', neg)
    sgd_calls = []
    real_ocall = optim.call

    def ocall(fn, *a):
        if fn == 'fsdet_sgd_step':
            sgd_calls.append((a[12], a[13] is not None))          # first step?, hyper-parameters from device memory?
        return real_ocall(fn, *a)
    monkeypatch.setattr(optim, 'call', ocall)
    m, L = _model(416, 3001)
    params = list(m.parameters())
    opt = FusedSGD(params, **sgd_hyper_parameters(1e-3, 0.9, 5e-4, bs, lr_factor(neg, cs)))
    red = GradAllReducer(m)
    assert red.world == 1 and m._det.grad_hook is None          # no collective: the second stream stays on
    gs = GraphedTrainStep(m, L, opt, red)
    twin, tL = _model(416, 3001)
    tparams = list(twin.parameters())
    tbufs = dict(twin.named_buffers())
    errors = []
    for k, (side, lr_scale) in enumerate(SCHEDULE):
        old_hyper = None
        if lr_scale != 1.0:                    # as MetaTrainer.adjust_learning_rate: group['lr'] rewritten in place
            g0 = opt.param_groups[0]
            old_hyper = (g0['lr'], g0['momentum'], g0['dampening'], g0['weight_decay'])
            for g in opt.param_groups:
                g['lr'] = g['lr'] * lr_scale
        before = _state(m, opt)
        hyper = tuple(opt.param_groups[0][h] for h in ('lr', 'momentum', 'dampening', 'weight_decay'))
        x, metax, mask, tgt = _batch(bs, cs, side, 3100 + k)
        n_calls = len(sgd_calls)
        t0 = time.time()
        random.seed(3200 + k)
        graph_loss = gs(x.cuda(), metax.cuda(), mask.cuda(), tgt).item()
        secs_graph = time.time() - t0
        calls = sgd_calls[n_calls:]
        grads = [p.grad for p in params]
        after = ([p.detach().clone() for p in params], [opt.state[p]['momentum_buffer'].detach().clone() for p in params])
        bn_graph = {n: b.detach().clone() for n, b in _bn_stats(m).items()}
        # the twin: the same state, seed and batch through a checked eager step
        with torch.no_grad():
            for tp, p0 in zip(tparams, before[0]):
                tp.copy_(p0)
            for n, b0 in before[2].items():
                tbufs[n].copy_(b0)
        for tp in tparams:
            tp.grad = None
        made = {}
        real = engine.call
        engine.call = checked(made)(real)
        t0 = time.time()
        try:
            random.seed(3200 + k)
            tloss = tL(twin(x.cuda(), metax.cuda(), mask.cuda()), tgt)
            tloss.backward()
            torch.cuda.synchronize()
        finally:
            engine.call = real
        secs_twin = time.time() - t0
        errors += report_checked(made, secs_twin)
        dg = [n for (n, _), g, tg in zip(twin.named_parameters(), grads, tparams) if not bit_equal(g, tg.grad)]
        db = [n for n, b in _bn_stats(twin).items() if not bit_equal(b, bn_graph[n])]
        first = k == 0
        worst, off, total = sgd_check(before, grads, after, hyper, first)
        path = 'first step, host arguments' if first else 'device hyper-parameters'
        print('step %d (side %d, %s, lr %.4g): graph vs checked twin: gradients %s, BatchNorm statistics %s; loss %.10g / '
              '%.10g; SGD (%s): worst %d ulp, %d of %d elements not bit-equal; %.2f s step, %.1f s checked twin' % (
                  k, side, 'eager' if first else 'graph', hyper[0], 'bit-equal' if not dg else 'first differing %s (%d)' % (dg[0], len(dg)),
                  'bit-equal' if not db else 'first differing %s (%d)' % (db[0], len(db)), graph_loss, tloss.item(), path,
                  worst, off, total, secs_graph, secs_twin))
        if dg:
            errors.append((k, side, 'gradient', dg[0], len(dg)))
        if db:
            errors.append((k, side, 'BatchNorm running statistic', db[0], len(db)))
        if worst > 1:
            errors.append((k, side, 'SGD update off by %d ulp' % worst))
        # the hyper-parameter path: host arguments on the eager first step, device memory (sync_hyper) in the graphs
        if first:
            ok = calls == [(1, False)] and not opt.capturable
        else:
            ok = opt.capturable and calls == ([] if k == 3 else [(0, True)])
        if not ok:
            errors.append((k, side, 'SGD launches (first, device hyper-parameters)', calls, opt.capturable))
        if old_hyper is not None:
            # the replay used the new rate: the chain with the old one misses
            stale = sgd_check(before, grads, after, old_hyper, first)[1]
            print('  the same replay against the previous rate %.4g: %d elements off' % (old_hyper[0], stale))
            if stale == 0:
                errors.append((k, side, 'replay after a learning-rate change matches the old rate'))
        del before, after, grads, bn_graph, tloss
        torch.cuda.empty_cache()
    gs.poll()
    print('captures: %d' % gs.captures)
    assert not errors, errors
    assert gs.captures == 2, gs.captures


# ------------------------------------------------------------------------------------------------------------ part 4
@pytest.mark.parametrize('two_streams', [True, False], ids=['two-streams', 'one-stream'])
def test_accumulated_gradients(two_streams, monkeypatch):
    """configs[1], two batches, two backward passes without zeroing in between (no reducer: .grad is a plain tensor, so
    every parameter takes the accumulating branch of NetRunner._param_grad): every gradient bit-equal to the fp32 sum of
    the two single-pass gradients."""
    from fewshot_detection_b200 import engine
    g1, g2 = single(SEED + 1).grads, single(SEED + 2).grads
    monkeypatch.setattr(engine, 'WGRAD_STREAM', two_streams)
    cnt = {}
    r = run(416, 64, 20, SEED, [SEED + 1, SEED + 2], lambda real: cnt.setdefault('c', StreamCount(real)))
    release(r)
    ref = accumulated_reference()
    dg = differing(r.grads, ref)
    nan = [n for n, g in r.grads.items() if not torch.isfinite(g).all()]
    print('\naccumulated gradients (%s, %d of %d launches on the second stream): %s%s; %.2f s' % (
        'two streams' if two_streams else 'one stream', cnt['c'].side, cnt['c'].total,
        'bit-equal to fl32(g1 + g2)' if not dg else 'first differing %s (%d of %d)' % (dg[0], len(dg), len(ref)),
        ', non-finite in %d tensors' % len(nan) if nan else '', r.secs))
    assert (cnt['c'].side > 0) == two_streams
    assert not dg, (dg[0], len(dg), nan[:3])
    assert len(g1) == len(g2) == N_PARAMS


def accumulated_reference():
    """fl32(g1 + g2) of the single-pass gradients of the configs[1] batches SEED + 1 and SEED + 2"""
    g1, g2 = single(SEED + 1).grads, single(SEED + 2).grads
    return {n: (g1[n].cuda() + g2[n].cuda()).cpu() for n in g1}


# ------------------------------------------------------------------------------------------------------------ part 5
class _Forgetful(list):
    """A NetRunner._keep that keeps nothing (the audit's teeth)."""

    def append(self, item):
        pass


class LifetimeAudit(object):
    """Makes a premature free on the second stream show up in the values, whatever the timing.

    engine.call is wrapped so that on the second stream each conv block's weight-gradient launches are preceded by a
    sleep (the first launch of the block) and each is followed by an event and another sleep; NetRunner._convbn_bwd is
    wrapped so that, once the block has returned and its Python references are gone, the main stream
    (1) NaN-fills every block the caching allocator lists as inactive in the main stream's segments of its default pool
        - while the second stream still sleeps before the block's first launch, so an input it is about to read that
        was released reads NaN;
    (2) waits for the event behind the block's last launch and poisons again - while the second stream sleeps before
        the torch operations queued behind that launch (the accumulation into .grad), so an output it wrote into a
        released block reads NaN.
    The fills go through views of the blocks' addresses on the main stream: only memory the allocator already holds
    and would hand to the next main-stream allocation is written, nothing is allocated or returned to the device.
    Every poisoning must have finished before the sleep it relies on ended (checked from the events' times), so a
    missed window fails the audit instead of passing it.  Sleeps: one per block plus one per launch, ~10 ms each."""

    def __init__(self, forget_keep=False):
        from fewshot_detection_b200 import engine
        self.main = torch.cuda.current_stream()
        self.forget = forget_keep
        self.real_convbn = engine.NetRunner._convbn_bwd
        self.real_call = None
        self.fork = None
        self.windows = []           # (what, event after a poisoning, event at the end of the sleep it must fit in)
        self.forks = self.sleeps = self.poisoned = 0
        self.t0 = self._event(self.main)

    @staticmethod
    def _event(stream):
        e = torch.cuda.Event(enable_timing=True)
        e.record(stream)
        return e

    def _sleep(self, stream):
        torch.cuda._sleep(SLEEP_CYCLES)
        self.sleeps += 1
        return self._event(stream)

    def wrap(self, real):
        self.real_call = real
        return self.call

    def call(self, fn, *a):
        cur = torch.cuda.current_stream()
        if cur == self.main:
            return self.real_call(fn, *a)
        if self.fork is None:
            raise AssertionError('second-stream launch outside a conv block backward: %s' % fn)
        if self.fork['held'] is None:
            self.fork['held'] = self._sleep(cur)
        rc = self.real_call(fn, *a)
        self.fork['done'] = self._event(cur)
        self.fork['resume'] = self._sleep(cur)
        return rc

    def convbn(self, runner, rec, st):
        if self.forget:
            runner._keep = _Forgetful()
        self.fork = {'held': None, 'done': None, 'resume': None}
        try:
            self.real_convbn(runner, rec, st)
        finally:
            fork, self.fork = self.fork, None
        if fork['held'] is None:
            return
        self.forks += 1
        self.windows.append(('before the first read', self._poison(), fork['held']))
        self.main.wait_event(fork['done'])
        self.windows.append(('after the last write', self._poison(), fork['resume']))

    def _poison(self):
        for seg in torch.cuda.memory_snapshot():
            if seg['stream'] != self.main.cuda_stream or tuple(seg.get('segment_pool_id', (0, 0))) != (0, 0):
                continue
            for blk in seg['blocks']:
                if blk['state'] == 'inactive':
                    dev(blk['address'], blk['size'] // 4).fill_(float('nan'))
                    self.poisoned += blk['size']
        return self._event(self.main)

    def margins(self):
        """ms from the end of each poisoning to the end of the sleep it fell in (negative: the window was missed)"""
        torch.cuda.synchronize()
        return [(what, self.t0.elapsed_time(end) - self.t0.elapsed_time(done)) for what, done, end in self.windows]


def audited_run(batch_seeds, monkeypatch, forget_keep=False, replicas=1):
    from fewshot_detection_b200 import engine
    audit = LifetimeAudit(forget_keep)
    monkeypatch.setattr(engine.NetRunner, '_convbn_bwd', lambda runner, rec, st: audit.convbn(runner, rec, st))
    try:
        r = run(416, 64, 20, SEED, batch_seeds, audit.wrap, replicas)
    finally:
        monkeypatch.setattr(engine.NetRunner, '_convbn_bwd', audit.real_convbn)
    margins = audit.margins()
    release(r)
    worst = min(margins, key=lambda w: w[1])
    print('audit of %d batch(es)%s: %d forks, %d sleeps, %.1f GB poisoned, smallest margin %.2f ms (%s), %.1f s' % (
        len(batch_seeds), ' with NetRunner._keep disabled' if forget_keep else '', audit.forks, audit.sleeps,
        audit.poisoned / 1e9, worst[1], worst[0], r.secs))
    assert audit.forks > 0
    return r, margins


def test_lifetime_audit(monkeypatch):
    """The plain and the accumulating configs[1] step under LifetimeAudit: both bit-equal to their unaudited results."""
    print()
    errors = []
    for batches, ref in (([SEED + 1], single(SEED + 1).grads), ([SEED + 1, SEED + 2], accumulated_reference())):
        r, margins = audited_run(batches, monkeypatch)
        missed = [w for w in margins if not w[1] > 0]
        dg = differing(r.grads, ref)
        nan = [n for n, g in r.grads.items() if not torch.isfinite(g).all()]
        print('  gradients: %s%s' % ('bit-equal' if not dg else 'first differing %s (%d of %d)' % (dg[0], len(dg), len(ref)),
                                     ', non-finite in %d tensors' % len(nan) if nan else ''))
        if missed:
            errors.append((len(batches), 'poisoning windows missed', len(missed), missed[:3]))
        if dg:
            errors.append((len(batches), 'gradients', dg[0], len(dg), nan[:3]))
        if len(batches) == 1:
            db = differing(r.bn, single(SEED + 1).bn)
            if db:
                errors.append((1, 'BatchNorm running statistic', db[0]))
    assert not errors, errors


def test_lifetime_audit_has_teeth(monkeypatch):
    """With NetRunner._keep disabled, the second stream reads dz and its planes after the main stream released them:
    the audit must report NaN or a mismatch."""
    print()
    r, margins = audited_run([SEED + 1], monkeypatch, forget_keep=True)
    dg = differing(r.grads, single(SEED + 1).grads)
    nan = [n for n, g in r.grads.items() if not torch.isfinite(g).all()]
    print('  %d gradients differ, %d non-finite (first: %s)' % (len(dg), len(nan), dg[:1]))
    assert nan or dg
