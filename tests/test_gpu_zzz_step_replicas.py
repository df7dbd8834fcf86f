"""The replica step (Darknet(..., replicas=R), the reference's four-replica nn.DataParallel step) at full size.

The replica step runs a second forward and backward path through the network: segmented BatchNorm passes (per-replica
statistics, [R][C] vectors), a per-replica head (one W (.) rw_r and one GEMM per replica over that replica's images, one
weight-gradient GEMM and one fsdet_head_param_grads per replica, dW summed through fsdet_copy_channels) and every
training GEMM without fused statistics rows.  This file gives it the evidence the one-replica step has.

  test_replica_step_checked        one eager step under both step checkers chained, bars unchanged, at R = 4, B = 64, 20
                                   classes, 416 (configs[1] as the reference trains it) and 608, at R = 4, B = 4, 3
                                   classes (one image per replica, support segments of 3 images) and at R = 2, B = 64:
                                   every segmented entry point against float64 per segment, RegionLossV2 on the head
                                   output (build_targets bit-exact, gradient within its first-order bound), the GEMM
                                   flavours reached equal to tests/test_tile_plans_replicas.py's pins, every seg-* kind
  test_replica_step_vs_float64_oracle   R = 4, B = 64, 20 classes, 416 against oracle.darknet.MetaDarknet in float64:
                                   R separate train-mode calls on the replicas' images and support sets, one
                                   region_loss_v2 over the concatenated outputs, one backward.  Head output and loss,
                                   running statistics (those of the oracle's first call), head weight and bias, drw row
                                   by row, and the layers after the last max-pool; bars from the one-replica step's own
                                   distance from float64 at the same weights and seeds
  test_seg_finalize_check_has_teeth   segment 1's statistics overwritten with segment 0's fail the segment check
  test_swapped_reweighting_rows_need_the_oracle   replica 1's head built from replica 0's vectors passes every
                                   per-kernel check and fails the float64 oracle comparison
  test_two_stream_replica_lifetime_audit   the replica step with its weight gradients on the second stream under
                                   test_gpu_zz_step_shipped.LifetimeAudit, bit-equal to the one-stream replica step

The file name sorts after every other GPU test: the slowest tests run last, and test_gpu_zz_step_shipped's lifetime audit,
whose 10 ms windows depend on how much free memory the allocator holds, runs before these steps have grown its cache.
"""
import math

import pytest
import torch

from test_gpu_zz_step_gemms import run_step
from test_gpu_zz_step_memops import dev
from test_gpu_zz_step_scales import check_region
from test_gpu_zz_step_shipped import _model, audited_run, checked, differing, release, report_checked, run
from test_tile_plans_replicas import REPLICA_FLAVOURS, SHAPES
from test_tile_plans_scales import FLAVOURS

pytestmark = pytest.mark.gpu

SEEDS = {SHAPES[0]: 2101, SHAPES[1]: 2111, SHAPES[2]: 2121, SHAPES[3]: 2131}
IDS = ['r4-416', 'r4-608', 'r4-b4', 'r2-416']
# every kind of segmented pass a replica step reaches (test_gpu_zz_step_memops.MemChecker's names)
SEG_KINDS = {'seg-colstats', 'seg-finalize', 'seg-fwd-full', 'seg-fwd-pool', 'seg-fwd-pool+full', 'seg-fwd-f32',
             'seg-fwd-planes', 'seg-fwd-odd', 'seg-bwd-finalize', 'seg-bwd-pool-only', 'seg-bwd-general-full',
             'seg-bwd-general-full+pool', 'seg-bwd-odd'}
# the one-segment BatchNorm passes: a replica step runs none of them (the network has no conv + bias block)
PLAIN_KINDS = {'fwd-full', 'fwd-pool', 'fwd-pool+full', 'bwd-pool-only', 'bwd-general-full', 'bwd-general-full+pool'}
GEMM_KINDS = {'fwd', 'dgrad', 'wgrad', 'head', 'head-dgrad', 'head-wgrad', 'first-fwd', 'first-wgrad', 'weight-prep'}
E2E_FACTOR = 2.0        # end-to-end bar: this many times the one-replica step's distance from float64 ...
E2E_CAP = 2e-4          # ... at most the evaluation pass's cap
RUNNING_BAR = 1e-4      # running statistics against the oracle's state after its first call (relative L2)
WHICH_CALL = 100.0      # ... and at least this many times closer to it than to the state after the second call
REPLICA_SLEEP_CYCLES = 200000000    # LifetimeAudit's sleeps for the replica step: about 100 ms each


def chained(made, inject=None):
    """wrap() chaining both step checkers (test_gpu_zz_step_shipped.checked), with `inject` (a wrap of the engine's
    own call) underneath them: an injected error is what the checkers see the kernel produce"""
    chain = checked(made)
    return chain if inject is None else (lambda real: chain(inject(real)))


# ------------------------------------------------------------------------------------------------------------ part 3
@pytest.mark.parametrize('shape', SHAPES, ids=IDS)
def test_replica_step_checked(shape):
    from test_gpu_zz_step_gemms import report as report_gemms
    from test_gpu_zz_step_memops import report as report_mem
    side, bs, cs, R = shape
    print('\n==== R = %d, side %d, B = %d, %d classes' % (R, side, bs, cs))
    made = {}
    out, L, tgt, secs = run_step(side, bs, cs, SEEDS[shape], chained(made), replicas=R)
    gchk, mchk = made['gemm'], made['mem']
    errors = []
    for rep, chk in ((report_gemms, gchk), (report_mem, mchk)):
        try:
            rep(chk, secs)
        except AssertionError as e:
            errors.append(e)
    fails, row = check_region(out, L, tgt, 'full', None)
    print(row)
    errors += fails
    reached = gchk.cov & set(FLAVOURS)
    heads = [l['shape'] for l in gchk.log if l['kind'] == 'head']
    print('GEMM flavours reached %s; head GEMMs %s' % (sorted(reached), heads))
    print('segmented kinds covered: %s' % sorted(k for k in mchk.cov if k.startswith('seg-')))
    assert not errors, errors
    assert reached == REPLICA_FLAVOURS[shape], (sorted(reached), sorted(REPLICA_FLAVOURS[shape]))
    assert GEMM_KINDS <= gchk.cov, sorted(GEMM_KINDS - gchk.cov)
    # every training convolution without statistics rows: the segmented pass computes the statistics
    assert 'fwd-nostats' in gchk.cov and 'fwd-stats' not in gchk.cov and not mchk.stat_src
    assert SEG_KINDS <= mchk.cov, sorted(SEG_KINDS - mchk.cov)
    assert not PLAIN_KINDS & mchk.cov, sorted(PLAIN_KINDS & mchk.cov)
    # one head GEMM per replica, each over B / R images
    assert len(heads) == R and all(h.startswith('%dx' % (bs // R)) for h in heads), heads


# ------------------------------------------------------------------------------------------------------------ part 4
def rel_errors(got, ref):
    """(relative L2, max element-wise error relative to max |ref|) against float64"""
    d = got.double().cpu() - ref.cpu()
    return (d.norm() / ref.norm().clamp_min(1e-300)).item(), (d.abs().max() / ref.abs().max().clamp_min(1e-300)).item()


def relt(a, b):
    return ((a.double().cpu() - b.double().cpu()).norm() / b.double().cpu().norm().clamp_min(1e-300)).item()


class DrwCapture(object):
    """Copies each fsdet_head_param_grads call's drw output ([n_cls][K], one call per replica) after the call."""

    def __init__(self, real):
        self.real = real
        self.drw = []

    def __call__(self, fn, *a):
        rc = self.real(fn, *a)
        if fn == 'fsdet_head_param_grads':
            dweff, Wp, rw, dW, drw, n_cls, O, K, st = a
            self.drw.append(dev(drw, n_cls * K).view(n_cls, K).clone())
        return rc


def last_pool_index(blocks):
    """module index of the detector's last stride-2 max-pool: the layers after it see no arg-max flip"""
    ind, last = -2, None
    for b in blocks:
        ind += 1
        if b['type'] == 'maxpool' and b['stride'] == '2':
            last = ind
    return last


def oracle_detect(om, x, dw, grad_from):
    """oracle.darknet._run_blocks of the detector, the modules before `grad_from` under no_grad: their outputs are
    constants, so memory stays at one replica's activations while the gradients of the later layers are exact"""
    from oracle import darknet as ODK
    ind, outputs = -2, {}
    for block in om.blocks:
        ind += 1
        t = block['type']
        with torch.set_grad_enabled(ind >= grad_from):
            if t in ('net', 'learnet', 'region'):
                continue
            if t in ('convolutional', 'maxpool', 'reorg', 'globalmax'):
                x = om.models[ind]((x, dw)) if ODK.is_dynamic(block) else om.models[ind](x)
            elif t == 'route':
                layers = [int(i) if int(i) > 0 else int(i) + ind for i in block['layers'].split(',')]
                x = outputs[layers[0]] if len(layers) == 1 else torch.cat([outputs[l] for l in layers], 1)
            else:
                raise NotImplementedError(t)
            outputs[ind] = x
    return x


def running_state(om):
    return {n: b.detach().clone() for n, b in om.named_buffers() if n.endswith(('running_mean', 'running_var'))}


def oracle_replica_step(state, blocks, learnet_blocks, x, metax, mask, tgt, R, seen, out_step):
    """The reference's R-replica step in float64: R train-mode calls (support net, then detector) on x[r B/R:(r+1) B/R]
    with support set r, one region_loss_v2 over the concatenated outputs, one backward.  The backward starts from
    region_loss_v2's gradient at the step's own output `out_step`: build_targets' IoU thresholds then take the decisions
    the step took (part 3 checks its build_targets bit-exact on that output), so a box within the output error of a
    threshold cannot move the comparison; the oracle's own output gives the loss.  Returns the output, the loss, the
    oracle model (its gradients), the drw of each replica, the running statistics after each call and the index of the
    first module after the last max-pool."""
    from oracle import darknet as ODK
    om = ODK.MetaDarknet([dict(b) for b in blocks], [dict(b) for b in learnet_blocks])
    om.load_state_dict(state)
    om = om.to(device='cuda', dtype=torch.float64).train()
    grad_from = last_pool_index(om.blocks) + 1
    nb, cs = x.shape[0] // R, metax.shape[0] // R
    outs, rws, snaps = [], [], []
    for r in range(R):
        with torch.no_grad():
            rw = om.meta_forward(metax[r * cs:(r + 1) * cs].cuda().double(), mask[r * cs:(r + 1) * cs].cuda().double())[0]
        rw = rw.detach().requires_grad_()
        outs.append(oracle_detect(om, x[r * nb:(r + 1) * nb].cuda().double(), rw, grad_from))
        rws.append(rw)
        snaps.append(running_state(om))
    out = torch.cat(outs, 0)
    loss = oracle_loss(out, tgt, om, seen)[0]
    out.backward(oracle_loss(out_step, tgt, om, seen)[1])
    return out.detach(), loss, om, [rw.grad.reshape(cs, -1) for rw in rws], snaps, grad_from


def oracle_loss(out, tgt, om, seen):
    """oracle.region_loss.region_loss_v2 (a float32 restatement, on the host) of `out` rounded to float32: (the loss,
    its gradient w.r.t. the output in float64).  Rounding moves both by about 1e-7 relative, far below the end-to-end
    bars."""
    from oracle import region_loss as ORL
    o32 = out.detach().float().cpu().requires_grad_()
    loss = ORL.region_loss_v2(o32, tgt, om.anchors, om.num_anchors, om.num_classes, seen=seen)
    loss.backward()
    return loss.item(), o32.grad.to(device=out.device, dtype=torch.float64)


def head_side_gradients(r, om, grad_from):
    """{name: relative L2 distance} of the gradients of every module after the last max-pool (run r against oracle om)"""
    return {n: relt(r.grads[n], p.grad) for n, p in om.named_parameters()
            if n.startswith('models.') and int(n.split('.')[1]) >= grad_from}


def one_replica_distance(side, bs, cs, seed, bseed):
    """The one-replica step's own distance from its float64 oracle at the same seeded weights and batch seed: (relative
    L2, max element) of the head output, the loss's relative error, and the head-side gradients' relative L2"""
    from test_gpu_zz_configs import _batch
    state = {k: v.clone() for k, v in _model(side, seed)[0].state_dict().items()}
    r = run(side, bs, cs, seed, [bseed])
    x, metax, mask, tgt = _batch(bs, cs, side, bseed)
    o64, l64, om, _, _, grad_from = oracle_replica_step(state, r.model.blocks, r.model.learnet_blocks, x, metax, mask, tgt,
                                                        1, r.L.seen, r.out)
    e = rel_errors(r.out, o64)
    le = abs(r.loss - l64) / abs(l64)
    grads = head_side_gradients(r, om, grad_from)
    release(r)
    del om, o64
    torch.cuda.empty_cache()
    return e, le, grads


def end_to_end(shape, seed, r, drw, state):
    """Compare the R-replica run `r` (its model started from `state`; drw: the per-replica drw it computed) with the
    float64 oracle step.  Returns (failures, printed lines)."""
    from test_gpu_zz_configs import _batch
    side, bs, cs, R = shape
    bseed = seed + 1
    e1, le1, g1 = one_replica_distance(side, bs, cs, seed, bseed)
    bar = tuple(min(E2E_CAP, E2E_FACTOR * e) for e in e1)
    x, metax, mask, tgt = _batch(bs, cs, side, bseed, replicas=R)
    m = r.model
    o64, l64, om, drw64, snaps, grad_from = oracle_replica_step(state, m.blocks, m.learnet_blocks, x, metax, mask, tgt, R,
                                                                r.L.seen, r.out)
    first, second = snaps[0], snaps[1]
    fails, lines = [], []
    eo = rel_errors(r.out, o64)
    le = abs(r.loss - l64) / abs(l64)
    lines.append('one-replica step from float64: head output %.2e relative L2, %.2e max element; loss %.2e' % (e1 + (le1,)))
    lines.append('replica step from float64:     head output %.2e relative L2, %.2e max element; loss %.2e (bars %.2e, %.2e)'
                 % (eo + (le, bar[0], bar[1])))
    if not (eo[0] <= bar[0] and eo[1] <= bar[1]):
        fails.append(('head output', eo, bar))
    if not le <= bar[0]:
        fails.append(('loss', r.loss, l64, le, bar[0]))
    # running statistics: replica 0's (the oracle's first call), far from what a second replica would have added
    worst_first, worst_ratio = 0.0, math.inf
    for n, got in r.bn.items():
        d1, d2 = relt(got, first[n]), relt(got, second[n])
        worst_first = max(worst_first, d1)
        worst_ratio = min(worst_ratio, d2 / max(d1, 1e-300))
        if not (d1 <= RUNNING_BAR and d2 >= WHICH_CALL * d1):
            fails.append(('running statistic', n, d1, d2))
    lines.append('running statistics (%d tensors): worst %.2e from the first call, at least %.0fx closer to it than to '
                 'the second' % (len(r.bn), worst_first, worst_ratio))
    # head-side gradients: the layers after the last max-pool (the head's W and bias among them) against the same bar
    # as the head output, or twice the one-replica step's own distance for that tensor where that is larger
    worst = []
    for n, e in head_side_gradients(r, om, grad_from).items():
        gbar = max(bar[0], E2E_FACTOR * g1[n])
        worst.append((e / gbar, e, g1[n], n))
        if not e <= gbar:
            fails.append(('gradient', n, e, gbar))
    worst.sort(reverse=True)
    lines.append('gradients of the %d tensors after the last max-pool, (replica step, one-replica step) from float64:' % len(worst))
    lines += ['  %-28s %.2e %.2e  ratio to the bar %.3f' % (n, e, e1_, q) for q, e, e1_, n in worst]
    rows = []
    for k in range(R):
        for c in range(cs):
            rows.append((relt(drw[k][c], drw64[k][c]), k, c))
    rows.sort(reverse=True)
    lines.append('drw, %d rows: worst %.2e (replica %d, row %d)' % (len(rows), rows[0][0], rows[0][1], rows[0][2]))
    if not rows[0][0] <= bar[0]:
        fails.append(('drw rows over the bar', [t for t in rows if t[0] > bar[0]][:5]))
    del om
    torch.cuda.empty_cache()
    return fails, lines


def replica_run_vs_oracle(shape, inject=None, made=None):
    """The seeded R-replica step and its end-to-end comparison; checked when `made` is a dict, with `inject` (a wrap
    of engine.call) above the checkers: what it changes is what the engine asked the kernels for.  Returns (failures,
    printed lines)."""
    from fewshot_detection_b200.cfg import cfg
    side, bs, cs, R = shape
    seed = SEEDS[shape]
    state = {k: v.clone() for k, v in _model(side, seed, R)[0].state_dict().items()}
    cap = {}

    def wrap(real):
        cap['drw'] = DrwCapture(real)
        inner = cap['drw'] if made is None else checked(made)(cap['drw'])
        return inner if inject is None else inject(inner)
    old = cfg.neg_ratio
    cfg.neg_ratio = 'full'
    try:
        r = run(side, bs, cs, seed, [seed + 1], wrap, replicas=R)
        drw = cap['drw'].drw
        assert len(drw) == R, len(drw)
        fails, lines = end_to_end(shape, seed, r, drw, state)
    finally:
        cfg.neg_ratio = old
    release(r)
    return fails, lines


def test_replica_step_vs_float64_oracle():
    """R = 4, B = 64, 20 classes, 416: the replica step against the float64 four-replica oracle."""
    fails, lines = replica_run_vs_oracle(SHAPES[0])
    print('\n' + '\n'.join(lines))
    assert not fails, fails


# ------------------------------------------------------------------------------------------------------------ part 5
class _Stop(Exception):
    pass


def test_seg_finalize_check_has_teeth():
    """fsdet_bn_seg_finalize's segment-1 mean, invstd, scale and shift overwritten with segment 0's (under the checkers,
    so they see it as the kernel's output): the segment check of the first BatchNorm layer reports segment 1."""
    made = {}

    def inject(real):
        def call(fn, *a):
            rc = real(fn, *a)
            if fn == 'fsdet_bn_seg_finalize':
                C = a[17]
                for p in a[10:14]:
                    dev(p + 4 * C, C).copy_(dev(p, C))
            return rc
        return call

    def stop_after_first(real):
        chk = chained(made, inject)(real)

        def call(fn, *a):
            rc = chk(fn, *a)
            if fn == 'fsdet_bn_seg_finalize':
                raise _Stop()
            return rc
        return call
    side, bs, cs, R = SHAPES[2]
    with pytest.raises(_Stop):
        run_step(side, bs, cs, SEEDS[SHAPES[2]], stop_after_first, replicas=R)
    f = made['mem'].failures
    print('\nreported:', f)
    assert any(w[0] == 'bn_finalize mean / invstd' and w[5] == 1 for w in f), f
    assert not any(w[0] == 'bn_finalize mean / invstd' and w[5] != 1 for w in f), f


def test_swapped_reweighting_rows_need_the_oracle():
    """Replica 1's fsdet_head_weff given replica 0's reweighting rows: each kernel computes what it was asked to (every
    per-kernel check passes), but the step is another step - only the end-to-end comparison reports it."""
    def inject(real):
        first = []

        def call(fn, *a):
            if fn == 'fsdet_head_weff':
                a = list(a)
                if first:
                    a[2] = first[0]
                else:
                    first.append(a[2])
            return real(fn, *a)
        return call
    made = {}
    fails, lines = replica_run_vs_oracle(SHAPES[2], inject, made)
    print('\n' + '\n'.join(lines))
    errors = report_checked(made, 0.0)
    assert not errors, errors
    print('end-to-end failures:', fails)
    assert any(f[0] == 'head output' for f in fails), fails


# ------------------------------------------------------------------------------------------------------------ part 6
def test_two_stream_replica_lifetime_audit(monkeypatch):
    """R = 4, B = 64, 416 with the weight gradients on the second stream (NetRunner._side_ok without its replica guard)
    under LifetimeAudit: gradients and BatchNorm running statistics bit-equal to the one-stream replica step."""
    import test_gpu_zz_step_shipped as shipped
    from fewshot_detection_b200 import engine
    from test_gpu_zz_step_shipped import SEED
    # the replica step's main stream holds more free blocks (R support sets), and listing and filling them takes longer
    # than the one-replica step's 10 ms windows: every poisoning must still finish inside the sleep it relies on
    monkeypatch.setattr(shipped, 'SLEEP_CYCLES', REPLICA_SLEEP_CYCLES)
    print()
    one = run(416, 64, 20, SEED, [SEED + 1], replicas=4)
    release(one)
    real = engine.NetRunner._side_ok

    def side_ok(runner):
        seg, runner._bwd_segments = runner._bwd_segments, 1
        try:
            return real(runner)
        finally:
            runner._bwd_segments = seg
    monkeypatch.setattr(engine.NetRunner, '_side_ok', side_ok)
    r, margins = audited_run([SEED + 1], monkeypatch, replicas=4)
    missed = [w for w in margins if not w[1] > 0]
    dg, db = differing(r.grads, one.grads), differing(r.bn, one.bn)
    nan = [n for n, g in r.grads.items() if not torch.isfinite(g).all()]
    print('  two-stream replica step vs one stream: gradients %s, BatchNorm statistics %s%s' % (
        'bit-equal' if not dg else 'first differing %s (%d of %d)' % (dg[0], len(dg), len(r.grads)),
        'bit-equal' if not db else 'first differing %s (%d)' % (db[0], len(db)),
        ', non-finite in %d tensors' % len(nan) if nan else ''))
    print('  smallest margin %.1f ms' % min(w[1] for w in margins))
    assert not missed, missed[:3]
    assert not dg and not db and not nan, (dg[:3], db[:3], nan[:3])
