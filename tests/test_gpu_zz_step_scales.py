"""The training step at every multi-scale input side: each kernel against float64, and the per-side step graphs against
eager steps.

Multi-scale base training (dataset.multiscale_width) draws the query side from 320, 352, ..., 608, so most steps run at a
side other than 416.  The kernels take different paths at each side: the first layer's last 104-column tile is partial
everywhere but at 416 (and its unrolled row walk ends on another remainder), the halo-tile kernel's last 16-row tile
hangs past the image at side / 4 in {88, 104, 120, 136, 152}, every im2col GEMM and weight-gradient split ends on another
short tile or slice, and from 512 up the first layer's pre-BatchNorm output is 2^31 bytes or more.

  test_step_at_side            one full-batch eager step per side (B = 64, 15 classes; and configs[4]: 608x608, 80
                               classes) under both step checkers chained - every GEMM (test_gpu_zz_step_gemms) and every
                               BatchNorm, pooling, head and data-movement kernel (test_gpu_zz_step_memops) against float64
                               with their bars unchanged; the flavours reached must be exactly those the C planner predicts
                               for the side's layer list (tests/test_tile_plans_scales.py).  Then the step's real head
                               output goes through RegionLossV2 at neg = full and at neg = 1: build_targets bit-exact
                               against the oracle, the six loss parts and every gradient element against float64
  test_graph_steps_match_eager_steps   GraphedTrainStep over all ten sides in schedule order (one graph per side, one
                               shared memory pool, sides revisited after other graphs were captured) against an eager
                               trajectory from the same seeds: parameters and momentum buffers bit-equal after every step
  test_trainer_losses_are_per_step_values   MetaTrainer.losses on the graph path equals the eager losses step by step
"""
import math
import random
import sys

import numpy as np
import pytest
import torch

from test_gpu_zz_step_gemms import COVERAGE as GEMM_COVERAGE, StepChecker, report as report_gemms, run_step
from test_gpu_zz_step_memops import COVERAGE as MEM_COVERAGE, MemChecker, dev, report as report_mem
from test_tile_plans_scales import FLAVOURS, SIDES, first_layer_tail, planned_flavours, query_gemms, support_gemms

pytestmark = pytest.mark.gpu

U = 2.0 ** -24          # fp32 unit roundoff
# CUDA's expf is within 2 ulp (at most 4 U relative), logf within 1 ulp (2 U), division and sqrtf are correctly rounded
# (the library is built without fast-math); see derive_bar_* below
EXP_ERR, LOG_ERR = 4 * U, 2 * U

CASES = [pytest.param(s, 64, 15, id='voc%d' % s) for s in SIDES if s != 416] + [pytest.param(608, 64, 80, id='configs4')]


# ------------------------------------------------------------------------------------------------------ region loss
class RegionCapture(object):
    """Wraps region_loss.call: each region kernel runs as launched, then its outputs are copied (they are freed when the
    loss returns), together with the launch arguments."""

    def __init__(self, real):
        self.real = real
        self.got = {}

    def __call__(self, fn, *a):
        rc = self.real(fn, *a)
        torch.cuda.synchronize()
        if fn == 'fsdet_region_decode':
            out, inds, nB, nb_dev, A, nC, H, W, anc, pred, st = a
            self.got['pred'] = dev(pred, nB * A * H * W * 4).view(-1, 4).clone()
            self.got['inds'] = dev(inds, nB, torch.int32).long().clone() if inds else torch.arange(nB, device='cuda')
        elif fn == 'fsdet_build_targets':
            pred, tgt, anc, nB, A, H, W, max_boxes, noobj, obj, thresh, seen = a[:12]
            self.got['bt'] = dict(tgt=dev(tgt, nB * 250, torch.float64).view(nB, 250).clone(), anchors=dev(anc, 2 * A, torch.float64).tolist(),
                                  A=A, H=H, W=W, noobj=noobj, obj=obj, thresh=thresh, seen=seen, max_boxes=max_boxes,
                                  planes=[dev(p, nB * A * H * W).view(nB, A, H * W).clone() for p in a[12:21]],
                                  counters=dev(a[21], 4, torch.int32).tolist())
        elif fn == 'fsdet_region_loss_grad':
            (out, grad, inds, nb_dev, imgs, rows_total, nB, bs, cs, A, nC, H, W) = a[:13]
            coord_scale, class_scale, mode, metayolo, losses = a[22:27]
            self.got['loss'] = dict(out=dev(out, rows_total * A * (5 + nC) * H * W).view(rows_total, A, 5 + nC, H * W).clone(),
                                    grad=dev(grad, rows_total * A * (5 + nC) * H * W).view(rows_total, A, 5 + nC, H * W).clone(),
                                    img_start=dev(imgs, bs + 1, torch.int32).long().clone(), nB=nB, bs=bs, cs=cs, nC=nC,
                                    coord_scale=coord_scale, class_scale=class_scale, mode=mode,
                                    losses=dev(losses, 8, torch.float64).clone())
        return rc


def sigmoid_err(s):
    """|fl(1 / (1 + expf(-v))) - sigmoid(v)| <= 6 U sigmoid(v): expf (4 U), the sum (U) and the division (U), each a
    relative error of the result to first order (the expf error enters scaled by e / (1 + e) <= 1)."""
    return 6 * U * s + 2.0 ** -149


def derive_bar_box(o, m, M, tx, ty, tw, th, tconf, cscale):
    """float64 gradient of channels 0..4 (x, y, w, h, objectness) of the kept rows and its element-wise bar.

    The kernel evaluates g_x = ((((c * dx) * m) * x) * (1 - x)) with dx = x m - tx m, x = sigmoid in fp32.  To first
    order, a product of factors f_i each off by e_i is off by sum_i e_i prod_{j != i} |f_j|, plus one rounding U |g| per
    multiplication; a difference a - b of computed values is off by their errors plus U |a - b| (U |a| + U |b| for the
    two products it is formed from: an fma contraction only removes roundings).  So
        e(x) = 6 U x,  e(1 - x) = e(x) + U |1 - x|,  e(dx) = |m| e(x) + U (|x m| + |tx m| + |dx|)
        e(g_x) = |c m| (e(dx) |x (1 - x)| + |dx| e(x) |1 - x| + |dx x| e(1 - x)) + 4 U |g_x|
    w, h are the raw outputs: e(dw) = U (|w m| + |tw m| + |dw|), e(g_w) = |c m| e(dw) + 2 U |g_w|.  Objectness uses
    sM = sqrtf(M) (e = U sM), dc = conf sM - tconf sM and g = ((dc sM) conf)(1 - conf), expanded the same way.
    The bar is twice that first-order bound (the second-order terms are ~1e-7 of it)."""
    g = torch.zeros(o.shape[:2] + (5,) + o.shape[3:], dtype=torch.float64, device=o.device)
    bar = torch.zeros_like(g)
    parts, pbar = [], []
    for c, (t, sig) in enumerate(((tx, True), (ty, True), (tw, False), (th, False))):
        v = o[:, :, c].double()
        if sig:
            x = torch.sigmoid(v)
            ex = sigmoid_err(x)
            dx = x * m - t * m
            edx = m.abs() * ex + U * ((x * m).abs() + (t * m).abs() + dx.abs())
            gx = cscale * dx * m * x * (1 - x)
            e1 = ex + U * (1 - x).abs()
            eg = abs(cscale) * m.abs() * (edx * (x * (1 - x)).abs() + dx.abs() * ex * (1 - x).abs() + (dx * x).abs() * e1) \
                + 4 * U * gx.abs()
        else:
            dx = v * m - t * m
            edx = U * ((v * m).abs() + (t * m).abs() + dx.abs())
            gx = cscale * dx * m
            eg = abs(cscale) * m.abs() * edx + 2 * U * gx.abs()
        g[:, :, c], bar[:, :, c] = gx, 2 * eg
        parts.append(0.5 * cscale * (dx * dx).sum().item())
        pbar.append(2 * abs(cscale) * (dx.abs() * edx).sum().item())     # d(dx^2 / 2) = dx e(dx)
    conf = torch.sigmoid(o[:, :, 4].double())
    ec = sigmoid_err(conf)
    sM = M.sqrt()
    esM = U * sM
    dc = conf * sM - tconf * sM
    edc = ec * sM + (conf.abs() + tconf.abs()) * esM + U * ((conf * sM).abs() + (tconf * sM).abs() + dc.abs())
    gc = dc * sM * conf * (1 - conf)
    e1 = ec + U * (1 - conf).abs()
    eg = (edc * (sM * conf * (1 - conf)).abs() + dc.abs() * esM * (conf * (1 - conf)).abs() + (dc * sM).abs() * ec * (1 - conf).abs()
          + (dc * sM * conf).abs() * e1 + 3 * U * gc.abs())
    g[:, :, 4], bar[:, :, 4] = gc, 2 * eg
    parts.append(0.5 * (dc * dc).sum().item())
    pbar.append(2 * (dc.abs() * edc).sum().item())
    return g, bar, parts, pbar


def derive_bar_cls(z, tc, cscale):
    """float64 softmax-across-classes gradient of the class channel, z [n, cs] logits of the positions whose class mask
    sums to one, tc [n] the target class, and its element-wise bar.

    The kernel: mx = max z (exact), t_c = expf(fl(z_c - mx)) (off by t_c (4 U + U |z_c - mx|)), se = sum_c t_c in order
    (cs - 1 roundings of at most U se), lse = fl(mx + logf(se)), so e(lse) = e(se) / se + 2 U |log se| + U |lse|;
    p_c = expf(fl(z_c - lse)) is off by p_c (e(lse) + U |z_c - lse| + 4 U), and g_c = fl(c (fl(p_c - [c = tc]))) by
    that plus U |p_c - [c = tc]| + U |g_c|.  The loss term lse - z_tc is off by e(lse) + U |lse - z_tc|.  The bar is
    twice the first-order bound."""
    cs = z.shape[1]
    mx = z.max(1, keepdim=True).values
    d = z - mx
    t = d.exp()
    se = t.sum(1, keepdim=True)
    lse = mx + se.log()
    e_lse = ((t * (EXP_ERR + U * d.abs())).sum(1, keepdim=True) + (cs - 1) * U * se) / se + LOG_ERR * se.log().abs() + U * lse.abs()
    p = (z - lse).exp()
    onehot = torch.zeros_like(p)
    ok = (tc >= 0) & (tc < cs)
    onehot[ok.nonzero().squeeze(1), tc[ok]] = 1.0
    g = cscale * (p - onehot)
    bar = 2 * (abs(cscale) * (p * (e_lse + U * (z - lse).abs() + EXP_ERR) + U * (p - onehot).abs()) + U * g.abs())
    zt = z.gather(1, tc.clamp(0, cs - 1).view(-1, 1))
    loss = (cscale * (lse - zt))[ok].sum().item()
    lbar = 2 * abs(cscale) * (e_lse + U * (lse - zt).abs())[ok].sum().item()
    return g, bar, loss, lbar


def ratio(got, ref, bar):
    """max |got - ref| / bar; exact agreement is 0, a difference where the bar is 0 (or a NaN) is infinite"""
    d = (got.double() - ref).abs()
    r = torch.where(d == 0, torch.zeros_like(d), d / bar)
    return torch.nan_to_num(r, nan=math.inf, posinf=math.inf).max().item()


def check_region(out, L, tgt, neg, seed):
    """One RegionLossV2 call on the step's head output at cfg.neg_ratio = neg (Python `random` seeded with `seed`);
    returns (failures, table row)."""
    from oracle import region_loss as ORL
    from fewshot_detection_b200 import region_loss as RL
    from fewshot_detection_b200.cfg import cfg
    cap = RegionCapture(RL.call)
    old_neg, old_call = cfg.neg_ratio, RL.call
    cfg.neg_ratio = neg
    RL.call = cap
    random.seed(seed)
    try:
        L(out, tgt)
        torch.cuda.synchronize()
    finally:
        RL.call, cfg.neg_ratio = old_call, old_neg
    fails = []
    bt, ls, inds = cap.got['bt'], cap.got['loss'], cap.got['inds']
    nB, bs, cs = ls['nB'], ls['bs'], ls['cs']
    rows_total = bs * cs
    G = bt['H']
    # build_targets against the oracle, from the kernel's own decoded boxes and the kept label rows
    assert torch.equal(bt['tgt'].cpu(), tgt.view(-1, 250)[inds.cpu()])
    ref = ORL.build_targets(cap.got['pred'].cpu().numpy(), bt['tgt'].cpu().numpy(), bt['anchors'], bt['A'], G, G,
                            bt['noobj'], bt['obj'], bt['thresh'], bt['seen'], bt['max_boxes'])
    if tuple(bt['counters'][:2]) != (ref[0], ref[1]):
        fails.append(('build_targets nGT / nCorrect', G, neg, bt['counters'][:2], ref[:2]))
    names = ['coord_mask', 'conf_mask', 'cls_mask', 'tx', 'ty', 'tw', 'th', 'tconf', 'tcls']
    for k, v, r in zip(names, bt['planes'], ref[2:]):
        v = v.cpu().numpy().reshape(r.shape)
        ok = np.allclose(v, r, rtol=0, atol=1e-6) if k in ('tw', 'th') else np.array_equal(v.view(np.uint32), r.view(np.uint32))
        if not ok:
            fails.append(('build_targets', k, G, neg))
    # float64 loss parts and gradient from the same output, masks and targets
    m, M, _, tx, ty, tw, th, tconf, tcls = [p.view(nB, bt['A'], G * G).double() for p in bt['planes']]
    cmask = bt['planes'][2].view(nB, bt['A'], G * G)
    o = ls['out'][inds]                                      # [nB, A, 6, HW] kept rows, slot order
    gbox, bbox, parts, pbar = derive_bar_box(o, m, M, tx, ty, tw, th, tconf, ls['coord_scale'])
    gref = torch.zeros(ls['grad'].shape, dtype=torch.float64, device='cuda')
    gbar = torch.zeros_like(gref)
    gref[inds, :, :5] = gbox
    gbar[inds, :, :5] = bbox
    # class channel: per (image, anchor, cell) the class mask and target class summed over the image's kept rows (fp32
    # sums of small integers: exact), softmax across the image's cs rows of the FULL output where the mask sums to one
    img = torch.repeat_interleave(torch.arange(bs, device='cuda'), (ls['img_start'][1:] - ls['img_start'][:-1]))
    msum = torch.zeros(bs, bt['A'], G * G, device='cuda').index_add_(0, img, cmask)
    tsum = torch.zeros(bs, bt['A'], G * G, device='cuda').index_add_(0, img, bt['planes'][8].view(nB, bt['A'], G * G))
    pos = (msum == 1).nonzero()                              # (b, a, cell)
    z = ls['out'].view(bs, cs, bt['A'], 6, G * G)[pos[:, 0], :, pos[:, 1], 5, pos[:, 2]].double()   # [n, cs]
    gcls, bcls, loss_cls, lbar_cls = derive_bar_cls(z, tsum[pos[:, 0], pos[:, 1], pos[:, 2]].long(), ls['class_scale'])
    gv = gref.view(bs, cs, bt['A'], 6, G * G)
    bv = gbar.view(bs, cs, bt['A'], 6, G * G)
    gv[pos[:, 0], :, pos[:, 1], 5, pos[:, 2]] = gcls
    bv[pos[:, 0], :, pos[:, 1], 5, pos[:, 2]] = bcls
    r_grad = ratio(ls['grad'], gref, gbar)
    # the bar has teeth: the element with the largest bar moved by four times it is reported
    moved = ls['grad'].clone()
    i = gbar.flatten().argmax().item()
    moved.view(-1)[i] = (gref.view(-1)[i] + 4 * gbar.view(-1)[i]).float()
    if not ratio(moved, gref, gbar) > 3.0:
        fails.append(('region gradient bar without teeth', G, neg))
    if not r_grad <= 1.0:
        fails.append(('region gradient', G, neg, r_grad))
    dropped = torch.ones(rows_total, dtype=torch.bool, device='cuda')
    dropped[inds] = False
    if dropped.any() and ls['grad'][dropped][:, :, :5].abs().max().item() != 0:
        fails.append(('box / objectness gradient of a dropped row', G, neg))
    got = ls['losses'].tolist()
    r_loss = 0.0
    # double accumulation of fp32 terms in any order: 1e-12 of the part on top of the fp32 bound
    for k, (want, b) in enumerate(zip(parts + [loss_cls], pbar + [lbar_cls])):
        d = abs(got[k] - want)
        r_loss = max(r_loss, 0.0 if d == 0 else d / (b + 1e-12 * abs(want)))
    if not r_loss <= 1.0:
        fails.append(('region loss parts', G, neg, got[:6], parts + [loss_cls]))
    row = '  region G=%d neg=%-4s seed %-5s kept %4d/%d rows  nGT %d  grad %.3f  loss parts %.3f  dropped rows %d' % (
        G, neg, seed, nB, rows_total, bt['counters'][0], r_grad, r_loss, int(dropped.sum()))
    return fails, row


# ------------------------------------------------------------------------------------------------- part 1 + part 2
@pytest.mark.parametrize('side,bs,cs', CASES)
def test_step_at_side(side, bs, cs):
    """One full-batch eager step at `side` under both step checkers (every bar as in test_gpu_zz_step_gemms and
    test_gpu_zz_step_memops), the flavours reached equal to the planner's, then the region loss of its head output."""
    from fewshot_detection_b200 import _lib
    made = {}

    def chain(real):
        made['gemm'] = StepChecker(real, _lib.lib)
        made['mem'] = MemChecker(made['gemm'], _lib.lib)
        return made['mem']
    print('\n==== side %d, B = %d, %d classes' % (side, bs, cs))
    out, L, tgt, secs = run_step(side, bs, cs, 1000 + side + cs, chain)
    gchk, mchk = made['gemm'], made['mem']
    errors = []
    for rep, chk in ((report_gemms, gchk), (report_mem, mchk)):
        try:
            rep(chk, secs)
        except AssertionError as e:
            errors.append(e)
    planned = planned_flavours(_lib.lib, query_gemms(side, bs, cs) + support_gemms(cs))
    reached = gchk.cov & set(FLAVOURS)
    wn, rem = first_layer_tail(side)
    query_first = [f for f in gchk.first_fwd if f == (bs, side, side)]
    print('side %d: flavours reached %s; first-layer forward: last column tile %d of 104 columns, wn %% 3 = %d' % (
        side, sorted(reached), wn, rem))
    rows = []
    for neg, seed in (('full', None), (1, 7000 + side)):
        f, row = check_region(out, L, tgt, neg, seed)
        errors += f
        rows.append(row)
    print('\n'.join(rows))
    sys.stdout.flush()
    assert not errors, errors
    assert reached == planned, ('flavours reached', sorted(reached), 'planned', sorted(planned))
    assert GEMM_COVERAGE <= gchk.cov, sorted(GEMM_COVERAGE - gchk.cov)
    assert MEM_COVERAGE <= mchk.cov, sorted(MEM_COVERAGE - mchk.cov)
    assert len(query_first) == 1 and (wn < 104) == (side != 416), (gchk.first_fwd, wn)


# ----------------------------------------------------------------------------------------------------------- part 3
# starts at 608 (an eager step), captures one graph at each of the ten sides, then replays 320, 480, 352 and 416 after
# the other sides' graphs were captured into the shared pool
GRAPH_SIDES = (608, 416, 320, 352, 384, 448, 480, 512, 544, 576, 608, 320, 480, 352, 416)


def _digest(tensors):
    """one int64 per tensor: the sum of its float32 bit patterns weighted by position, on the device"""
    out = []
    for t in tensors:
        b = t.detach().reshape(-1).view(torch.int32).long()
        out.append((b * torch.arange(1, b.numel() + 1, device=b.device)).sum())
    return torch.stack(out).cpu()


def _trajectory(graph, bs=8, cs=15):
    from fewshot_detection_b200 import netcfg
    from fewshot_detection_b200.darknet_meta import Darknet
    from fewshot_detection_b200.distributed import GradAllReducer
    from fewshot_detection_b200.graph import GraphedTrainStep
    from fewshot_detection_b200.optim import FusedSGD
    from fewshot_detection_b200.trainer import lr_factor, sgd_hyper_parameters
    from seeding import seeded_init
    from test_gpu_zz_configs import _batch
    m = Darknet(netcfg.darknet_dynamic_blocks(416, 416), netcfg.reweighting_net_blocks())
    seeded_init(m, 91)
    m = m.cuda().train()
    params = list(m.parameters())
    names = [n for n, _ in m.named_parameters()]
    # the training driver's SGD settings for base training (cfg rate 1e-3, neg = 1): larger rates diverge at this batch
    opt = FusedSGD(params, **sgd_hyper_parameters(1e-3, 0.9, 5e-4, bs, lr_factor(1, cs)))
    L = m.models[len(m.models) - 1]
    L.verbose = False
    L.seen = 20000
    red = GradAllReducer(m)
    gs = GraphedTrainStep(m, L, opt, red) if graph else None
    random.seed(4242)
    losses, digests = [], []
    for it, side in enumerate(GRAPH_SIDES):
        x, metax, mask, tgt = _batch(bs, cs, side, 500 + it)
        x, metax, mask = x.cuda(), metax.cuda(), mask.cuda()
        L.seen += bs
        if graph:
            loss = gs(x, metax, mask, tgt)
        else:
            red.begin_step()
            loss = L(m(x, metax, mask), tgt)
            loss.backward()
            red.finish()
            opt.step()
        losses.append(loss.item())
        digests.append(_digest(params + [opt.state[p]['momentum_buffer'] for p in params]))
    captures = 0
    if graph:
        gs.poll()
        captures = gs.captures
    final = [t.detach().cpu().clone() for t in params + [opt.state[p]['momentum_buffer'] for p in params]]
    names = names + ['momentum of ' + n for n in names]
    draw = random.random()
    del m, opt, gs, red, params, L
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return losses, digests, final, names, captures, draw


def test_graph_steps_match_eager_steps():
    """Full network, B = 8, 15 classes, neg = 1: the graphed trajectory over all ten sides equals the eager one bit for
    bit after every step (every kernel of the step is deterministic and a replay issues the same launches; only the
    loss, a sum of double atomics in another row order, may differ in its last bits)."""
    from fewshot_detection_b200.cfg import cfg
    old = cfg.neg_ratio
    cfg.neg_ratio = 1
    try:
        eager = _trajectory(False)
        graph = _trajectory(True)
    finally:
        cfg.neg_ratio = old
    (l0, d0, f0, names, _, r0), (l1, d1, f1, _, captures, r1) = eager, graph
    assert r0 == r1                                  # the same number of neg_filter draws
    assert captures == 10, captures
    assert all(math.isfinite(l) for l in l0 + l1), (l0, l1)
    assert all(torch.isfinite(t).all() for t in f0), 'the eager trajectory diverged'
    for it, (side, a, b) in enumerate(zip(GRAPH_SIDES, d0, d1)):
        diff = (a != b).nonzero().flatten().tolist()
        assert not diff, ('step %d (side %d): first tensors that differ' % (it, side), [names[i] for i in diff[:5]])
    for n, a, b in zip(names, f0, f1):
        assert torch.equal(a, b), n
    for it, (a, b) in enumerate(zip(l0, l1)):
        assert abs(a - b) <= 1e-6 * abs(a), (it, GRAPH_SIDES[it], a, b)
    print('\n%d steps over sides %s: parameters and momentum bit-equal after every step; worst loss difference %.1e' % (
        len(GRAPH_SIDES), GRAPH_SIDES, max(abs(a - b) / abs(a) for a, b in zip(l0, l1))))


def test_trainer_losses_are_per_step_values():
    """MetaTrainer.losses holds one value per step on the graph path too: a replay returns the graph's static loss buffer,
    which the next replay of that graph overwrites (and, allocated in the graphs' shared pool, another graph's scratch may
    overwrite), so the trainer must keep a copy.  The query side changes every batch; the graph run's losses equal the
    eager run's step by step."""
    from fewshot_detection_b200 import netcfg, trainer as T
    from fewshot_detection_b200.darknet_meta import Darknet
    from fewshot_detection_b200.optim import FusedSGD
    from seeding import seeded_init, synth_targets, synth_masks
    bs, cs = 6, 5
    sides = (128, 96, 160, 128, 192, 96, 160, 128, 192, 96)

    def batch(it):
        g = torch.Generator().manual_seed(100 + it)
        x = torch.rand(bs, 3, sides[it], sides[it], generator=g).cuda()
        metax = torch.rand(cs, 3, 64, 64, generator=g).cuda()
        return x, metax, torch.from_numpy(synth_masks(cs, 64, 200 + it)).cuda(), torch.from_numpy(synth_targets(bs, cs, 300 + it, max_gt=2))

    class Queries(object):
        def __len__(self):
            return len(sides)

        def __iter__(self):
            for i in range(len(sides)):
                x, _, _, tgt = batch(i)
                yield x, tgt

    class Supports(object):
        batch_size = cs

        def batch(self, r):
            return batch(r.start // cs)[1:3]

    def run(use_graph):
        m = Darknet(netcfg.mini_dynamic_blocks(128, 8), netcfg.mini_reweighting_blocks(64, 8, 256))
        seeded_init(m, 11)
        m = m.cuda().train()
        opt = FusedSGD(m.parameters(), lr=1e-3, momentum=0.9, dampening=0, weight_decay=5e-4)
        tr = T.MetaTrainer(m, opt, 1e-3, bs, [0], [1], lambda seen: Queries(), Supports, save_interval=10 ** 6,
                           log=lambda s: None, use_graph=use_graph)
        assert (tr.graphed is not None) == use_graph
        m.models[len(m.models) - 1].verbose = False
        tr.region_loss.seen = 20000
        random.seed(5)
        tr.train_epoch(0)
        if use_graph:
            tr.graphed.poll()
            assert tr.graphed.captures == 4
        return [l.item() for l in tr.losses]
    eager, graph = run(False), run(True)
    assert len(eager) == len(graph) == len(sides)
    for it, (a, b) in enumerate(zip(eager, graph)):
        assert abs(a - b) <= 1e-6 * abs(a), (it, sides[it], eager, graph)
