"""The evaluation pass at full size: every eval-mode kernel against float64 at the batch sizes evaluation runs, and the
detections against a float64 model.

Every AP the project reports comes from an eval-mode forward of the full network, which is not the training forward
without gradients: BatchNorm takes the running statistics (fsdet_bn_finalize with training = 0), the convolutions
write no statistics rows, every block writes fp32 output that the next convolution re-splits into fp16 planes under a
fresh per-tensor amax, and the batch sizes are those of evaluation (64 and the tails 24, 8, 32 and 1), where the planner
picks other kernels and every im2col layer ends on another partial tile (tests/test_tile_plans_eval.py).

Model: the full detector and reweighting net at 416 (seeded_init), with BatchNorm running statistics that fit real
activations: every momentum set to 1, one train-mode forward under no_grad on a calibration batch of its own seed (the
running statistics become that batch's statistics), momenta restored, eval().  A second model keeps seeded_init's raw
buffers (mean 0.1 N(0, 1), var U(0.5, 1.5)), which do not fit, so its activations drift off unit scale through the
layers: the per-tensor amax scaling then works on unnormalised data.

  test_eval_pass   valid.ensemble_dynamic_weights and valid.detect, the production entry points, with engine.call
                   replaced by both step checkers chained (test_gpu_zz_step_gemms.StepChecker inside
                   test_gpu_zz_step_memops.MemChecker), every bar unchanged: coverage of the eval kernels, no batch
                   statistics anywhere, the flavour of every GEMM equal to the planner's, parameters and BatchNorm buffers
                   bit-unchanged, a second pass bit-identical.  For voc64 and coco8 also the end-to-end comparison with
                   oracle.darknet.MetaDarknet in float64 on the GPU: ensembled dynamic weights and head output within
                   max(1e-5, 8 e32) (at most 2e-4), e32 being the same oracle's float32 distance from float64 (TF32 off),
                   and the decoded, NMS-ed detections of both outputs
  test_end_to_end_bar_reports_one_moved_head_element   the end-to-end bar has teeth
"""
import sys
import time

import numpy as np
import pytest
import torch

from test_gpu_detect import _match
from test_gpu_zz_step_gemms import StepChecker, report as report_gemms
from test_gpu_zz_step_memops import MemChecker, dev, report as report_mem
from test_tile_plans_eval import flavour, query_eval_gemms, support_eval_gemms
from test_tile_plans_scales import FLAVOURS, planned_flavours

pytestmark = pytest.mark.gpu

SIDE = 416
CONF_THRESH, NMS_THRESH = 0.005, 0.45
# end-to-end bar: max(E2E_FLOOR, E2E_FACTOR e32), at most E2E_CAP, e32 the float32 oracle's distance from float64.  The
# forward amplifies per-layer rounding several hundredfold: the float32 oracle is 2.6e-5 (torch's own convolutions) to
# 3.4e-5 (cuDNN) from float64 at the head output.  The tensor-core GEMMs are fp32-grade, not fp32-exact (three fp16
# products, tensor-core accumulation: up to 2.8e-6 relative L2 per GEMM in their own check), so the pass sits 3 to 7 e32
# from float64 - 1.1e-4 at the head output at every batch size and class count, with every kernel inside its own bar.
# Hence 8 e32, and a cap of 2e-4: 1e-4 does not hold.
E2E_FLOOR, E2E_FACTOR, E2E_CAP = 1e-5, 8, 2e-4
QUERY_CHUNK = 16                     # images per float64 oracle forward

# support batch sizes, query batch size, classes, model
CASES = [pytest.param((64, 8), 64, 20, 'calibrated', id='voc64'),
         pytest.param((64,), 24, 20, 'calibrated', id='voc24'),
         pytest.param((64,), 1, 20, 'calibrated', id='voc1'),
         pytest.param((64, 32), 8, 80, 'calibrated', id='coco8'),
         pytest.param((64,), 24, 20, 'raw', id='raw-stats')]
END_TO_END = ('voc64', 'coco8')

# what every evaluation pass must reach
MEM_COVERAGE = {'finalize-eval', 'fwd-f32', 'fwd-pool', 'amax', 'split-f16', 'globalmax', 'head-weff'}
GEMM_COVERAGE = {'first-fwd', 'fwd', 'head'}


# ----------------------------------------------------------------------------------------------------------- models
def make_model(seed, calibrate):
    """The full model at 416 in eval mode; `calibrate`: running statistics of one train-mode forward (momentum 1)."""
    from fewshot_detection_b200 import netcfg
    from fewshot_detection_b200.darknet_meta import Darknet
    from seeding import seeded_init, synth_masks
    m = Darknet(netcfg.darknet_dynamic_blocks(SIDE, SIDE), netcfg.reweighting_net_blocks())
    seeded_init(m, seed)
    m = m.cuda()
    if calibrate:
        bns = [b for b in m.modules() if isinstance(b, torch.nn.BatchNorm2d)]
        moms = [b.momentum for b in bns]
        for b in bns:
            b.momentum = 1.0
        g = torch.Generator().manual_seed(seed + 1)
        x = torch.rand(16, 3, SIDE, SIDE, generator=g)
        metax = torch.rand(20, 3, SIDE, SIDE, generator=g)
        mask = torch.from_numpy(synth_masks(20, SIDE, seed + 2))
        m.train()
        with torch.no_grad():
            m(x.cuda(), metax.cuda(), mask.cuda())
        torch.cuda.synchronize()
        for b, mo in zip(bns, moms):
            b.momentum = mo
    return m.eval()


@pytest.fixture(scope='module')
def models():
    return {'calibrated': make_model(501, True), 'raw': make_model(502, False)}


def support_batches(sizes, n_cls, seed):
    """(metax, mask, class ids) per support batch; the class ids run through the classes in turn"""
    from seeding import synth_masks
    g = torch.Generator().manual_seed(seed)
    out, k = [], 0
    for i, n in enumerate(sizes):
        out.append((torch.rand(n, 3, SIDE, SIDE, generator=g), torch.from_numpy(synth_masks(n, SIDE, seed + 1 + i)),
                    [(k + j) % n_cls for j in range(n)]))
        k += n
    return out


def query_batch(B, seed):
    return torch.rand(B, 3, SIDE, SIDE, generator=torch.Generator().manual_seed(seed))


def snapshot(m):
    return dict((k, v.detach().clone()) for k, v in m.state_dict().items())


# ------------------------------------------------------------------------------------------------------ pass runner
class AmaxLog(object):
    """Outermost wrapper of engine.call: the value of every fsdet_amax (the scale an fp32 tensor is re-split under)."""

    def __init__(self, inner):
        self.inner = inner
        self.amax = []

    def __call__(self, fn, *a):
        rc = self.inner(fn, *a)
        if fn == 'fsdet_amax':
            src, ld, C, n, out, st = a
            torch.cuda.synchronize()
            self.amax.append((n, C, dev(out, 1).item()))
        return rc


def eval_pass(m, support, query, n_cls, wrap=None):
    """The evaluation twin of test_gpu_zz_step_gemms.run_step: valid.ensemble_dynamic_weights over the support
    batches, then valid.detect on each query batch, while engine.call is replaced by wrap(engine.call) (when given).
    Returns the ensembled dynamic weights [n_cls, C], the head output of each query batch, the detections of each and
    the seconds the pass took."""
    from fewshot_detection_b200 import engine, valid
    outs = []
    real_detect_forward = m.detect_forward

    def detect_forward(x, dw):            # keeps the head output valid.detect decodes
        out = real_detect_forward(x, dw)
        outs.append(out)
        return out
    m.detect_forward = detect_forward
    real = engine.call
    if wrap is not None:
        engine.call = wrap(real)
    torch.cuda.synchronize()
    t0 = time.time()
    try:
        dw = valid.ensemble_dynamic_weights(m, support, n_cls)[0]
        dets = [valid.detect(m, x.cuda(), dw, n_cls) for x in query]
        torch.cuda.synchronize()
    finally:
        engine.call = real
        del m.detect_forward
    return dw.view(n_cls, -1), outs, dets, time.time() - t0


def predicted_gemms(support, query, n_cls):
    """(shape, flavour) of every tensor-core GEMM of the pass, in launch order, as StepChecker logs them"""
    from fewshot_detection_b200 import _lib
    gemms = [g for metax, _, _ in support for g in support_eval_gemms(metax.shape[0])]
    gemms += [g for x in query for g in query_eval_gemms(x.shape[0], n_cls)]
    return [('%dx%dx%dx%d->%d k%d m%d' % g[1:], flavour(_lib.lib, g)) for g in gemms], gemms


# ------------------------------------------------------------------------------------------------------- end to end
def rel_errors(got, ref):
    """(relative L2, max element-wise error relative to max |ref|) against float64"""
    d = got.double() - ref
    return (d.norm() / ref.norm()).item(), (d.abs().max() / ref.abs().max()).item()


def bars(e32):
    return tuple(min(E2E_CAP, max(E2E_FLOOR, E2E_FACTOR * e)) for e in e32)


def oracle_pass(m, support, query, n_cls, dtype):
    """oracle.darknet.MetaDarknet with m's parameters and BatchNorm buffers, in eval mode and `dtype` on the GPU:
    the ensembled dynamic weights (oracle.utils.ensemble_reweights) and the head output of the query batch."""
    from oracle import darknet as ODK, utils as OU
    om = ODK.MetaDarknet([dict(b) for b in m.blocks], [dict(b) for b in m.learnet_blocks])
    om.load_state_dict(m.state_dict())
    om = om.to(device='cuda', dtype=dtype).eval()
    with torch.no_grad():
        vecs = [(om.meta_forward(metax.cuda().to(dtype), mask.cuda().to(dtype))[0].reshape(len(ids), -1), ids)
                for metax, mask, ids in support]
        dw = OU.ensemble_reweights(vecs, n_cls, dtype)
        x = query[0]
        out = torch.cat([om.detect_forward(x[b:b + QUERY_CHUNK].cuda().to(dtype), [dw.view(n_cls, -1, 1, 1)])
                         for b in range(0, x.shape[0], QUERY_CHUNK)])
    del om
    torch.cuda.empty_cache()
    return dw, out


def confidences64(o64, n_cls):
    """float64 det_conf * cls_conf of every anchor-cell, [rows, A*H*W] in the decode's a*HW + cell order (the class
    score of a row is the softmax across the n_cls rows of its image)"""
    N, ch, H, W = o64.shape
    o = o64.view(N // n_cls, n_cls, 5, ch // 5, H * W)
    conf = torch.sigmoid(o[:, :, :, 4]) * torch.softmax(o[:, :, :, 5], dim=1)
    return conf.reshape(N, 5 * H * W)


def candidate_slots(d):
    """per row the set of anchor-cells (a*HW + cell) above the confidence threshold"""
    count, cand = d.count.cpu().numpy(), d.cand.cpu().numpy()
    return [set(cand[n, :count[n], 7].view(np.int32).tolist()) for n in range(d.N)]


def end_to_end(m, support, query, n_cls, dw, out, dets, move_element=False):
    """The pass's dynamic weights, head output and detections against the float64 oracle.  Returns (failures, lines).
    move_element: one head-output element is moved by four times its element-wise bar first."""
    from fewshot_detection_b200 import utils as U
    t0 = time.time()
    dw64, o64 = oracle_pass(m, support, query, n_cls, torch.float64)
    t64 = time.time() - t0
    dw32, o32 = oracle_pass(m, support, query, n_cls, torch.float32)
    fails, lines = [], []
    if move_element:
        out = out.clone()
        i = o64.abs().flatten().argmax().item() // 2
        out.view(-1)[i] = (o64.view(-1)[i] + 4 * bars(rel_errors(o32, o64))[1] * o64.abs().max()).float()
    worst = 0.0
    for what, got, ref, f32 in (('dynamic weights', dw, dw64, dw32), ('head output', out, o64, o32)):
        e32, e = rel_errors(f32, ref), rel_errors(got, ref)
        bar = bars(e32)
        ratio = max(e[0] / bar[0], e[1] / bar[1])
        worst = max(worst, ratio)
        lines.append('  %-15s rel L2 %.2e (fp32 oracle %.2e, bar %.2e)  max element %.2e (fp32 oracle %.2e, bar %.2e)'
                     '  ratio %.3f' % (what, e[0], e32[0], bar[0], e[1], e32[1], bar[1], ratio))
        if not ratio <= 1.0:
            fails.append(('end to end', what, e, e32, bar))
    # detections: the same decode + NMS kernels on the pass's output and on the float64 output rounded to float32
    d64 = U.region_detections(o64.float().contiguous(), CONF_THRESH, m.num_classes, m.anchors, m.num_anchors, 0, 1,
                              n_models=n_cls).nms(NMS_THRESH)
    d = dets[0]
    delta = (out.double() - o64).abs().max().item()      # |d conf| <= 0.75 max |d logit| (sigmoid and softmax slopes)
    conf = confidences64(o64, n_cls).cpu().numpy()
    flipped = far = 0
    for n, (a, b) in enumerate(zip(candidate_slots(d), candidate_slots(d64))):
        for s in a ^ b:
            flipped += 1
            if abs(conf[n, s] - CONF_THRESH) > delta:
                far += 1
    if far:
        fails.append(('candidates differ away from the threshold', far, delta))
    # box entries move by at most max |d logit| relative to max(1, |entry|) to first order (x, y: sigmoid slope / W;
    # w, h: exp; det_conf, cls_conf: sigmoid and softmax slopes), so that is _match's tolerance
    tol = max(1e-5, 2 * delta)
    kept, kept64 = d.kept_boxes(NMS_THRESH), d64.kept_boxes(NMS_THRESH)
    rows_bad = miss = extra = 0
    for got, want in zip(kept, kept64):
        slack = max(1, len(want) // 100)
        a, b = _match(got, want, tol), _match(want, got, tol)
        miss, extra = miss + a, extra + b
        if abs(len(got) - len(want)) > slack or a > slack or b > slack:
            rows_bad += 1
    if rows_bad:
        fails.append(('kept boxes differ beyond the 1 % slack', rows_bad))
    lines.append('  detections: %d rows, %d candidates (float64: %d), %d differ (all within %.1e of the threshold: %s); '
                 '%d / %d kept boxes; unmatched at %.1e: %d / %d; rows beyond the slack %d' % (
                     d.N, int(d.count.sum()), int(d64.count.sum()), flipped, delta, far == 0, sum(map(len, kept)),
                     sum(map(len, kept64)), tol, miss, extra, rows_bad))
    lines.append('  float64 and float32 oracles %.1f s + %.1f s' % (t64, time.time() - t0 - t64))
    return fails, lines, worst


# ------------------------------------------------------------------------------------------------------------ tests
@pytest.mark.parametrize('sup,B,n_cls,which', CASES)
def test_eval_pass(request, models, sup, B, n_cls, which):
    """One evaluation pass under both step checkers, then the same pass again unchecked, then (voc64, coco8) the
    float64 model."""
    from fewshot_detection_b200 import _lib
    case = request.node.callspec.id
    m = models[which]
    support = support_batches(sup, n_cls, 300 + n_cls)
    query = [query_batch(B, 400 + B)]
    before = snapshot(m)
    made = {}

    def chain(real):
        made['gemm'] = StepChecker(real, _lib.lib)
        made['mem'] = MemChecker(made['gemm'], _lib.lib)
        made['amax'] = AmaxLog(made['mem'])
        return made['amax']
    print('\n==== %s: support batches %s, query B = %d, %d classes, %s running statistics' % (case, sup, B, n_cls, which))
    dw, outs, dets, secs = eval_pass(m, support, query, n_cls, chain)
    gchk, mchk, alog = made['gemm'], made['mem'], made['amax']
    errors = []
    for rep, chk in ((report_gemms, gchk), (report_mem, mchk)):
        try:
            rep(chk, secs)
        except AssertionError as e:
            errors.append(e)
    # eval must run no batch statistics: no train-mode finalize, no statistics rows from any convolution, no fp16
    # planes written by the BatchNorm pass (they need the batch-range amax_y)
    if 'finalize-train' in mchk.cov or mchk.stat_src or 'fwd-planes' in mchk.cov:
        errors.append(('batch statistics in eval', sorted(mchk.cov), len(mchk.stat_src)))
    want, gemms = predicted_gemms(support, query, n_cls)
    got = [(l['shape'], l['flavour']) for l in gchk.log if l['kind'] in ('fwd', 'head')]
    reached = gchk.cov & set(FLAVOURS)
    print('flavours reached %s; tensor-core GEMMs %d (predicted %d)' % (sorted(reached), len(got), len(want)))
    print('per-tensor amax of every fp32 tensor re-split into planes (rows x channels: amax), in launch order:\n  %s' % (
        '  '.join('%dx%d: %.3g' % t for t in alog.amax)))
    # the same pass again, unchecked: bit-identical dynamic weights, head output and detections
    dw2, outs2, dets2, secs2 = eval_pass(m, support, query, n_cls)
    after = snapshot(m)
    changed = [k for k in before if not torch.equal(before[k], after[k])]
    t_e2e = time.time()
    same = (torch.equal(dw, dw2) and torch.equal(outs[0], outs2[0]) and torch.equal(dets[0].count, dets2[0].count)
            and torch.equal(dets[0].keep_count, dets2[0].keep_count))
    print('checked pass %.1f s, unchecked pass %.2f s; second pass bit-identical: %s' % (secs, secs2, same))
    e2e = []
    if case in END_TO_END:
        fails, lines, worst = end_to_end(m, support, query, n_cls, dw, outs[0], dets)
        e2e = fails
        print('end to end against float64 (%.1f s in all), worst ratio to the bar %.3f:' % (time.time() - t_e2e, worst))
        print('\n'.join(lines))
    sys.stdout.flush()
    assert not errors, errors
    assert MEM_COVERAGE <= mchk.cov, sorted(MEM_COVERAGE - mchk.cov)
    assert GEMM_COVERAGE <= gchk.cov, sorted(GEMM_COVERAGE - gchk.cov)
    assert got == want, ('GEMMs and flavours reached differ from the planner', [(a, b) for a, b in zip(got, want)
                                                                                if a != b][:5], len(got), len(want))
    assert reached == planned_flavours(_lib.lib, gemms), (sorted(reached), sorted(planned_flavours(_lib.lib, gemms)))
    assert not changed, ('eval changed parameters or BatchNorm buffers', changed[:5])
    assert same, 'a second evaluation pass gave other bits'
    assert not e2e, e2e


def test_end_to_end_bar_reports_one_moved_head_element(models):
    """The end-to-end element-wise bar has teeth: on a real pass (B = 2, 20 support images, 20 classes), the comparison
    holds, and one head-output element moved by four times its element-wise bar is reported."""
    m = models['calibrated']
    support, query = support_batches((20,), 20, 77), [query_batch(2, 78)]
    dw, outs, dets, _ = eval_pass(m, support, query, 20)
    fails, lines, worst = end_to_end(m, support, query, 20, dw, outs[0], dets)
    print('\n' + '\n'.join(lines))
    assert not fails, fails
    fails, lines, worst = end_to_end(m, support, query, 20, dw, outs[0], dets, move_element=True)
    print('\n'.join(lines))
    assert worst > 3.0, worst
    assert any(f[:2] == ('end to end', 'head output') for f in fails), fails
    assert all(f[1] != 'dynamic weights' for f in fails if f[0] == 'end to end'), fails
