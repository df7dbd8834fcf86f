#!/usr/bin/env python
"""Time of an evaluation batch under a test-time augmentation plan (valid.detect_tta), broken into its stages, for
B = 64 images and 20 classes at conf 0.005 / NMS 0.45 (the evaluation's thresholds):

    plans   one pass [(416, 0)], 416 + flip, and the six passes of 416 / 544 / 608 with flips
    stages  forward (detect_forward of every pass), decode + merge (fsdet_region_detect + fsdet_tta_merge of every
            pass), NMS (fsdet_nms_merged) and gather (fsdet_voc_gather_merged into a VOC pool)

and the wide NMS alone on a merged table of about 8k candidates per row.

    python tools/tta_bench.py [--iters 10] [--warmup 2] [--json PATH]

CUDA events around each stage, averaged over `iters` batches after `warmup`; the stages of a batch run back to back
on one stream, so their sum is the batch time.  The model is the detection bench's (seeded, calibrated BatchNorm
statistics); inputs are random images.  The GPU name, power limit and SM clocks are printed with the numbers, because
the numbers depend on them.  The gain in AP of a plan is a property of a trained model and a dataset; it is not
measured here.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests', 'golden'))
sys.path.insert(0, os.path.join(ROOT, 'tools'))
sys.path.insert(0, os.path.join(ROOT, 'tests'))

B, N_CLS, CONF, NMS = 64, 20, 0.005, 0.45
PLANS = [('one pass', [416], False), ('416 + flip', [416], True), ('six passes', [416, 544, 608], True)]


def run_plan(m, dw, inputs, passes, ev, names, sizes):
    """One batch through the plan, a CUDA event at each stage boundary: {stage: ms}, survivors per row (tensor)."""
    import torch
    from fewshot_detection_b200 import valid as VA
    from fewshot_detection_b200.utils import MergedDetections, region_detections
    ev_ = [torch.cuda.Event(enable_timing=True) for _ in range(2 * len(passes) + 3)]
    merged = MergedDetections(B * N_CLS, VA.tta_capacity(m, passes), inputs[0].device)
    k = 0
    ev_[k].record()
    fwd = dec = 0.0
    marks = []
    for (side, flip), x in zip(passes, inputs):
        with torch.no_grad():
            out = m.detect_forward(x, dw)
        k += 1
        ev_[k].record()
        d = region_detections(out, CONF, m.num_classes, m.anchors, m.num_anchors, 0, 1, n_models=N_CLS)
        merged.add_pass(d, side, flip)
        k += 1
        ev_[k].record()
        marks.append((k - 2, k - 1, k))
    merged.nms(NMS)
    ev_[k + 1].record()
    ev.add(merged, names, sizes)
    ev_[k + 2].record()
    torch.cuda.synchronize()
    for a, b, c in marks:
        fwd += ev_[a].elapsed_time(ev_[b])
        dec += ev_[b].elapsed_time(ev_[c])
    return {'forward': fwd, 'decode+merge': dec, 'nms': ev_[k].elapsed_time(ev_[k + 1]),
            'gather': ev_[k + 1].elapsed_time(ev_[k + 2])}, merged


def wide_nms_alone(iters, warmup):
    """fsdet_nms_merged on B*20 rows of about 8k candidates (six passes' worth), boxes in a few clusters per row."""
    import numpy as np
    import torch
    from fewshot_detection_b200.utils import MergedDetections, tta_record_dtype
    rs = np.random.RandomState(0)
    N, cap, n = B * N_CLS, 8190, 8000
    rec = np.zeros((N, cap), dtype=tta_record_dtype())
    centre = rs.uniform(0.1, 0.9, (N, 40, 2))
    pick = rs.randint(0, 40, (N, n))
    xy = np.take_along_axis(centre, pick[..., None].repeat(2, -1), 1) + rs.normal(0, 0.02, (N, n, 2))
    rec['x'][:, :n], rec['y'][:, :n] = xy[..., 0], xy[..., 1]
    rec['w'][:, :n], rec['h'][:, :n] = rs.uniform(0.05, 0.3, (N, n)), rs.uniform(0.05, 0.3, (N, n))
    rec['det'][:, :n] = rs.uniform(0.005, 1, (N, n))
    rec['cls'][:, :n] = 1.0
    md = MergedDetections(N, cap, torch.device('cuda', 0))
    md.merged.copy_(torch.from_numpy(rec.view(np.uint8).reshape(N, cap, -1)))
    md.count.fill_(n)
    times = []
    for i in range(warmup + iters):
        md._nms_thresh = None
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        md.nms(NMS)
        b.record()
        torch.cuda.synchronize()
        if i >= warmup:
            times.append(a.elapsed_time(b))
    kc = md.keep_count.float()
    return {'rows': N, 'candidates_per_row': n, 'ms': sum(times) / len(times),
            'survivors_per_row_mean': float(kc.mean()), 'survivors_per_row_max': int(kc.max())}


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--json', default=None)
    args = ap.parse_args(argv)
    import torch
    from detect_bench import gpu_info, make_model
    from test_gpu_eval_shard import make_set, voc_recs
    from fewshot_detection_b200 import valid as VA, voc_eval as V
    torch.cuda.set_device(0)
    info = gpu_info()
    m = make_model(3)
    from test_gpu_zz_eval_pass import support_batches
    dw = VA.ensemble_dynamic_weights(m, support_batches((64,), N_CLS, 4), N_CLS)
    gt, sizes, _, names, classes, _ = make_set(1, B, N_CLS)
    recs = voc_recs(gt, names, classes)
    g = torch.Generator().manual_seed(5)
    base = dict((s, torch.rand(B, 3, s, s, generator=g).cuda()) for s in (416, 544, 608))
    results = {'gpu': info, 'B': B, 'n_cls': N_CLS, 'conf': CONF, 'nms': NMS, 'plans': []}
    for title, sides, flip in PLANS:
        passes = VA.tta_plan(sides, flip)
        inputs = [torch.flip(base[s], dims=[3]) if f else base[s] for s, f in passes]
        acc = None
        for i in range(args.warmup + args.iters):
            ev = V.DeviceVocEval(classes, names, recs)
            t, merged = run_plan(m, dw, inputs, passes, ev, names, sizes)
            if i >= args.warmup:
                acc = t if acc is None else dict((k, acc[k] + t[k]) for k in acc)
        t = dict((k, v / args.iters) for k, v in acc.items())
        counts, kc = merged.count.float(), merged.keep_count.float()
        row = {'plan': title, 'passes': passes, 'ms': t, 'total_ms': sum(t.values()),
               'candidates_per_row_mean': float(counts.mean()), 'candidates_per_row_max': int(counts.max()),
               'survivors_per_row_mean': float(kc.mean())}
        results['plans'].append(row)
    results['wide_nms'] = wide_nms_alone(args.iters, args.warmup)
    print('GPU %s, power limit %s, SM clock %s (max %s)' % (info['name'], info['power_limit'], info['sm_clock'],
                                                             info['sm_clock_max']))
    print('B = %d images x %d classes, conf %g, NMS %g; ms per batch (mean of %d after %d warm-up)'
          % (B, N_CLS, CONF, NMS, args.iters, args.warmup))
    print('%-12s %9s %13s %8s %8s %9s %12s %10s' % ('plan', 'forward', 'decode+merge', 'nms', 'gather', 'total',
                                                     'cand/row max', 'kept/row'))
    for r in results['plans']:
        t = r['ms']
        print('%-12s %9.2f %13.2f %8.2f %8.2f %9.2f %12d %10.1f' % (r['plan'], t['forward'], t['decode+merge'], t['nms'],
                                                                    t['gather'], r['total_ms'],
                                                                    r['candidates_per_row_max'],
                                                                    r['survivors_per_row_mean']))
    w = results['wide_nms']
    print('wide NMS alone: %d rows x %d candidates: %.2f ms (survivors per row: mean %.1f, max %d)'
          % (w['rows'], w['candidates_per_row'], w['ms'], w['survivors_per_row_mean'], w['survivors_per_row_max']))
    info2 = gpu_info()
    print('after: SM clock %s, power limit %s' % (info2['sm_clock'], info2['power_limit']))
    if args.json:
        with open(args.json, 'w') as f:
            json.dump(results, f, indent=1)
    return 0


if __name__ == '__main__':
    sys.exit(main())
