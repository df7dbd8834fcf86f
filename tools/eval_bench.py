#!/usr/bin/env python
"""Time the two ways of scoring one evaluation pass over a VOC2007-test-sized set (4,952 images, 20 classes):

  files   valid.write_detections for every batch, then voc_eval.mean_ap on the written result files
  device  voc_eval.DeviceVocEval: .add for every batch, then .result (csrc/voc_eval.cu)

    python tools/eval_bench.py [--images 4952] [--kept 30] [--device-passes 5] [--out result.json]

The annotations are a synthetic devkit (tools/e2e_train_synth.make_devkit, seeded), parsed once before timing.  The
Detections come from the full-size meta detector's forward (416x416, seeded random weights) on random images: its
output keeps its class scores, and the objectness and box channels of each (image, class) row are rewritten so that
`--kept` distinct cells pass conf_thresh 0.005 with boxes of 0.6-1.4 cells, most of which survive NMS, and one more
anchor per annotated object of that class predicts a box within a few % of it.  Both paths
score the same Detections; neither time includes the forward.  Prints one JSON line: seconds per pass of each path,
the AP per class from both, detections scored, and the GPU's name and power limit read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))


def gpu_info():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(',')]
        return name, power
    except (OSError, IndexError, ValueError, subprocess.TimeoutExpired):
        import torch
        return torch.cuda.get_device_name(0), 'unknown'


def rewrite_head(out, n_cls, kept, A, anchors, rs):
    """Row r of the head output [rows, A*6, H, W]: `kept` distinct cells get objectness logit 3 on one anchor with
    box logits for 0.6-1.4 cells; every other anchor-cell gets -30 (confidence ~1e-13, below conf_thresh)."""
    import torch
    rows, _, H, W = out.shape
    o = out.view(rows, A, 6, H, W)
    o[:, :, 4] = -30.0
    cells = np.stack([rs.choice(H * W, kept, replace=False) for _ in range(rows)])
    a = rs.randint(0, A, (rows, kept))
    size = rs.uniform(0.6, 1.4, (rows, kept, 2))
    aw = np.array(anchors[0::2])[a]
    ah = np.array(anchors[1::2])[a]
    r_idx = np.repeat(np.arange(rows), kept)
    dev = out.device
    r_t, a_t = torch.from_numpy(r_idx).to(dev), torch.from_numpy(a.ravel()).to(dev)
    cy = torch.from_numpy(cells.ravel() // W).to(dev)
    cx = torch.from_numpy(cells.ravel() % W).to(dev)
    vals = lambda v: torch.from_numpy(np.asarray(v, dtype=np.float32).ravel()).to(dev)
    o[r_t, a_t, 4, cy, cx] = 3.0
    o[r_t, a_t, 0, cy, cx] = vals(rs.uniform(-2, 2, rows * kept))
    o[r_t, a_t, 1, cy, cx] = vals(rs.uniform(-2, 2, rows * kept))
    o[r_t, a_t, 2, cy, cx] = vals(np.log(size[..., 0] / aw))
    o[r_t, a_t, 3, cy, cx] = vals(np.log(size[..., 1] / ah))
    return out


def place_on_truth(out, batch_names, recs, sizes, classes, A, anchors, rs):
    """For every annotated object, one anchor of the row (image, its class) predicts a box within a few % of it, so
    the APs are not trivially zero."""
    import torch
    rows, _, H, W = out.shape
    n_cls = len(classes)
    cidx = dict((c, i) for i, c in enumerate(classes))
    r_, a_, cy_, cx_, v = [], [], [], [], []
    for b, n in enumerate(batch_names):
        iw, ih = sizes[n]
        for o in recs[n]:
            if o['name'] not in cidx:
                continue
            x1, y1, x2, y2 = o['bbox']
            cx, cy = (x1 + x2) / 2.0 / iw * W, (y1 + y2) / 2.0 / ih * H
            w, h = (x2 - x1) / float(iw) * W, (y2 - y1) / float(ih) * H
            cx, cy = cx * (1 + rs.normal(0, 0.02)), cy * (1 + rs.normal(0, 0.02))
            w, h = w * (1 + rs.normal(0, 0.04)), h * (1 + rs.normal(0, 0.04))
            gx, gy = min(int(cx), W - 1), min(int(cy), H - 1)
            fx, fy = np.clip(cx - gx, 0.02, 0.98), np.clip(cy - gy, 0.02, 0.98)
            a = rs.randint(0, A)
            r_.append(b * n_cls + cidx[o['name']])
            a_.append(a)
            cy_.append(gy)
            cx_.append(gx)
            v.append([np.log(fx / (1 - fx)), np.log(fy / (1 - fy)), np.log(max(w, 0.05) / anchors[2 * a]),
                      np.log(max(h, 0.05) / anchors[2 * a + 1]), 3.0])
    if not r_:
        return out
    o = out.view(rows, A, 6, H, W)
    dev = out.device
    idx = [torch.tensor(t, dtype=torch.long, device=dev) for t in (r_, a_, cy_, cx_)]
    v = torch.tensor(np.array(v), dtype=torch.float32, device=dev)
    for k in range(5):
        o[idx[0], idx[1], k, idx[2], idx[3]] = v[:, k]
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--images', type=int, default=4952)
    ap.add_argument('--kept', type=int, default=30, help='cells per (image, class) row above conf_thresh')
    ap.add_argument('--batch', type=int, default=64)
    ap.add_argument('--device-passes', type=int, default=5)
    ap.add_argument('--seed', type=int, default=0)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()

    import torch
    from e2e_train_synth import VOC, make_devkit
    from fewshot_detection_b200 import netcfg, valid as VA, voc_eval as VE
    from fewshot_detection_b200.darknet_meta import Darknet
    from fewshot_detection_b200.utils import region_detections
    if not torch.cuda.is_available():
        raise SystemExit('eval_bench.py measures the GPU path: no CUDA device')
    torch.cuda.set_device(0)
    name, power = gpu_info()
    work = tempfile.mkdtemp(prefix='fsdet_eval_bench_')
    names, sizes = make_devkit(os.path.join(work, 'VOCdevkit'), args.images, seed=args.seed)
    voc = os.path.join(work, 'VOCdevkit', 'VOC2007')
    annopath = os.path.join(voc, 'Annotations', '{}.xml')
    imagesetfile = os.path.join(voc, 'ImageSets', 'Main', 'test.txt')
    cachedir = os.path.join(work, 'VOCdevkit', 'annotations_cache')
    recs = VE.load_annotations(annopath, names, cachedir)        # parsed and cached once, outside both timings
    classes, n_cls = list(VOC), len(VOC)

    torch.manual_seed(args.seed)
    m = Darknet(netcfg.darknet_dynamic_blocks(), netcfg.reweighting_net_blocks()).cuda().eval()
    g = torch.Generator(device='cuda').manual_seed(args.seed)
    with torch.no_grad():
        metax = torch.rand(n_cls, 3, 416, 416, device='cuda', generator=g)
        mask = (torch.rand(n_cls, 1, 416, 416, device='cuda', generator=g) > 0.5).float()
        dw = m.meta_forward(metax, mask)
    rs = np.random.RandomState(args.seed + 1)
    batches = []
    for s in range(0, len(names), args.batch):
        ids = names[s:s + args.batch]
        with torch.no_grad():
            out = m.detect_forward(torch.rand(len(ids), 3, 416, 416, device='cuda', generator=g), dw)
        out = rewrite_head(out.detach().float().contiguous(), n_cls, args.kept, m.num_anchors, m.anchors, rs)
        out = place_on_truth(out, ids, recs, sizes, classes, m.num_anchors, m.anchors, rs)
        d = region_detections(out, VA.CONF_THRESH, m.num_classes, m.anchors, m.num_anchors, 0, 1, n_models=n_cls)
        batches.append((d.nms(VA.NMS_THRESH), ids, [sizes[n] for n in ids]))
    torch.cuda.synchronize()
    kept_total = int(sum(int(d.keep_count.sum()) for d, _, _ in batches))
    rows = len(names) * n_cls

    # file path: result files, then mean_ap over them
    res = os.path.join(work, 'results')
    os.makedirs(res)
    detpath = os.path.join(res, 'comp4_det_test_{}.txt')
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fps = [open(detpath.format(c), 'w') for c in classes]
    for d, ids, sz in batches:
        VA.write_detections(fps, d, ids, sz, n_cls)
    for f in fps:
        f.close()
    t1 = time.perf_counter()
    files = VE.mean_ap(detpath, annopath, imagesetfile, classes, cachedir, True)
    t_files = time.perf_counter() - t0
    t_write = t1 - t0

    # device path
    def device_pass():
        ev = VE.DeviceVocEval(classes, names, recs)
        for d, ids, sz in batches:
            ev.add(d, ids, sz)
        r = ev.result(True)
        torch.cuda.synchronize()
        return r
    device = device_pass()                                        # warm-up: module load, allocator
    times = []
    for _ in range(args.device_passes):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        device = device_pass()
        times.append(time.perf_counter() - t0)
    t_dev = float(np.median(times))

    tied = []
    for c in classes:
        with open(detpath.format(c)) as f:
            conf = [l.split(' ')[1] for l in f]
        if len(set(conf)) != len(conf):
            tied.append(c)
    diff = dict((c, abs(files['ap'][c] - device['ap'][c])) for c in classes)
    line = {'gpu': name, 'power_limit': power, 'images': len(names), 'classes': n_cls, 'rows': rows,
            'cells_per_row': args.kept, 'kept_per_row_mean': kept_total / float(rows), 'detections': kept_total,
            'files_s_per_pass': t_files, 'files_write_s': t_write, 'files_mean_ap_s': t_files - t_write,
            'device_s_per_pass': t_dev, 'device_s_all_passes': times, 'speedup': t_files / t_dev,
            'mean_ap_files': files['mean'], 'mean_ap_device': device['mean'],
            'ap_files': files['ap'], 'ap_device': device['ap'],
            'max_ap_abs_diff': max(diff.values()), 'classes_equal': sum(1 for c in classes if diff[c] == 0.0),
            'classes_with_tied_confidences': len(tied)}
    print(json.dumps(line))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(line, f)
    return 0


if __name__ == '__main__':
    sys.exit(main())
