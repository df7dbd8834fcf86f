#!/usr/bin/env python
"""Time one COCO minival-sized evaluation pass (5,000 images x 80 classes) on the two paths:

  device  coco_eval.DeviceCocoEval: .add for every batch of Detections, then .result (csrc/coco_eval.cu)
  host    coco_eval.load_coco_annotations on the instances json + coco_eval.coco_evaluate on the results json,
          for `--host-classes` classes only (default 8: the host path takes minutes for all 80)

    python tools/coco_eval_bench.py [--images 5000] [--kept 30] [--host-classes 8] [--device-passes 5] [--out f.json]

The instances json is synthetic and seeded: 1-13 objects per image, 1% crowd, sizes log-uniform from 6 pixels to
2/3 of the image (small, medium and large objects), json area = box area x U(0.6, 1).  Each (image, class) row
holds kept/2 .. 3*kept/2 NMS survivors (float32 candidates as decode + NMS leave them), one near each object of that
class, scores rounded to 1/4096 so that they tie.  Prints one JSON line: seconds per pass of each path, the host
time scaled to 80 classes, the per-class AP of the host classes from both paths (they must be equal) and the GPU's
name and power limit read in the same run.
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

A, H, W = 5, 3, 3                                     # 45 candidate slots per row


def synthetic_instances(n_img, classes, seed):
    rs = np.random.RandomState(seed)
    sizes = np.stack([rs.randint(300, 641, n_img), rs.randint(300, 641, n_img)], 1)
    images = [{'id': 10 * i + 7, 'file_name': 'COCO_val2014_%012d.jpg' % (10 * i + 7), 'width': int(sizes[i, 0]),
               'height': int(sizes[i, 1])} for i in range(n_img)]
    anns = []
    for i in range(n_img):
        iw, ih = sizes[i]
        n = rs.randint(1, 14)
        for c in rs.randint(0, len(classes), n):
            w, h = np.exp(rs.uniform(np.log(6), np.log(iw / 1.5))), np.exp(rs.uniform(np.log(6), np.log(ih / 1.5)))
            x, y = rs.uniform(0, iw - w), rs.uniform(0, ih - h)
            anns.append({'id': len(anns) + 1, 'image_id': 10 * i + 7, 'category_id': int(c) + 1,
                         'bbox': [float(x), float(y), float(w), float(h)], 'area': float(w * h * rs.uniform(0.6, 1.0)),
                         'iscrowd': int(rs.rand() < 0.01)})
    from fewshot_detection_b200.coco_eval import COCO_ALIASES
    cats = [{'id': k + 1, 'name': COCO_ALIASES.get(c, c)} for k, c in enumerate(classes)]
    return {'images': images, 'annotations': anns, 'categories': cats}, sizes


def synthetic_detections(data, sizes, n_cls, kept, batch, seed):
    """Per batch: (image indices, cand [N, 45, 8], keep, keep_count) on the host."""
    rs = np.random.RandomState(seed + 1)
    n_img = len(sizes)
    by_img = [[] for _ in range(n_img)]
    for a in data['annotations']:
        by_img[(a['image_id'] - 7) // 10].append(a)
    out = []
    for b0 in range(0, n_img, batch):
        imgs = list(range(b0, min(b0 + batch, n_img)))
        N = len(imgs) * n_cls
        kc = rs.randint(kept // 2, 3 * kept // 2 + 1, N).astype(np.int32)
        cand = np.zeros((N, A * H * W, 8), dtype=np.float32)
        wh = sizes[imgs].repeat(n_cls, 0)[:, None, :]
        size = np.exp(rs.uniform(np.log(4), np.log(300), (N, A * H * W, 2)))
        ctr = rs.uniform(0, 1, (N, A * H * W, 2)) * wh
        for j, i in enumerate(imgs):
            for a in by_img[i]:
                r = j * n_cls + a['category_id'] - 1
                s = rs.randint(0, kc[r])
                x, y, w, h = a['bbox']
                ctr[r, s] = np.array([x + w / 2, y + h / 2]) * rs.normal(1, 0.03, 2)
                size[r, s] = np.array([w, h]) * rs.normal(1, 0.06, 2)
        cand[..., 0:2] = ctr / wh * np.array([W, H])
        cand[..., 2:4] = size / wh * np.array([W, H])
        cand[..., 4] = np.round(rs.uniform(0, 1, cand.shape[:2]) * 4096) / 4096
        cand[..., 5] = 1.0
        keep = np.tile(np.arange(A * H * W, dtype=np.int32), (N, 1))
        out.append((imgs, cand, keep, kc))
    return out


def host_results(batches, sizes, n_cls, classes, image_ids):
    """detection_records' arithmetic (vectorised) for the rows of `classes`, as results json dicts."""
    res = []
    for imgs, cand, keep, kc in batches:
        v = cand.astype(np.float64)
        bx, by, bw, bh = v[..., 0] / W, v[..., 1] / H, v[..., 2] / W, v[..., 3] / H
        width, height = sizes[imgs].repeat(n_cls, 0)[:, 0:1].astype(np.float64), sizes[imgs].repeat(n_cls, 0)[:, 1:2].astype(np.float64)
        x1, y1 = (bx - bw / 2.0) * width, (by - bh / 2.0) * height
        x2, y2 = (bx + bw / 2.0) * width, (by + bh / 2.0) * height
        score = v[..., 4] * v[..., 5]
        for j, i in enumerate(imgs):
            for c in classes:
                r = j * n_cls + c
                for s in np.argsort(-score[r, :kc[r]], kind='mergesort')[:100]:
                    res.append({'image_id': image_ids[i], 'category_id': c + 1, 'score': float(score[r, s]),
                                'bbox': [float(x1[r, s]), float(y1[r, s]), float(x2[r, s] - x1[r, s]),
                                         float(y2[r, s] - y1[r, s])]})
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--images', type=int, default=5000)
    ap.add_argument('--kept', type=int, default=30, help='mean NMS survivors per (image, class) row')
    ap.add_argument('--batch', type=int, default=64)
    ap.add_argument('--host-classes', type=int, default=8, help='classes scored on the host path')
    ap.add_argument('--device-passes', type=int, default=5)
    ap.add_argument('--seed', type=int, default=0)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()

    import torch
    from eval_bench import gpu_info
    from fewshot_detection_b200 import coco_eval as C, utils as U
    from fewshot_detection_b200.cfg import COCO_NAMES
    if not torch.cuda.is_available():
        raise SystemExit('coco_eval_bench.py measures the GPU path: no CUDA device')
    torch.cuda.set_device(0)
    name, power = gpu_info()
    classes, n_cls = list(COCO_NAMES), len(COCO_NAMES)
    data, sizes = synthetic_instances(args.images, classes, args.seed)
    work = tempfile.mkdtemp(prefix='fsdet_coco_bench_')
    ann_path = os.path.join(work, 'instances_synth.json')
    with open(ann_path, 'w') as f:
        json.dump(data, f)
    names = [os.path.splitext(im['file_name'])[0] for im in data['images']]
    image_ids = [im['id'] for im in data['images']]
    gt = C.load_coco_annotations(ann_path, names, classes)
    host_batches = synthetic_detections(data, sizes, n_cls, args.kept, args.batch, args.seed)
    batches = []
    for imgs, cand, keep, kc in host_batches:
        d = U.Detections(torch.from_numpy(cand).cuda(), torch.from_numpy(kc).cuda(), None, len(kc), A, 1, H, W, False,
                         True, 0.005)
        d.keep, d.keep_count = torch.from_numpy(keep).cuda(), torch.from_numpy(kc).cuda()
        batches.append((d, [names[i] for i in imgs], [tuple(float(v) for v in sizes[i]) for i in imgs]))
    torch.cuda.synchronize()

    def device_pass():
        ev = C.DeviceCocoEval(classes, names, gt)
        for d, ids, sz in batches:
            ev.add(d, ids, sz)
        r = ev.result()
        torch.cuda.synchronize()
        return r, int(ev.counters[0])
    device, n_det = device_pass()                                 # warm-up: module load, allocator
    times = []
    for _ in range(args.device_passes):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        device, _ = device_pass()
        times.append(time.perf_counter() - t0)
    t_dev = float(np.median(times))

    pick = sorted(np.random.RandomState(args.seed + 2).choice(n_cls, args.host_classes, replace=False).tolist())
    res_path = os.path.join(work, 'results.json')
    with open(res_path, 'w') as f:
        json.dump(host_results(host_batches, sizes, n_cls, pick, image_ids), f)
    t0 = time.perf_counter()
    sub = [classes[c] for c in pick]
    with open(ann_path) as f:
        full = json.load(f)
    full['categories'] = [c for c in full['categories'] if c['id'] - 1 in pick]
    full['annotations'] = [a for a in full['annotations'] if a['category_id'] - 1 in pick]
    sub_path = os.path.join(work, 'instances_sub.json')
    with open(sub_path, 'w') as f:
        json.dump(full, f)
    host_gt = C.load_coco_annotations(sub_path, names, sub)
    with open(res_path) as f:
        results = json.load(f)
    host = C.coco_evaluate(host_gt, results, names, sub)
    t_host = time.perf_counter() - t0
    equal = bool(np.array_equal(device['precision'][:, :, pick].view(np.uint64), host['precision'].view(np.uint64)) and
                 np.array_equal(device['recall'][:, pick].view(np.uint64), host['recall'].view(np.uint64)))
    line = {'gpu': name, 'power_limit': power, 'images': len(names), 'classes': n_cls, 'gt_objects': len(data['annotations']),
            'detections': n_det, 'device_s_per_pass': t_dev, 'device_s_all_passes': times,
            'host_classes': sub, 'host_s': t_host, 'host_s_per_80_classes_estimate': t_host * n_cls / len(pick),
            'precision_recall_bit_equal': equal, 'ap_device': dict((c, device['ap'][c]) for c in sub),
            'ap_host': host['ap'], 'stats_device_all_classes': device['all']}
    print(json.dumps(line))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(line, f)
    return 0 if equal else 1


if __name__ == '__main__':
    sys.exit(main())
