"""COCO box AP / AR (the twelve numbers of pycocotools' COCOeval.summarize) for the COCO few-shot setting.

Host evaluator, written from the COCO box-evaluation definition.  It follows pycocotools `COCOeval` with
iouType='bbox', useCats=1 and default `Params`, with the same evaluate / evaluateImg / accumulate / summarize structure,
so that it can be read against pycocotools line by line.  pycocotools itself is not used.

  * IoU is maskApi's bbIou on (x, y, w, h) in float64: a crowd ground truth divides by the detection's area only;
  * per (image, class) the detections are stable-sorted by score (descending) and cut to maxDets[-1] = 100;
  * per area range a ground truth is ignored if it is crowd or its json `area` lies outside the (inclusive) range, and
    the non-ignored ones come first; a detection is greedily matched at each IoU threshold to the best remaining
    ground truth (a later one wins an equal IoU), inherits its ignore flag, and an unmatched detection outside the
    area range is ignored;
  * per (class, area, maxDets) the first maxDets detections of every image are ranked by a stable sort on score, in
    image-set order, and the interpolated precision is read at the 101 recall thresholds.

Images are taken in image-set order where pycocotools takes ascending image ids; the two agree whenever the image
list is sorted by id (as COCO file names are).  Detection boxes are the reference's result-line corners, unclipped to
the image, as `valid.detection_lines` computes them.  `write_coco_results` writes the standard results json, so the
numbers can be cross-checked with pycocotools wherever it is installed.

The same numbers without copying detections to the host: `DeviceCocoEval` (csrc/coco_eval.cu).
"""
import json
import os

import numpy as np

from . import eval_pool
from .eval_pool import DetectionPool, _ptr, check_pool_flags

# coco.names (cfg.coco_classes) spells six classes the VOC way
COCO_ALIASES = {'motorbike': 'motorcycle', 'aeroplane': 'airplane', 'sofa': 'couch', 'pottedplant': 'potted plant',
                'diningtable': 'dining table', 'tvmonitor': 'tv'}
STAT_NAMES = ['AP', 'AP50', 'AP75', 'APs', 'APm', 'APl', 'AR1', 'AR10', 'AR100', 'ARs', 'ARm', 'ARl']


class Params(object):
    """pycocotools Params(iouType='bbox') defaults."""

    def __init__(self):
        self.iouThrs = np.linspace(.5, 0.95, int(np.round((0.95 - .5) / .05)) + 1, endpoint=True)
        self.recThrs = np.linspace(.0, 1.00, int(np.round((1.00 - .0) / .01)) + 1, endpoint=True)
        self.maxDets = [1, 10, 100]
        self.areaRng = [[0 ** 2, 1e5 ** 2], [0 ** 2, 32 ** 2], [32 ** 2, 96 ** 2], [96 ** 2, 1e5 ** 2]]
        self.areaRngLbl = ['all', 'small', 'medium', 'large']


# ---- input / output ---------------------------------------------------------------------------------------------------
def load_coco_annotations(json_path, imagenames, classes):
    """An instances_*.json -> {'image_ids', 'category_ids', 'anns'}.

    imagenames are file-name stems (COCO_val2014_000000000042) matched to images[].file_name; class i of `classes`
    (coco.names order) is the i-th category by ascending id, and the names must agree up to COCO_ALIASES.
    anns[k] lists image k's objects in json order as (class index, [x, y, w, h] float64, area, iscrowd)."""
    with open(json_path, 'r') as f:
        data = json.load(f)
    cats = sorted(data['categories'], key=lambda c: c['id'])
    if len(cats) != len(classes):
        raise ValueError('%d categories in %s, %d classes' % (len(cats), json_path, len(classes)))
    for name, c in zip(classes, cats):
        if COCO_ALIASES.get(name, name) != c['name']:
            raise ValueError('class %r does not match category %d %r' % (name, c['id'], c['name']))
    cat_index = dict((c['id'], i) for i, c in enumerate(cats))
    by_stem = dict((os.path.splitext(im['file_name'])[0], im['id']) for im in data['images'])
    missing = [n for n in imagenames if n not in by_stem]
    if missing:
        raise KeyError('images not in %s: %s' % (json_path, missing[:5]))
    image_ids = [by_stem[n] for n in imagenames]
    index = dict((i, k) for k, i in enumerate(image_ids))
    anns = [[] for _ in imagenames]
    for a in data['annotations']:
        k = index.get(a['image_id'])
        if k is not None:
            anns[k].append((cat_index[a['category_id']], [float(v) for v in a['bbox']], a['area'], int(a['iscrowd'])))
    return {'image_ids': image_ids, 'category_ids': [c['id'] for c in cats], 'anns': anns}


def detection_records(dets, imgids, sizes, n_cls, max_det=100):
    """The kept boxes of one batch (utils.Detections after .nms()) in valid.detection_lines order: image b, class i,
    then the row's first `max_det` boxes by a stable sort on score, descending.  score = det_conf * cls_conf and the
    corners are detection_lines' (float64, unclipped); bbox = [x1, y1, x2 - x1, y2 - y1].
    Returns [(imgid, class index, score, bbox)]."""
    kept = dets.kept_boxes(dets._nms_thresh)
    bs = dets.N // n_cls
    assert len(imgids) == bs and len(sizes) == bs
    out = []
    for b in range(bs):
        width, height = sizes[b]
        for i in range(n_cls):
            row = []
            for box in kept[b * n_cls + i]:
                x1 = (box[0] - box[2] / 2.0) * width
                y1 = (box[1] - box[3] / 2.0) * height
                x2 = (box[0] + box[2] / 2.0) * width
                y2 = (box[1] + box[3] / 2.0) * height
                det_conf = box[4]
                for j in range((len(box) - 5) // 2):
                    row.append((imgids[b], i, det_conf * box[5 + 2 * j], [x1, y1, x2 - x1, y2 - y1]))
            order = np.argsort([-r[2] for r in row], kind='mergesort')[:max_det]
            out.extend(row[k] for k in order)
    return out


def write_coco_results(fp, records, image_ids, category_ids):
    """The results json [{"image_id", "category_id", "bbox", "score"}] of detection_records' tuples.  image_ids maps
    an imgid to its COCO id, category_ids[i] is class i's category id.  Floats are written with repr (exact)."""
    json.dump([{'image_id': image_ids[r[0]], 'category_id': category_ids[r[1]], 'bbox': [float(v) for v in r[3]],
                'score': float(r[2])} for r in records], fp)


# ---- evaluation ---------------------------------------------------------------------------------------------------
def bbox_iou(d, g, iscrowd):
    """maskApi.c bbIou: [D, G] IoU of (x, y, w, h) boxes, float64."""
    d = np.asarray(d, dtype=np.float64).reshape(-1, 4)
    g = np.asarray(g, dtype=np.float64).reshape(-1, 4)
    crowd = np.asarray(iscrowd, dtype=bool)
    da = (d[:, 2] * d[:, 3])[:, None]
    ga = (g[:, 2] * g[:, 3])[None, :]
    w = np.minimum(d[:, 2:3] + d[:, 0:1], (g[:, 2] + g[:, 0])[None]) - np.maximum(d[:, 0:1], g[None, :, 0])
    h = np.minimum(d[:, 3:4] + d[:, 1:2], (g[:, 3] + g[:, 1])[None]) - np.maximum(d[:, 1:2], g[None, :, 1])
    i = w * h
    u = np.where(crowd[None, :], da, da + ga - i)
    with np.errstate(divide='ignore', invalid='ignore'):
        o = i / u
    return np.where((w > 0) & (h > 0), o, 0.0)


def evaluate_img(dt, gt, aRng, maxDet, p):
    """COCOeval.evaluateImg for one (image, class, area range).  dt: [(score, bbox)], gt: [(bbox, area, iscrowd)]."""
    if len(gt) == 0 and len(dt) == 0:
        return None
    gt_ignore = np.array([bool(g[2]) or g[1] < aRng[0] or g[1] > aRng[1] for g in gt], dtype=bool)
    gtind = np.argsort(gt_ignore, kind='mergesort')
    gt = [gt[i] for i in gtind]
    dtind = np.argsort([-d[0] for d in dt], kind='mergesort')
    dt = [dt[i] for i in dtind[0:maxDet]]
    iscrowd = np.array([int(g[2]) for g in gt], dtype=bool)
    gtIg = gt_ignore[gtind]
    T, G, D = len(p.iouThrs), len(gt), len(dt)
    gtm = np.zeros((T, G), dtype=bool)
    dtm = np.zeros((T, D), dtype=bool)
    dtIg = np.zeros((T, D), dtype=bool)
    if G and D:
        ious = bbox_iou([d[1] for d in dt], [g[0] for g in gt], iscrowd)
        for dind in range(D):
            # the threshold loop of pycocotools, all thresholds at once
            iou = np.minimum(p.iouThrs, 1 - 1e-10)
            m = np.full(T, -1)
            done = np.zeros(T, dtype=bool)
            for gind in range(G):
                live = ~done & ~(gtm[:, gind] & ~iscrowd[gind])                    # taken, not crowd: continue
                brk = live & (m > -1) & ~gtIg[np.maximum(m, 0)] & gtIg[gind]      # break
                done |= brk
                live &= ~brk
                take = live & ~(ious[dind, gind] < iou)                           # < iou: continue
                iou = np.where(take, ious[dind, gind], iou)
                m = np.where(take, gind, m)
            hit = m > -1
            dtIg[hit, dind] = gtIg[m[hit]]
            dtm[hit, dind] = True
            gtm[np.nonzero(hit)[0], m[hit]] = True
    a = np.array([d[1][2] * d[1][3] < aRng[0] or d[1][2] * d[1][3] > aRng[1] for d in dt], dtype=bool).reshape(1, D)
    dtIg = np.logical_or(dtIg, np.logical_and(~dtm, np.repeat(a, T, 0)))
    return {'dtScores': np.array([d[0] for d in dt], dtype=np.float64), 'dtMatches': dtm, 'dtIgnore': dtIg,
            'gtIgnore': gtIg}


def accumulate(evalImgs, n_cls, n_img, p):
    """COCOeval.accumulate: precision [T, R, K, A, M] and recall [T, K, A, M], -1 where undefined.
    evalImgs[k][a][i] is evaluate_img's result for class k, area a, image i (image-set order)."""
    T, R, K, A, M = len(p.iouThrs), len(p.recThrs), n_cls, len(p.areaRng), len(p.maxDets)
    precision = -np.ones((T, R, K, A, M))
    recall = -np.ones((T, K, A, M))
    for k in range(K):
        for a in range(A):
            E = [e for e in evalImgs[k][a] if e is not None]
            if len(E) == 0:
                continue
            for m, maxDet in enumerate(p.maxDets):
                dtScores = np.concatenate([e['dtScores'][0:maxDet] for e in E])
                inds = np.argsort(-dtScores, kind='mergesort')
                dtm = np.concatenate([e['dtMatches'][:, 0:maxDet] for e in E], axis=1)[:, inds]
                dtIg = np.concatenate([e['dtIgnore'][:, 0:maxDet] for e in E], axis=1)[:, inds]
                gtIg = np.concatenate([e['gtIgnore'] for e in E])
                npig = np.count_nonzero(gtIg == 0)
                if npig == 0:
                    continue
                tps = np.logical_and(dtm, np.logical_not(dtIg))
                fps = np.logical_and(np.logical_not(dtm), np.logical_not(dtIg))
                tp_sum = np.cumsum(tps, axis=1).astype(dtype=np.float64)
                fp_sum = np.cumsum(fps, axis=1).astype(dtype=np.float64)
                for t, (tp, fp) in enumerate(zip(tp_sum, fp_sum)):
                    nd = len(tp)
                    rc = tp / npig
                    pr = tp / (fp + tp + np.spacing(1))
                    recall[t, k, a, m] = rc[-1] if nd else 0
                    q = np.zeros((R,))
                    if nd:
                        pr = np.maximum.accumulate(pr[::-1])[::-1]        # pycocotools' backward running max
                        pi = np.searchsorted(rc, p.recThrs, side='left')
                        ok = pi < nd                                       # past the end: 0 (pycocotools' IndexError)
                        q[ok] = pr[pi[ok]]
                    precision[t, :, k, a, m] = q
    return precision, recall


def _mean_defined(s):
    return -1.0 if len(s[s > -1]) == 0 else float(np.mean(s[s > -1]))


def summarize(precision, recall, classes, novel_classes=(), params=None):
    """COCOeval.summarize's 12 stats over all classes, the base and the novel classes ({'all', 'base', 'novel'}:
    lists in STAT_NAMES order, None for an empty subset) and the AP@[.5:.95] of each class ({'ap'})."""
    p = params or Params()

    def stats(ks):
        if not ks:
            return None

        def one(ap, iouThr=None, areaRng='all', maxDets=100):
            aind = [i for i, aRng in enumerate(p.areaRngLbl) if aRng == areaRng]
            mind = [i for i, mDet in enumerate(p.maxDets) if mDet == maxDets]
            s = precision if ap else recall
            if iouThr is not None:
                s = s[np.where(iouThr == p.iouThrs)[0]]
            s = s[:, :, ks][..., aind, mind] if ap else s[:, ks][..., aind, mind]
            return _mean_defined(s)
        md = p.maxDets[2]
        return [one(1), one(1, .5, maxDets=md), one(1, .75, maxDets=md), one(1, areaRng='small', maxDets=md),
                one(1, areaRng='medium', maxDets=md), one(1, areaRng='large', maxDets=md), one(0, maxDets=p.maxDets[0]),
                one(0, maxDets=p.maxDets[1]), one(0, maxDets=md), one(0, areaRng='small', maxDets=md),
                one(0, areaRng='medium', maxDets=md), one(0, areaRng='large', maxDets=md)]
    classes = list(classes)
    novel = [k for k, c in enumerate(classes) if c in novel_classes]
    base = [k for k, c in enumerate(classes) if c not in novel_classes]
    ap = dict((c, _mean_defined(precision[:, :, k, 0, -1])) for k, c in enumerate(classes))
    return {'all': stats(list(range(len(classes)))), 'base': stats(base), 'novel': stats(novel), 'ap': ap}


def coco_evaluate(gt, results, imagenames, classes, params=None, novel_classes=()):
    """COCOeval(iouType='bbox').evaluate(); accumulate(); summarize() on the results json's list of dicts.
    Returns {'precision', 'recall'} plus summarize's dict."""
    p = params or Params()
    n_img, n_cls = len(imagenames), len(classes)
    img_index = dict((i, k) for k, i in enumerate(gt['image_ids']))
    cat_index = dict((c, k) for k, c in enumerate(gt['category_ids']))
    dts = {}
    for r in results:
        if r['image_id'] not in img_index:
            raise ValueError('result for image id %r outside the evaluated set' % r['image_id'])
        key = (img_index[r['image_id']], cat_index[r['category_id']])
        dts.setdefault(key, []).append((float(r['score']), [float(v) for v in r['bbox']]))
    gts = {}
    for i, objs in enumerate(gt['anns']):
        for c, bbox, area, crowd in objs:
            gts.setdefault((i, c), []).append((bbox, area, crowd))
    evalImgs = [[[None] * n_img for _ in p.areaRng] for _ in range(n_cls)]
    for (i, c) in set(dts) | set(gts):
        for a, aRng in enumerate(p.areaRng):
            evalImgs[c][a][i] = evaluate_img(dts.get((i, c), []), gts.get((i, c), []), aRng, p.maxDets[-1], p)
    precision, recall = accumulate(evalImgs, n_cls, n_img, p)
    out = {'precision': precision, 'recall': recall}
    out.update(summarize(precision, recall, classes, novel_classes, p))
    return out


def format_stats(stats, p=None):
    """The lines COCOeval.summarize prints."""
    p = p or Params()
    lines = []
    for k, v in enumerate(stats):
        ap = k < 6
        iou = {1: '0.50', 2: '0.75'}.get(k, '%0.2f:%0.2f' % (p.iouThrs[0], p.iouThrs[-1]))
        area = {3: 'small', 4: 'medium', 5: 'large', 9: 'small', 10: 'medium', 11: 'large'}.get(k, 'all')
        md = {6: p.maxDets[0], 7: p.maxDets[1]}.get(k, p.maxDets[2])
        lines.append(' {:<18} {} @[ IoU={:<9} | area={:>6s} | maxDets={:>3d} ] = {:0.3f}'.format(
            'Average Precision' if ap else 'Average Recall', '(AP)' if ap else '(AR)', iou, area, md, v))
    return lines


# --------------------------------------------------------------------------------------------------------------------
# The same numbers with the detections kept on the device (csrc/coco_eval.cu).
def gt_tables(gt, n_cls):
    """Ground truth as CSR over (class, image): ptr int32 [n_cls*n_images + 1], box float64 [n, 4] (x, y, w, h),
    area float64 [n], iscrowd uint8 [n]; objects of an (image, class) in json order."""
    n_img = len(gt['anns'])
    objs = [(o[0] * n_img + i, o[1], o[2], o[3]) for i, objs in enumerate(gt['anns']) for o in objs]
    cell = np.array([o[0] for o in objs], dtype=np.int64)
    order = np.argsort(cell, kind='stable')                      # (class, image) rows, json order inside
    ptr = np.concatenate(([0], np.cumsum(np.bincount(cell, minlength=n_cls * n_img))))
    box = np.array([o[1] for o in objs], dtype=np.float64).reshape(-1, 4)[order]
    area = np.array([float(o[2]) for o in objs], dtype=np.float64)[order]
    crowd = np.array([1 if o[3] else 0 for o in objs], dtype=np.uint8)[order]
    return ptr.astype(np.int32), box, area, crowd


def device_params(p=None):
    """The Params arrays the device takes: iouThrs [10], recThrs [101], maxDets [3] int32, areaRng [4, 2]."""
    p = p or Params()
    arrs = (np.ascontiguousarray(p.iouThrs, dtype=np.float64), np.ascontiguousarray(p.recThrs, dtype=np.float64),
            np.ascontiguousarray(p.maxDets, dtype=np.int32), np.ascontiguousarray(p.areaRng, dtype=np.float64))
    if [a.size for a in arrs] != [10, 101, 3, 8]:
        raise ValueError('the device evaluates 10 IoU thresholds, 101 recall thresholds, 3 maxDets and 4 areas')
    return arrs


class DeviceCocoEval(DetectionPool):
    """coco_evaluate over detections that never leave the device.

        ev = DeviceCocoEval(classes, imagenames, load_coco_annotations(json_path, imagenames, classes))
        for each batch:  ev.add(dets, image_indices, sizes)     # Detections after .nms(0.45), nC = 1 (meta detector)
        ev.result(novel_classes=())                              # coco_evaluate's dict

    `add` appends each row's first 100 kept boxes by score (csrc/coco_eval.cu), with detection_records' float64
    scores and boxes.  `result` matches and ranks on the device; only precision [T, R, K, A, M] and recall
    [T, K, A, M] come back, and the summary is computed from them on the host.  Every image of the set counts with
    its ground truth, added or not; each image may be added once.  `last` keeps the device arrays of the last result.
    `merge` and `gather` combine the pools of several evaluators (eval_pool.DetectionPool)."""
    KEY_DTYPE, MERGE_FN = 'float64', 'fsdet_coco_merge'

    def __init__(self, classes, imagenames, gt, device=None, params=None):
        import torch
        DetectionPool.__init__(self, classes, imagenames, device)
        if len(gt['anns']) != len(self.imagenames):
            raise ValueError('ground truth of %d images for %d names' % (len(gt['anns']), len(self.imagenames)))
        self.params = params or Params()
        self.image_ids, self.category_ids = list(gt['image_ids']), list(gt['category_ids'])
        self.iou_thrs, self.rec_thrs, self.max_dets, self.area_rng = device_params(self.params)
        self.max_det = int(self.max_dets[-1])
        ptr, box, area, crowd = gt_tables(gt, len(self.classes))
        self.n_gt = int(len(area))
        self.gt_ptr = torch.from_numpy(ptr).to(self.device)
        self.gt_box = torch.from_numpy(box).to(self.device)
        self.gt_area = torch.from_numpy(area).to(self.device)
        self.gt_crowd = torch.from_numpy(crowd).to(self.device)

    def _row_bound(self, cap):
        return min(cap, self.max_det)

    def _gather(self, dets, cap, image_index, image_size):
        if eval_pool._is_merged(dets):
            eval_pool._call('fsdet_coco_gather_merged', _ptr(dets.merged), _ptr(dets.keep), _ptr(dets.keep_count),
                            dets.N, cap, len(self.classes), _ptr(image_index), _ptr(image_size), self.max_det,
                            _ptr(self.key), _ptr(self.box), self.pool_cap, _ptr(self.groups), self.group_cap,
                            _ptr(self.counters), eval_pool._stream())
            return
        eval_pool._call('fsdet_coco_gather', _ptr(dets.cand), _ptr(dets.keep), _ptr(dets.keep_count), dets.N, cap,
                        dets.H, dets.W, dets.nC, len(self.classes), _ptr(image_index), _ptr(image_size), self.max_det,
                        _ptr(self.key), _ptr(self.box), self.pool_cap, _ptr(self.groups), self.group_cap,
                        _ptr(self.counters), eval_pool._stream())

    def result_file_part(self, dets, imgids, sizes):
        """The results-json records of one added batch: detection_records' tuples."""
        return detection_records(dets, imgids, sizes, len(self.classes), self.max_det)

    def write_result_file(self, fp, parts):
        """Write result_file_part's batches, in order, to the open file `fp` as one results json."""
        ids = dict((n, i) for n, i in zip(self.imagenames, self.image_ids))
        write_coco_results(fp, [r for part in parts for r in part], ids, self.category_ids)

    def evaluate(self):
        """Run the device evaluation; returns the dict of device tensors (also kept in `last`)."""
        import torch
        n_det, n_groups, _, overflow = [int(v) for v in self.counters.cpu()]
        check_pool_flags(overflow)
        n_cls, n_img, dev = len(self.classes), len(self.imagenames), self.device
        T, R, A, M = len(self.iou_thrs), len(self.rec_thrs), len(self.area_rng), len(self.max_dets)
        ws = torch.empty(max(1, eval_pool._call_size('fsdet_coco_workspace_bytes', n_det, self.n_gt, n_cls, n_img)),
                         dtype=torch.uint8, device=dev)
        out = dict(dt_flags=torch.empty(A, max(n_det, 1), dtype=torch.int32, device=dev),
                   order=torch.empty(max(n_det, 1), dtype=torch.int32, device=dev),
                   precision=torch.empty(T, R, n_cls, A, M, dtype=torch.float64, device=dev),
                   recall=torch.empty(T, n_cls, A, M, dtype=torch.float64, device=dev))
        eval_pool._call('fsdet_coco_evaluate', _ptr(self.key) if n_det else None, _ptr(self.box) if n_det else None,
                        n_det, _ptr(self.groups), n_groups, _ptr(self.gt_ptr), _ptr(self.gt_box) if self.n_gt else None,
                        _ptr(self.gt_area) if self.n_gt else None, _ptr(self.gt_crowd) if self.n_gt else None,
                        self.n_gt, n_cls, n_img, self.iou_thrs.ctypes.data, self.rec_thrs.ctypes.data,
                        self.max_dets.ctypes.data, self.area_rng.ctypes.data, _ptr(ws), ws.numel(),
                        _ptr(out['dt_flags']), _ptr(out['order']), _ptr(out['precision']), _ptr(out['recall']),
                        eval_pool._stream())
        self.last = out
        return out

    def result(self, novel_classes=()):
        """coco_evaluate's dict: precision, recall (numpy) and the summary."""
        out = self.evaluate()
        precision, recall = out['precision'].cpu().numpy(), out['recall'].cpu().numpy()
        r = {'precision': precision, 'recall': recall}
        r.update(summarize(precision, recall, self.classes, novel_classes, self.params))
        return r
