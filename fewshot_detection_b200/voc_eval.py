"""PASCAL VOC detection AP from per-class result files (SURVEY.md 8f row 4).

Host-side companion of `valid.write_detections`: consumes the `imgid prob x1 y1 x2 y2` files and the VOC XML
annotations and returns (recall, precision, AP) per class - the numbers the reference reports through
scripts/voc_eval.py (voc_ap :63-94, voc_eval :96-243; itself the py-faster-rcnn evaluator).  Same function names,
arguments and return values; written from the PASCAL VOC devkit definition:

  * detections of a class are ranked by confidence (descending);
  * a detection is a true positive if its best-overlapping ground-truth box of that class in its image has
    IoU > ovthresh (pixel-inclusive areas: width = xmax - xmin + 1), is not `difficult`, and has not been claimed by a
    higher-ranked detection; a match to a `difficult` box is ignored; anything else is a false positive;
  * AP = area under the monotone precision envelope (VOC10+) or the 11-point average (VOC07).

This is small host work (text parsing + a few thousand IoUs per class): numpy on the CPU, like the reference.
"""
import os
import pickle
import xml.etree.ElementTree as ET

import numpy as np

from . import eval_pool
from .eval_pool import DetectionPool, _ptr, check_pool_flags


def parse_rec(filename):
    """One VOC annotation file -> list of {'name', 'pose', 'truncated', 'difficult', 'bbox': [xmin, ymin, xmax, ymax]}."""
    objects = []
    for node in ET.parse(filename).getroot().iter('object'):
        box = node.find('bndbox')
        objects.append({
            'name': node.findtext('name'),
            'pose': node.findtext('pose'),
            'truncated': int(node.findtext('truncated')),
            'difficult': int(node.findtext('difficult')),
            'bbox': [int(box.findtext(k)) for k in ('xmin', 'ymin', 'xmax', 'ymax')],
        })
    return objects


def voc_ap(rec, prec, use_07_metric=False):
    """AP of a precision/recall curve (arrays ordered by decreasing confidence)."""
    rec = np.asarray(rec, dtype=np.float64)
    prec = np.asarray(prec, dtype=np.float64)
    if use_07_metric:
        ap = 0.
        for t in np.arange(0., 1.1, 0.1):
            above = rec >= t
            ap = ap + (np.max(prec[above]) if above.any() else 0) / 11.
        return ap
    r = np.concatenate(([0.], rec, [1.]))
    p = np.concatenate(([0.], prec, [0.]))
    p = np.maximum.accumulate(p[::-1])[::-1]          # precision envelope: best precision at any higher recall
    step = np.nonzero(r[1:] != r[:-1])[0]
    return np.sum((r[step + 1] - r[step]) * p[step + 1])


def load_annotations(annopath, imagenames, cachedir=None):
    """{imagename: parse_rec(annopath.format(imagename))}, cached as <cachedir>/annots.pkl like the reference."""
    cachefile = os.path.join(cachedir, 'annots.pkl') if cachedir else None
    if cachefile and os.path.isfile(cachefile):
        with open(cachefile, 'rb') as f:
            return pickle.load(f)
    recs = dict((name, parse_rec(annopath.format(name))) for name in imagenames)
    if cachefile:
        if not os.path.isdir(cachedir):
            os.mkdir(cachedir)
        with open(cachefile, 'wb') as f:
            pickle.dump(recs, f)
    return recs


def match_detections(image_ids, confidence, boxes, gt, ovthresh=0.5):
    """Rank the detections and mark true / false positives.

    gt: {image id: (bbox int/float [k, 4], difficult bool [k])}.  Returns (tp, fp) float arrays in rank order."""
    order = np.argsort(-np.asarray(confidence, dtype=np.float64))
    boxes = np.asarray(boxes, dtype=np.float64).reshape(-1, 4)
    claimed = dict((k, np.zeros(len(v[0]), dtype=bool)) for k, v in gt.items())
    tp = np.zeros(len(order))
    fp = np.zeros(len(order))
    for rank, d in enumerate(order):
        img = image_ids[d]
        gboxes, difficult = gt[img]
        best, j = -np.inf, -1
        if len(gboxes):
            g = np.asarray(gboxes, dtype=np.float64)
            b = boxes[d]
            iw = np.minimum(g[:, 2], b[2]) - np.maximum(g[:, 0], b[0]) + 1.
            ih = np.minimum(g[:, 3], b[3]) - np.maximum(g[:, 1], b[1]) + 1.
            inter = np.maximum(iw, 0.) * np.maximum(ih, 0.)
            union = (b[2] - b[0] + 1.) * (b[3] - b[1] + 1.) + (g[:, 2] - g[:, 0] + 1.) * (g[:, 3] - g[:, 1] + 1.) - inter
            iou = inter / union
            j = int(np.argmax(iou))
            best = iou[j]
        if best > ovthresh:
            if difficult[j]:
                continue                      # neither TP nor FP
            if claimed[img][j]:
                fp[rank] = 1.
            else:
                tp[rank] = 1.
                claimed[img][j] = True
        else:
            fp[rank] = 1.
    return tp, fp


def voc_eval(detpath, annopath, imagesetfile, classname, cachedir, ovthresh=0.5, use_07_metric=False):
    """rec, prec, ap = voc_eval(...) as scripts/voc_eval.py:96-243: `detpath.format(classname)` is the result file,
    `annopath.format(imagename)` the XML annotation, `imagesetfile` the list of image names."""
    with open(imagesetfile, 'r') as f:
        imagenames = [x.strip() for x in f.readlines()]
    recs = load_annotations(annopath, imagenames, cachedir)
    gt, npos = {}, 0
    for name in imagenames:
        objs = [o for o in recs[name] if o['name'] == classname]
        difficult = np.array([o['difficult'] for o in objs]).astype(bool)
        gt[name] = (np.array([o['bbox'] for o in objs]), difficult)
        npos += int(np.sum(~difficult))
    with open(detpath.format(classname), 'r') as f:
        rows = [x.strip().split(' ') for x in f.readlines()]
    image_ids = [r[0] for r in rows]
    confidence = np.array([float(r[1]) for r in rows])
    boxes = np.array([[float(z) for z in r[2:]] for r in rows])
    tp, fp = match_detections(image_ids, confidence, boxes, gt, ovthresh)
    tp, fp = np.cumsum(tp), np.cumsum(fp)
    rec = tp / float(npos)
    prec = tp / np.maximum(tp + fp, np.finfo(np.float64).eps)
    return rec, prec, voc_ap(rec, prec, use_07_metric)


def mean_ap(detpath, annopath, imagesetfile, classes, cachedir, use_07_metric=True, novel_classes=()):
    """Per-class AP plus the base / novel means the reference prints (scripts/voc_eval.py:_do_python_eval)."""
    aps = dict((c, voc_eval(detpath, annopath, imagesetfile, c, cachedir, 0.5, use_07_metric)[2]) for c in classes)
    return _ap_summary(classes, aps, novel_classes)


def _ap_summary(classes, aps, novel_classes):
    base = [aps[c] for c in classes if c not in novel_classes]
    novel = [aps[c] for c in classes if c in novel_classes]
    return {'ap': aps, 'mean': float(np.mean(list(aps.values()))), 'mean_base': float(np.mean(base)) if base else None,
            'mean_novel': float(np.mean(novel)) if novel else None}


# --------------------------------------------------------------------------------------------------------------------
# The same numbers without the result files: detections stay on the device (csrc/voc_eval.cu).
VOC07_THRESHOLDS = np.arange(0., 1.1, 0.1)          # voc_ap's thresholds, handed to the device as computed here


def gt_tables(classes, imagenames, recs):
    """Ground truth as CSR over (class, image): gt_ptr int32 [n_cls*n_images + 1], boxes int32 [n_gt, 4] and
    difficult uint8 [n_gt], objects in annotation order (the order voc_eval builds `R`)."""
    cidx = dict((c, i) for i, c in enumerate(classes))
    per = [[[] for _ in imagenames] for _ in classes]
    for k, name in enumerate(imagenames):
        for o in recs[name]:
            i = cidx.get(o['name'])
            if i is not None:
                per[i][k].append(o)
    ptr, boxes, diff = [0], [], []
    for i in range(len(classes)):
        for objs in per[i]:
            boxes.extend([int(v) for v in o['bbox']] for o in objs)
            diff.extend(1 if o['difficult'] else 0 for o in objs)
            ptr.append(len(boxes))
    return (np.array(ptr, dtype=np.int32), np.array(boxes, dtype=np.int32).reshape(-1, 4),
            np.array(diff, dtype=np.uint8))


class DeviceVocEval(DetectionPool):
    """voc_eval / mean_ap over detections that never leave the device.

        ev = DeviceVocEval(classes, imagenames, load_annotations(annopath, imagenames, cachedir))
        for each batch:  ev.add(dets, image_indices, sizes)     # Detections after .nms(0.45), nC = 1 (meta detector)
        ev.result(use_07_metric=True, novel_classes=())          # the dict mean_ap returns

    `add` appends the batch's kept boxes in the order write_detections writes lines and computes them as those lines
    read back: float64, the reference's operation order, '%f' rounding (csrc/voc_eval.cu).  `result` matches, ranks
    and scores every class on the device; only per-class numbers come back (and, with curves=True, rec / prec).
    Ranking differs from the file path in one deliberate way: detections with equal printed confidences keep
    result-file order (a stable sort), where np.argsort's order at ties depends on numpy's sort implementation.
    Each image of the set may be added once.

    Sharded over ranks (shard.py): each rank adds its own contiguous block of batches, then `gather` merges the pools
    in rank order on one rank and scores them there; `merge` does the same for several evaluators on one device."""
    KEY_DTYPE, MERGE_FN = 'int32', 'fsdet_voc_merge'

    def __init__(self, classes, imagenames, recs, device=None, ovthresh=0.5):
        import torch
        DetectionPool.__init__(self, classes, imagenames, device)
        self.ovthresh = float(ovthresh)
        ptr, boxes, diff = gt_tables(self.classes, self.imagenames, recs)
        self.n_gt = int(len(diff))
        self.gt_ptr = torch.from_numpy(ptr).to(self.device)
        self.gt_box = torch.from_numpy(boxes).to(self.device)
        self.gt_difficult = torch.from_numpy(diff).to(self.device)

    def _gather(self, dets, cap, image_index, image_size):
        if eval_pool._is_merged(dets):
            eval_pool._call('fsdet_voc_gather_merged', _ptr(dets.merged), _ptr(dets.keep), _ptr(dets.keep_count), dets.N,
                            cap, len(self.classes), _ptr(image_index), _ptr(image_size), _ptr(self.key),
                            _ptr(self.box), self.pool_cap, _ptr(self.groups), self.group_cap, _ptr(self.counters),
                            eval_pool._stream())
            return
        eval_pool._call('fsdet_voc_gather', _ptr(dets.cand), _ptr(dets.keep), _ptr(dets.keep_count), dets.N, cap,
                        dets.H, dets.W, dets.nC, len(self.classes), _ptr(image_index), _ptr(image_size), _ptr(self.key),
                        _ptr(self.box), self.pool_cap, _ptr(self.groups), self.group_cap, _ptr(self.counters),
                        eval_pool._stream())

    def result_file_part(self, dets, imgids, sizes):
        """The result-file lines of one added batch: valid.detection_lines' {class index: [lines]}."""
        from .valid import detection_lines
        return detection_lines(dets, imgids, sizes, len(self.classes))

    def write_result_file(self, fps, parts):
        """Write result_file_part's batches, in order, to the per-class files `fps` (write_detections' files)."""
        for i in range(len(self.classes)):
            for part in parts:
                fps[i].writelines(part[i])

    def result(self, use_07_metric=True, novel_classes=(), curves=False):
        """The dict mean_ap returns; with curves=True also 'rec' / 'prec': {class: float64 array in rank order}.
        The device results of the last call stay in `self.last` (flags, order, rec, prec, ... as tensors)."""
        import torch
        n_det, n_groups, _, overflow = [int(v) for v in self.counters.cpu()]
        check_pool_flags(overflow)
        n_cls, dev = len(self.classes), self.device
        ws = torch.empty(max(1, eval_pool._call_size('fsdet_voc_workspace_bytes', n_det, self.n_gt)), dtype=torch.uint8,
                         device=dev)
        out = dict(flags=torch.empty(n_det, dtype=torch.uint8, device=dev),
                   order=torch.empty(n_det, dtype=torch.int32, device=dev),
                   rec=torch.empty(n_det, dtype=torch.float64, device=dev),
                   prec=torch.empty(n_det, dtype=torch.float64, device=dev),
                   cls_count=torch.empty(n_cls, dtype=torch.int32, device=dev),
                   npos=torch.empty(n_cls, dtype=torch.int32, device=dev),
                   ap07=torch.empty(n_cls, dtype=torch.float64, device=dev),
                   ap_area=torch.empty(n_cls, dtype=torch.float64, device=dev))
        th = np.ascontiguousarray(VOC07_THRESHOLDS, dtype=np.float64)
        eval_pool._call('fsdet_voc_evaluate', _ptr(self.key) if n_det else None, _ptr(self.box) if n_det else None,
                        n_det, _ptr(self.groups), n_groups, _ptr(self.gt_ptr), _ptr(self.gt_box) if self.n_gt else None,
                        _ptr(self.gt_difficult) if self.n_gt else None, self.n_gt, n_cls, len(self.imagenames),
                        self.ovthresh, th.ctypes.data, _ptr(ws), ws.numel(), _ptr(out['flags']), _ptr(out['order']),
                        _ptr(out['rec']), _ptr(out['prec']), _ptr(out['cls_count']), _ptr(out['npos']),
                        _ptr(out['ap07']), _ptr(out['ap_area']), eval_pool._stream())
        self.last = out
        ap = (out['ap07'] if use_07_metric else out['ap_area']).cpu().numpy()
        aps = dict((c, float(ap[i])) for i, c in enumerate(self.classes))
        r = _ap_summary(self.classes, aps, novel_classes)
        if curves:
            cnt = out['cls_count'].cpu().numpy().astype(np.int64)
            starts = np.concatenate(([0], np.cumsum(cnt)))
            rec, prec = out['rec'].cpu().numpy(), out['prec'].cpu().numpy()
            r['rec'] = dict((c, rec[starts[i]:starts[i + 1]]) for i, c in enumerate(self.classes))
            r['prec'] = dict((c, prec[starts[i]:starts[i + 1]]) for i, c in enumerate(self.classes))
        return r

