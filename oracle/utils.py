"""Oracle restatement of the reference's detection decode + NMS (TEST INFRASTRUCTURE ONLY).

Follows /root/reference/utils.py and valid_ensemble.py:
  nms                   utils.py:85-104
  get_region_boxes      utils.py:112-193
  get_region_boxes_v2   utils.py:195-290
  ensemble_reweights    valid_ensemble.py:86-100   (running mean of reweighting vectors per class)
  detection_lines       valid_ensemble.py:153-178  (per-class result lines `imgid prob x1 y1 x2 y2`)

torch-0.3.1 semantics kept (requirements.txt:3): indexing a 1-D tensor with an int yields a *Python float*, so
every box entry, the `det_conf * cls_conf > conf_thresh` test, the `1 - conf` NMS key (then rounded to float32 by the
store into a FloatTensor) and the NMS IoUs are float64 arithmetic on values promoted exactly from float32.
Tensor math (sigmoid / exp / softmax / max) is torch CPU float32, as at the reference's call sites.

Pinned by tests/golden/detect_*.npz, minted from the reference's own utils.py by tests/golden/make_golden_detect.py.
"""
import numpy as np
import torch

from .region_loss import bbox_iou


def nms(boxes, nms_thresh):
    """utils.py:85-104.  `boxes`: list of lists [x, y, w, h, det_conf, ...]; returns the kept boxes in descending
    det_conf order.  Like the reference, suppressed boxes get box[4] = 0 IN PLACE.  The sort key is
    float32(1 - det_conf) ascending (det_confs is a FloatTensor, :89-91); ties keep list order (stable sort)."""
    if len(boxes) == 0:
        return boxes
    keys = np.empty(len(boxes), dtype=np.float32)
    for i in range(len(boxes)):
        keys[i] = 1 - boxes[i][4]
    order = np.argsort(keys, kind='stable')
    out = []
    for i in range(len(boxes)):
        box_i = boxes[order[i]]
        if box_i[4] > 0:
            out.append(box_i)
            for j in range(i + 1, len(boxes)):
                box_j = boxes[order[j]]
                if bbox_iou(box_i, box_j) > nms_thresh:
                    box_j[4] = 0
    return out


def _decode(output, anchors, num_anchors):
    """Shared tensor prologue of utils.py:112-150 / :224-243: float32 xs, ys, ws, hs, det_confs, flat index
    ind = b*A*HW + a*HW + cy*W + cx."""
    batch, _, h, w = output.shape
    nA = num_anchors
    step = len(anchors) // nA
    o = output.view(batch * nA, -1, h * w).transpose(0, 1).contiguous().view(-1, batch * nA * h * w)
    gx = torch.linspace(0, w - 1, w).repeat(h, 1).repeat(batch * nA, 1, 1).view(-1)
    gy = torch.linspace(0, h - 1, h).repeat(w, 1).t().repeat(batch * nA, 1, 1).view(-1)
    xs = torch.sigmoid(o[0]) + gx
    ys = torch.sigmoid(o[1]) + gy
    an = torch.Tensor(anchors).view(nA, step)
    aw = an[:, 0:1].repeat(batch, 1).repeat(1, 1, h * w).view(-1)
    ah = an[:, 1:2].repeat(batch, 1).repeat(1, 1, h * w).view(-1)
    ws = torch.exp(o[2]) * aw
    hs = torch.exp(o[3]) * ah
    det = torch.sigmoid(o[4])
    return o, xs, ys, ws, hs, det


def _collect(batch, h, w, nA, nC, xs, ys, ws, hs, det, cmax, cid, cls_confs, conf_thresh, only_objectness, validation):
    """The triple loop of utils.py:167-185 / :262-280 on Python floats."""
    xs, ys, ws, hs, det, cmax = [t.tolist() for t in (xs, ys, ws, hs, det, cmax)]
    cid = cid.tolist()
    if validation:
        cls_confs = cls_confs.view(-1, nC).tolist()
    sz_hw = h * w
    sz_hwa = sz_hw * nA
    all_boxes = []
    for b in range(batch):
        boxes = []
        for cy in range(h):
            for cx in range(w):
                for i in range(nA):
                    ind = b * sz_hwa + i * sz_hw + cy * w + cx
                    det_conf = det[ind]
                    conf = det_conf if only_objectness else det_conf * cmax[ind]
                    if conf > conf_thresh:
                        box = [xs[ind] / w, ys[ind] / h, ws[ind] / w, hs[ind] / h, det_conf, cmax[ind], cid[ind]]
                        if (not only_objectness) and validation:
                            for c in range(nC):
                                tmp = cls_confs[ind][c]
                                if c != cid[ind] and det_conf * tmp > conf_thresh:
                                    box.append(tmp)
                                    box.append(c)
                        boxes.append(box)
        all_boxes.append(boxes)
    return all_boxes


def region_arrays(output, num_classes, anchors, num_anchors, n_models=None):
    """The float32 tensors both decode functions compute before their triple loop, flat in the reference's
    `ind = b*A*HW + a*HW + cy*W + cx` order: (xs, ys, ws, hs, det_confs, cls_max_confs, cls_max_ids, cls_confs).
    n_models=None: get_region_boxes (utils.py:121-143); else get_region_boxes_v2 (utils.py:211-243)."""
    output = torch.as_tensor(output, dtype=torch.float32)
    if output.dim() == 3:
        output = output.unsqueeze(0)
    batch, ch, h, w = output.shape
    nA, nC = num_anchors, num_classes
    assert ch == (5 + nC) * nA
    o, xs, ys, ws, hs, det = _decode(output, anchors, nA)
    if n_models is None:
        cls_confs = torch.softmax(o[5:5 + nC].transpose(0, 1), dim=1)
    else:
        cs = n_models
        assert batch % cs == 0
        bs = batch // cs
        cls = output.view(batch, nA, 5 + nC, h, w)[:, :, 5:5 + nC].squeeze()
        cls = cls.reshape(bs, cs, nA * nC * h * w).transpose(1, 2).contiguous().view(bs * nA * nC * h * w, cs)
        cls = torch.softmax(cls, dim=1)
        cls_confs = cls.view(bs, nA * nC * h * w, cs).transpose(1, 2).contiguous().view(bs * cs * nA, nC, h * w) \
            .transpose(1, 2).reshape(bs * cs * nA * h * w, nC)
    cmax, cid = torch.max(cls_confs, 1)
    return xs, ys, ws, hs, det, cmax.view(-1), cid.view(-1), cls_confs


def get_region_boxes(output, conf_thresh, num_classes, anchors, num_anchors, only_objectness=1, validation=False):
    """utils.py:112-193 (plain detector: softmax over the nC class logits of each anchor-cell)."""
    output = torch.as_tensor(output, dtype=torch.float32)
    if output.dim() == 3:
        output = output.unsqueeze(0)
    batch, ch, h, w = output.shape
    xs, ys, ws, hs, det, cmax, cid, cls_confs = region_arrays(output, num_classes, anchors, num_anchors)
    return _collect(batch, h, w, num_anchors, num_classes, xs, ys, ws, hs, det, cmax, cid, cls_confs,
                    conf_thresh, only_objectness, validation)


def get_region_boxes_v2(output, n_models, conf_thresh, num_classes, anchors, num_anchors, only_objectness=1,
                        validation=False):
    """utils.py:195-290 (meta detector: rows are (image, class) pairs, image-major; the class score of a row is the
    softmax ACROSS the n_models class rows of its image, per anchor-cell)."""
    output = torch.as_tensor(output, dtype=torch.float32)
    if output.dim() == 3:
        output = output.unsqueeze(0)
    batch, ch, h, w = output.shape
    xs, ys, ws, hs, det, cmax, cid, cls_confs = region_arrays(output, num_classes, anchors, num_anchors, n_models)
    return _collect(batch, h, w, num_anchors, num_classes, xs, ys, ws, hs, det, cmax, cid, cls_confs,
                    conf_thresh, only_objectness, validation)


def ensemble_reweights(batches, n_cls, dtype=torch.float32):
    """valid_ensemble.py:86-100: running mean of the support net's vectors per class.  `batches` yields
    (dw [n, C], clsids [n]).  Returns [n_cls, C] in `dtype` (float32 as in the reference; float64 for a float64
    oracle of the whole evaluation pass)."""
    enews = [0.0] * n_cls
    cnt = [0.0] * n_cls
    for dw, clsids in batches:
        dw = torch.as_tensor(dw, dtype=dtype)
        for ci, c in enumerate(clsids):
            c = int(c)
            enews[c] = enews[c] * cnt[c] / (cnt[c] + 1) + dw[ci] / (cnt[c] + 1)
            cnt[c] += 1
    return torch.stack(enews)


def detection_lines(boxes, imgid, width, height):
    """valid_ensemble.py:163-178: the result-file lines of one (image, class) row after NMS."""
    lines = []
    for box in boxes:
        x1 = (box[0] - box[2] / 2.0) * width
        y1 = (box[1] - box[3] / 2.0) * height
        x2 = (box[0] + box[2] / 2.0) * width
        y2 = (box[1] + box[3] / 2.0) * height
        det_conf = box[4]
        for j in range((len(box) - 5) // 2):
            cls_conf = box[5 + 2 * j]
            prob = det_conf * cls_conf
            lines.append('%s %f %f %f %f %f\n' % (imgid, prob, x1, y1, x2, y2))
    return lines
