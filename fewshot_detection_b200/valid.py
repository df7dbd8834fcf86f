"""Evaluation path of the meta detector (valid_ensemble.py:13-181) on device-resident tensors.

The reference's `valid()` interleaves four things: dataset / file IO (dataset.listDataset, dataset.MetaDataset: the
input pipeline, SURVEY.md 8f row 3, not part of this build), the ensembling of the support net's reweighting vectors
(:86-100), the query forward + decode + NMS (:140-162) and the result-file format (:163-178).  This module provides the
last three with the loaders replaced by plain iterables of tensors, so a caller that owns a data pipeline gets the
same files:

    dw   = ensemble_dynamic_weights(m, meta_batches, n_cls)             # [ [n_cls, C, 1, 1] ]
    dets = detect(m, data, dw, n_cls)                                    # Detections, NMS done, still on the device
    write_detections(fps, dets, imgids, sizes, n_cls)                    # 'imgid prob x1 y1 x2 y2' per class file

or, without the files, scores them where they are (voc_eval.DeviceVocEval, coco_eval.DeviceCocoEval):

    evaluator.add(dets, imgids, sizes); ...; evaluator.result()          # the dict voc_eval.mean_ap returns

`score_batches` runs that whole pass, in one process or sharded over the ranks of a process group.

CUDA only (libfsdet.so); no host fallback.
"""
import os

import torch

from ._lib import call, ptr
from .utils import region_detections

CONF_THRESH = 0.005   # valid_ensemble.py:137
NMS_THRESH = 0.45     # valid_ensemble.py:138


def _st():
    return torch.cuda.current_stream().cuda_stream


class ReweightEnsembler(object):
    """Running mean of the reweighting vectors per class (valid_ensemble.py:86-100):
    enews[c] = enews[c]*cnt[c]/(cnt[c]+1) + dw[ci]/(cnt[c]+1); cnt[c] += 1, in sample order, float32."""

    def __init__(self, n_cls, channels, device):
        self.n_cls, self.C = n_cls, channels
        self.enews = torch.zeros(n_cls, channels, dtype=torch.float32, device=device)
        self._cnt = [torch.zeros(n_cls, dtype=torch.int32, device=device) for _ in range(2)]
        self._cur = 0

    def update(self, dw, clsids):
        """dw: CUDA float32 [n, C(,1,1)]; clsids: n class indices (list / tensor)."""
        n = int(dw.size(0))
        dw = dw.detach().reshape(n, -1).float().contiguous()
        assert dw.size(1) == self.C
        ids = torch.as_tensor([int(c) for c in clsids], dtype=torch.int32).to(dw.device)
        assert ids.numel() == n
        if n and (int(ids.min()) < 0 or int(ids.max()) >= self.n_cls):
            raise IndexError('class id out of range')        # the reference's `enews[c]` raises IndexError too
        cin, cout = self._cnt[self._cur], self._cnt[1 - self._cur]
        call('fsdet_rw_running_mean', ptr(self.enews), ptr(cin), ptr(cout), ptr(dw), ptr(ids), n, self.n_cls, self.C, _st())
        self._cur = 1 - self._cur

    @property
    def counts(self):
        return self._cnt[self._cur]

    def result(self):
        """`[torch.stack(enews)]`: [ [n_cls, C, 1, 1] ]."""
        return [self.enews.view(self.n_cls, self.C, 1, 1)]


def ensemble_dynamic_weights(m, meta_batches, n_cls):
    """valid_ensemble.py:86-100.  `meta_batches` yields (metax [n,3,S,S], mask [n,1,S,S], clsids [n]) like the
    reference's MetaDataset(ensemble=True, with_ids=True) loader."""
    ens = None
    with torch.no_grad():
        for metax, mask, clsids in meta_batches:
            dev = next(m.parameters()).device
            dw = m.meta_forward(metax.to(dev), mask.to(dev))[0]
            if ens is None:
                ens = ReweightEnsembler(n_cls, dw[0].numel(), dw.device)
            ens.update(dw, clsids)
    if ens is None:
        raise ValueError('no support batches')
    return ens.result()


def detect(m, data, dynamic_weights, n_cls, conf_thresh=CONF_THRESH, nms_thresh=NMS_THRESH):
    """valid_ensemble.py:140-162 for one batch: detect_forward -> get_region_boxes_v2(only_objectness=0,
    validation=1) -> nms for every (image, class) row.  Returns utils.Detections (device resident)."""
    with torch.no_grad():
        output = m.detect_forward(data, dynamic_weights)
    dets = region_detections(output, conf_thresh, m.num_classes, m.anchors, m.num_anchors, 0, 1, n_models=n_cls)
    return dets.nms(nms_thresh)


def detection_lines(dets, imgids, sizes, n_cls, nms_thresh=NMS_THRESH):
    """valid_ensemble.py:153-178: {class index: [lines]} with `imgid prob x1 y1 x2 y2` per surviving box.
    imgids[b], sizes[b] = (width, height) of image b of the batch."""
    kept = dets.kept_boxes(nms_thresh)
    bs = dets.N // n_cls
    assert len(imgids) == bs and len(sizes) == bs
    out = dict((i, []) for i in range(n_cls))
    for b in range(bs):
        width, height = sizes[b]
        for i in range(n_cls):
            for box in kept[b * n_cls + i]:
                x1 = (box[0] - box[2] / 2.0) * width
                y1 = (box[1] - box[3] / 2.0) * height
                x2 = (box[0] + box[2] / 2.0) * width
                y2 = (box[1] + box[3] / 2.0) * height
                det_conf = box[4]
                for j in range((len(box) - 5) // 2):
                    prob = det_conf * box[5 + 2 * j]
                    out[i].append('%s %f %f %f %f %f\n' % (imgids[b], prob, x1, y1, x2, y2))
    return out


def write_detections(fps, dets, imgids, sizes, n_cls, nms_thresh=NMS_THRESH):
    """Append the batch's lines to the per-class files `fps[i]` (valid_ensemble.py:128-131, :178)."""
    lines = detection_lines(dets, imgids, sizes, n_cls, nms_thresh)
    for i in range(n_cls):
        fps[i].writelines(lines[i])


def valid_batches(m, meta_batches, image_batches, class_names, prefix, outfile):
    """The body of valid_ensemble.valid() (:86-181) over iterables: `meta_batches` as in ensemble_dynamic_weights,
    `image_batches` yields (data [b,3,H,W], imgids, sizes).  Writes `<prefix>/<outfile><class>.txt`."""
    n_cls = len(class_names)
    m.eval()
    dynamic_weights = ensemble_dynamic_weights(m, meta_batches, n_cls)
    if not os.path.exists(prefix):
        os.makedirs(prefix)
    fps = [open('%s/%s%s.txt' % (prefix, outfile, name), 'w') for name in class_names]
    try:
        dev = next(m.parameters()).device
        for data, imgids, sizes in image_batches:
            dets = detect(m, data.to(dev), dynamic_weights, n_cls)
            write_detections(fps, dets, imgids, sizes, n_cls)
    finally:
        for fp in fps:
            fp.close()
    return dynamic_weights


def score_batches(m, support_batches, image_batches, evaluator, out=None, sharded=False, process_group=None, dst=0,
                  **result_kwargs):
    """valid_batches scored on the device: `evaluator` is a voc_eval.DeviceVocEval or coco_eval.DeviceCocoEval over
    the evaluated image set, `support_batches` are as ensemble_dynamic_weights' meta_batches, `image_batches` yields
    (data, imgids, sizes) with imgids names of that set.  Returns evaluator.result(**result_kwargs): mean_ap's dict
    (use_07_metric=, novel_classes=, curves=) or coco_evaluate's (novel_classes=).

    out (optional) also receives the result files of the same detections, copied to the host for them: for VOC the
    per-class files valid_batches writes (a list of open files), for COCO the standard results json (an open file).

    sharded=True: collective over `process_group`, each rank running its own block of the single-process support and
    query batches (shard.shard_range).  The pools are merged in rank order and scored once on rank `dst`; every rank
    returns the single-process dict.  `out` is open on `dst` and True on the other ranks, whose parts go to `dst`,
    which writes every rank's in rank order: the single-process files.  None on every rank for no files."""
    n_cls = len(evaluator.classes)
    m.eval()
    if sharded:
        dynamic_weights = sharded_ensemble_dynamic_weights(m, support_batches, n_cls, process_group)
    else:
        dynamic_weights = ensemble_dynamic_weights(m, support_batches, n_cls)
    dev = next(m.parameters()).device
    parts = []
    for data, imgids, sizes in image_batches:
        dets = detect(m, data.to(dev), dynamic_weights, n_cls)
        evaluator.add(dets, imgids, sizes)
        if out is not None:
            parts.append(evaluator.result_file_part(dets, imgids, sizes))
    if out is not None:
        if sharded:
            ranks = gather_to(parts, process_group, dst)                # None except on `dst`
            parts = None if ranks is None else [p for r in ranks for p in r]
        if parts is not None:
            evaluator.write_result_file(out, parts)
    if sharded:
        return evaluator.gather(process_group, dst, **result_kwargs)
    return evaluator.result(**result_kwargs)


# ---- the sharded pieces of the pass (shard.py) ----------------------------------------------------------------------
def sharded_ensemble_dynamic_weights(m, meta_batches, n_cls, process_group=None):
    """ensemble_dynamic_weights over every rank's support batches, in rank order.  `meta_batches` are this rank's
    block of the single-process batches (shard.shard_range).  Each rank runs the reweighting net on its own batches;
    the vectors, class ids and batch sizes are all-gathered and every rank applies the running mean batch by batch in
    the single-process order, so every rank returns the single-process result, bit for bit."""
    import numpy as np
    from .shard import all_gather_padded, group_info
    world, _ = group_info(process_group)
    dev = next(m.parameters()).device
    rows, ids, sizes = [], [], []
    with torch.no_grad():
        for metax, mask, clsids in meta_batches:
            dw = m.meta_forward(metax.to(dev), mask.to(dev))[0]
            rows.append(dw.detach().reshape(dw.size(0), -1).float())
            ids.extend(int(c) for c in clsids)
            sizes.append(int(dw.size(0)))
    C = int(rows[0].size(1)) if rows else 0
    shape = torch.tensor([[len(sizes), len(ids), C]], dtype=torch.int64, device=dev)
    shapes = all_gather_padded(shape, 1, process_group).reshape(world, 3).cpu().numpy()
    C = int(shapes[:, 2].max())
    if C == 0:
        raise ValueError('no support batches')
    if any(c not in (0, C) for c in shapes[:, 2]):
        raise ValueError('ranks disagree on the reweighting vector size: %s' % shapes[:, 2].tolist())
    nb, nr = max(1, int(shapes[:, 0].max())), max(1, int(shapes[:, 1].max()))
    local = torch.cat(rows) if rows else torch.zeros(0, C, dtype=torch.float32, device=dev)
    all_rows = all_gather_padded(local, nr, process_group)
    all_ids = all_gather_padded(torch.tensor(ids, dtype=torch.int64).reshape(-1).to(dev), nr, process_group).cpu().numpy()
    all_sizes = all_gather_padded(torch.tensor(sizes, dtype=torch.int64).reshape(-1).to(dev), nb, process_group).cpu().numpy()
    ens = ReweightEnsembler(n_cls, C, dev)
    for r in range(world):
        off = 0
        for b in range(int(shapes[r, 0])):
            n = int(all_sizes[r, b])
            ens.update(all_rows[r, off:off + n], np.asarray(all_ids[r, off:off + n]).tolist())
            off += n
    return ens.result()


def gather_to(obj, process_group, dst):
    """The objects of every rank, in rank order, on rank `dst` (None elsewhere)."""
    import torch.distributed as dist
    from .shard import global_rank, group_info
    world, rank = group_info(process_group)
    out = [None] * world if rank == dst else None
    dist.gather_object(obj, out, dst=global_rank(process_group, dst), group=process_group)
    return out
