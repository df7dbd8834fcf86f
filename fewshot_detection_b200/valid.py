"""Evaluation path of the meta detector (valid_ensemble.py:13-181) on device-resident tensors.

The reference's `valid()` interleaves four things: dataset / file IO (dataset.listDataset, dataset.MetaDataset: the
input pipeline, SURVEY.md 8f row 3, not part of this build), the ensembling of the support net's reweighting vectors
(:86-100), the query forward + decode + NMS (:140-162) and the result-file format (:163-178).  This module provides the
last three with the loaders replaced by plain iterables of tensors, so a caller that owns a data pipeline gets the
same files:

    dw   = ensemble_dynamic_weights(m, meta_batches, n_cls)             # [ [n_cls, C, 1, 1] ]
    dets = detect(m, data, dw, n_cls)                                    # Detections, NMS done, still on the device
    write_detections(fps, dets, imgids, sizes, n_cls)                    # 'imgid prob x1 y1 x2 y2' per class file

or, for the boxes of each image rather than the evaluation files, detect_images (per-image top max_det over all
classes, on the device; graph.GraphedDetect replays the same pass as one CUDA graph).

or, with test-time augmentation (several sides, mirrored or not, merged into one NMS on the device):

    inputs = tta_inputs(batcher, indices, passes)                        # one input per pass (side, flip)
    dets = detect_tta(m, inputs, dw, n_cls, passes)                      # utils.MergedDetections, NMS done

which every consumer below takes in place of Detections,

or, without the files, scores them where they are (voc_eval.DeviceVocEval, coco_eval.DeviceCocoEval):

    evaluator.add(dets, imgids, sizes); ...; evaluator.result()          # the dict voc_eval.mean_ap returns

`score_batches` runs that whole pass, in one process or sharded over the ranks of a process group.  Both passes can
write the ensembled vectors to the reference's vectors file and detect with the base-class rows of a stored one
(valid_ensemble.py:102-119, `use_baserw`): evaluation_dynamic_weights.

CUDA only (libfsdet.so); no host fallback.
"""
import os

import torch

from ._lib import call, ptr
from .utils import MergedDetections, region_detections

CONF_THRESH = 0.005   # valid_ensemble.py:137
NMS_THRESH = 0.45     # valid_ensemble.py:138
DETECT_CONF_THRESH = 0.5    # detect.py's do_detect(m, img, 0.5, 0.4)
DETECT_NMS_THRESH = 0.4
MAX_DET = 100


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


# ---- stored reweighting vectors (valid_ensemble.py:102-119) ----------------------------------------------------------
# The file is the reference's: a pickled list with one float32 numpy array [n_cls, C, 1, 1] per dynamic layer, rows in
# the order of the evaluated class list.  Its `use_baserw` mode replaces the base-class rows of the ensembled vectors
# with the stored ones, so that after k-shot fine-tuning the base classes keep vectors averaged over a large support set.
def reweighting_vector_shapes(learnet_blocks, n_cls):
    """The shapes of the vectors a model with these reweighting-net blocks ensembles for n_cls classes: one layer,
    [n_cls, C, 1, 1] with C the filters of the net's last convolution (what meta_forward returns per support image)."""
    convs = [b for b in learnet_blocks if b['type'] == 'convolutional']
    if not convs:
        raise ValueError('the reweighting net has no convolution')
    return [(int(n_cls), int(convs[-1]['filters']), 1, 1)]


def save_reweighting_vectors(path, dynamic_weights):
    """Pickle `[x.cpu().numpy() for x in dynamic_weights]` to `path` (the reference's commented-out writer,
    valid_ensemble.py:102-106)."""
    import pickle
    arrays = [x.detach().to('cpu', torch.float32).contiguous().numpy() for x in dynamic_weights]
    with open(path, 'wb') as f:
        pickle.dump(arrays, f)


def load_reweighting_vectors(path, shapes=None):
    """The list save_reweighting_vectors wrote, or a Python 2 pickle of the same list.  `shapes`: the shape of every
    layer the evaluated model has (reweighting_vector_shapes); anything else raises ValueError, as does anything that
    is not a list of finite float32 arrays."""
    import pickle
    import numpy as np
    with open(path, 'rb') as f:
        try:
            rws = pickle.load(f, encoding='latin1')    # Python 2 pickles hold the array bytes as 8-bit str
        except Exception as e:
            raise ValueError('%s: not a pickled list of vectors: %s: %s' % (path, type(e).__name__, e))
    want = 'float32 arrays of shapes %s' % [tuple(s) for s in shapes] if shapes is not None else \
        'float32 arrays [n_cls, C, 1, 1]'
    if not isinstance(rws, list) or not all(isinstance(a, np.ndarray) for a in rws):
        got = type(rws).__name__ if not isinstance(rws, list) else 'a list of %s' % [type(a).__name__ for a in rws]
        raise ValueError('%s: expected a list of %s, got %s' % (path, want, got))
    got = [tuple(a.shape) for a in rws]
    if shapes is not None and got != [tuple(s) for s in shapes]:
        raise ValueError('%s: the model needs %s, the file has shapes %s' % (path, want, got))
    for i, a in enumerate(rws):
        if a.dtype != np.float32 or a.ndim != 4 or a.shape[2:] != (1, 1):
            raise ValueError('%s: expected %s, layer %d is %s %s' % (path, want, i, a.dtype, a.shape))
        if not np.isfinite(a).all():
            raise ValueError('%s: layer %d %s has non-finite values' % (path, i, a.shape))
    return rws


def substitute_base_rows(dynamic_weights, stored, base_rows):
    """dynamic_weights[i][base_rows] = stored[i][base_rows] in place, in every layer (valid_ensemble.py:117-119).
    `stored` is load_reweighting_vectors' list; `base_rows` are the indices of the evaluated classes that are not
    novel (cfg._real_base_ids for cfg.classes).  The other rows keep their ensembled values."""
    if len(stored) != len(dynamic_weights):
        raise ValueError('%d stored layers for %d dynamic layers' % (len(stored), len(dynamic_weights)))
    rows = torch.as_tensor(list(base_rows), dtype=torch.int64)
    for dw, rw in zip(dynamic_weights, stored):
        src = torch.as_tensor(rw)
        if tuple(src.shape) != tuple(dw.shape):
            raise ValueError('stored vectors %s do not fit the ensembled %s' % (tuple(src.shape), tuple(dw.shape)))
        dw[rows.to(dw.device)] = src[rows].to(dw.device, dw.dtype)      # only the base rows go to the device
    return dynamic_weights


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


def evaluation_dynamic_weights(m, meta_batches, n_cls, sharded=False, process_group=None, dst=0, base_rw=None,
                               base_rows=None, save_rw=None):
    """The vectors an evaluation pass detects with: the ensemble over `meta_batches` (sharded=True: this rank's block,
    gathered so that every rank holds the single-process vectors), written to the file `save_rw` by one process
    (rank `dst` when sharded) before any substitution, then with the `base_rows` of the stored `base_rw`
    (load_reweighting_vectors) substituted on every rank."""
    if base_rw is not None and base_rows is None:
        raise ValueError('base_rw needs base_rows: the indices of the evaluated classes that are not novel')
    if sharded:
        from .shard import group_info
        dynamic_weights = sharded_ensemble_dynamic_weights(m, meta_batches, n_cls, process_group)
        writer = group_info(process_group)[1] == dst
    else:
        dynamic_weights = ensemble_dynamic_weights(m, meta_batches, n_cls)
        writer = True
    if save_rw is not None and writer:
        save_reweighting_vectors(save_rw, dynamic_weights)
    if base_rw is not None:
        substitute_base_rows(dynamic_weights, base_rw, base_rows)
    return dynamic_weights


def detect(m, data, dynamic_weights, n_cls, conf_thresh=CONF_THRESH, nms_thresh=NMS_THRESH, anchors_dev=None):
    """valid_ensemble.py:140-162 for one batch: detect_forward -> get_region_boxes_v2(only_objectness=0,
    validation=1) -> nms for every (image, class) row.  Returns utils.Detections (device resident).
    anchors_dev: see utils.region_detections."""
    with torch.no_grad():
        output = m.detect_forward(data, dynamic_weights)
    dets = region_detections(output, conf_thresh, m.num_classes, m.anchors, m.num_anchors, 0, 1, n_models=n_cls,
                             anchors_dev=anchors_dev)
    return dets.nms(nms_thresh)


# ---- test-time augmentation ------------------------------------------------------------------------------------------
# A plan is an ordered list of passes (side, flip): the images resized to side x side (side a multiple of 32), mirrored
# left-right when flip = 1.  The candidates of every pass are merged per (image, class) row in pass order, the flipped
# passes' boxes mirrored back (x = 1 - x), and suppressed together by one NMS.  [(m.width, 0)] is the plain evaluation.
def tta_plan(sides, flip=False):
    """The passes of `sides` (in order), each followed by its mirrored pass when flip.  Raises ValueError on an empty
    list, a side that is not a positive multiple of 32, or a repeated side."""
    sides = [int(s) for s in sides]
    if not sides:
        raise ValueError('no test-time augmentation sides')
    for side in sides:
        if side <= 0 or side % 32:
            raise ValueError('side %d is not a positive multiple of 32' % side)
    if len(set(sides)) != len(sides):
        raise ValueError('repeated side in %s' % sides)
    return [(side, f) for side in sides for f in ((0, 1) if flip else (0,))]


def parse_tta_sides(text):
    """`416,544,608` -> [416, 544, 608] (ValueError on anything tta_plan refuses)."""
    try:
        sides = [int(t) for t in str(text).split(',') if t.strip()]
    except ValueError:
        raise ValueError('sides must be integers separated by commas, got %r' % text)
    tta_plan(sides)
    return sides


def check_tta_passes(passes):
    """The passes as a list of (side, flip) int pairs; ValueError on an empty plan, a bad side or flag, or a pass twice."""
    out = []
    for p in passes:
        side, flip = int(p[0]), int(p[1])
        if side <= 0 or side % 32:
            raise ValueError('side %d is not a positive multiple of 32' % side)
        if flip not in (0, 1):
            raise ValueError('flip must be 0 or 1, got %d' % flip)
        out.append((side, flip))
    if not out:
        raise ValueError('no test-time augmentation passes')
    if len(set(out)) != len(out):
        raise ValueError('repeated pass in %s' % out)
    return out


def tta_inputs(batcher, indices, passes):
    """The input of every pass for the images `indices` of a dataset.DetectionBatcher (evaluation: train=False),
    decoded once: per side exactly what the batcher's batch() makes at shape (side, side) (the same resize through
    fsdet_augment_batch), and for a flipped pass torch.flip of that along the width."""
    from . import image as I
    passes = check_tta_passes(passes)
    entries = [batcher._entry(i) for i in indices]
    arrays = I.decode_many([e.item if e._arr is None else e._arr for e in entries])
    base = {}
    for side, _ in passes:
        if side in base:
            continue
        params = [I.identity_augmentation(int(a.shape[1]), int(a.shape[0])) for a in arrays]
        for p in params:
            p['shape'] = (side, side)
        pixels = I.PackedImages(arrays).marshal(params, side, side)
        base[side] = I.augment_batch(pixels, (side, side), params, filter=batcher.filter)
    return [torch.flip(base[side], dims=[3]) if flip else base[side] for side, flip in passes]


def tta_capacity(m, passes):
    """Candidates per merged row of a plan: the sum of the passes' A * (side/32)^2."""
    return sum(int(m.num_anchors) * (side // 32) ** 2 for side, _ in passes)


def detect_tta_pass(m, merged, data, dynamic_weights, n_cls, side, flip, conf_thresh=CONF_THRESH, anchors_dev=None):
    """One pass of a plan: detect_forward, the decode of detect(), and fsdet_tta_merge into `merged`."""
    with torch.no_grad():
        output = m.detect_forward(data, dynamic_weights)
    if tuple(output.shape[2:]) != (side // 32, side // 32):
        raise ValueError('pass (%d, %d): head grid %s, expected %d x %d' % (side, flip, tuple(output.shape[2:]),
                                                                           side // 32, side // 32))
    dets = region_detections(output, conf_thresh, m.num_classes, m.anchors, m.num_anchors, 0, 1, n_models=n_cls,
                             anchors_dev=anchors_dev)
    return merged.add_pass(dets, side, flip)


def detect_tta(m, batch, dynamic_weights, n_cls, passes, conf_thresh=CONF_THRESH, nms_thresh=NMS_THRESH):
    """detect() under a test-time augmentation plan: `batch` holds the input of every pass (tta_inputs), each run
    through detect_forward with the same vectors and decoded as detect() decodes; the candidates are merged per
    (image, class) row in pass order (flipped passes mirrored back) and suppressed by one NMS (fsdet_nms_merged).
    Returns utils.MergedDetections (device resident).  For the plan [(m.width, 0)] every consumer writes what it
    writes for detect()."""
    passes = check_tta_passes(passes)
    batch = list(batch)
    if len(batch) != len(passes):
        raise ValueError('%d inputs for %d passes' % (len(batch), len(passes)))
    merged = None
    for (side, flip), data in zip(passes, batch):
        if tuple(data.shape[2:]) != (side, side):
            raise ValueError('pass (%d, %d) got an input of %s' % (side, flip, tuple(data.shape)))
        if merged is None:
            merged = MergedDetections(data.size(0) * n_cls, tta_capacity(m, passes), data.device)
        detect_tta_pass(m, merged, data, dynamic_weights, n_cls, side, flip, conf_thresh)
    return merged.nms(nms_thresh)


def detect_images(m, data, dynamic_weights, n_cls, sizes, conf_thresh=DETECT_CONF_THRESH, nms_thresh=DETECT_NMS_THRESH,
                  max_det=MAX_DET):
    """The boxes of every image of a batch: detect, then Detections.select.  sizes[b] = (width, height) of image b
    (or an int32 [B, 2] device tensor).  Returns utils.ImageDetections, on the device: per image the first max_det
    boxes over all classes, by prob descending, in pixels; `.lists(class_names)` brings them to the host.  The
    thresholds default to those of the reference's single-image detection (do_detect: conf 0.5, NMS 0.4)."""
    return detect(m, data, dynamic_weights, n_cls, conf_thresh, nms_thresh).select(n_cls, sizes, max_det)


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
    """Append the batch's lines to the per-class files `fps[i]` (valid_ensemble.py:128-131, :178).  dets: Detections,
    or the MergedDetections of detect_tta."""
    lines = detection_lines(dets, imgids, sizes, n_cls, nms_thresh)
    for i in range(n_cls):
        fps[i].writelines(lines[i])


def valid_batches(m, meta_batches, image_batches, class_names, prefix, outfile, base_rw=None, base_rows=None,
                  save_rw=None, tta=None):
    """The body of valid_ensemble.valid() (:86-181) over iterables: `meta_batches` as in ensemble_dynamic_weights,
    `image_batches` yields (data [b,3,H,W], imgids, sizes).  Writes `<prefix>/<outfile><class>.txt`.
    base_rw, base_rows, save_rw: the stored-vector mode and the vectors file, as in evaluation_dynamic_weights.
    tta: a test-time augmentation plan; `data` is then the list of the passes' inputs (tta_inputs)."""
    n_cls = len(class_names)
    m.eval()
    dynamic_weights = evaluation_dynamic_weights(m, meta_batches, n_cls, base_rw=base_rw, base_rows=base_rows,
                                                 save_rw=save_rw)
    if not os.path.exists(prefix):
        os.makedirs(prefix)
    fps = [open('%s/%s%s.txt' % (prefix, outfile, name), 'w') for name in class_names]
    try:
        dev = next(m.parameters()).device
        for data, imgids, sizes in image_batches:
            write_detections(fps, _detect_batch(m, data, dev, dynamic_weights, n_cls, tta), imgids, sizes, n_cls)
    finally:
        for fp in fps:
            fp.close()
    return dynamic_weights


def _detect_batch(m, data, dev, dynamic_weights, n_cls, tta):
    """detect() of one batch, or detect_tta() of its passes' inputs under the plan `tta`."""
    if tta is None:
        return detect(m, data.to(dev), dynamic_weights, n_cls)
    return detect_tta(m, [d.to(dev) for d in data], dynamic_weights, n_cls, tta)


def score_batches(m, support_batches, image_batches, evaluator, out=None, sharded=False, process_group=None, dst=0,
                  base_rw=None, base_rows=None, save_rw=None, tta=None, **result_kwargs):
    """valid_batches scored on the device: `evaluator` is a voc_eval.DeviceVocEval or coco_eval.DeviceCocoEval over
    the evaluated image set, `support_batches` are as ensemble_dynamic_weights' meta_batches, `image_batches` yields
    (data, imgids, sizes) with imgids names of that set.  Returns evaluator.result(**result_kwargs): mean_ap's dict
    (use_07_metric=, novel_classes=, curves=) or coco_evaluate's (novel_classes=).

    out (optional) also receives the result files of the same detections, copied to the host for them: for VOC the
    per-class files valid_batches writes (a list of open files), for COCO the standard results json (an open file).

    sharded=True: collective over `process_group`, each rank running its own block of the single-process support and
    query batches (shard.shard_range).  The pools are merged in rank order and scored once on rank `dst`; every rank
    returns the single-process dict.  `out` is open on `dst` and True on the other ranks, whose parts go to `dst`,
    which writes every rank's in rank order: the single-process files.  None on every rank for no files.

    base_rw, base_rows, save_rw: the stored-vector mode and the vectors file, as in evaluation_dynamic_weights (the
    file is written on `dst` when sharded).

    tta: a test-time augmentation plan (detect_tta); `data` is then the list of the passes' inputs (tta_inputs).  The
    merged detections go to the same pools, so a sharded evaluation merges them as it merges single-pass ones."""
    n_cls = len(evaluator.classes)
    m.eval()
    dynamic_weights = evaluation_dynamic_weights(m, support_batches, n_cls, sharded, process_group, dst, base_rw,
                                                 base_rows, save_rw)
    dev = next(m.parameters()).device
    parts = []
    for data, imgids, sizes in image_batches:
        dets = _detect_batch(m, data, dev, dynamic_weights, n_cls, tta)
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
