"""Small host helpers of the reference's utils.py that the training driver uses."""
import struct
import time


def read_data_cfg(datacfg):
    """`.data` file -> dict (utils.py:460-475), same defaults."""
    options = dict()
    options['gpus'] = '0,1,2,3'
    options['num_workers'] = '10'
    with open(datacfg, 'r') as fp:
        for line in fp.readlines():
            line = line.strip()
            if line == '':
                continue
            key, value = line.split('=')
            options[key.strip()] = value.strip()
    return options


def logging(message):
    print('%s %s' % (time.strftime("%Y-%m-%d %H:%M:%S", time.localtime()), message))


def load_class_names(namesfile):
    """utils.py:392-399: one class name per line, trailing whitespace stripped (blank lines included)."""
    with open(namesfile, 'r') as fp:
        return [line.rstrip() for line in fp.readlines()]


def _image_type(head):
    """The type `imghdr.what` reports for the first bytes of a file, for the types get_image_size reads."""
    if head[:8] == b'\x89PNG\r\n\x1a\n':
        return 'png'
    if head[:6] in (b'GIF87a', b'GIF89a'):
        return 'gif'
    if head[6:10] in (b'JFIF', b'Exif') or head[:4] == b'\xff\xd8\xff\xdb':
        return 'jpeg'
    return None


def get_image_size(fname):
    """utils.py:536-569: (width, height) from the header of a PNG, GIF or JPEG file, without decoding it; None for
    any other file, a file shorter than 24 bytes or a JPEG without a frame header."""
    with open(fname, 'rb') as fhandle:
        head = fhandle.read(24)
        if len(head) != 24:
            return None
        kind = _image_type(head)
        if kind == 'png':
            if struct.unpack('>i', head[4:8])[0] != 0x0d0a1a0a:
                return None
            width, height = struct.unpack('>ii', head[16:24])
        elif kind == 'gif':
            width, height = struct.unpack('<HH', head[6:10])
        elif kind == 'jpeg':
            try:
                fhandle.seek(0)                     # walk the segments up to the first SOFn marker
                size, ftype = 2, 0
                while not 0xc0 <= ftype <= 0xcf:
                    fhandle.seek(size, 1)
                    byte = fhandle.read(1)
                    while ord(byte) == 0xff:
                        byte = fhandle.read(1)
                    ftype = ord(byte)
                    size = struct.unpack('>H', fhandle.read(2))[0] - 2
                fhandle.seek(1, 1)                  # the sample precision byte
                height, width = struct.unpack('>HH', fhandle.read(4))
            except Exception:
                return None
        else:
            return None
        return width, height


# --------------------------------------------------------------------------------------------------------------------
# Detection decode + NMS (evaluation; SURVEY.md 8f row 1).  Same names, arguments and return values as the reference's
# utils.py; the tensor prologue, the confidence filter and the O(n^2) suppression loops run in libfsdet.so
# (csrc/detect.cu) for ALL rows of the batch at once.  CUDA only: there is no host fallback.
def bbox_iou(box1, box2, x1y1x2y2=True):
    """utils.py:21-52 on Python floats (host helper, e.g. for train_meta.test()'s recall count)."""
    if x1y1x2y2:
        mx, Mx = min(box1[0], box2[0]), max(box1[2], box2[2])
        my, My = min(box1[1], box2[1]), max(box1[3], box2[3])
        w1, h1, w2, h2 = box1[2] - box1[0], box1[3] - box1[1], box2[2] - box2[0], box2[3] - box2[1]
    else:
        mx = min(box1[0] - box1[2] / 2.0, box2[0] - box2[2] / 2.0)
        Mx = max(box1[0] + box1[2] / 2.0, box2[0] + box2[2] / 2.0)
        my = min(box1[1] - box1[3] / 2.0, box2[1] - box2[3] / 2.0)
        My = max(box1[1] + box1[3] / 2.0, box2[1] + box2[3] / 2.0)
        w1, h1, w2, h2 = box1[2], box1[3], box2[2], box2[3]
    cw = w1 + w2 - (Mx - mx)
    ch = h1 + h2 - (My - my)
    if cw <= 0 or ch <= 0:
        return 0.0
    carea = cw * ch
    return carea / (w1 * h1 + w2 * h2 - carea)


def _stream():
    import torch
    return torch.cuda.current_stream().cuda_stream


class Detections(object):
    """Device-resident result of the decode (+ NMS) of one head output.

    cand   float32 [N, A*H*W, 8]: per row the candidates above the confidence threshold in the reference's loop order,
           {xs, ys, ws, hs (grid units), det_conf, cls_max_conf, int32 cls_max_id, int32 a*H*W+cell}
    count  int32 [N]
    keep / keep_count (after `.nms(thresh)`): candidate slots of the NMS survivors per row, best first.
    Nothing is copied to the host until `.boxes()` / `.kept_boxes()` / `.lines()` is called."""

    def __init__(self, cand, count, cls_dense, N, A, nC, H, W, only_objectness, validation, conf_thresh):
        self.cand, self.count, self.cls_dense = cand, count, cls_dense
        self.N, self.A, self.nC, self.H, self.W = N, A, nC, H, W
        self.only_objectness, self.validation, self.conf_thresh = only_objectness, validation, conf_thresh
        self.keep = self.keep_count = None
        self._nms_thresh = None
        self._host = None
        self._rows = None

    # ---- device side
    def nms(self, nms_thresh):
        """utils.nms (utils.py:85-104) for every row in one launch.  Returns self."""
        import torch
        from ._lib import call, ptr
        if self._nms_thresh != nms_thresh:
            cap = self.A * self.H * self.W
            self.keep = torch.empty(self.N, cap, dtype=torch.int32, device=self.cand.device)
            self.keep_count = torch.zeros(self.N, dtype=torch.int32, device=self.cand.device)
            call('fsdet_nms', ptr(self.cand), ptr(self.count), self.N, cap, self.H, self.W, float(nms_thresh),
                 ptr(self.keep), ptr(self.keep_count), _stream())
            self._nms_thresh = nms_thresh
            self._kept_host = None
        return self

    # ---- host side (one D2H copy each)
    def _fetch(self):
        if self._host is None:
            count = self.count.cpu().numpy()
            mx = int(count.max()) if self.N else 0
            cand = self.cand[:, :mx].cpu().numpy()
            dense = self.cls_dense.cpu().numpy() if (self.cls_dense is not None and self.validation
                                                     and not self.only_objectness and self.nC > 1) else None
            self._host = (count, cand, dense)
        return self._host

    def _box(self, n, slot, cand, dense):
        """One box in the reference's list form (utils.py:175-181 / :270-276), Python floats."""
        import numpy as np
        v = cand[n, slot]
        ints = v[6:8].view(np.int32)
        det, cid = float(v[4]), int(ints[0])
        box = [float(v[0]) / self.W, float(v[1]) / self.H, float(v[2]) / self.W, float(v[3]) / self.H, det, float(v[5]), cid]
        if dense is not None:
            row = dense[n * self.A * self.H * self.W + int(ints[1])]
            for c in range(self.nC):
                tmp = float(row[c])
                if c != cid and det * tmp > self.conf_thresh:
                    box.append(tmp)
                    box.append(c)
        return box

    def boxes(self):
        """all_boxes of get_region_boxes(_v2): list (rows) of lists (boxes) of Python numbers."""
        if self._rows is None:
            count, cand, dense = self._fetch()
            self._rows = [_Row([self._box(n, s, cand, dense) for s in range(int(count[n]))], self, n)
                          for n in range(self.N)]
        return self._rows

    def kept_boxes(self, nms_thresh):
        """[nms(row, nms_thresh) for row in boxes()] without building the un-kept boxes' lists."""
        self.nms(nms_thresh)
        count, cand, dense = self._fetch()
        kc = self.keep_count.cpu().numpy()
        mx = int(kc.max()) if self.N else 0
        keep = self.keep[:, :mx].cpu().numpy()
        return [[self._box(n, int(keep[n, i]), cand, dense) for i in range(int(kc[n]))] for n in range(self.N)]

    def _nms_row(self, index, row, nms_thresh):
        """Reference semantics for one row of boxes(): survivors returned best first (the same list objects),
        suppressed boxes get box[4] = 0 in place."""
        self.nms(nms_thresh)
        if getattr(self, '_kept_host', None) is None:
            self._kept_host = (self.keep_count.cpu().numpy(), self.keep.cpu().numpy())
        kc, keep = self._kept_host
        slots = [int(s) for s in keep[index, :int(kc[index])]]
        alive = set(slots)
        for s, box in enumerate(row):
            if s not in alive:
                box[4] = 0
        return [row[s] for s in slots]

    # ---- per-image result (meta detector)
    def select(self, n_cls, sizes, max_det=100, out=None):
        """The first `max_det` NMS survivors of every image, over all its class rows, ordered by prob = det_conf *
        cls_conf descending, then class, then NMS rank, with the boxes in pixels (fsdet_detect_select): an
        ImageDetections, still on the device, of fixed shape.  Rows are (image, class) pairs, image-major, as
        get_region_boxes_v2 makes them; `.nms()` must have run.  sizes: (width, height) per image, a sequence or an
        int32 [B, 2] tensor on the device.  out (optional): an ImageDetections of the same B and max_det to write into
        (a CUDA graph's static result)."""
        import torch
        from ._lib import call, lib, ptr
        if self.keep is None:
            raise ValueError('select needs the NMS survivors: call .nms(thresh) first')
        if self.nC != 1:
            raise ValueError('select takes the meta detector\'s rows (one class channel per row), not nC = %d' % self.nC)
        dev = self.cand.device
        n_cls, max_det, sizes, out = _select_args(self, n_cls, sizes, max_det, out, dev)
        cap = self.A * self.H * self.W
        ws_bytes = int(lib.fsdet_detect_select_workspace_bytes(self.N, cap))
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        call('fsdet_detect_select', ptr(self.cand), ptr(self.keep), ptr(self.keep_count), self.N, cap, self.H, self.W,
             n_cls, ptr(sizes), max_det, ptr(ws), ws_bytes, ptr(out.score), ptr(out.box), ptr(out.cls), ptr(out.count),
             ptr(out.total), _stream())
        return out


def _select_args(dets, n_cls, sizes, max_det, out, dev):
    """The checked arguments of Detections.select / MergedDetections.select: n_cls, max_det, the int32 [B, 2] sizes on
    the device and the ImageDetections to write."""
    import torch
    if dets.keep is None:
        raise ValueError('select needs the NMS survivors: call .nms(thresh) first')
    n_cls, max_det = int(n_cls), int(max_det)
    if n_cls <= 0 or dets.N % n_cls or dets.N == 0:
        raise ValueError('%d rows are not images x %d classes' % (dets.N, n_cls))
    if max_det <= 0:
        raise ValueError('max_det must be positive, got %d' % max_det)
    B = dets.N // n_cls
    if not torch.is_tensor(sizes):
        sizes = torch.tensor([[int(w), int(h)] for w, h in sizes], dtype=torch.int32).to(dev)
    if tuple(sizes.shape) != (B, 2) or sizes.dtype != torch.int32 or sizes.device != dev:
        raise ValueError('sizes must be int32 [%d, 2] on %s, got %s %s on %s'
                         % (B, dev, sizes.dtype, tuple(sizes.shape), sizes.device))
    if out is None:
        out = ImageDetections.empty(B, max_det, dev)
    elif (out.B, out.max_det) != (B, max_det):
        raise ValueError('out holds %d x %d results, the batch needs %d x %d' % (out.B, out.max_det, B, max_det))
    return n_cls, max_det, sizes.contiguous(), out


# --------------------------------------------------------------------------------------------------------------------
# Test-time augmentation (valid.detect_tta): the candidates of several passes over the same images (other sides,
# mirrored) in one table per (image, class) row, suppressed together.
TTA_RECORD_BYTES = 48
NMS_MERGED_MAX_CAP = 65536       # candidates per merged row fsdet_nms_merged accepts


def tta_record_dtype():
    """numpy dtype of one merged record (include/fsdet.h): the normalised float64 box (x mirrored for a flipped pass),
    float32 det_conf and cls_conf, the class id and src = pass << 20 | the pass's candidate slot."""
    import numpy as np
    return np.dtype([('x', '<f8'), ('y', '<f8'), ('w', '<f8'), ('h', '<f8'), ('det', '<f4'), ('cls', '<f4'),
                     ('cid', '<i4'), ('src', '<i4')])


class MergedDetections(object):
    """Device-resident candidates of a test-time augmentation plan, merged per row (fsdet_tta_merge).

    merged    uint8 [N, cap, 48]: per row the candidates of every pass added, pass order then candidate order, as
              records of tta_record_dtype()
    count     int32 [N]
    overflow  int32 [1]: set when a pass did not fit a row's capacity (that pass is then missing from the row)
    keep / keep_count (after `.nms(thresh)`): merged slots of the NMS survivors per row, best first.
    Rows are (image, class) pairs of the meta detector (nC = 1).  `passes` lists the (side, flip) of every pass added.
    Nothing is copied to the host until `.kept_boxes()` / `.records()` / `.overflowed()` is called."""
    nC = 1

    def __init__(self, N, cap, device):
        import torch
        if not 0 < cap <= NMS_MERGED_MAX_CAP:
            raise ValueError('%d candidates per merged row (1..%d)' % (cap, NMS_MERGED_MAX_CAP))
        self.N, self.cap = int(N), int(cap)
        self.merged = torch.empty(self.N, self.cap, TTA_RECORD_BYTES, dtype=torch.uint8, device=device)
        self.count = torch.zeros(self.N, dtype=torch.int32, device=device)
        self.overflow = torch.zeros(1, dtype=torch.int32, device=device)
        self.passes = []
        self.keep = self.keep_count = None
        self._nms_thresh = None

    @property
    def device(self):
        return self.merged.device

    def add_pass(self, dets, side, flip):
        """Append the candidates of one pass (utils.Detections of the meta detector, before or after its own NMS) to
        every row; flip: the pass's input was mirrored left-right, so its boxes are mirrored back (x = 1 - x)."""
        from ._lib import call, ptr
        if dets.N != self.N or dets.nC != 1:
            raise ValueError('a pass of %d rows x nC = %d, the table holds %d rows x nC = 1' % (dets.N, dets.nC, self.N))
        call('fsdet_tta_merge', ptr(dets.cand), ptr(dets.count), dets.N, dets.A * dets.H * dets.W, dets.H, dets.W,
             int(bool(flip)), len(self.passes), ptr(self.merged), ptr(self.count), self.cap, ptr(self.overflow),
             _stream())
        self.passes.append((int(side), int(bool(flip))))
        self.keep = self.keep_count = None
        self._nms_thresh = None
        return self

    def nms(self, nms_thresh):
        """utils.nms over every merged row (fsdet_nms_merged).  Returns self."""
        import torch
        from ._lib import call, lib, ptr
        if self._nms_thresh != nms_thresh:
            ws_bytes = int(lib.fsdet_nms_merged_workspace_bytes(self.N, self.cap))
            ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=self.device)
            self.keep = torch.empty(self.N, self.cap, dtype=torch.int32, device=self.device)
            self.keep_count = torch.zeros(self.N, dtype=torch.int32, device=self.device)
            call('fsdet_nms_merged', ptr(self.merged), ptr(self.count), self.N, self.cap, float(nms_thresh), ptr(ws),
                 ws_bytes, ptr(self.keep), ptr(self.keep_count), _stream())
            self._nms_thresh = nms_thresh
        return self

    def overflowed(self):
        """Whether a pass did not fit (one 4-byte device-to-host copy)."""
        return bool(int(self.overflow.item()))

    def _check(self):
        if self.overflowed():
            raise RuntimeError('merged detections overflow: a pass did not fit %d candidates per row' % self.cap)

    def records(self):
        """(count int32 [N], numpy records [N, max count] of tta_record_dtype()), one device-to-host copy."""
        self._check()
        count = self.count.cpu().numpy()
        mx = int(count.max()) if self.N else 0
        host = self.merged[:, :mx].cpu().numpy()
        return count, host.reshape(self.N * mx * TTA_RECORD_BYTES).view(tta_record_dtype()).reshape(self.N, mx)

    def kept_boxes(self, nms_thresh):
        """Per row the survivors in the reference's box-list form [x, y, w, h, det_conf, cls_conf, cls_id] (Python
        floats), best first: what Detections.kept_boxes gives for one pass, so valid.detection_lines and
        coco_eval.detection_records print merged rows unchanged."""
        self.nms(nms_thresh)
        _, rec = self.records()
        kc = self.keep_count.cpu().numpy()
        mx = int(kc.max()) if self.N else 0
        keep = self.keep[:, :mx].cpu().numpy()
        out = []
        for n in range(self.N):
            row = []
            for i in range(int(kc[n])):
                q = rec[n, int(keep[n, i])]
                row.append([float(q['x']), float(q['y']), float(q['w']), float(q['h']), float(q['det']), float(q['cls']),
                            int(q['cid'])])
            out.append(row)
        return out

    def select(self, n_cls, sizes, max_det=100, out=None):
        """Detections.select on the merged rows (fsdet_detect_select_merged): per image the first max_det survivors
        over all its class rows, by prob descending, then class, then NMS rank, in pixels."""
        import torch
        from ._lib import call, lib, ptr
        n_cls, max_det, sizes, out = _select_args(self, n_cls, sizes, max_det, out, self.device)
        ws_bytes = int(lib.fsdet_detect_select_workspace_bytes(self.N, self.cap))
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=self.device)
        call('fsdet_detect_select_merged', ptr(self.merged), ptr(self.keep), ptr(self.keep_count), self.N, self.cap,
             n_cls, ptr(sizes), max_det, ptr(ws), ws_bytes, ptr(out.score), ptr(out.box), ptr(out.cls), ptr(out.count),
             ptr(out.total), _stream())
        return out


class ImageDetections(object):
    """Per-image detections of a batch (Detections.select), device resident, fixed shape:
    score float64 [B, max_det], box float64 [B, max_det, 4] (x1, y1, x2, y2 in pixels), cls int32 [B, max_det],
    count int32 [B] (valid slots, best first), total int32 [B] (NMS survivors before the max_det cap).
    Slots past count hold score 0, box 0, class -1.  All five are views of one device buffer, so `.lists()` costs
    one device-to-host copy.  `n_images` <= B: the images that are results (a padded batch's real images)."""

    def __init__(self, buf, B, max_det, n_images=None):
        self.buf, self.B, self.max_det = buf, B, max_det
        self.n_images = B if n_images is None else n_images
        self.score, self.box, self.cls, self.count, self.total = self._views(buf, B, max_det)

    @staticmethod
    def _bytes(B, max_det):
        return B * max_det * 5 * 8 + B * max_det * 4 + 2 * B * 4

    @staticmethod
    def _views(buf, B, max_det):
        import torch
        K = B * max_det
        f64 = buf[:K * 40].view(torch.float64) if torch.is_tensor(buf) else buf[:K * 40].view('<f8')
        i32 = buf[K * 40:].view(torch.int32) if torch.is_tensor(buf) else buf[K * 40:].view('<i4')
        return (f64[:K].reshape(B, max_det), f64[K:].reshape(B, max_det, 4), i32[:K].reshape(B, max_det),
                i32[K:K + B], i32[K + B:K + 2 * B])

    @classmethod
    def empty(cls, B, max_det, device):
        import torch
        return cls(torch.empty(cls._bytes(B, max_det), dtype=torch.uint8, device=device), B, max_det)

    def narrow(self, n_images):
        """The same buffer with only the first n_images images as results."""
        return ImageDetections(self.buf, self.B, self.max_det, n_images)

    def host(self):
        """numpy (score, box, cls, count, total) of the result images, one device-to-host copy."""
        score, box, cls, count, total = self._views(self.buf.cpu().numpy(), self.B, self.max_det)
        n = self.n_images
        return score[:n], box[:n], cls[:n], count[:n], total[:n]

    def lists(self, class_names=None):
        """One list per image of (name, prob, x1, y1, x2, y2), best first; the class index instead of the name when
        class_names is None."""
        score, box, cls, count, _ = self.host()
        out = []
        for b in range(self.n_images):
            rows = []
            for k in range(int(count[b])):
                c = int(cls[b, k])
                x1, y1, x2, y2 = (float(v) for v in box[b, k])
                rows.append((class_names[c] if class_names is not None else c, float(score[b, k]), x1, y1, x2, y2))
            out.append(rows)
        return out


class _Row(list):
    """A row of get_region_boxes(_v2)'s result that remembers where it came from, so that `nms(row, t)` can use
    the batched device NMS instead of re-uploading the boxes."""

    def __init__(self, boxes, parent, index):
        super(_Row, self).__init__(boxes)
        self._parent, self._index, self._n0 = parent, index, len(boxes)
        self._sig = [b[4] for b in boxes]

    def _pristine(self):
        return len(self) == self._n0 and all(b[4] == s for b, s in zip(self, self._sig))


def _detect(output, n_models, v2, conf_thresh, num_classes, anchors, num_anchors, only_objectness, validation,
            anchors_dev=None):
    import torch
    from ._lib import call, ptr
    if not torch.is_tensor(output) or not output.is_cuda:
        raise TypeError('get_region_boxes runs on the GPU only; `output` must be a CUDA tensor (no CPU fallback)')
    if output.dim() == 3:
        output = output.unsqueeze(0)
    output = output.detach().float().contiguous()
    N, ch, H, W = output.shape
    A, nC = int(num_anchors), int(num_classes)
    assert ch == (5 + nC) * A
    assert len(anchors) // A == 2, 'anchor_step must be 2'
    if v2:
        assert N % n_models == 0
    dev = output.device
    cap = A * H * W
    cand = torch.empty(N, cap, 8, dtype=torch.float32, device=dev)
    count = torch.zeros(N, dtype=torch.int32, device=dev)
    want_dense = bool(validation) and not only_objectness and nC > 1
    dense = torch.empty(N * cap, nC, dtype=torch.float32, device=dev) if want_dense else None
    if anchors_dev is None:
        anc = torch.tensor([float(a) for a in anchors], dtype=torch.float32).to(dev)
    else:                                             # staged by the caller: no host-to-device copy here
        anc = anchors_dev
        assert anc.dtype == torch.float32 and anc.device == dev and anc.numel() == len(anchors) and anc.is_contiguous()
    call('fsdet_region_detect', ptr(output), ptr(anc), N, A, nC, H, W, int(n_models), int(v2), int(bool(only_objectness)),
         float(conf_thresh), ptr(cand), ptr(count), ptr(dense), _stream())
    return Detections(cand, count, dense, N, A, nC, H, W, bool(only_objectness), bool(validation), float(conf_thresh))


def region_detections(output, conf_thresh, num_classes, anchors, num_anchors, only_objectness=1, validation=False,
                      n_models=None, anchors_dev=None):
    """Device-resident form of get_region_boxes (n_models=None) / get_region_boxes_v2: returns `Detections`.
    anchors_dev (optional): the anchors as a float32 device tensor, staged once by a caller that captures the decode
    in a CUDA graph (otherwise they are uploaded from the host on every call)."""
    if n_models is None:
        return _detect(output, 1, 0, conf_thresh, num_classes, anchors, num_anchors, only_objectness, validation,
                       anchors_dev)
    return _detect(output, n_models, 1, conf_thresh, num_classes, anchors, num_anchors, only_objectness, validation,
                   anchors_dev)


def get_region_boxes(output, conf_thresh, num_classes, anchors, num_anchors, only_objectness=1, validation=False):
    """utils.py:112-193: list (images) of lists of [x, y, w, h, det_conf, cls_max_conf, cls_max_id(, conf, id)*]."""
    return region_detections(output, conf_thresh, num_classes, anchors, num_anchors, only_objectness, validation).boxes()


def get_region_boxes_v2(output, n_models, conf_thresh, num_classes, anchors, num_anchors, only_objectness=1,
                        validation=False):
    """utils.py:195-290: rows are (image, class) pairs, image-major (`oi = b * n_cls + i`, valid_ensemble.py:158)."""
    return region_detections(output, conf_thresh, num_classes, anchors, num_anchors, only_objectness, validation,
                             n_models=n_models).boxes()


def nms(boxes, nms_thresh):
    """utils.py:85-104.  A row of get_region_boxes(_v2) uses the batched device NMS of its batch (computed once for
    all rows); any other list of boxes is uploaded as float64 and suppressed by the same kernel."""
    if len(boxes) == 0:
        return boxes
    if isinstance(boxes, _Row) and boxes._pristine():
        return boxes._parent._nms_row(boxes._index, boxes, nms_thresh)
    import numpy as np
    import torch
    from ._lib import call, ptr
    if not torch.cuda.is_available():
        raise RuntimeError('nms runs on the GPU only (no CPU fallback)')
    n = len(boxes)
    if n > 4096:
        raise ValueError('nms: %d boxes in one row (max 4096)' % n)
    host = np.array([[float(b[0]), float(b[1]), float(b[2]), float(b[3]), float(b[4])] for b in boxes], dtype=np.float64)
    dev = torch.device('cuda', torch.cuda.current_device())
    b64 = torch.from_numpy(host).to(dev)
    count = torch.tensor([n], dtype=torch.int32, device=dev)
    keep = torch.empty(1, n, dtype=torch.int32, device=dev)
    kc = torch.zeros(1, dtype=torch.int32, device=dev)
    call('fsdet_nms_boxes64', ptr(b64), ptr(count), 1, n, float(nms_thresh), ptr(keep), ptr(kc), _stream())
    slots = keep[0, :int(kc.item())].tolist()
    alive = set(slots)
    for s, box in enumerate(boxes):
        if s not in alive:
            box[4] = 0
    return [boxes[s] for s in slots]
