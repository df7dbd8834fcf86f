"""fsdet_detect_select (csrc/detect.cu) without a GPU: the kernel source compiled by g++ against
tools/host_emul/cuda_host_emul.h, on seeded candidate tables, bit for bit against the Python reference below.

The reference is built from utils.Detections.kept_boxes with valid.detection_lines' formulas: every NMS survivor of an
image's class rows, ordered by prob = det_conf * cls_conf descending, then class, then NMS rank, cut to max_det."""
import ctypes

import numpy as np
import pytest
import torch

from emul_util import build_emul


def P(a):
    return a.ctypes.data_as(ctypes.c_void_p) if a is not None else None


@pytest.fixture(scope='module')
def emul():
    return build_emul('detect', 'detect.cu')


def reference_select(dets, n_cls, sizes, max_det):
    """Per image: (total, [(class, prob, x1, y1, x2, y2)] of the first max_det), from Detections.kept_boxes."""
    kept = dets.kept_boxes(dets._nms_thresh)
    out = []
    for b in range(dets.N // n_cls):
        width, height = sizes[b]
        recs = []
        for i in range(n_cls):
            for rank, box in enumerate(kept[b * n_cls + i]):
                x1 = (box[0] - box[2] / 2.0) * width
                y1 = (box[1] - box[3] / 2.0) * height
                x2 = (box[0] + box[2] / 2.0) * width
                y2 = (box[1] + box[3] / 2.0) * height
                prob = box[4] * box[5]
                recs.append(((-prob, i, rank), (i, prob, x1, y1, x2, y2)))
        recs.sort(key=lambda r: r[0])
        out.append((len(recs), [r[1] for r in recs[:max_det]]))
    return out


def assert_select_equals(got, want, max_det):
    """got: numpy (score, box, cls, count, total) of fsdet_detect_select; want: reference_select.  Bit for bit."""
    score, box, cls, count, total = got
    assert len(count) == len(want)
    for b, (tot, rows) in enumerate(want):
        assert int(total[b]) == tot and int(count[b]) == len(rows) == min(tot, max_det)
        for k, (c, prob, x1, y1, x2, y2) in enumerate(rows):
            assert int(cls[b, k]) == c, (b, k)
            assert score[b, k] == prob and score[b, k].tobytes() == np.float64(prob).tobytes(), (b, k)
            assert box[b, k].tobytes() == np.array([x1, y1, x2, y2], np.float64).tobytes(), (b, k)
        assert (score[b, len(rows):] == 0).all() and (box[b, len(rows):] == 0).all() and (cls[b, len(rows):] == -1).all()


def synthetic_table(seed, B, n_cls, cap, kept, ties=False):
    """cand [N, cap, 8] / keep / keep_count with kept[b][i] survivors in row (b, i), each a distinct candidate slot.
    ties: det_conf and cls_conf from a few binary fractions, so equal probs occur within and across classes (some
    from different factors: 0.5 * 0.25 == 0.25 * 0.5)."""
    rs = np.random.RandomState(seed)
    N = B * n_cls
    cand = np.zeros((N, cap, 8), dtype=np.float32)
    count = np.zeros(N, dtype=np.int32)
    keep = np.full((N, cap), -1, dtype=np.int32)
    kc = np.zeros(N, dtype=np.int32)
    for n in range(N):
        k = kept[n // n_cls][n % n_cls]
        cnt = min(cap, k + rs.randint(0, 4))
        count[n] = cnt
        cand[n, :cnt, 0:2] = rs.uniform(0, 13, (cnt, 2))
        cand[n, :cnt, 2:4] = rs.uniform(0.05, 6, (cnt, 2))
        if ties:
            cand[n, :cnt, 4] = rs.choice([0.5, 0.25, 0.75, 0.125], cnt)
            cand[n, :cnt, 5] = rs.choice([0.5, 0.25, 1.0], cnt)
        else:
            cand[n, :cnt, 4] = rs.uniform(0.01, 1, cnt)
            cand[n, :cnt, 5] = rs.uniform(0.01, 1, cnt)
        cand[n, :cnt, 6:8] = np.zeros((cnt, 2), np.int32).view(np.float32)
        keep[n, :k] = rs.permutation(cnt)[:k]
        kc[n] = k
    return cand, count, keep, kc


def run_select(emul, cand, keep, kc, n_cls, H, W, sizes, max_det):
    N, cap, _ = cand.shape
    B = N // n_cls
    emul.emul_detect_select_workspace_bytes.restype = ctypes.c_size_t
    nbytes = emul.emul_detect_select_workspace_bytes(N, cap)
    ws = np.zeros(nbytes + 256, dtype=np.uint8)
    base = (ws.ctypes.data + 255) // 256 * 256
    score = np.full((B, max_det), np.nan)
    box = np.full((B, max_det, 4), np.nan)
    cls = np.full((B, max_det), 7, dtype=np.int32)
    count = np.full(B, -9, dtype=np.int32)
    total = np.full(B, -9, dtype=np.int32)
    sz = np.ascontiguousarray(np.array(sizes, dtype=np.int32).reshape(B, 2))
    rc = emul.emul_detect_select(P(cand), P(keep), P(kc), N, cap, H, W, n_cls, P(sz), max_det, ctypes.c_void_p(base),
                                 P(score), P(box), P(cls), P(count), P(total))
    assert rc == 0
    return score, box, cls, count, total


def detections(cand, count, keep, kc, H, W):
    from fewshot_detection_b200 import utils as U
    N, cap, _ = cand.shape
    d = U.Detections(torch.from_numpy(cand), torch.from_numpy(count), None, N, cap // (H * W), 1, H, W, False, True, 0.0)
    d.keep, d.keep_count, d._nms_thresh, d._kept_host = torch.from_numpy(keep), torch.from_numpy(kc), 0.45, None
    return d


H = W = 13
CAP = 5 * H * W          # 845: the meta detector's candidates per row at 416


@pytest.mark.parametrize('name,B,n_cls,kept,max_det,ties', [
    # image 1 has no survivor, rows 0 and 2 of image 0 are empty; totals 5 < max_det and 0
    ('empty', 3, 4, [[0, 3, 0, 2], [0, 0, 0, 0], [1, 0, 0, 0]], 10, False),
    # totals below (9), at (12) and above (30) max_det = 12
    ('below-at-above', 3, 3, [[3, 3, 3], [4, 4, 4], [10, 10, 10]], 12, False),
    # 3 x 845 = 2535 survivors in image 0: more than one block (256 threads) and one radix tile (2048 items) hold
    ('many', 2, 3, [[CAP, CAP, CAP], [700, 0, 5]], 100, False),
    # equal probs within a class and across classes: class, then NMS rank decide
    ('ties', 2, 5, [[40, 40, 40, 40, 40], [7, 0, 30, 1, 12]], 60, True),
    # max_det = 1
    ('max-det-1', 4, 2, [[5, 5], [0, 1], [0, 0], [2, 9]], 1, True),
    # one image of one class (no image pass in the sort)
    ('one-image', 1, 1, [[300]], 50, True),
])
def test_emulated_select_equals_reference(emul, name, B, n_cls, kept, max_det, ties):
    cand, count, keep, kc = synthetic_table(len(name) * 7 + B, B, n_cls, CAP, kept, ties)
    rs = np.random.RandomState(B)
    sizes = [(int(rs.randint(50, 1000)), int(rs.randint(50, 1000))) for _ in range(B)]
    got = run_select(emul, cand, keep, kc, n_cls, H, W, sizes, max_det)
    want = reference_select(detections(cand, count, keep, kc, H, W), n_cls, sizes, max_det)
    if ties:
        probs = [p for _, rows in want for _, p, *_ in rows]
        assert len(set(probs)) < len(probs)                 # the case does contain ties
    assert_select_equals(got, want, max_det)


def test_emulated_select_of_real_nms_survivors(emul):
    """The emulated decode and NMS of a random head output feed the selection, as on the device."""
    from test_detect_host_emul import _random_head, P as P2
    rs = np.random.RandomState(3)
    B, n_cls, A = 2, 3, 5
    out = _random_head(rs, B * n_cls, A, 1, H, W, 0.0)
    anchors = np.array(rs.uniform(0.5, 6.0, 2 * A).round(3), dtype=np.float32)
    N, K = B * n_cls, A * H * W
    cand = np.zeros((N, K, 8), dtype=np.float32)
    count = np.zeros(N, dtype=np.int32)
    emul.emul_region_detect(P2(out), P2(anchors), N, A, 1, H, W, n_cls, 1, 0, ctypes.c_double(0.005), P2(cand), P2(count),
                            None)
    keep = np.full((N, K), -1, dtype=np.int32)
    kc = np.zeros(N, dtype=np.int32)
    emul.emul_nms(P2(cand), None, P2(count), N, K, H, W, ctypes.c_double(0.45), P2(keep), P2(kc))
    assert kc.sum() > 20
    sizes = [(500, 375), (333, 640)]
    got = run_select(emul, cand, keep, kc, n_cls, H, W, sizes, 15)
    assert_select_equals(got, reference_select(detections(cand, count, keep, kc, H, W), n_cls, sizes, 15), 15)
