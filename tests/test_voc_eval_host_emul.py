"""csrc/voc_eval.cu (device VOC AP) without a GPU: the kernel source and the library's launch sequence are compiled by
g++ against tools/host_emul/cuda_host_emul.h and run on the CPU.  Checked against
  * tests/golden/voc_eval.npz (the reference's scripts/voc_eval.py on the same annotations and result lines);
  * voc_eval.match_detections / voc_ap on synthetic sets with heavy ties, through a copy that ranks with a stable sort
    (the device's definition at ties);
  * '%f' % x -> float() for the rounding of confidences and corners;
  * valid.detection_lines for the gather of kept boxes from decode + NMS buffers.
The GPU runs the same checks through the C ABI (tests/test_gpu_voc_eval.py)."""
import ctypes
import os

import numpy as np
import pytest

from emul_util import build_emul
from fewshot_detection_b200 import voc_eval as V

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
KEY_MASK = (1 << 20) - 1


@pytest.fixture(scope='module')
def emul():
    return build_emul('voc_eval', 'voc_eval.cu')


def P(a):
    return a.ctypes.data_as(ctypes.c_void_p) if a is not None and a.size else None


# ---- helpers shared with tests/test_gpu_voc_eval.py ----------------------------------------------------------------
def match_detections_stable(image_ids, confidence, boxes, gt, ovthresh=0.5):
    """voc_eval.match_detections with np.argsort(..., kind='stable'): ties keep result-file order."""
    order = np.argsort(-np.asarray(confidence, dtype=np.float64), kind='stable')
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
                continue
            if claimed[img][j]:
                fp[rank] = 1.
            else:
                tp[rank] = 1.
                claimed[img][j] = True
        else:
            fp[rank] = 1.
    return tp, fp


def host_class_eval(lines, recs, imagenames, classname, match=match_detections_stable):
    """voc_eval.voc_eval's body on parsed lines [(imgname, conf, x1, y1, x2, y2)]: tp, fp, rec, prec, ap07, ap_area."""
    gt, npos = {}, 0
    for name in imagenames:
        objs = [o for o in recs[name] if o['name'] == classname]
        difficult = np.array([o['difficult'] for o in objs]).astype(bool)
        gt[name] = (np.array([o['bbox'] for o in objs]), difficult)
        npos += int(np.sum(~difficult))
    tp, fp = match([l[0] for l in lines], np.array([l[1] for l in lines]), np.array([l[2:] for l in lines]), gt)
    ctp, cfp = np.cumsum(tp), np.cumsum(fp)
    with np.errstate(divide='ignore', invalid='ignore'):
        rec = ctp / float(npos)
    prec = ctp / np.maximum(ctp + cfp, np.finfo(np.float64).eps)
    with np.errstate(invalid='ignore'):
        return tp, fp, rec, prec, V.voc_ap(rec, prec, True), V.voc_ap(rec, prec, False)


def pack_lines(per_class, imagenames):
    """Records + groups of per-class line lists [(imgname, conf, x1, y1, x2, y2)] whose images form contiguous runs
    (as the gather writes them).  conf must be a '%f' value."""
    index = dict((n, k) for k, n in enumerate(imagenames))
    keys, boxes, groups = [], [], []
    for c, lines in enumerate(per_class):
        seen = set()
        for k, l in enumerate(lines):
            if k == 0 or l[0] != lines[k - 1][0]:
                assert l[0] not in seen, 'image runs must be contiguous'
                seen.add(l[0])
                groups.append([len(keys), 0, index[l[0]], c])
            groups[-1][1] += 1
            n = int(round(l[1] * 1e6))
            assert 0 <= n <= 1000000 and n / 1e6 == l[1]
            keys.append((c << 20) | (KEY_MASK - n))
            boxes.append(l[2:])
    return (np.array(keys, dtype=np.uint32), np.array(boxes, dtype=np.float64).reshape(-1, 4),
            np.array(groups, dtype=np.int32).reshape(-1, 4))


def emul_evaluate(emul, per_class, classes, imagenames, recs, ovthresh=0.5):
    keys, boxes, groups = pack_lines(per_class, imagenames)
    gt_ptr, gt_box, gt_diff = V.gt_tables(classes, imagenames, recs)
    n, n_cls, n_gt = len(keys), len(classes), len(gt_diff)
    ws = np.zeros(max(1, emul.emul_voc_workspace_bytes(n, n_gt)), dtype=np.uint8)
    emul.emul_voc_workspace_bytes.restype = ctypes.c_size_t
    out = dict(flags=np.full(n, 9, np.uint8), order=np.full(n, -1, np.int32), rec=np.full(n, -7.0), prec=np.full(n, -7.0),
               cls_count=np.full(n_cls, -1, np.int32), npos=np.full(n_cls, -1, np.int32), ap07=np.full(n_cls, -7.0),
               ap_area=np.full(n_cls, -7.0))
    th = np.ascontiguousarray(V.VOC07_THRESHOLDS)
    emul.emul_voc_evaluate(P(keys), P(boxes), n, P(groups), len(groups), P(gt_ptr), P(gt_box), P(gt_diff), n_gt, n_cls,
                           len(imagenames), ctypes.c_double(ovthresh), P(th), P(ws), P(out['flags']), P(out['order']),
                           P(out['rec']), P(out['prec']), P(out['cls_count']), P(out['npos']), P(out['ap07']),
                           P(out['ap_area']))
    return out


def check_against_host(out, per_class, classes, imagenames, recs):
    """Flags in rank order, rec / prec bit-equal, VOC07 AP equal, area AP within 1e-12 (NaN where numpy gives NaN)."""
    start = 0
    for c, name in enumerate(classes):
        lines = per_class[c]
        n = len(lines)
        assert out['cls_count'][c] == n
        tp, fp, rec, prec, ap07, ap_area = host_class_eval(lines, recs, imagenames, name)
        order = out['order'][start:start + n]
        assert np.array_equal(np.sort(order - start), np.arange(n))      # class c's records, packed class by class
        f = out['flags'][order]
        assert np.array_equal((f == 1).astype(float), tp), name
        assert np.array_equal((f == 2).astype(float), fp), name
        assert np.array_equal(out['rec'][start:start + n], rec, equal_nan=True), name
        assert np.array_equal(out['prec'][start:start + n], prec), name
        assert out['ap07'][c] == ap07, (name, out['ap07'][c], ap07)
        if np.isnan(ap_area):
            assert np.isnan(out['ap_area'][c]), name
        else:
            assert abs(out['ap_area'][c] - ap_area) <= 1e-12, (name, out['ap_area'][c], ap_area)
        start += n


# ---- the '%f' round trip --------------------------------------------------------------------------------------------
def round_trip_inputs(n, seed=0):
    rs = np.random.RandomState(seed)
    parts = [rs.uniform(0, 1, n // 4),                                    # confidences
             rs.uniform(-60, 700, n // 4),                                # corners, some negative
             (rs.randint(0, 2 ** 20, n // 8) + 0.5) / 2.0 ** rs.randint(7, 21, n // 8),   # exact binary halves of 1e-6 steps
             (rs.randint(-10 ** 9, 10 ** 9, n // 8) + 0.5) / 1e6,         # nearest doubles to decimal halves
             rs.uniform(-1e-6, 1e-6, n // 16),                            # '-0.000000'
             np.ldexp(rs.uniform(1, 2, n // 16), rs.randint(-40, 40, n // 16)),
             np.array([0.0078125, 0.0234375, -0.0078125, 0.5, 2.5e-7, 5e-7, -5e-7, 1.5e-6, 4503599627.3705, 2.0 ** 33 + 0.25,
                       1e300, -0.0, 0.0, 1.0, 1e-300])]
    return np.concatenate(parts)


def expected_round_trip(x):
    return np.char.mod('%f', x).astype(np.float64)


def test_round6_equals_printf_round_trip(emul):
    x = round_trip_inputs(2000000)
    y = np.empty_like(x)
    nn = np.empty_like(x)
    emul.emul_voc_round6(P(x), P(y), P(nn), ctypes.c_longlong(len(x)))
    want = expected_round_trip(x)
    bad = np.nonzero(y.view(np.uint64) != want.view(np.uint64))[0]
    assert bad.size == 0, [(repr(x[i]), repr(y[i]), repr(want[i])) for i in bad[:10]]
    small = np.abs(x) < 2.0 ** 33
    assert np.array_equal(nn[small] / 1e6, y[small])
    # the two exact binary ties of the issue's examples
    k = len(x) - 15
    assert y[k] == 0.007812 and y[k + 1] == 0.023438 and y[k + 2] == -0.007812


# ---- against the reference's own evaluator --------------------------------------------------------------------
def golden_case(gold):
    names = [str(n) for n in gold['names']]
    recs = dict((n, []) for n in names)
    for n, c, df, x1, y1, x2, y2 in gold['gt']:
        recs[str(n)].append({'name': str(c), 'pose': 'Unspecified', 'truncated': 0, 'difficult': int(df),
                             'bbox': [int(x1), int(y1), int(x2), int(y2)]})
    classes = [str(c) for c in gold['classes']]
    index = dict((n, k) for k, n in enumerate(names))
    per_class = []
    for c in classes:
        rows = [str(l).split(' ') for l in gold['det/' + c]]
        lines = [(r[0], float(r[1])) + tuple(float(z) for z in r[2:]) for r in rows]
        per_class.append(sorted(lines, key=lambda l: index[l[0]]))           # stable: image runs, file order inside
    return names, recs, classes, per_class


def test_golden_reference_voc_eval(emul):
    gold = np.load(os.path.join(G, 'voc_eval.npz'), allow_pickle=False)
    names, recs, classes, per_class = golden_case(gold)
    for lines in per_class:
        assert len(set(l[1] for l in lines)) == len(lines)                    # no tied confidences in this fixture
    out = emul_evaluate(emul, per_class, classes, names, recs)
    start = 0
    for c, name in enumerate(classes):
        n = len(per_class[c])
        assert np.array_equal(out['rec'][start:start + n], gold['rec/%s/1' % name])
        assert np.array_equal(out['prec'][start:start + n], gold['prec/%s/1' % name])
        assert out['ap07'][c] == float(gold['ap/%s/1' % name])
        assert abs(out['ap_area'][c] - float(gold['ap/%s/0' % name])) <= 1e-12
        start += n
    check_against_host(out, per_class, classes, names, recs)


# ---- synthetic sets with heavy ties and every matching rule -----------------------------------------------------------
def synthetic_case(seed, n_img=40, classes=('a', 'b', 'c', 'd', 'e'), per_img=12, n_conf=7):
    """Images with 0-4 objects per class (some difficult), detections near them, duplicates, far-off boxes, and
    confidences drawn from n_conf values.  Class 'd' has only difficult objects (npos = 0); class 'e' never gets a
    detection."""
    rs = np.random.RandomState(seed)
    names = ['%06d' % (7 * k + 3) for k in range(n_img)]
    recs = {}
    for n in names:
        objs = []
        for c in classes:
            for _ in range(rs.randint(0, 3) if c != 'e' else rs.randint(0, 2)):
                x1, y1 = rs.randint(0, 300, 2)
                w, h = rs.randint(10, 150, 2)
                objs.append({'name': c, 'pose': 'Unspecified', 'truncated': 0,
                             'difficult': 1 if (c == 'd' or rs.rand() < 0.15) else 0,
                             'bbox': [int(x1), int(y1), int(x1 + w), int(y1 + h)]})
        recs[n] = objs
    confs = np.round(rs.uniform(0.005, 1.0, n_conf), 6)
    per_class = []
    for c in classes:
        lines = []
        if c == 'e':
            per_class.append(lines)
            continue
        for n in names:
            if rs.rand() < 0.2:
                continue                                                    # image without detections of c
            gts = [o['bbox'] for o in recs[n] if o['name'] == c]
            for _ in range(rs.randint(1, per_img)):
                if gts and rs.rand() < 0.7:
                    g = np.array(gts[rs.randint(len(gts))], dtype=np.float64)
                    b = g + rs.normal(0, rs.choice([1.0, 8.0, 25.0]), 4)    # near a ground truth: TP / duplicate / miss
                else:
                    x1, y1 = rs.uniform(-20, 400, 2)
                    b = np.array([x1, y1, x1 + rs.uniform(5, 120), y1 + rs.uniform(5, 120)])
                b = np.array([float('%f' % v) for v in b])
                lines.append((n, float(confs[rs.randint(n_conf)])) + tuple(b))
        per_class.append(lines)
    return names, recs, list(classes), per_class


@pytest.mark.parametrize('seed', [0, 1, 2])
def test_heavy_ties_against_stable_host_copy(emul, seed):
    names, recs, classes, per_class = synthetic_case(seed)
    assert sum(len(l) for l in per_class) > 500
    out = emul_evaluate(emul, per_class, classes, names, recs)
    check_against_host(out, per_class, classes, names, recs)
    assert out['npos'][classes.index('d')] == 0 and np.isnan(out['ap_area'][classes.index('d')])
    assert out['ap07'][classes.index('d')] == 0.0
    assert out['cls_count'][classes.index('e')] == 0 and out['ap07'][classes.index('e')] == 0.0
    assert out['ap_area'][classes.index('e')] == 0.0


def test_more_than_one_radix_tile(emul):
    """> 2048 records of one class: the sort's tiles and the scans' partial sums are exercised."""
    names, recs, classes, per_class = synthetic_case(5, n_img=160, classes=('a', 'b'), per_img=40, n_conf=40)
    assert len(per_class[0]) > 2048
    out = emul_evaluate(emul, per_class, classes, names, recs)
    check_against_host(out, per_class, classes, names, recs)


def test_matching_rules(emul):
    """voc_eval's rules one by one: TP, duplicate of a claimed box, a difficult match, an image without ground truth,
    no overlap, the first of two equal IoUs, IoU exactly at the threshold (not a match)."""
    names = ['a', 'b', 'c']
    recs = {'a': [{'name': 'x', 'difficult': 0, 'bbox': [10, 10, 50, 50]}, {'name': 'x', 'difficult': 1, 'bbox': [100, 100, 150, 150]}],
            'b': [], 'c': [{'name': 'x', 'difficult': 0, 'bbox': [0, 0, 9, 9]}, {'name': 'x', 'difficult': 0, 'bbox': [0, 0, 9, 9]},
                           {'name': 'x', 'difficult': 0, 'bbox': [200, 200, 209, 219]}]}
    lines = [('a', 0.9, 10., 10., 50., 50.), ('a', 0.8, 12., 12., 50., 50.), ('a', 0.7, 100., 100., 150., 150.),
             ('a', 0.5, 300., 300., 320., 320.), ('b', 0.6, 0., 0., 10., 10.),
             ('c', 0.4, 0., 0., 9., 9.), ('c', 0.4, 0., 0., 9., 9.), ('c', 0.4, 0., 0., 9., 9.),
             ('c', 0.3, 200., 200., 209., 209.)]                             # IoU = 100 / 200 = 0.5: not > 0.5
    out = emul_evaluate(emul, [lines], ['x'], names, recs)
    f = out['flags'][out['order']]
    assert f.tolist() == [1, 2, 0, 2, 2, 1, 2, 2, 2]
    check_against_host(out, [lines], ['x'], names, recs)
    tp, fp = V.match_detections([l[0] for l in lines], [l[1] for l in lines], [l[2:] for l in lines],
                                dict((n, (np.array([o['bbox'] for o in recs[n]]).reshape(-1, 4),
                                          np.array([o['difficult'] for o in recs[n]], bool))) for n in names))
    assert sorted(tp.tolist()) == sorted((f == 1).astype(float).tolist())


def test_no_detections_at_all(emul):
    names = ['a']
    recs = {'a': [{'name': 'x', 'difficult': 0, 'bbox': [1, 1, 5, 5]}]}
    out = emul_evaluate(emul, [[], []], ['x', 'y'], names, recs)
    assert out['ap07'].tolist() == [0.0, 0.0] and out['ap_area'].tolist() == [0.0, 0.0]
    assert out['npos'].tolist() == [1, 0] and out['cls_count'].tolist() == [0, 0]
    assert V.voc_ap(np.array([]), np.array([]), True) == 0.0


# ---- gather: decode + NMS buffers -> records, against valid.detection_lines ---------------------------------------
def test_gather_equals_result_lines(emul):
    import torch
    from fewshot_detection_b200 import utils as U, valid as VA
    from test_detect_host_emul import run_detect
    from test_gpu_detect import params
    detect_emul = build_emul('detect', 'detect.cu', opt='-O1')
    gold = np.load(os.path.join(G, 'detect.npz'), allow_pickle=False)
    tag = 'v2_g13'
    p = params(gold, tag)
    out = gold[tag + '/output']
    N, _, H, W = out.shape
    K = p['nA'] * H * W
    n_cls = p['cs']
    bs = N // n_cls
    cand, count, dense = run_detect(detect_emul, out, p)
    keep = np.full((N, K), -1, dtype=np.int32)
    kc = np.full(N, -1, dtype=np.int32)
    detect_emul.emul_nms(P(cand), None, P(count), N, K, H, W, ctypes.c_double(p['nms']), P(keep), P(kc))
    d = U.Detections(torch.from_numpy(cand), torch.from_numpy(count), torch.from_numpy(dense) if dense is not None else None,
                     N, p['nA'], p['nC'], H, W, bool(p['only_obj']), p['val'], p['thr'])
    d.keep, d.keep_count, d._nms_thresh, d._kept_host = torch.from_numpy(keep), torch.from_numpy(kc), p['nms'], None
    imgids, sizes = ['000017', '000004'][:bs], [(500, 375), (353, 481)][:bs]
    lines = VA.detection_lines(d, imgids, sizes, n_cls, p['nms'])
    # two batches: the same images under other indices second time round, to check appending
    cap_pool = 2 * int(kc.sum()) + 5
    keys = np.zeros(cap_pool, dtype=np.uint32)
    boxes = np.zeros((cap_pool, 4))
    groups = np.full((4 * N, 4), -1, dtype=np.int32)
    counters = np.zeros(4, dtype=np.int64)
    for batch, idx in enumerate(([3, 1], [0, 2])):
        idx = np.array(idx[:bs], dtype=np.int32)
        size = np.array(sizes, dtype=np.float64)
        emul.emul_voc_gather(P(cand), P(keep), P(kc), N, K, H, W, n_cls, P(idx), P(size), P(keys), P(boxes),
                             ctypes.c_longlong(cap_pool), P(groups), len(groups), P(counters))
        assert counters[3] == 0 and counters[1] == (batch + 1) * N and counters[2] == batch * N
    assert counters[0] == 2 * kc.sum()
    half = int(kc.sum())
    for r in range(N):
        for batch, idx in enumerate(([3, 1], [0, 2])):
            g = groups[batch * N + r]
            assert g[1] == kc[r] and g[2] == idx[r // n_cls] and g[3] == r % n_cls
            assert g[0] == batch * half + kc[:r].sum()
    for i in range(n_cls):
        want = [l.split(' ') for l in lines[i]]
        got = [(r, k) for r in range(N) if r % n_cls == i for k in range(groups[r][0], groups[r][0] + groups[r][1])]
        assert len(got) == len(want) > 0
        for (r, k), w in zip(got, want):
            assert w[0] == imgids[r // n_cls]
            assert keys[k] >> 20 == i and KEY_MASK - (keys[k] & KEY_MASK) == int(w[1].replace('.', ''))
            assert boxes[k].tolist() == [float(z) for z in w[2:6]]
        assert np.array_equal(keys[half:2 * half], keys[:half]) and np.array_equal(boxes[half:2 * half], boxes[:half])
    # a batch that does not fit is dropped and flagged, and so is everything after it
    counters2 = np.zeros(4, dtype=np.int64)
    emul.emul_voc_gather(P(cand), P(keep), P(kc), N, K, H, W, n_cls, P(np.array([0, 1], np.int32)), P(np.array(sizes, np.float64)),
                         P(keys), P(boxes), ctypes.c_longlong(int(kc.sum()) - 1), P(groups), len(groups), P(counters2))
    assert counters2.tolist() == [0, 0, 0, 1]


def test_device_pool_glue_and_merge_on_emulated_kernels(emul, monkeypatch):
    """DeviceVocEval's host side (ground-truth tables, capacity growth, argument lists, result dict, merging) with the
    C-ABI calls routed to the emulated kernels and CPU tensors; same dict as mean_ap on the files write_detections
    writes, and the same pool and dict from two evaluators given half the batches each and merged."""
    import torch
    from fewshot_detection_b200 import eval_pool, utils as U
    gold = np.load(os.path.join(G, 'voc_eval.npz'), allow_pickle=False)
    names, recs, classes, per_class = golden_case(gold)
    calls = []
    V_ = ctypes.c_void_p

    def fake_call(name, *a):
        calls.append(name)
        if name == 'fsdet_voc_gather':
            a = list(a)
            del a[7]                                                         # nC (checked by the library)
            a = [V_(x) if isinstance(x, int) and k in (0, 1, 2, 8, 9, 10, 11, 13, 15) else x for k, x in enumerate(a[:-1])]
            a[12] = ctypes.c_longlong(a[12])
            return emul.emul_voc_gather(*a)
        if name == 'fsdet_voc_evaluate':
            a = list(a)
            del a[14]                                                        # workspace bytes
            ptrs = (0, 1, 3, 5, 6, 7, 12, 13, 14, 15, 16, 17, 18, 19, 20, 21)
            a = [V_(x) if k in ptrs else x for k, x in enumerate(a[:-1])]
            a[11] = ctypes.c_double(a[11])
            return emul.emul_voc_evaluate(*a)
        if name == 'fsdet_voc_merge':
            a = list(a[:-1])
            del a[9]                                                         # workspace bytes
            a = [V_(x) if k in (1, 2, 3, 5, 8, 9, 10, 12, 14) else x for k, x in enumerate(a)]
            a[4], a[6], a[11] = ctypes.c_longlong(a[4]), ctypes.c_longlong(a[6]), ctypes.c_longlong(a[11])
            return emul.emul_voc_merge(*a)
        raise AssertionError(name)
    emul.emul_voc_workspace_bytes.restype = ctypes.c_size_t
    emul.emul_eval_merge_workspace_bytes.restype = ctypes.c_size_t
    monkeypatch.setattr(eval_pool, '_call', fake_call)
    monkeypatch.setattr(eval_pool, '_call_size', lambda name, *a: getattr(emul, name.replace('fsdet_', 'emul_'))(*a))
    monkeypatch.setattr(eval_pool, '_stream', lambda *a: None)
    ev = V.DeviceVocEval(classes, names, recs, device='cpu')
    # Detections whose kept boxes print exactly as the golden lines: one batch per image, grid 1x1, W = H = 1, A = the
    # most lines of one image and class, det = 1, cls = prob, (xs, ys, ws, hs) chosen so that the corners come back
    index = dict((n, k) for k, n in enumerate(names))
    by_img = dict((n, [[] for _ in classes]) for n in names)
    for c, lines in enumerate(per_class):
        for l in lines:
            by_img[l[0]][c].append(l)
    A = max(len(v) for img in by_img.values() for v in img)
    size = (1000, 1000)
    batches = []
    for n in names:
        rows = by_img[n]
        cand = np.zeros((len(classes), A, 8), dtype=np.float32)
        keep = np.zeros((len(classes), A), dtype=np.int32)
        kc = np.array([len(r) for r in rows], dtype=np.int32)
        for c, r in enumerate(rows):
            for s, l in enumerate(r):
                x1, y1, x2, y2 = l[2:]
                cand[c, s, :6] = [(x1 + x2) / 2 / size[0], (y1 + y2) / 2 / size[1], (x2 - x1) / size[0], (y2 - y1) / size[1],
                                  1.0, l[1]]
                keep[c, s] = s
        d = U.Detections(torch.from_numpy(cand), torch.from_numpy(kc.copy()), None, len(classes), A, 1, 1, 1, False, True, 0.005)
        d.keep, d.keep_count = torch.from_numpy(keep), torch.from_numpy(kc)
        ev.add(d, [n], [size])
        batches.append((d, n))
        # what the device computed from these float32 values, as lines: overwrite the host copy with it
        for c, r in enumerate(rows):
            g = ev.groups[int(ev.counters[2]) + c].numpy()
            for s in range(len(r)):
                k = g[0] + s
                key = int(ev.key[k]) & 0xffffffff
                r[s] = (n, (KEY_MASK - (key & KEY_MASK)) / 1e6) + tuple(ev.box[k].tolist())
    with pytest.raises(ValueError):
        ev.add(d, [names[-1]], [size])                                      # an image twice
    res = ev.result(True, novel_classes=('cow',), curves=True)
    res_area = ev.result(False)
    assert calls.count('fsdet_voc_gather') == len(names) and calls.count('fsdet_voc_evaluate') == 2
    per_class2 = [[l for n in names for l in by_img[n][c]] for c in range(len(classes))]
    for c, name in enumerate(classes):
        _, _, rec, prec, ap07, ap_area = host_class_eval(per_class2[c], recs, names, name)
        assert res['ap'][name] == ap07 and abs(res_area['ap'][name] - ap_area) <= 1e-12
        assert np.array_equal(res['rec'][name], rec) and np.array_equal(res['prec'][name], prec)
    assert res['mean_novel'] == res['ap']['cow']
    assert res['mean'] == float(np.mean([res['ap'][c] for c in classes]))
    # the same batches over two evaluators, merged in order
    halves = [ev.empty_like(), ev.empty_like()]
    for k, (d, n) in enumerate(batches):
        halves[2 * k // len(batches)].add(d, [n], [size])
    assert all(int(h.counters[0]) > 0 for h in halves)
    merged = V.DeviceVocEval.merge(halves)
    assert calls.count('fsdet_voc_merge') == 1
    n, g = int(ev.counters[0]), int(ev.counters[1])
    assert [int(v) for v in merged.counters[[0, 1, 3]]] == [n, g, 0]
    assert torch.equal(merged.key[:n], ev.key[:n]) and torch.equal(merged.box[:n], ev.box[:n])
    assert torch.equal(merged.groups[:g], ev.groups[:g])
    res2, res2_area = merged.result(True, novel_classes=('cow',), curves=True), merged.result(False)
    assert res2_area == res_area
    assert [res2[k] for k in ('ap', 'mean', 'mean_base', 'mean_novel')] == \
        [res[k] for k in ('ap', 'mean', 'mean_base', 'mean_novel')]
    for k in ('rec', 'prec'):
        assert all(np.array_equal(res2[k][c], res[k][c]) for c in classes)
