"""csrc/coco_eval.cu (device COCO AP / AR) without a GPU: the kernel source and the library's launch sequence are
compiled by g++ against tools/host_emul/cuda_host_emul.h and run on the CPU.  The gather must reproduce
coco_eval.detection_records and the evaluation coco_eval.coco_evaluate bit for bit, on seeded synthetic sets with
more than 100 survivors in a row, heavy score ties within and across images, crowd ground truth, areas on the range
boundaries, images without detections, classes without ground truth and batches appended out of image order.
The GPU runs the same checks through the C ABI (tests/test_gpu_coco_eval.py)."""
import ctypes

import numpy as np
import pytest

from emul_util import build_emul
from fewshot_detection_b200 import coco_eval as C

A_, H_, W_ = 5, 13, 13                                  # anchors and grid of the synthetic Detections


@pytest.fixture(scope='module')
def emul():
    lib = build_emul('coco_eval', 'coco_eval.cu')
    lib.emul_coco_workspace_bytes.restype = ctypes.c_size_t
    return lib


def P(a):
    return a.ctypes.data_as(ctypes.c_void_p) if a is not None and a.size else None


# ---- synthetic sets (shared with tests/test_gpu_coco_eval.py) ---------------------------------------------------------
def synthetic_set(seed, n_img=24, n_cls=6, big_rows=3, n_scores=6):
    """Ground truth {'image_ids', 'category_ids', 'anns'}, image sizes and per (image, class) row the NMS survivors
    as float32 candidates (xs, ys, ws, hs in grid units, det_conf, cls_conf).  The last class has no ground truth;
    about one image in six has no detections; `big_rows` rows hold 101-140 survivors; scores come from `n_scores`
    products (ties within and across images); some objects are crowd and some json areas sit exactly on 32^2 and
    96^2."""
    rs = np.random.RandomState(seed)
    sizes = [(int(rs.randint(200, 640)), int(rs.randint(200, 640))) for _ in range(n_img)]
    anns = []
    for i in range(n_img):
        W, H = sizes[i]
        objs = []
        for c in range(n_cls - 1):
            for _ in range(rs.randint(0, 4)):
                w, h = rs.uniform(4, W / 2.0), rs.uniform(4, H / 2.0)
                x, y = rs.uniform(0, W - w), rs.uniform(0, H - h)
                area = w * h * rs.uniform(0.5, 1.0)
                u = rs.rand()
                if u < 0.1:
                    area = 32.0 ** 2
                elif u < 0.2:
                    area = 96.0 ** 2
                elif u < 0.3:
                    area = int(area)
                objs.append((c, [float(x), float(y), float(w), float(h)], area, int(rs.rand() < 0.12)))
        objs = [objs[k] for k in rs.permutation(len(objs))]
        anns.append(objs)
    gt = {'image_ids': [5000 + 3 * i for i in range(n_img)], 'category_ids': [1 + 2 * c for c in range(n_cls)],
          'anns': anns}
    dets = np.asarray(rs.uniform(0.05, 1.0, n_scores), dtype=np.float32)
    clsc = np.asarray(rs.uniform(0.3, 1.0, n_scores), dtype=np.float32)
    rows = []
    big = set(rs.choice(n_img * n_cls, big_rows, replace=False).tolist())
    for i in range(n_img):
        W, H = sizes[i]
        empty = rs.rand() < 0.17
        for c in range(n_cls):
            n = 0 if empty else (rs.randint(101, 141) if i * n_cls + c in big else rs.randint(0, 25))
            gts = [o[1] for o in anns[i] if o[0] == c]
            row = []
            for _ in range(n):
                if gts and rs.rand() < 0.6:
                    x, y, w, h = gts[rs.randint(len(gts))]
                    x, y = x + rs.normal(0, w * 0.1), y + rs.normal(0, h * 0.1)
                    w, h = w * np.exp(rs.normal(0, 0.15)), h * np.exp(rs.normal(0, 0.15))
                else:
                    w, h = rs.uniform(3, W / 1.5), rs.uniform(3, H / 1.5)
                    x, y = rs.uniform(-10, W - w / 2), rs.uniform(-10, H - h / 2)
                k = rs.randint(n_scores)
                row.append([(x + w / 2) / W * W_, (y + h / 2) / H * H_, w / W * W_, h / H * H_, dets[k], clsc[k]])
            rows.append(np.array(row, dtype=np.float32).reshape(-1, 6))
    return gt, sizes, rows


def detections(rows, images, n_cls):
    """cand / keep / keep_count of a batch of images (rows of those images, class-major within an image), survivors
    in a shuffled slot order so that `keep` is not the identity."""
    cap = A_ * H_ * W_
    N = len(images) * n_cls
    cand = np.zeros((N, cap, 8), dtype=np.float32)
    keep = np.full((N, cap), -1, dtype=np.int32)
    kc = np.zeros(N, dtype=np.int32)
    rs = np.random.RandomState(len(images) + images[0])
    for b, i in enumerate(images):
        for c in range(n_cls):
            r, row = b * n_cls + c, rows[i * n_cls + c]
            slots = rs.permutation(cap)[:len(row)]
            cand[r, slots, :6] = row
            keep[r, :len(row)] = slots
            kc[r] = len(row)
    return cand, keep, kc


def host_detections(cand, keep, kc, n_cls):
    import torch
    from fewshot_detection_b200 import utils as U
    N = len(kc)
    count = torch.full((N,), cand.shape[1], dtype=torch.int32)                  # every slot a candidate
    d = U.Detections(torch.from_numpy(cand), count, None, N, A_, 1, H_, W_, False, True, 0.005)
    d.keep, d.keep_count, d._nms_thresh = torch.from_numpy(keep), torch.from_numpy(kc), 0.45
    return d


def batches_of(n_img, seed):
    """Images in batches of 1-5, batches in a shuffled order: records are appended out of image order."""
    rs = np.random.RandomState(seed + 100)
    order = rs.permutation(n_img).tolist()
    out = []
    while order:
        k = rs.randint(1, 6)
        out.append(order[:k])
        order = order[k:]
    return out


def host_reference(gt, sizes, rows, names, n_cls, batches):
    """detection_records of every batch (in batch order) and coco_evaluate over them."""
    records = []
    for images in batches:
        cand, keep, kc = detections(rows, images, n_cls)
        d = host_detections(cand, keep, kc, n_cls)
        records.extend(C.detection_records(d, [names[i] for i in images], [sizes[i] for i in images], n_cls))
    index = dict((n, gt['image_ids'][k]) for k, n in enumerate(names))
    results = [{'image_id': index[r[0]], 'category_id': gt['category_ids'][r[1]], 'bbox': r[3], 'score': r[2]}
               for r in records]
    return records, C.coco_evaluate(gt, results, names, ['c%d' % k for k in range(n_cls)])


# ---- the emulated kernels ---------------------------------------------------------------------------------------------
def emul_gather(emul, gt, sizes, rows, n_cls, batches, pool_cap=None, group_cap=None):
    total = sum(min(len(r), 100) for r in rows)
    pool_cap = total if pool_cap is None else pool_cap
    group_cap = len(rows) if group_cap is None else group_cap
    score = np.full(max(pool_cap, 1), -7.0)
    box = np.full((max(pool_cap, 1), 4), -7.0)
    groups = np.full((max(group_cap, 1), 4), -1, dtype=np.int32)
    counters = np.zeros(4, dtype=np.int64)
    for images in batches:
        cand, keep, kc = detections(rows, images, n_cls)
        idx = np.array(images, dtype=np.int32)
        size = np.array([sizes[i] for i in images], dtype=np.float64)
        emul.emul_coco_gather(P(cand), P(keep), P(kc), len(kc), keep.shape[1], H_, W_, n_cls, P(idx), P(size), 100,
                              P(score), P(box), ctypes.c_longlong(pool_cap), P(groups), group_cap, P(counters))
    return score, box, groups, counters


def emul_evaluate(emul, score, box, groups, counters, gt, n_cls):
    n_det, n_groups = int(counters[0]), int(counters[1])
    ptr, gbox, garea, crowd = C.gt_tables(gt, n_cls)
    n_img, n_gt = len(gt['anns']), len(garea)
    iou, rec, md, area = C.device_params()
    ws = np.zeros(max(1, emul.emul_coco_workspace_bytes(n_det, n_gt, n_cls, n_img)), dtype=np.uint8)
    out = dict(dt_flags=np.full((4, max(n_det, 1)), 0x7fffffff, np.int32), order=np.full(max(n_det, 1), -1, np.int32),
               precision=np.full((10, 101, n_cls, 4, 3), -7.0), recall=np.full((10, n_cls, 4, 3), -7.0))
    emul.emul_coco_evaluate(P(score), P(box), n_det, P(groups), n_groups, P(ptr), P(gbox), P(garea), P(crowd), n_gt,
                            n_cls, n_img, P(iou), P(rec), P(md), P(area), P(ws), P(out['dt_flags']), P(out['order']),
                            P(out['precision']), P(out['recall']))
    return out


def check_gather(score, box, groups, counters, records, names, n_cls, batches):
    """The pool holds detection_records' records, group by group in batch order, bit for bit."""
    assert counters[3] == 0 and counters[1] == sum(len(b) for b in batches) * n_cls
    assert counters[0] == len(records)
    k = 0
    for gi in range(int(counters[1])):
        first, count, img, cls = groups[gi]
        b = next(j for j, bb in enumerate(batches) if img in bb)
        assert gi == sum(len(bb) for bb in batches[:b]) * n_cls + batches[b].index(img) * n_cls + cls
        for j in range(count):
            name, c, s, bb = records[k]
            assert (name, c) == (names[img], cls) and first + j == k
            assert score[k] == s and box[k].tolist() == bb, (k, score[k], s, box[k], bb)
            k += 1
    assert k == len(records)


def check_bit_equal(out, ref):
    for key in ('precision', 'recall'):
        a, b = out[key], ref[key]
        bad = np.nonzero(a.view(np.uint64) != b.view(np.uint64))
        assert len(bad[0]) == 0, (key, list(zip(*bad))[:5], a[bad][:5], b[bad][:5])


@pytest.mark.parametrize('seed', [0, 1, 2])
def test_gather_and_evaluate_equal_the_host(emul, seed):
    n_cls = 6
    gt, sizes, rows = synthetic_set(seed, n_cls=n_cls)
    names = ['COCO_val2014_%012d' % i for i in gt['image_ids']]
    batches = batches_of(len(names), seed)
    records, ref = host_reference(gt, sizes, rows, names, n_cls, batches)
    assert max(len(r) for r in rows) > 100 and any(len(r) == 0 for r in rows)
    score, box, groups, counters = emul_gather(emul, gt, sizes, rows, n_cls, batches)
    check_gather(score, box, groups, counters, records, names, n_cls, batches)
    out = emul_evaluate(emul, score, box, groups, counters, gt, n_cls)
    check_bit_equal(out, ref)
    assert (ref['precision'][:, :, n_cls - 1] == -1).all()                    # no ground truth
    assert (ref['precision'][:, :, :n_cls - 1] > 0).any() and (ref['precision'][:, :, :n_cls - 1] < 1).any()
    assert ref['all'][0] > 0


def test_every_image_counts_without_detections(emul):
    """Images never added keep their ground truth: recall falls accordingly."""
    n_cls = 4
    gt, sizes, rows = synthetic_set(5, n_img=12, n_cls=n_cls, big_rows=1)
    names = ['n%d' % i for i in range(12)]
    batches = [[3, 1], [7], [0, 2, 4]]
    records, ref = host_reference(gt, sizes, rows, names, n_cls, batches)
    score, box, groups, counters = emul_gather(emul, gt, sizes, rows, n_cls, batches)
    out = emul_evaluate(emul, score, box, groups, counters, gt, n_cls)
    check_bit_equal(out, ref)


def test_no_detections_at_all(emul):
    n_cls = 3
    gt, sizes, rows = synthetic_set(6, n_img=5, n_cls=n_cls, big_rows=0)
    out = emul_evaluate(emul, np.zeros(1), np.zeros((1, 4)), np.zeros((1, 4), np.int32), np.zeros(4, np.int64), gt, n_cls)
    ref = C.coco_evaluate(gt, [], ['n%d' % i for i in range(5)], ['a', 'b', 'c'])
    check_bit_equal(out, ref)
    assert set(np.unique(out['precision'])) <= {-1.0, 0.0}


def test_pool_and_group_overflow(emul):
    n_cls = 3
    gt, sizes, rows = synthetic_set(7, n_img=6, n_cls=n_cls, big_rows=1)
    total = sum(min(len(r), 100) for r in rows)
    batches = [[0, 1, 2], [3, 4, 5]]
    first = sum(min(len(r), 100) for r in rows[:3 * n_cls])
    # the second batch does not fit the pool: it is dropped, flagged, and the first stays
    _, _, _, counters = emul_gather(emul, gt, sizes, rows, n_cls, batches, pool_cap=total - 1)
    assert counters.tolist() == [first, 3 * n_cls, 0, 1]
    _, _, _, counters = emul_gather(emul, gt, sizes, rows, n_cls, batches, group_cap=len(rows) - 1)
    assert counters.tolist() == [first, 3 * n_cls, 0, 1]
    # and nothing is appended after an overflow
    _, _, _, counters = emul_gather(emul, gt, sizes, rows, n_cls, [[0], [1, 2, 3, 4, 5], [0]], pool_cap=total)
    assert counters[3] == 1 and counters[1] == 6 * n_cls


def test_device_pool_glue_and_merge_on_emulated_kernels(emul, monkeypatch):
    """DeviceCocoEval's host side (ground-truth tables, capacity growth, argument lists, summary, merging) with the
    C-ABI calls routed to the emulated kernels and CPU tensors: the same dict as coco_evaluate, and the same pool and
    dict from two evaluators given half the batches each and merged."""
    import torch
    from fewshot_detection_b200 import eval_pool
    n_cls = 5
    gt, sizes, rows = synthetic_set(3, n_img=14, n_cls=n_cls)
    names = ['n%d' % i for i in range(14)]
    classes = ['c%d' % k for k in range(n_cls)]
    batches = batches_of(14, 3)
    _, ref = host_reference(gt, sizes, rows, names, n_cls, batches)
    V_ = ctypes.c_void_p
    calls = []

    def fake_call(name, *a):
        calls.append(name)
        a = list(a[:-1])
        if name == 'fsdet_coco_gather':
            del a[7]                                                          # nC (checked by the library)
            a = [V_(x) if isinstance(x, int) and k in (0, 1, 2, 8, 9, 11, 12, 14, 16) else x for k, x in enumerate(a)]
            a[13] = ctypes.c_longlong(a[13])
            return emul.emul_coco_gather(*a)
        if name == 'fsdet_coco_evaluate':
            del a[17]                                                         # workspace bytes
            ptrs = (0, 1, 3, 5, 6, 7, 8, 12, 13, 14, 15, 16, 17, 18, 19, 20)
            return emul.emul_coco_evaluate(*[V_(x) if k in ptrs else x for k, x in enumerate(a)])
        if name == 'fsdet_coco_merge':
            del a[9]                                                          # workspace bytes
            a = [V_(x) if k in (1, 2, 3, 5, 8, 9, 10, 12, 14) else x for k, x in enumerate(a)]
            a[4], a[6], a[11] = ctypes.c_longlong(a[4]), ctypes.c_longlong(a[6]), ctypes.c_longlong(a[11])
            return emul.emul_coco_merge(*a)
        raise AssertionError(name)
    emul.emul_eval_merge_workspace_bytes.restype = ctypes.c_size_t
    monkeypatch.setattr(eval_pool, '_call', fake_call)
    monkeypatch.setattr(eval_pool, '_call_size', lambda name, *a: getattr(emul, name.replace('fsdet_', 'emul_'))(*a))
    monkeypatch.setattr(eval_pool, '_stream', lambda *a: None)
    ev = C.DeviceCocoEval(classes, names, gt, device='cpu')
    for images in batches:
        cand, keep, kc = detections(rows, images, n_cls)
        ev.add(host_detections(cand, keep, kc, n_cls), [names[i] for i in images], [sizes[i] for i in images])
    with pytest.raises(ValueError):
        ev.add(host_detections(cand, keep, kc, n_cls), [names[i] for i in images], [sizes[i] for i in images])
    res = ev.result(novel_classes=('c1', 'c4'))
    assert calls.count('fsdet_coco_gather') == len(batches) and calls.count('fsdet_coco_evaluate') == 1
    check_bit_equal(res, ref)
    want = C.summarize(ref['precision'], ref['recall'], classes, ('c1', 'c4'))
    assert res['all'] == ref['all'] == want['all'] and res['novel'] == want['novel'] and res['ap'] == want['ap']
    assert res['ap']['c4'] == -1.0
    # the same batches over two evaluators, merged in order
    halves = [ev.empty_like(), ev.empty_like()]
    for k, images in enumerate(batches):
        cand, keep, kc = detections(rows, images, n_cls)
        halves[2 * k // len(batches)].add(host_detections(cand, keep, kc, n_cls), [names[i] for i in images],
                                          [sizes[i] for i in images])
    assert all(int(h.counters[0]) > 0 for h in halves)
    merged = type(ev).merge(halves)
    assert calls.count('fsdet_coco_merge') == 1
    n, g = int(ev.counters[0]), int(ev.counters[1])
    assert [int(v) for v in merged.counters[[0, 1, 3]]] == [n, g, 0]
    assert torch.equal(merged.key[:n], ev.key[:n]) and torch.equal(merged.box[:n], ev.box[:n])
    assert torch.equal(merged.groups[:g], ev.groups[:g])
    res2 = merged.result(novel_classes=('c1', 'c4'))
    check_bit_equal(res2, res)
    assert all(res2[k] == res[k] for k in ('all', 'base', 'novel', 'ap'))
