"""Device COCO AP / AR (csrc/coco_eval.cu) through the C ABI and coco_eval.DeviceCocoEval, on the GPU.

  * the synthetic sets of the host-emulation test: gather and evaluation bit-equal to coco_eval.detection_records and
    coco_eval.coco_evaluate, and the overflow flag;
  * a mini meta model on a synthetic COCO set: valid.score_batches equals the results json scored by the host
    evaluator, with no per-detection data copied to the host;
  * a minival-sized pass (5,000 images x 80 classes, ~30 survivors per row): precision / recall of 8 random classes
    bit-equal to a host run over those classes alone (classes are evaluated independently)."""
import io
import json
import os
import sys

import numpy as np
import pytest
import torch

from test_coco_eval_host_emul import (batches_of, check_bit_equal, check_gather, detections, host_reference,
                                      synthetic_set, H_, W_)

pytestmark = pytest.mark.gpu

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def _st():
    return torch.cuda.current_stream().cuda_stream


def device_gather(sizes, rows, n_cls, batches, pool_cap=None):
    from fewshot_detection_b200 import _lib
    total = sum(min(len(r), 100) for r in rows)
    pool_cap = total if pool_cap is None else pool_cap
    score = torch.full((max(pool_cap, 1),), -7.0, dtype=torch.float64, device='cuda')
    box = torch.full((max(pool_cap, 1), 4), -7.0, dtype=torch.float64, device='cuda')
    groups = torch.full((len(rows), 4), -1, dtype=torch.int32, device='cuda')
    counters = torch.zeros(4, dtype=torch.int64, device='cuda')
    for images in batches:
        cand, keep, kc = [torch.from_numpy(a).cuda() for a in detections(rows, images, n_cls)]
        idx = torch.tensor(images, dtype=torch.int32, device='cuda')
        size = torch.tensor([sizes[i] for i in images], dtype=torch.float64, device='cuda')
        _lib.call('fsdet_coco_gather', cand.data_ptr(), keep.data_ptr(), kc.data_ptr(), len(kc), keep.shape[1], H_, W_,
                  1, n_cls, idx.data_ptr(), size.data_ptr(), 100, score.data_ptr(), box.data_ptr(), pool_cap,
                  groups.data_ptr(), len(rows), counters.data_ptr(), _st())
    return score, box, groups, counters


def device_evaluate(score, box, groups, counters, gt, n_cls):
    from fewshot_detection_b200 import _lib, coco_eval as C
    n_det, n_groups = int(counters[0]), int(counters[1])
    ptr, gbox, garea, crowd = [torch.from_numpy(a).cuda() for a in C.gt_tables(gt, n_cls)]
    n_img, n_gt = len(gt['anns']), garea.numel()
    iou, rec, md, area = C.device_params()
    nbytes = _lib.lib.fsdet_coco_workspace_bytes(n_det, n_gt, n_cls, n_img)
    ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device='cuda')
    out = dict(dt_flags=torch.empty(4, max(n_det, 1), dtype=torch.int32, device='cuda'),
               order=torch.empty(max(n_det, 1), dtype=torch.int32, device='cuda'),
               precision=torch.full((10, 101, n_cls, 4, 3), -7.0, dtype=torch.float64, device='cuda'),
               recall=torch.full((10, n_cls, 4, 3), -7.0, dtype=torch.float64, device='cuda'))
    p = lambda t: t.data_ptr() if t.numel() else None
    _lib.call('fsdet_coco_evaluate', score.data_ptr(), box.data_ptr(), n_det, groups.data_ptr(), n_groups, p(ptr),
              p(gbox), p(garea), p(crowd), n_gt, n_cls, n_img, iou.ctypes.data, rec.ctypes.data, md.ctypes.data,
              area.ctypes.data, ws.data_ptr(), nbytes, out['dt_flags'].data_ptr(), out['order'].data_ptr(),
              out['precision'].data_ptr(), out['recall'].data_ptr(), _st())
    return dict((k, v.cpu().numpy()) for k, v in out.items())


@pytest.mark.parametrize('seed,n_img,n_cls', [(0, 24, 6), (1, 24, 6), (2, 24, 6), (9, 300, 12)])
def test_gather_and_evaluate_equal_the_host(seed, n_img, n_cls):
    gt, sizes, rows = synthetic_set(seed, n_img=n_img, n_cls=n_cls, big_rows=max(3, n_img // 20))
    names = ['COCO_val2014_%012d' % i for i in gt['image_ids']]
    batches = batches_of(n_img, seed)
    records, ref = host_reference(gt, sizes, rows, names, n_cls, batches)
    score, box, groups, counters = device_gather(sizes, rows, n_cls, batches)
    check_gather(score.cpu().numpy(), box.cpu().numpy(), groups.cpu().numpy(), counters.cpu().numpy(), records, names,
                 n_cls, batches)
    out = device_evaluate(score, box, groups, counters, gt, n_cls)
    check_bit_equal(out, ref)


def test_pool_overflow_is_flagged():
    n_cls = 3
    gt, sizes, rows = synthetic_set(7, n_img=6, n_cls=n_cls, big_rows=1)
    total = sum(min(len(r), 100) for r in rows)
    first = sum(min(len(r), 100) for r in rows[:3 * n_cls])
    _, _, _, counters = device_gather(sizes, rows, n_cls, [[0, 1, 2], [3, 4, 5]], pool_cap=total - 1)
    assert counters.cpu().tolist() == [first, 3 * n_cls, 0, 1]


# ---- end to end: mini meta model on a synthetic COCO set ------------------------------------------------------------
class _CopyLog(object):
    """Records the element count of every CUDA tensor read on the host through the Tensor API."""

    def __init__(self, monkeypatch):
        self.sizes = []
        for name in ('cpu', 'item', 'tolist', 'numpy', '__int__', '__float__', '__bool__', '__index__'):
            orig = getattr(torch.Tensor, name)

            def wrap(t, *a, _orig=orig, **k):
                if t.is_cuda:
                    self.sizes.append(t.numel())
                return _orig(t, *a, **k)
            monkeypatch.setattr(torch.Tensor, name, wrap)
        orig_to = torch.Tensor.to

        def to(t, *a, **k):
            r = orig_to(t, *a, **k)
            if t.is_cuda and not r.is_cuda:
                self.sizes.append(t.numel())
            return r
        monkeypatch.setattr(torch.Tensor, 'to', to)


def test_score_batches_device_equals_results_json(tmp_path, monkeypatch):
    sys.path.insert(0, G)
    from seeding import seeded_init, synth_masks
    from fewshot_detection_b200 import coco_eval as C, netcfg, valid as VA
    from fewshot_detection_b200.darknet_meta import Darknet
    torch.manual_seed(0)
    det, ler = netcfg.mini_dynamic_blocks(128, 16), netcfg.mini_reweighting_blocks(64, 16, 512)
    m = Darknet([dict(b) for b in det], [dict(b) for b in ler])
    seeded_init(m, 3)
    m = m.cuda().eval()
    classes = ['bird', 'bus', 'cow']
    n_cls, bs, n_img = len(classes), 4, 26
    rs = np.random.RandomState(4)
    names = ['COCO_val2014_%012d' % (3 * k + 1) for k in range(n_img)]
    sizes = dict((n, (500, 375) if k % 3 else (353, 500)) for k, n in enumerate(names))
    g = torch.Generator().manual_seed(5)
    meta = [(torch.rand(n_cls, 3, 64, 64, generator=g).cuda(), torch.from_numpy(synth_masks(n_cls, 64, 6)).cuda(),
             list(range(n_cls))) for _ in range(2)]
    images = [(torch.rand(len(names[b:b + bs]), 3, 128, 128, generator=g).cuda(), names[b:b + bs],
               [sizes[n] for n in names[b:b + bs]]) for b in range(0, n_img, bs)]
    # ground truth that the random model partly finds: boxes near some of its own detections, plus random boxes
    dw = VA.ensemble_dynamic_weights(m, meta, n_cls)
    found = dict((n, []) for n in names)
    for x, ids, sz in images:
        for r in C.detection_records(VA.detect(m, x, dw, n_cls), ids, sz, n_cls):
            found[r[0]].append((r[1], r[3]))
    objs, k = [], 0
    for i, n in enumerate(names):
        W, H = sizes[n]
        picks = [found[n][j] for j in rs.choice(len(found[n]), min(len(found[n]), rs.randint(0, 5)), replace=False)]
        picks += [(rs.randint(n_cls), [rs.uniform(0, W / 2), rs.uniform(0, H / 2), rs.uniform(8, W / 2),
                                       rs.uniform(8, H / 2)]) for _ in range(rs.randint(0, 2))]
        for c, b in picks:
            b = [float(v) for v in np.array(b) + rs.normal(0, 3, 4)]
            k += 1
            objs.append({'id': k, 'image_id': 3 * i + 1, 'category_id': 2 * c + 1, 'bbox': b,
                         'area': abs(b[2] * b[3]) * rs.uniform(0.6, 1.0), 'iscrowd': int(rs.rand() < 0.1)})
    data = {'images': [{'id': 3 * i + 1, 'file_name': n + '.jpg'} for i, n in enumerate(names)],
            'categories': [{'id': 2 * c + 1, 'name': classes[c]} for c in range(n_cls)], 'annotations': objs}
    path = str(tmp_path / 'instances_synth.json')
    with open(path, 'w') as f:
        json.dump(data, f)
    gt = C.load_coco_annotations(path, names, classes)
    torch.cuda.synchronize()
    # device path, host reads logged
    ev = C.DeviceCocoEval(classes, names, gt)
    log = _CopyLog(monkeypatch)
    dev = VA.score_batches(m, meta, images, ev, novel_classes=('cow',))
    monkeypatch.undo()
    assert max(log.sizes) <= 10 * 101 * n_cls * 4 * 3, log.sizes              # counters, precision, recall, scalars
    n_det = int(ev.counters[0])
    assert n_det > 300 and not any(s == n_det or s == 4 * n_det for s in log.sizes)
    # results json of the same detections, scored on the host
    ev2 = C.DeviceCocoEval(classes, names, gt)
    f = io.StringIO()
    again = VA.score_batches(m, meta, images, ev2, out=f, novel_classes=('cow',))
    results = json.loads(f.getvalue())
    assert len(results) == n_det
    host = C.coco_evaluate(gt, results, names, classes, novel_classes=('cow',))
    check_bit_equal(dev, host)
    check_bit_equal(again, host)
    assert dev['all'] == host['all'] and dev['base'] == host['base'] and dev['novel'] == host['novel']
    assert dev['ap'] == host['ap'] and 0 < dev['all'][0] < 1
    print('device COCO stats', dev['all'])


# ---- a minival-sized pass ---------------------------------------------------------------------------------------------
MA, MH, MW = 5, 3, 3                                   # anchors and grid of the minival rows: 45 slots per row


def minival_set(n_img=5000, n_cls=80, kept=30, seed=0):
    """Ground truth (about 7 objects per image, crowd ~1%, json area = box area x [0.6, 1]) and per batch of 64 images
    the survivors as cand [N, kept, 8] / keep / keep_count: ~`kept` boxes per row, some near the row's objects, scores
    rounded to 1/4096 (ties)."""
    rs = np.random.RandomState(seed)
    sizes = np.stack([rs.randint(300, 641, n_img), rs.randint(300, 641, n_img)], 1)
    anns = []
    for i in range(n_img):
        W, H = sizes[i]
        n = rs.randint(1, 14)
        cls = rs.randint(0, n_cls, n)
        wh = np.exp(rs.uniform(np.log(6), np.log(W / 1.5), (n, 2)))
        xy = rs.uniform(0, 1, (n, 2)) * (np.array([W, H]) - wh)
        anns.append([(int(c), [float(v) for v in np.r_[p, s]], float(s[0] * s[1] * rs.uniform(0.6, 1.0)),
                      int(rs.rand() < 0.01)) for c, p, s in zip(cls, xy, wh)])
    gt = {'image_ids': list(range(1, n_img + 1)), 'category_ids': list(range(1, n_cls + 1)), 'anns': anns}
    batches = []
    for b0 in range(0, n_img, 64):
        imgs = list(range(b0, min(b0 + 64, n_img)))
        N = len(imgs) * n_cls
        kc = rs.randint(kept // 2, 3 * kept // 2 + 1, N).astype(np.int32)
        cand = np.zeros((N, MA * MH * MW, 8), dtype=np.float32)
        wh = sizes[imgs].repeat(n_cls, 0)[:, None, :]                              # [N, 1, 2] image (W, H)
        size = np.exp(rs.uniform(np.log(4), np.log(300), (N, cand.shape[1], 2)))
        ctr = rs.uniform(0, 1, (N, cand.shape[1], 2)) * wh
        for j, i in enumerate(imgs):
            for c, box, _, _ in anns[i]:
                r = j * n_cls + c
                s = rs.randint(0, kc[r])
                ctr[r, s] = [box[0] + box[2] / 2, box[1] + box[3] / 2] * rs.normal(1, 0.03, 2)
                size[r, s] = np.array(box[2:]) * rs.normal(1, 0.06, 2)
        cand[..., 0:2] = ctr / wh * np.array([MW, MH])
        cand[..., 2:4] = size / wh * np.array([MW, MH])
        cand[..., 4] = np.round(rs.uniform(0, 1, cand.shape[:2]) * 4096) / 4096
        cand[..., 5] = 1.0
        keep = np.tile(np.arange(cand.shape[1], dtype=np.int32), (N, 1))
        batches.append((imgs, cand, keep, kc, sizes[imgs].astype(np.float64)))
    return gt, batches


def host_records(batches, n_cls, classes):
    """detection_records' arithmetic, vectorised, for the rows of `classes` only: results json dicts."""
    for imgs, cand, keep, kc, size in batches:
        v = cand.astype(np.float64)
        bx, by, bw, bh = v[..., 0] / MW, v[..., 1] / MH, v[..., 2] / MW, v[..., 3] / MH
        width = size.repeat(n_cls, 0)[:, 0:1]
        height = size.repeat(n_cls, 0)[:, 1:2]
        x1, y1 = (bx - bw / 2.0) * width, (by - bh / 2.0) * height
        x2, y2 = (bx + bw / 2.0) * width, (by + bh / 2.0) * height
        score = v[..., 4] * v[..., 5]
        for j, i in enumerate(imgs):
            for c in classes:
                r = j * n_cls + c
                for s in np.argsort(-score[r, :kc[r]], kind='mergesort')[:100]:
                    yield {'image_id': i + 1, 'category_id': c + 1, 'score': float(score[r, s]),
                           'bbox': [float(x1[r, s]), float(y1[r, s]), float(x2[r, s] - x1[r, s]), float(y2[r, s] - y1[r, s])]}


def test_minival_sized_pass_equals_the_host_on_sampled_classes():
    import time
    from fewshot_detection_b200 import coco_eval as C
    from fewshot_detection_b200 import utils as U
    n_img, n_cls = 5000, 80
    gt, batches = minival_set(n_img, n_cls)
    names = ['COCO_val2014_%012d' % i for i in gt['image_ids']]
    classes = ['c%d' % k for k in range(n_cls)]
    ev = C.DeviceCocoEval(classes, names, gt)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for imgs, cand, keep, kc, size in batches:
        N = len(kc)
        d = U.Detections(torch.from_numpy(cand).cuda(), torch.from_numpy(kc).cuda(), None, N, MA, 1, MH, MW, False, True,
                         0.005)
        d.keep, d.keep_count = torch.from_numpy(keep).cuda(), torch.from_numpy(kc).cuda()
        ev.add(d, [names[i] for i in imgs], [tuple(s) for s in size])
    dev = ev.result()
    t_dev = time.perf_counter() - t0
    n_det = int(ev.counters[0])
    assert n_det > 25 * n_img * n_cls
    pick = sorted(np.random.RandomState(1).choice(n_cls, 8, replace=False).tolist())
    sub_gt = {'image_ids': gt['image_ids'], 'category_ids': [gt['category_ids'][c] for c in pick],
              'anns': [[(pick.index(c), b, a, cr) for c, b, a, cr in objs if c in pick] for objs in gt['anns']]}
    t0 = time.perf_counter()
    host = C.coco_evaluate(sub_gt, host_records(batches, n_cls, pick), names, [classes[c] for c in pick])
    t_host = time.perf_counter() - t0
    check_bit_equal({'precision': dev['precision'][:, :, pick], 'recall': dev['recall'][:, pick]}, host)
    assert (host['precision'] > 0).any()
    print('minival-sized pass: %d records, device %.3f s (80 classes), host %.1f s (8 classes)' % (n_det, t_dev, t_host))
