"""Device VOC AP (csrc/voc_eval.cu) through the C ABI and voc_eval.DeviceVocEval, on the GPU.

  * '%f' % x -> float() of millions of doubles, bit-exact;
  * tests/golden/voc_eval.npz (the reference's scripts/voc_eval.py): rec / prec equal, VOC07 AP equal, area AP within
    1e-12; synthetic sets with heavy ties against a stable-ranking copy of match_detections;
  * a mini meta model on a synthetic devkit: valid.score_batches against valid_batches + voc_eval.mean_ap on the
    written files (equal wherever a class has no tied confidences) and against the stable-ranking copy on the same
    lines (equal everywhere), with no per-detection data copied to the host."""
import os

import numpy as np
import pytest
import torch

from test_voc_eval_host_emul import (check_against_host, expected_round_trip, golden_case, host_class_eval,
                                     pack_lines, round_trip_inputs, synthetic_case)

pytestmark = pytest.mark.gpu

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
XML = '<annotation><filename>{name}.jpg</filename>{objs}</annotation>'
OBJ = ('<object><name>{cls}</name><pose>Unspecified</pose><truncated>0</truncated><difficult>{df}</difficult>'
       '<bndbox><xmin>{x1}</xmin><ymin>{y1}</ymin><xmax>{x2}</xmax><ymax>{y2}</ymax></bndbox></object>')


def _st():
    return torch.cuda.current_stream().cuda_stream


def device_evaluate(per_class, classes, imagenames, recs, ovthresh=0.5):
    from fewshot_detection_b200 import _lib, voc_eval as V
    keys, boxes, groups = pack_lines(per_class, imagenames)
    gt_ptr, gt_box, gt_diff = V.gt_tables(classes, imagenames, recs)
    n, n_cls, n_gt = len(keys), len(classes), len(gt_diff)
    d = dict((k, torch.from_numpy(np.ascontiguousarray(a)).cuda()) for k, a in
             (('keys', keys.view(np.int32)), ('boxes', boxes), ('groups', groups), ('gt_ptr', gt_ptr), ('gt_box', gt_box),
              ('gt_diff', gt_diff)))
    nbytes = _lib.lib.fsdet_voc_workspace_bytes(n, n_gt)
    ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device='cuda')
    out = dict(flags=torch.full((n,), 9, dtype=torch.uint8), order=torch.full((n,), -1, dtype=torch.int32),
               rec=torch.full((n,), -7.0, dtype=torch.float64), prec=torch.full((n,), -7.0, dtype=torch.float64),
               cls_count=torch.full((n_cls,), -1, dtype=torch.int32), npos=torch.full((n_cls,), -1, dtype=torch.int32),
               ap07=torch.full((n_cls,), -7.0, dtype=torch.float64), ap_area=torch.full((n_cls,), -7.0, dtype=torch.float64))
    out = dict((k, v.cuda()) for k, v in out.items())
    th = np.ascontiguousarray(V.VOC07_THRESHOLDS)
    p = lambda t: t.data_ptr() if t.numel() else None
    _lib.call('fsdet_voc_evaluate', p(d['keys']), p(d['boxes']), n, p(d['groups']), len(groups), p(d['gt_ptr']),
              p(d['gt_box']), p(d['gt_diff']), n_gt, n_cls, len(imagenames), ovthresh, th.ctypes.data, ws.data_ptr(), nbytes,
              p(out['flags']), p(out['order']), p(out['rec']), p(out['prec']), p(out['cls_count']), p(out['npos']),
              p(out['ap07']), p(out['ap_area']), _st())
    return dict((k, v.cpu().numpy()) for k, v in out.items())


def test_round6_equals_printf_round_trip():
    from fewshot_detection_b200 import _lib
    x = round_trip_inputs(4000000, seed=1)
    xd = torch.from_numpy(x).cuda()
    y = torch.empty_like(xd)
    n = torch.empty_like(xd)
    _lib.call('fsdet_voc_round6', xd.data_ptr(), y.data_ptr(), n.data_ptr(), len(x), _st())
    y, n = y.cpu().numpy(), n.cpu().numpy()
    want = expected_round_trip(x)
    bad = np.nonzero(y.view(np.uint64) != want.view(np.uint64))[0]
    assert bad.size == 0, [(repr(x[i]), repr(y[i]), repr(want[i])) for i in bad[:10]]
    small = np.abs(x) < 2.0 ** 33
    assert np.array_equal(n[small] / 1e6, y[small])
    k = len(x) - 15
    assert y[k] == 0.007812 and y[k + 1] == 0.023438 and y[k + 2] == -0.007812


def test_golden_reference_voc_eval():
    gold = np.load(os.path.join(G, 'voc_eval.npz'), allow_pickle=False)
    names, recs, classes, per_class = golden_case(gold)
    out = device_evaluate(per_class, classes, names, recs)
    start = 0
    for c, name in enumerate(classes):
        n = len(per_class[c])
        assert np.array_equal(out['rec'][start:start + n], gold['rec/%s/1' % name])
        assert np.array_equal(out['prec'][start:start + n], gold['prec/%s/1' % name])
        assert out['ap07'][c] == float(gold['ap/%s/1' % name])
        assert abs(out['ap_area'][c] - float(gold['ap/%s/0' % name])) <= 1e-12
        start += n
    check_against_host(out, per_class, classes, names, recs)


@pytest.mark.parametrize('seed,n_img,per_img', [(0, 40, 12), (1, 40, 12), (7, 600, 60)])
def test_heavy_ties_against_stable_host_copy(seed, n_img, per_img):
    names, recs, classes, per_class = synthetic_case(seed, n_img=n_img, per_img=per_img)
    out = device_evaluate(per_class, classes, names, recs)
    check_against_host(out, per_class, classes, names, recs)
    d, e = classes.index('d'), classes.index('e')
    assert out['npos'][d] == 0 and np.isnan(out['ap_area'][d]) and out['ap07'][d] == 0.0
    assert out['cls_count'][e] == 0 and out['ap07'][e] == 0.0 and out['ap_area'][e] == 0.0


# ---- end to end: mini meta model on a synthetic devkit ----------------------------------------------------------------
def write_devkit(root, names, recs):
    os.makedirs(os.path.join(root, 'Annotations'))
    for n in names:
        objs = ''.join(OBJ.format(cls=o['name'], df=o['difficult'], x1=o['bbox'][0], y1=o['bbox'][1], x2=o['bbox'][2],
                                  y2=o['bbox'][3]) for o in recs[n])
        with open(os.path.join(root, 'Annotations', n + '.xml'), 'w') as f:
            f.write(XML.format(name=n, objs=objs))
    with open(os.path.join(root, 'test.txt'), 'w') as f:
        f.write('\n'.join(names) + '\n')


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


def test_score_batches_device_ap_equals_result_files(tmp_path, monkeypatch):
    import sys
    sys.path.insert(0, G)
    from seeding import seeded_init, synth_masks
    from fewshot_detection_b200 import netcfg, valid as VA, voc_eval as V
    from fewshot_detection_b200.darknet_meta import Darknet
    torch.manual_seed(0)
    det, ler = netcfg.mini_dynamic_blocks(128, 16), netcfg.mini_reweighting_blocks(64, 16, 512)
    m = Darknet([dict(b) for b in det], [dict(b) for b in ler])
    seeded_init(m, 3)
    m = m.cuda().eval()
    classes = ['bird', 'bus', 'cow']
    n_cls, bs, n_img = len(classes), 4, 26                       # the last batch holds 2 images
    rs = np.random.RandomState(4)
    names = ['%06d' % (3 * k + 1) for k in range(n_img)]
    sizes = dict((n, (500, 375) if k % 3 else (353, 500)) for k, n in enumerate(names))
    root = str(tmp_path)
    g = torch.Generator().manual_seed(5)
    meta = [(torch.rand(n_cls, 3, 64, 64, generator=g).cuda(), torch.from_numpy(synth_masks(n_cls, 64, 6)).cuda(),
             list(range(n_cls))) for _ in range(2)]
    images = [(torch.rand(len(names[b:b + bs]), 3, 128, 128, generator=g).cuda(), names[b:b + bs],
               [sizes[n] for n in names[b:b + bs]]) for b in range(0, n_img, bs)]
    # ground truth that the random model partly finds: boxes near some of its own detections, plus random boxes
    VA.valid_batches(m, meta, images, classes, os.path.join(root, 'pre'), 'p_')
    found = dict((n, []) for n in names)
    for c in classes:
        with open(os.path.join(root, 'pre', 'p_%s.txt' % c)) as f:
            for l in f:
                r = l.split(' ')
                found[r[0]].append((c, [float(z) for z in r[2:6]]))
    recs = {}
    for n in names:
        W, H = sizes[n]
        objs = []
        picks = [found[n][k] for k in rs.choice(len(found[n]), min(len(found[n]), rs.randint(0, 4)), replace=False)]
        for _ in range(rs.randint(0, 2)):
            w, h = rs.randint(W // 3, W), rs.randint(H // 3, H)
            x1, y1 = rs.randint(1, W - w + 1), rs.randint(1, H - h + 1)
            picks.append((classes[rs.randint(n_cls)], [x1, y1, x1 + w - 1, y1 + h - 1]))
        for c, b in picks:
            b = np.array(b) + rs.normal(0, 3, 4)
            x1, y1 = int(np.clip(b[0], 1, W - 2)), int(np.clip(b[1], 1, H - 2))
            x2, y2 = int(np.clip(b[2], x1 + 1, W)), int(np.clip(b[3], y1 + 1, H))
            objs.append({'name': c, 'pose': 'Unspecified', 'truncated': 0, 'difficult': int(rs.rand() < 0.1),
                         'bbox': [x1, y1, x2, y2]})
        recs[n] = objs
    write_devkit(root, names, recs)
    torch.cuda.synchronize()
    # file path
    VA.valid_batches(m, meta, images, classes, os.path.join(root, 'results'), 'comp4_det_test_')
    detpath = os.path.join(root, 'results', 'comp4_det_test_{}.txt')
    annopath = os.path.join(root, 'Annotations', '{}.xml')
    files07 = V.mean_ap(detpath, annopath, os.path.join(root, 'test.txt'), classes, os.path.join(root, 'cache'), True)
    files_area = V.mean_ap(detpath, annopath, os.path.join(root, 'test.txt'), classes, os.path.join(root, 'cache'), False)
    # device path, host reads logged
    recs_loaded = V.load_annotations(annopath, names, os.path.join(root, 'cache'))
    ev = V.DeviceVocEval(classes, names, recs_loaded)
    log = _CopyLog(monkeypatch)
    dev07 = VA.score_batches(m, meta, images, ev, use_07_metric=True, novel_classes=('cow',))
    monkeypatch.undo()
    assert max(log.sizes) <= max(n_cls, 4), log.sizes          # counters, per-class results, scalars of the ensembling
    # the accumulator alone, from the CUDA trace: its only device-to-host copies are the record count read when the
    # pool is first sized, the counters and the per-class APs
    from torch.profiler import ProfilerActivity, profile
    dw = VA.ensemble_dynamic_weights(m, meta, n_cls)
    dets = [VA.detect(m, x, dw, n_cls) for x, _, _ in images]
    ev2 = V.DeviceVocEval(classes, names, recs_loaded)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for d, (_, ids, sz) in zip(dets, images):
            ev2.add(d, ids, sz)
        again = ev2.result(True, novel_classes=('cow',))
        torch.cuda.synchronize()
    names_seen = [e.name for e in prof.events()]
    dtoh = [n for n in names_seen if 'Memcpy' in n and ('DtoH' in n or 'Device -> P' in n)]
    assert len(dtoh) <= 3, dtoh
    assert any(n.startswith('void fsdet::voc_') or 'voc_match_kernel' in n for n in names_seen), sorted(set(names_seen))[:40]
    assert again == dev07
    dev_area = ev.result(False, curves=True)
    # the same lines, ranked stably on the host
    n_lines, tied = 0, []
    for c, name in enumerate(classes):
        with open(detpath.format(name)) as f:
            rows = [l.strip().split(' ') for l in f.readlines()]
        lines = [(r[0], float(r[1])) + tuple(float(z) for z in r[2:]) for r in rows]
        n_lines += len(lines)
        _, _, rec, prec, ap07, ap_area = host_class_eval(lines, recs_loaded, names, name)
        assert dev07['ap'][name] == ap07, name
        assert abs(dev_area['ap'][name] - ap_area) <= 1e-12, name
        assert np.array_equal(dev_area['rec'][name], rec) and np.array_equal(dev_area['prec'][name], prec), name
        if len(set(l[1] for l in lines)) == len(lines):
            assert dev07['ap'][name] == files07['ap'][name], name
            assert abs(dev_area['ap'][name] - files_area['ap'][name]) <= 1e-12, name
        else:
            tied.append(name)
    assert n_lines > 300 and int(ev.counters[0]) == n_lines
    assert 0 < dev07['mean'] < 1 and dev07['mean_novel'] == dev07['ap']['cow']
    # the result files of the device pass are the files valid_batches writes, byte for byte
    import io
    fps = [io.StringIO() for _ in classes]
    with_files = VA.score_batches(m, meta, images, V.DeviceVocEval(classes, names, recs_loaded), out=fps,
                                  use_07_metric=True, novel_classes=('cow',))
    assert with_files == dev07
    for name, f in zip(classes, fps):
        with open(detpath.format(name)) as g:
            assert f.getvalue() == g.read(), name
    print('device AP %s, files AP %s, %d lines, classes with tied confidences: %s'
          % (dev07['ap'], files07['ap'], n_lines, tied))
