"""Test-time augmentation on the GPU (valid.detect_tta, utils.MergedDetections, the *_merged kernels):

  * the plan [(416, 0)] writes what the single-pass path writes: result lines, the VOC and COCO pools and result
    dicts, and the per-image selection, byte for byte;
  * tta_inputs: per side the evaluation batcher's input, a flipped pass torch.flip of it;
  * full-size head outputs (voc64, coco8, conf 0.005) at the passes {320, 416, 608} x flip: survivors, their order and
    the written lines equal the oracle built from the passes' own box lists (mirrored, concatenated in pass order,
    suppressed by the reference's nms);
  * device VOC AP of a TTA evaluation equals the host evaluator on its result files, and device COCO the host
    evaluator on its results json;
  * a TTA evaluation split over several evaluators and merged equals one evaluator, bit for bit;
  * the detection command with --tta-sides / --tta-flip end to end."""
import io
import json
import os
import sys

import numpy as np
import pytest
import torch

from test_gpu_eval_shard import bits, make_set, split, voc_recs

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


@pytest.fixture(scope='module')
def model():
    from test_gpu_zz_eval_pass import make_model
    return make_model(501, True)


def vectors(m, sup, n_cls, seed):
    from test_gpu_zz_eval_pass import support_batches
    from fewshot_detection_b200 import valid as VA
    return VA.ensemble_dynamic_weights(m, support_batches(sup, n_cls, seed), n_cls)


def pool_bytes(ev):
    """Records, groups, and the record / group counts and error flags (counters[2], the first group of the last batch
    added, is 0 after a merge)."""
    n, g = (int(v) for v in ev.counters[:2])
    c = ev.counters.cpu().numpy()
    return (ev.key[:n].cpu().numpy().tobytes(), ev.box[:n].cpu().numpy().tobytes(), ev.groups[:g].cpu().numpy().tobytes(),
            c[[0, 1, 3]].tobytes())


def test_one_pass_equals_the_single_pass_path(model):
    from test_gpu_zz_eval_pass import query_batch
    from fewshot_detection_b200 import coco_eval as C, valid as VA, voc_eval as V
    n_cls, B = 20, 16
    dw = vectors(model, (64,), n_cls, 41)
    x = query_batch(B, 42).cuda()
    gt, sizes, _, names, classes, _ = make_set(3, B, n_cls)
    one = VA.detect(model, x, dw, n_cls)
    tta = VA.detect_tta(model, [x], dw, n_cls, [(416, 0)])
    assert not tta.overflowed() and torch.equal(tta.count, one.count)
    assert VA.detection_lines(tta, names, sizes, n_cls) == VA.detection_lines(one, names, sizes, n_cls)
    assert C.detection_records(tta, names, sizes, n_cls) == C.detection_records(one, names, sizes, n_cls)
    for max_det in (100, 3):
        a, b = tta.select(n_cls, sizes, max_det).host(), one.select(n_cls, sizes, max_det).host()
        assert all(u.tobytes() == v.tobytes() for u, v in zip(a, b))
    recs = voc_recs(gt, names, classes)
    for make, kw in ((lambda: V.DeviceVocEval(classes, names, recs), dict(use_07_metric=True, curves=True)),
                     (lambda: C.DeviceCocoEval(classes, names, gt), {})):
        e1, e2 = make(), make()
        e1.add(one, names, sizes)
        e2.add(tta, names, sizes)
        assert pool_bytes(e1) == pool_bytes(e2) and int(e1.counters[0]) > 1000
        r1, r2 = e1.result(**kw), e2.result(**kw)
        assert repr(r1) == repr(r2)


def test_flipped_inputs_are_torch_flip():
    from fewshot_detection_b200 import valid as VA
    from fewshot_detection_b200.dataset import DetectionBatcher
    rs = np.random.RandomState(7)
    arrays = [rs.randint(0, 256, (h, w, 3)).astype(np.uint8) for w, h in ((500, 375), (97, 311), (640, 480))]
    db = DetectionBatcher([(a, np.zeros((0, 5))) for a in arrays], shape=(416, 416), shuffle=False, train=False,
                          batch_size=3)
    passes = [(416, 0), (416, 1), (320, 1), (608, 0), (320, 0)]
    got = VA.tta_inputs(db, range(3), passes)
    for (side, flip), x in zip(passes, got):
        want = DetectionBatcher([(a, np.zeros((0, 5))) for a in arrays], shape=(side, side), shuffle=False,
                                train=False, batch_size=3).batch(range(3))[0]
        if flip:
            want = torch.flip(want, dims=[3])
        assert x.shape == (3, 3, side, side) and torch.equal(x, want), (side, flip)


def fast_nms(row, thresh):
    """oracle.utils.nms restated with numpy float64 vectors (same operation order, IEEE, no contraction): kept indices."""
    box = np.array([b[:4] for b in row], dtype=np.float64).reshape(-1, 4)
    det = np.array([b[4] for b in row], dtype=np.float64)
    order = np.argsort((1 - det).astype(np.float32), kind='stable')
    alive = det[order] > 0
    b = box[order]
    x1, x2 = b[:, 0] - b[:, 2] / 2.0, b[:, 0] + b[:, 2] / 2.0
    y1, y2 = b[:, 1] - b[:, 3] / 2.0, b[:, 1] + b[:, 3] / 2.0
    out = []
    for i in range(len(row)):
        if not alive[i]:
            continue
        out.append(int(order[i]))
        j = slice(i + 1, None)
        uw = np.maximum(x2[i], x2[j]) - np.minimum(x1[i], x1[j])
        uh = np.maximum(y2[i], y2[j]) - np.minimum(y1[i], y1[j])
        cw = b[i, 2] + b[j, 2] - uw
        ch = b[i, 3] + b[j, 3] - uh
        carea = cw * ch
        with np.errstate(divide='ignore', invalid='ignore'):
            iou = np.where((cw <= 0) | (ch <= 0), 0.0, carea / (b[i, 2] * b[i, 3] + b[j, 2] * b[j, 3] - carea))
        alive[j] &= ~(iou > thresh)
    return out


# the oracle (Python lists) runs on the rows of a few images of each batch; the device runs every row
@pytest.mark.parametrize('sup,B,n_cls,images', [pytest.param((64, 8), 64, 20, (0, 37, 63), id='voc64'),
                                                pytest.param((64, 32), 8, 80, (0, 5), id='coco8')])
def test_plan_equals_the_oracle_on_full_size_head_outputs(model, sup, B, n_cls, images):
    from oracle import utils as OU
    from fewshot_detection_b200 import valid as VA
    from fewshot_detection_b200.utils import MergedDetections, region_detections
    passes = VA.tta_plan([320, 416, 608], True)
    dw = vectors(model, sup, n_cls, 51)
    g = torch.Generator().manual_seed(52)
    base = dict((s, torch.rand(B, 3, s, s, generator=g).cuda()) for s in (320, 416, 608))
    inputs = [torch.flip(base[s], dims=[3]) if f else base[s] for s, f in passes]
    N = B * n_cls
    merged = MergedDetections(N, VA.tta_capacity(model, passes), inputs[0].device)
    picked = [b * n_cls + i for b in images for i in range(n_cls)]
    rows = dict((n, []) for n in picked)
    with torch.no_grad():
        for p, ((side, flip), x) in enumerate(zip(passes, inputs)):
            d = region_detections(model.detect_forward(x, dw), 0.005, model.num_classes, model.anchors,
                                  model.num_anchors, 0, 1, n_models=n_cls)
            merged.add_pass(d, side, flip)
            count, cand, dense = d._fetch()                # the pass's box lists, as Detections.boxes() builds them
            for n in picked:
                for t in range(int(count[n])):
                    b = d._box(n, t, cand, dense) + [(p, t)]
                    if flip:
                        b[0] = 1.0 - b[0]
                    rows[n].append(b)
    merged.nms(0.45)
    public = VA.detect_tta(model, inputs, dw, n_cls, passes)
    assert torch.equal(public.keep_count, merged.keep_count) and torch.equal(public.count, merged.count)
    kc = merged.keep_count.cpu().numpy()
    keep = merged.keep.cpu().numpy()
    pk = public.keep.cpu().numpy()
    assert all(np.array_equal(pk[n, :kc[n]], keep[n, :kc[n]]) for n in range(N))
    counts = merged.count.cpu().numpy()
    assert [int(counts[n]) for n in picked] == [len(rows[n]) for n in picked]
    want = dict((n, fast_nms(rows[n], 0.45)) for n in picked)
    for n in picked:
        assert keep[n, :kc[n]].tolist() == want[n], n
    # the reference's own nms on the shortest non-empty rows and on one long row pins the restatement
    lengths = sorted((len(rows[n]), n) for n in picked if rows[n])
    for _, n in lengths[:6] + [lengths[len(lengths) // 2]]:
        ref = OU.nms([list(b) for b in rows[n]], 0.45)
        assert [b[7] for b in ref] == [rows[n][s][7] for s in want[n]], n
    # written values: the result lines of the merged survivors are the oracle's lines of its survivors
    sizes = [(int(w), int(h)) for w, h in np.random.RandomState(B).randint(32, 1200, (B, 2))]
    ids = ['img%03d' % b for b in range(B)]
    lines = VA.detection_lines(merged, ids, sizes, n_cls)
    for i in range(n_cls):
        ref = []
        for b in images:
            ref += OU.detection_lines([rows[b * n_cls + i][s][:7] for s in want[b * n_cls + i]], ids[b], *sizes[b])
        assert [l for l in lines[i] if int(l.split()[0][3:]) in images] == ref, i
    print('%s: merged rows up to %d candidates (%d over 4096), %d survivors' %
          (sys._getframe().f_code.co_name, counts.max(), (counts > 4096).sum(), kc.sum()))


def mini_model():
    sys.path.insert(0, G)
    from seeding import seeded_init
    from fewshot_detection_b200 import netcfg
    from fewshot_detection_b200.darknet_meta import Darknet
    det, ler = netcfg.mini_dynamic_blocks(128, 16), netcfg.mini_reweighting_blocks(64, 16, 512)
    m = Darknet([dict(b) for b in det], [dict(b) for b in ler])
    seeded_init(m, 3)
    return m.cuda().eval()


MINI_PLAN = [(128, 0), (128, 1), (96, 0), (160, 1)]


def mini_batches(names, sizes, n_cls, bs, seed):
    from seeding import synth_masks
    g = torch.Generator().manual_seed(seed)
    meta = [(torch.rand(n_cls, 3, 64, 64, generator=g).cuda(), torch.from_numpy(synth_masks(n_cls, 64, 6)).cuda(),
             list(range(n_cls))) for _ in range(2)]
    images = []
    for b in range(0, len(names), bs):
        k = len(names[b:b + bs])
        base = dict((s, torch.rand(k, 3, s, s, generator=g).cuda()) for s, _ in MINI_PLAN)
        images.append(([torch.flip(base[s], dims=[3]) if f else base[s] for s, f in MINI_PLAN], names[b:b + bs],
                       [sizes[n] for n in names[b:b + bs]]))
    return meta, images


def test_device_scores_equal_the_host_on_tta_result_files(tmp_path):
    from test_voc_eval_host_emul import host_class_eval
    from fewshot_detection_b200 import coco_eval as C, valid as VA, voc_eval as V
    m = mini_model()
    classes = ['bird', 'bus', 'cow']
    n_cls, bs, n_img = 3, 4, 22
    gt, _, _, names, _, _ = make_set(5, n_img, n_cls)
    sizes = dict((n, (500, 375) if k % 3 else (353, 500)) for k, n in enumerate(names))
    meta, images = mini_batches(names, sizes, n_cls, bs, 6)
    # VOC: the TTA result files, scored on the host, against the device pool
    recs = voc_recs(gt, names, classes)
    prefix = str(tmp_path / 'res')
    VA.valid_batches(m, meta, images, classes, prefix, 'comp4_det_test_', tta=MINI_PLAN)
    dev = VA.score_batches(m, meta, images, V.DeviceVocEval(classes, names, recs), tta=MINI_PLAN, use_07_metric=True)
    n_lines = 0
    for c in classes:
        with open(os.path.join(prefix, 'comp4_det_test_%s.txt' % c)) as f:
            rows = [l.strip().split(' ') for l in f]
        lines = [(r[0], float(r[1])) + tuple(float(z) for z in r[2:]) for r in rows]
        n_lines += len(lines)
        assert dev['ap'][c] == host_class_eval(lines, recs, names, c)[4], c
    assert n_lines > 300
    # COCO: the results json of the same detections, scored on the host
    f = io.StringIO()
    dev = VA.score_batches(m, meta, images, C.DeviceCocoEval(classes, names, gt), out=f, tta=MINI_PLAN)
    host = C.coco_evaluate(gt, json.loads(f.getvalue()), names, classes)
    assert np.array_equal(bits(dev['precision']), bits(host['precision']))
    assert np.array_equal(bits(dev['recall']), bits(host['recall']))
    assert dev['all'] == host['all'] and dev['ap'] == host['ap']


@pytest.mark.parametrize('world', [2, 3])
def test_split_tta_evaluation_merges_to_one_evaluator(world):
    from fewshot_detection_b200 import coco_eval as C, valid as VA, voc_eval as V
    m = mini_model()
    classes = ['bird', 'bus', 'cow']
    n_cls, bs, n_img = 3, 3, 15
    gt, _, _, names, _, _ = make_set(8, n_img, n_cls)
    sizes = dict((n, (640, 480)) for n in names)
    meta, images = mini_batches(names, sizes, n_cls, bs, 9)
    dw = VA.ensemble_dynamic_weights(m, meta, n_cls)
    dets = [(VA.detect_tta(m, x, dw, n_cls, MINI_PLAN), ids, sz) for x, ids, sz in images]
    recs = voc_recs(gt, names, classes)
    for make, kw in ((lambda: V.DeviceVocEval(classes, names, recs), dict(use_07_metric=False, curves=True)),
                     (lambda: C.DeviceCocoEval(classes, names, gt), {})):
        one = make()
        for d, ids, sz in dets:
            one.add(d, ids, sz)
        parts = []
        for block in split(dets, world):
            ev = make()
            for d, ids, sz in block:
                ev.add(d, ids, sz)
            parts.append(ev)
        merged = type(one).merge(parts)
        assert pool_bytes(merged) == pool_bytes(one)
        assert repr(merged.result(**kw)) == repr(one.result(**kw))


def test_detect_command_with_tta_end_to_end(tmp_path):
    from PIL import Image
    from test_detect_command import tool
    from seeding import seeded_init
    from fewshot_detection_b200 import netcfg, valid as VA
    from fewshot_detection_b200.cfg import cfg, parse_cfg
    from fewshot_detection_b200.darknet_meta import Darknet
    from fewshot_detection_b200.dataset import DetectionBatcher
    from fewshot_detection_b200.image import decode_many
    saved = dict(cfg)
    try:
        root = str(tmp_path)
        det, ler = os.path.join(root, 'det.cfg'), os.path.join(root, 'ler.cfg')
        netcfg.write_cfg(netcfg.mini_dynamic_blocks(128, 16), det)
        netcfg.write_cfg(netcfg.mini_reweighting_blocks(64, 16, 512), ler)
        cfg.config_meta(parse_cfg(ler)[0])
        cfg.config_net(parse_cfg(det)[0])
        m = Darknet(parse_cfg(det), parse_cfg(ler))
        seeded_init(m, 7)
        weights = os.path.join(root, 'w.weights')
        m.save_weights(weights)
        names = ['cat', 'dog']
        with open(os.path.join(root, 'c.names'), 'w') as f:
            f.write('\n'.join(names) + '\n')
        rw = os.path.join(root, 'rw.pkl')
        VA.save_reweighting_vectors(rw, [torch.randn(2, 512, 1, 1, generator=torch.Generator().manual_seed(8)) * 0.1])
        rs = np.random.RandomState(9)
        paths = []
        for k, (w, h) in enumerate([(200, 150), (97, 311), (640, 480)]):
            p = os.path.join(root, 'im%d.png' % k)
            Image.fromarray(rs.randint(0, 256, (h, w, 3)).astype(np.uint8)).save(p)
            paths.append(p)
        out = os.path.join(root, 'out')
        args = [det, ler, weights] + paths + ['--rw', rw, '--names', os.path.join(root, 'c.names'), '--conf', '0.005',
                                             '--max-det', '9', '--out', out, '--tta-sides', '128,96', '--tta-flip']
        assert tool('detect_b200').main(args) == 0
        assert not os.path.exists(out) and os.path.isdir(out + '_tta')
        # the same plan through the API
        m2 = Darknet(parse_cfg(det), parse_cfg(ler))
        m2.load_weights(weights)
        m2 = m2.cuda().eval()
        dw = [torch.from_numpy(a).cuda() for a in VA.load_reweighting_vectors(rw)]
        arrays = decode_many(paths)
        db = DetectionBatcher([(a, np.zeros((0, 5))) for a in arrays], shape=(128, 128), shuffle=False, train=False,
                              batch_size=3)
        plan = [(128, 0), (128, 1), (96, 0), (96, 1)]
        sizes = [(a.shape[1], a.shape[0]) for a in arrays]
        want = VA.detect_tta(m2, VA.tta_inputs(db, range(3), plan), dw, 2, plan, 0.005, 0.4).select(2, sizes, 9)
        n_lines = 0
        for p, rows in zip(paths, want.lists(names)):
            with open(os.path.join(out + '_tta', os.path.splitext(os.path.basename(p))[0] + '.txt')) as f:
                got = [l.rstrip('\n').rsplit(' ', 5) for l in f]
            assert [[g[0]] + [float(v) for v in g[1:]] for g in got] == [[r[0]] + list(r[1:]) for r in rows]
            n_lines += len(rows)
        assert n_lines > 0
    finally:
        cfg.clear()
        cfg.update(saved)
