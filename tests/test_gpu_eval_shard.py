"""Sharded evaluation on one device (fsdet_voc_merge / fsdet_coco_merge through DeviceVocEval.merge /
DeviceCocoEval.merge) and the trainer's checkpoint evaluation.

  * the seeded detection sets of the device-scoring tests (heavy score ties, rows with more than 100 survivors), their
    batches split in rank order over 2-4 evaluators and merged: AP, rec / prec and COCO precision / recall bit-equal
    to one evaluator given every batch;
  * an image added to two evaluators is reported by the merge, not scored;
  * MetaTrainer.fit over two checkpoint epochs of K graphed steps at neg = 1, with the evaluation callback run by
    train_epoch after each: the losses, parameters, momentum buffers, BatchNorm buffers and random-number states of
    the same run without the callback, bit for bit; the engine's weight planes are neither rebuilt nor moved."""
import random
import sys
import os

import numpy as np
import pytest
import torch

from test_coco_eval_host_emul import batches_of, detections, synthetic_set, A_, H_, W_

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def device_dets(rows, images, n_cls):
    from fewshot_detection_b200 import utils as U
    cand, keep, kc = detections(rows, images, n_cls)
    N = len(kc)
    d = U.Detections(torch.from_numpy(cand).cuda(), torch.full((N,), cand.shape[1], dtype=torch.int32).cuda(), None, N,
                     A_, 1, H_, W_, False, True, 0.005)
    d.keep, d.keep_count, d._nms_thresh = torch.from_numpy(keep).cuda(), torch.from_numpy(kc).cuda(), 0.45
    return d


def voc_recs(gt, names, classes):
    """The COCO set's ground truth as VOC annotations (crowd objects as `difficult`)."""
    recs = {}
    for i, n in enumerate(names):
        recs[n] = [{'name': classes[c], 'difficult': crowd,
                    'bbox': [int(b[0]), int(b[1]), int(b[0] + b[2]), int(b[1] + b[3])]} for c, b, _, crowd in gt['anns'][i]]
    return recs


def make_set(seed, n_img, n_cls):
    gt, sizes, rows = synthetic_set(seed, n_img=n_img, n_cls=n_cls, big_rows=max(3, n_img // 20))
    names = ['COCO_val2014_%012d' % i for i in gt['image_ids']]
    classes = ['c%d' % k for k in range(n_cls)]
    assert max(len(r) for r in rows) > 100
    return gt, sizes, rows, names, classes, batches_of(n_img, seed)


def fill(ev, rows, sizes, names, n_cls, batches):
    for images in batches:
        ev.add(device_dets(rows, images, n_cls), [names[i] for i in images], [sizes[i] for i in images])
    return ev


def split(batches, world):
    from fewshot_detection_b200.shard import shard_range
    return [batches[slice(*shard_range(len(batches), 1, world, r))] for r in range(world)]


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).reshape(-1).view(np.uint64)


@pytest.mark.parametrize('seed,n_img,n_cls,world', [(0, 24, 6, 2), (1, 24, 6, 3), (9, 300, 12, 4), (2, 24, 6, 16)])
def test_voc_merged_pool_equals_one_evaluator(seed, n_img, n_cls, world):
    from fewshot_detection_b200 import voc_eval as V
    gt, sizes, rows, names, classes, batches = make_set(seed, n_img, n_cls)
    recs = voc_recs(gt, names, classes)
    one = fill(V.DeviceVocEval(classes, names, recs), rows, sizes, names, n_cls, batches)
    parts = [fill(V.DeviceVocEval(classes, names, recs), rows, sizes, names, n_cls, b) for b in split(batches, world)]
    merged = V.DeviceVocEval.merge(parts)
    n = int(one.counters[0])
    assert merged.counters.tolist()[:2] == one.counters.tolist()[:2] and n > 1000
    assert torch.equal(merged.key[:n], one.key[:n]) and torch.equal(merged.box[:n], one.box[:n])
    for use07 in (True, False):
        a = merged.result(use07, novel_classes=('c1',), curves=True)
        b = one.result(use07, novel_classes=('c1',), curves=True)
        for k in ('mean', 'mean_base', 'mean_novel'):
            assert np.array_equal(bits(np.float64(a[k])), bits(np.float64(b[k]))), k
        assert np.array_equal(bits([a['ap'][c] for c in classes]), bits([b['ap'][c] for c in classes]))
        for c in classes:
            assert np.array_equal(bits(a['rec'][c]), bits(b['rec'][c])) and np.array_equal(bits(a['prec'][c]), bits(b['prec'][c]))
    assert 0 < b['ap']['c0'] < 1


@pytest.mark.parametrize('seed,n_img,n_cls,world', [(0, 24, 6, 2), (1, 24, 6, 4), (9, 300, 12, 3), (2, 24, 6, 16)])
def test_coco_merge_equals_one_evaluator(seed, n_img, n_cls, world):
    from fewshot_detection_b200 import coco_eval as C
    gt, sizes, rows, names, classes, batches = make_set(seed, n_img, n_cls)
    one = fill(C.DeviceCocoEval(classes, names, gt), rows, sizes, names, n_cls, batches)
    parts = [fill(C.DeviceCocoEval(classes, names, gt), rows, sizes, names, n_cls, b) for b in split(batches, world)]
    merged = C.DeviceCocoEval.merge(parts)
    a, b = merged.result(novel_classes=('c2',)), one.result(novel_classes=('c2',))
    assert np.array_equal(bits(a['precision']), bits(b['precision']))
    assert np.array_equal(bits(a['recall']), bits(b['recall']))
    assert a['all'] == b['all'] and a['novel'] == b['novel'] and a['ap'] == b['ap'] and b['all'][0] > 0


def test_merge_reports_an_image_on_two_evaluators():
    from fewshot_detection_b200 import coco_eval as C, voc_eval as V
    gt, sizes, rows, names, classes, _ = make_set(3, 12, 4)
    for ev in (V.DeviceVocEval(classes, names, voc_recs(gt, names, classes)), C.DeviceCocoEval(classes, names, gt)):
        p0 = fill(ev.empty_like(), rows, sizes, names, 4, [[0, 1], [2, 3]])
        p1 = fill(ev.empty_like(), rows, sizes, names, 4, [[3, 4]])
        merged = type(ev).merge([p0, p1])
        assert int(merged.counters[3]) == 2
        with pytest.raises(RuntimeError, match='two ranks'):
            merged.result()


# ---- the trainer's checkpoint evaluation leaves training as it was ---------------------------------------------------
def test_checkpoint_evaluation_leaves_training_unchanged():
    sys.path.insert(0, G)
    from fewshot_detection_b200 import netcfg, trainer as T, valid as VA
    from fewshot_detection_b200.cfg import cfg
    from fewshot_detection_b200.darknet_meta import Darknet
    from fewshot_detection_b200.optim import FusedSGD
    from seeding import seeded_init, synth_targets, synth_masks
    bs, cs, K = 6, 5, 3

    def batch(it):
        g = torch.Generator().manual_seed(100 + it)
        x = torch.rand(bs, 3, 128, 128, generator=g).cuda()
        metax = torch.rand(cs, 3, 64, 64, generator=g).cuda()
        return x, metax, torch.from_numpy(synth_masks(cs, 64, 200 + it)).cuda(), torch.from_numpy(synth_targets(bs, cs, 300 + it, max_gt=2))

    def evaluate(m, epoch):
        random.random()                                          # a loader that draws: restored by the trainer
        np.random.rand(3)
        g = torch.Generator().manual_seed(7)
        meta = [(torch.rand(cs, 3, 64, 64, generator=g).cuda(), torch.from_numpy(synth_masks(cs, 64, 9)).cuda(),
                 list(range(cs)))]
        dw = VA.ensemble_dynamic_weights(m, meta, cs)
        n = 0
        for k in range(2):
            d = VA.detect(m, torch.rand(4, 3, 128, 128, generator=g).cuda(), dw, cs)
            n += int(d.keep_count.sum())
        return 'detections %d' % n

    class Queries(object):                                       # the epoch's query batches
        def __init__(self, epoch):
            self.epoch = epoch

        def __len__(self):
            return K

        def __iter__(self):
            for i in range(K):
                x, _, _, tgt = batch(self.epoch * K + i)
                yield x, tgt

    class Supports(object):                                      # the epoch's support batches
        batch_size = cs

        def __init__(self, epoch):
            self.epoch = epoch

        def batch(self, r):
            return batch(self.epoch * K + r.start // cs)[1:3]

    def run(with_eval):
        m = Darknet(netcfg.mini_dynamic_blocks(128, 8), netcfg.mini_reweighting_blocks(64, 8, 256))
        seeded_init(m, 11)
        m = m.cuda().train()
        opt = FusedSGD(m.parameters(), lr=1e-3, momentum=0.9, dampening=0, weight_decay=5e-4)
        logs, epochs, results = [], [0, 0], []

        def queries(seen):
            epochs[0] += 1
            return Queries(epochs[0] - 1)

        def supports():
            epochs[1] += 1
            return Supports(epochs[1] - 1)
        tr = T.MetaTrainer(m, opt, 1e-3, bs, [0], [1], queries, supports, save_interval=1, world=1, log=logs.append,
                           use_graph=True, evaluate=evaluate if with_eval else None)
        assert tr.graphed is not None
        m.models[len(m.models) - 1].verbose = False
        tr.region_loss.seen = 20000
        unchecked = tr.evaluate_checkpoint

        def checked(epoch):                                      # what the hook in train_epoch must leave alone
            plans = [(r_, getattr(r_, '_wplan', None)) for r_ in (m._det, m._ler)]
            assert plans[0][1] is not None and plans[0][1]['n'] > 0          # the detector has tensor-core layers

            def plane_ptrs():
                return [[t.data_ptr() for v in (p or {}).get('by_id', {}).values() for part in v.values() if part
                         for t in part] for _, p in plans]
            planes = plane_ptrs()
            bn = [b.clone() for b in m.buffers()]
            r = unchecked(epoch)
            assert m.training
            assert all(torch.equal(a, b) for a, b in zip(bn, m.buffers()))          # BN statistics untouched
            assert all(getattr(r_, '_wplan', None) is p for r_, p in plans)         # the graphs' weight planes
            assert plane_ptrs() == planes and len(planes[0]) > 0
            results.append(r)
            return r
        tr.evaluate_checkpoint = checked
        random.seed(77)
        np.random.seed(78)
        tr.fit(0, 2)                                             # K steps, checkpoint epoch, K steps, checkpoint epoch
        torch.cuda.synchronize()
        if with_eval:
            assert len(results) == 2 and all(r.startswith('detections') for r in results)
            assert sum(1 for l in logs if l.startswith('evaluation at epoch')) == 2
        else:
            assert results == [None, None]
        return ([l.item() for l in tr.losses], [p.detach().clone() for p in m.parameters()],
                [opt.state[p]['momentum_buffer'].clone() for p in m.parameters()], [b.clone() for b in m.buffers()],
                random.random(), float(np.random.rand()))

    old = cfg.neg_ratio
    cfg.neg_ratio = 1
    try:
        plain, evald = run(False), run(True)
    finally:
        cfg.neg_ratio = old
    assert plain[0] == evald[0]
    for k in (1, 2, 3):
        assert len(plain[k]) == len(evald[k]) > 0
        assert all(torch.equal(a, b) for a, b in zip(plain[k], evald[k])), k
    assert plain[4:] == evald[4:]
