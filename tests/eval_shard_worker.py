"""Worker of tests/test_gpu_eval_shard_multi.py (one process per rank, launched with torch.distributed.run; argv[1] is
the backend: nccl with one GPU per rank, or gloo with the ranks sharing the GPUs there are).  On a mini meta model:
  1. valid.sharded_ensemble_dynamic_weights: the reweighting vectors bit-equal on every rank and to one process, also
     when a rank gets no support batch;
  2. valid.score_batches(sharded=True): the result dicts, the per-class result lines and the COCO results
     json equal those of one process, for an image count that is not a multiple of world x batch and for a set where
     a rank gets no batch;
  3. an image evaluated on two ranks raises on every rank (the error of the scoring rank is broadcast).
Prints 'SHARD_OK' on every rank on success."""
import contextlib
import io
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests', 'golden'))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402


def same(a, b):
    """Equal result dicts: arrays bit for bit, floats by repr (NaN equals NaN)."""
    if isinstance(a, dict):
        return set(a) == set(b) and all(same(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(same(x, y) for x, y in zip(a, b))
    if isinstance(a, np.ndarray):
        return a.shape == b.shape and np.array_equal(np.ascontiguousarray(a).view(np.uint8),
                                                     np.ascontiguousarray(b).view(np.uint8))
    return repr(a) == repr(b)


def main():
    backend = sys.argv[1]
    rank, world, local = int(os.environ['RANK']), int(os.environ['WORLD_SIZE']), int(os.environ['LOCAL_RANK'])
    dev = torch.device('cuda', local % torch.cuda.device_count())
    torch.cuda.set_device(dev)
    dist.init_process_group(backend, device_id=dev if backend == 'nccl' else None)
    from fewshot_detection_b200 import coco_eval as C, netcfg, valid as VA, voc_eval as V
    from fewshot_detection_b200.darknet_meta import Darknet
    from fewshot_detection_b200.shard import shard_range
    from seeding import seeded_init, synth_masks
    with contextlib.redirect_stdout(sys.stderr):
        m = Darknet(netcfg.mini_dynamic_blocks(128, 16), netcfg.mini_reweighting_blocks(64, 16, 512))
    seeded_init(m, 3)
    m = m.to(dev).eval()
    classes = ['bird', 'bus', 'cow']
    n_cls = len(classes)

    def support(s, e):
        g = torch.Generator().manual_seed(1000 + s)
        return (torch.rand(e - s, 3, 64, 64, generator=g).to(dev), torch.from_numpy(synth_masks(e - s, 64, s)).to(dev),
                [k % n_cls for k in range(s, e)])

    def supports(n, sb, r0, r1):
        return [support(s, min(s + sb, r1)) for s in range(r0, r1, sb)]

    # ---- 1. support ensemble
    for n_sup, sb in ((13, 3), (3, 4)):                         # 5 batches over 2 ranks; 1 batch: rank 1 idle
        single = VA.ensemble_dynamic_weights(m, supports(n_sup, sb, 0, n_sup), n_cls)[0]
        s0, s1 = shard_range(n_sup, sb, world, rank)
        sharded = VA.sharded_ensemble_dynamic_weights(m, supports(n_sup, sb, s0, s1), n_cls)[0]
        assert torch.equal(sharded, single), ('enews differ from one process', n_sup, sb)
        ref = sharded.clone()
        dist.broadcast(ref, 0)
        assert torch.equal(ref, sharded), 'enews differ between ranks'

    # ---- 2. VOC and COCO scoring
    for n_img, bs in ((26, 4), (3, 4)):                          # 7 batches (4 + 3); 1 batch: rank 1 idle
        rs = np.random.RandomState(n_img)
        names = ['COCO_val2014_%012d' % (3 * k + 1) for k in range(n_img)]
        sizes = [(500, 375) if k % 3 else (353, 500) for k in range(n_img)]
        recs, anns = {}, []
        for k, n in enumerate(names):
            W, H = sizes[k]
            objs = []
            for _ in range(rs.randint(1, 6)):
                w, h = int(rs.randint(W // 6, W // 2)), int(rs.randint(H // 6, H // 2))
                x, y = int(rs.randint(1, W - w)), int(rs.randint(1, H - h))
                objs.append((int(rs.randint(n_cls)), x, y, w, h, int(rs.rand() < 0.1)))
            recs[n] = [{'name': classes[c], 'difficult': d, 'bbox': [x, y, x + w - 1, y + h - 1]} for c, x, y, w, h, d in objs]
            anns.append([(c, [float(x), float(y), float(w), float(h)], float(w * h), d) for c, x, y, w, h, d in objs])
        gt = {'image_ids': [3 * k + 1 for k in range(n_img)], 'category_ids': [1, 3, 5], 'anns': anns}

        def images(q0, q1):
            out = []
            for s in range(q0, q1, bs):
                e = min(s + bs, q1)
                g = torch.Generator().manual_seed(5000 + s)
                out.append((torch.rand(e - s, 3, 128, 128, generator=g).to(dev), names[s:e], sizes[s:e]))
            return out
        sup = supports(13, 3, 0, 13)
        s0, s1 = shard_range(13, 3, world, rank)
        q0, q1 = shard_range(n_img, bs, world, rank)
        fps1 = [io.StringIO() for _ in classes]
        one = VA.score_batches(m, sup, images(0, n_img), V.DeviceVocEval(classes, names, recs), out=fps1,
                               use_07_metric=True, novel_classes=('cow',))
        fpsN = [io.StringIO() for _ in classes] if rank == 0 else True
        got = VA.score_batches(m, supports(13, 3, s0, s1), images(q0, q1), V.DeviceVocEval(classes, names, recs),
                               out=fpsN, sharded=True, use_07_metric=True, novel_classes=('cow',))
        assert same(got, one), ('sharded VOC result differs', n_img, got, one)
        if rank == 0:
            assert [f.getvalue() for f in fpsN] == [f.getvalue() for f in fps1], 'VOC result lines differ'
            assert sum(len(f.getvalue()) for f in fps1) > 0
        f1 = io.StringIO()
        one = VA.score_batches(m, sup, images(0, n_img), C.DeviceCocoEval(classes, names, gt), out=f1,
                               novel_classes=('cow',))
        fN = io.StringIO() if rank == 0 else True
        got = VA.score_batches(m, supports(13, 3, s0, s1), images(q0, q1), C.DeviceCocoEval(classes, names, gt),
                               out=fN, sharded=True, novel_classes=('cow',))
        assert same(got, one), ('sharded COCO result differs', n_img)
        if rank == 0:
            assert fN.getvalue() == f1.getvalue() and len(f1.getvalue()) > 2, 'COCO results json differs'

    # ---- 3. the same image on two ranks: the scoring rank's error reaches every rank
    ev = V.DeviceVocEval(classes, names, recs)
    dw = VA.ensemble_dynamic_weights(m, sup, n_cls)
    x, ids, sz = images(0, n_img)[0]
    ev.add(VA.detect(m, x[:1], dw, n_cls), ids[:1], sz[:1])          # both ranks: image 0 (the merged pool fits)
    try:
        ev.gather(None, 0)
        raise AssertionError('a duplicated image was scored')
    except RuntimeError as e:
        assert 'two ranks' in str(e), e

    dist.barrier()
    print('SHARD_OK rank %d (%s)' % (rank, backend), flush=True)
    torch.cuda.synchronize()
    dist.destroy_process_group()


if __name__ == '__main__':
    main()
