#!/usr/bin/env python
"""Time one evaluation pass end to end, on one GPU or sharded over the GPUs of a torchrun job:

    python tools/eval_shard_bench.py [--images 4952] [--support 2000] [--out result.json]
    torchrun --nproc-per-node N tools/eval_shard_bench.py ...

The full-size meta detector (416 x 416, 20 classes, seeded weights) evaluates a synthetic set sized like VOC2007 test:
seeded tensors stand in for the decoded query and support images (no JPEG decode is timed), random ground truth per
image.  Phases, each ended by a device synchronise and a barrier: the support ensemble (reweighting net over every
support image + running mean), the query pass (forward, decode, NMS, gather into the device VOC evaluator) and the
scoring (merge of the ranks' pools on rank 0, AP on the device, result broadcast).  Rank 0 prints one JSON line with
the times, the mean AP (equal for every N: the pass is sharded bit for bit) and the GPU model, power limit and clocks
read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests', 'golden'))


def gpu_info():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm,clocks.sm',
                              '--format=csv,noheader'], capture_output=True, text=True, timeout=30).stdout
        return [l.strip() for l in out.strip().splitlines()]
    except (OSError, subprocess.SubprocessError) as e:
        return ['nvidia-smi unavailable: %s' % e]


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--images', type=int, default=4952, help='query images (VOC2007 test: 4952)')
    ap.add_argument('--support', type=int, default=2000, help='support images of the ensemble')
    ap.add_argument('--batch-size', type=int, default=64)
    ap.add_argument('--support-batch', type=int, default=64)
    ap.add_argument('--out', default=None, help='also write the JSON result here (rank 0)')
    args = ap.parse_args()

    import numpy as np
    import torch
    import torch.distributed as dist
    world, rank = int(os.environ.get('WORLD_SIZE', '1')), int(os.environ.get('RANK', '0'))
    local = int(os.environ.get('LOCAL_RANK', '0'))
    torch.cuda.set_device(local)
    dev = torch.device('cuda', local)
    if world > 1:
        dist.init_process_group('nccl', device_id=dev)
    from fewshot_detection_b200 import netcfg, valid as VA, voc_eval as VE
    from fewshot_detection_b200.cfg import cfg
    from fewshot_detection_b200.darknet_meta import Darknet
    from fewshot_detection_b200.shard import shard_range
    from seeding import seeded_init, synth_masks

    classes = list(cfg.voc_classes)
    n_cls, side = len(classes), 416
    m = Darknet(netcfg.darknet_dynamic_blocks(side, side), netcfg.reweighting_net_blocks())
    seeded_init(m, 3)
    m = m.to(dev).eval()

    rs = np.random.RandomState(0)
    names = ['%06d' % (2 * k + 1) for k in range(args.images)]
    recs = {}
    for n in names:
        objs = []
        for _ in range(rs.randint(1, 4)):
            x1, y1 = rs.randint(0, 300, 2)
            w, h = rs.randint(20, 200, 2)
            objs.append({'name': classes[rs.randint(n_cls)], 'difficult': int(rs.rand() < 0.1),
                         'bbox': [int(x1), int(y1), int(x1 + w), int(y1 + h)]})
        recs[n] = objs

    def support_batch(s, e):
        g = torch.Generator(device=dev).manual_seed(10007 + s)
        metax = torch.rand(e - s, 3, side, side, generator=g, device=dev)
        mask = torch.from_numpy(synth_masks(e - s, side, s)).to(dev)
        return metax, mask, [k % n_cls for k in range(s, e)]

    def query_batch(s, e):
        g = torch.Generator(device=dev).manual_seed(20011 + s)
        return torch.rand(e - s, 3, side, side, generator=g, device=dev), names[s:e], [(500, 375)] * (e - s)

    s0, s1 = shard_range(args.support, args.support_batch, world, rank)
    q0, q1 = shard_range(args.images, args.batch_size, world, rank)

    def sync():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()

    # warm-up: one support and one query batch of the timed shapes
    dw = VA.ensemble_dynamic_weights(m, [support_batch(0, min(args.support_batch, args.support))], n_cls)
    VA.detect(m, query_batch(0, min(args.batch_size, args.images))[0], dw, n_cls)
    sync()

    t0 = time.perf_counter()
    meta = (support_batch(s, min(s + args.support_batch, s1)) for s in range(s0, s1, args.support_batch))
    if world > 1:
        dw = VA.sharded_ensemble_dynamic_weights(m, meta, n_cls)
    else:
        dw = VA.ensemble_dynamic_weights(m, meta, n_cls)
    sync()
    t1 = time.perf_counter()
    ev = VE.DeviceVocEval(classes, names, recs, device=dev)
    for s in range(q0, q1, args.batch_size):
        x, ids, sizes = query_batch(s, min(s + args.batch_size, q1))
        ev.add(VA.detect(m, x, dw, n_cls), ids, sizes)
    sync()
    t2 = time.perf_counter()
    r = ev.gather(None, 0, use_07_metric=True) if world > 1 else ev.result(True)
    sync()
    t3 = time.perf_counter()
    out = {'gpus': world, 'images': args.images, 'support': args.support, 'batch_size': args.batch_size,
           'support_batch': args.support_batch, 'support_ensemble_s': round(t1 - t0, 4),
           'query_forward_nms_s': round(t2 - t1, 4), 'scoring_s': round(t3 - t2, 4), 'wall_s': round(t3 - t0, 4),
           'detections_rank0': int(ev.counters[0]), 'mean_ap': r['mean'],
           'enews_checksum': float(dw[0].double().sum()), 'gpu': gpu_info()}
    if rank == 0:
        print(json.dumps(out), flush=True)
        if args.out:
            with open(args.out, 'w') as f:
                json.dump(out, f)
    if world > 1:
        torch.cuda.synchronize()
        dist.destroy_process_group()
    return 0


if __name__ == '__main__':
    sys.exit(main())
