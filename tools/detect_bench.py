#!/usr/bin/env python
"""Throughput and latency of the detection pass (valid.detect_images: forward, decode, NMS, per-image selection) of
the full model at 416x416, launched eagerly and replayed as a CUDA graph (graph.GraphedDetect), at B = 1 and 64 and
20 and 80 classes.

    python tools/detect_bench.py [--iters 50] [--warmup 5] [--conf 0.5] [--json PATH]

Batches per second: CUDA events around `iters` back-to-back calls after `warmup` calls.  Latency: the mean of CUDA
events around single calls, each followed by a synchronise (what one request waits for, before the host copy of its
boxes).  The model is seeded at random with calibrated BatchNorm statistics; inputs are random images.  The GPU name,
power limit and SM clocks are printed with the numbers, because the numbers depend on them.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests', 'golden'))

SIDE = 416


def gpu_info():
    import torch
    info = {'name': torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader',
                            '-i', '0'], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30)
        info['power_limit'], info['sm_clock'], info['sm_clock_max'] = [v.strip() for v in q.stdout.strip().split(',')]
    except Exception as e:                             # reported, not guessed
        info['power_limit'] = info['sm_clock'] = info['sm_clock_max'] = 'unavailable (%s)' % type(e).__name__
    return info


def make_model(seed):
    """The full 416 model in eval mode, BatchNorm statistics of one train-mode forward (momentum 1)."""
    import torch
    from fewshot_detection_b200 import netcfg
    from fewshot_detection_b200.cfg import cfg, parse_cfg  # noqa: F401
    from fewshot_detection_b200.darknet_meta import Darknet
    from seeding import seeded_init, synth_masks
    m = Darknet(netcfg.darknet_dynamic_blocks(SIDE, SIDE), netcfg.reweighting_net_blocks())
    seeded_init(m, seed)
    m = m.cuda()
    bns = [b for b in m.modules() if isinstance(b, torch.nn.BatchNorm2d)]
    for b in bns:
        b.momentum = 1.0
    g = torch.Generator().manual_seed(seed + 1)
    m.train()
    with torch.no_grad():
        m(torch.rand(16, 3, SIDE, SIDE, generator=g).cuda(), torch.rand(20, 3, SIDE, SIDE, generator=g).cuda(),
          torch.from_numpy(synth_masks(20, SIDE, seed + 2)).cuda())
    for b in bns:
        b.momentum = 0.1
    return m.eval()


def vectors(m, n_cls, seed):
    import torch
    from fewshot_detection_b200 import valid as VA
    from seeding import synth_masks
    g = torch.Generator().manual_seed(seed)
    n = max(n_cls, 20)
    batch = (torch.rand(n, 3, SIDE, SIDE, generator=g), torch.from_numpy(synth_masks(n, SIDE, seed + 1)),
             [j % n_cls for j in range(n)])
    return VA.ensemble_dynamic_weights(m, [batch], n_cls)


def time_calls(fn, iters, warmup):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    e.synchronize()
    per_s = iters / (s.elapsed_time(e) / 1e3)
    lat = []
    for _ in range(iters):
        s.record()
        fn()
        e.record()
        e.synchronize()
        lat.append(s.elapsed_time(e))
    return per_s, sum(lat) / len(lat)


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--conf', type=float, default=0.5)
    ap.add_argument('--nms', type=float, default=0.4)
    ap.add_argument('--max-det', type=int, default=100)
    ap.add_argument('--json', default=None, help='also write the results here')
    args = ap.parse_args(argv)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('detect_bench needs a GPU')
    torch.cuda.set_device(0)
    from fewshot_detection_b200 import valid as VA
    from fewshot_detection_b200.graph import GraphedDetect
    info = gpu_info()
    print('GPU %s, power limit %s, SM clock %s (max %s)' % (info['name'], info['power_limit'], info['sm_clock'],
                                                             info['sm_clock_max']))
    m = make_model(501)
    rows = []
    print('%7s %4s %8s %12s %12s' % ('classes', 'B', 'mode', 'batches/s', 'latency ms'))
    for n_cls in (20, 80):
        dw = vectors(m, n_cls, 7)
        for B in (1, 64):
            x = torch.rand(B, 3, SIDE, SIDE, generator=torch.Generator().manual_seed(B)).cuda()
            sizes = [(500, 375)] * B
            sizes_dev = torch.tensor(sizes, dtype=torch.int32).cuda()
            gd = GraphedDetect(m, dw, B, SIDE, n_cls, args.conf, args.nms, args.max_det)
            modes = (('eager', lambda: VA.detect_images(m, x, dw, n_cls, sizes_dev, args.conf, args.nms, args.max_det)),
                     ('graph', lambda: gd(x, sizes)))
            res = {}
            for mode, fn in modes:
                per_s, lat = time_calls(fn, args.iters, args.warmup)
                res[mode] = per_s
                rows.append(dict(classes=n_cls, B=B, mode=mode, batches_per_s=per_s, latency_ms=lat))
                print('%7d %4d %8s %12.1f %12.3f' % (n_cls, B, mode, per_s, lat))
            print('%7d %4d %8s %11.2fx' % (n_cls, B, 'speedup', res['graph'] / res['eager']))
            del gd
    if args.json:
        with open(args.json, 'w') as f:
            json.dump(dict(gpu=info, conf=args.conf, nms=args.nms, max_det=args.max_det, side=SIDE, rows=rows), f, indent=1)
    return 0


if __name__ == '__main__':
    sys.exit(main())
