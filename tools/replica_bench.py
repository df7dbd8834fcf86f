#!/usr/bin/env python
"""Cost of the reference's replica step on one GPU: the graph-replayed meta-training step (forward, RegionLossV2,
backward, FusedSGD) with Darknet(..., replicas=R).

    python tools/replica_bench.py [--steps K] [--warmup W] [--runs N]

Runs B = 64 query images, 20 classes at 416x416 with R = 1 (one support set of 20 images, BatchNorm over the whole
batch) and R = 4 (the reference's four nn.DataParallel replicas: four support sets, BatchNorm per 16 images),
alternating, N runs each; then one run at 608x608 with R = 4 and one of COCO base training (60 classes, R = 4).
Each line: images/s, ms/step, peak device memory; the card's name, power limit and the median SM clock sampled during
the timed steps are printed first and last.  Every model is built, captured and freed inside its run."""
import argparse
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests', 'golden'))

import numpy as np  # noqa: E402
import torch  # noqa: E402


def smi(query):
    r = subprocess.run(['nvidia-smi', '--query-gpu=' + query, '--format=csv,noheader,nounits', '-i',
                        str(torch.cuda.current_device())], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
    return r.stdout.strip() if r.returncode == 0 else 'n/a'


class ClockSampler(object):
    def __init__(self):
        self.samples, self._stop = [], threading.Event()
        self._t = threading.Thread(target=self._run, daemon=True)

    def _run(self):
        while not self._stop.is_set():
            v = smi('clocks.sm')
            if v.isdigit():
                self.samples.append(int(v))
            self._stop.wait(0.2)

    def __enter__(self):
        self._t.start()
        return self

    def __exit__(self, *a):
        self._stop.set()
        self._t.join()


def run(bs, cs, side, R, steps, warmup, seed=7):
    from fewshot_detection_b200 import netcfg
    from fewshot_detection_b200.cfg import cfg
    from fewshot_detection_b200.darknet_meta import Darknet
    from fewshot_detection_b200.distributed import GradAllReducer
    from fewshot_detection_b200.graph import GraphedTrainStep
    from fewshot_detection_b200.optim import FusedSGD
    from fewshot_detection_b200.trainer import lr_factor, sgd_hyper_parameters
    from seeding import seeded_init, synth_masks, synth_targets
    cfg.neg_ratio = 1
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    m = Darknet(netcfg.darknet_dynamic_blocks(side, side), netcfg.reweighting_net_blocks(), replicas=R)
    seeded_init(m, seed)
    m = m.cuda().train()
    L = m.models[len(m.models) - 1]
    L.seen, L.verbose = 20000, False
    opt = FusedSGD(list(m.parameters()), **sgd_hyper_parameters(1e-3, 0.9, 5e-4, bs, lr_factor(1, cs)))
    gs = GraphedTrainStep(m, L, opt, GradAllReducer(m), strict=True)
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(bs, 3, side, side, generator=g).cuda()
    metax = torch.rand(R * cs, 3, 416, 416, generator=g).cuda()
    mask = torch.from_numpy(synth_masks(R * cs, 416, seed + 1)).cuda()
    tgt = torch.from_numpy(synth_targets(bs, cs, seed + 2))
    for _ in range(warmup):
        gs(x, metax, mask, tgt)
    torch.cuda.synchronize()
    with ClockSampler() as clk:
        t0 = time.time()
        for _ in range(steps):
            loss = gs(x, metax, mask, tgt)
        torch.cuda.synchronize()
        dt = time.time() - t0
    assert torch.isfinite(loss).item()
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    del gs, opt, m, L, x, metax, mask
    torch.cuda.empty_cache()
    return dict(img_s=bs * steps / dt, ms=1e3 * dt / steps, peak_gib=peak,
                sm_mhz=float(np.median(clk.samples)) if clk.samples else float('nan'))


def line(name, r):
    print('%-34s %8.1f img/s %8.2f ms/step  peak %6.1f GiB  median SM clock %s MHz'
          % (name, r['img_s'], r['ms'], r['peak_gib'], '%.0f' % r['sm_mhz']), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--runs', type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('replica_bench needs a CUDA device')
    card = 'card %s, power limit %s W, max SM clock %s MHz' % (smi('name'), smi('power.limit'), smi('clocks.max.sm'))
    print(card, flush=True)
    res = {1: [], 4: []}
    for k in range(a.runs):
        for R in (1, 4):
            r = run(64, 20, 416, R, a.steps, a.warmup)
            res[R].append(r)
            line('voc 416, B 64, R %d (run %d)' % (R, k + 1), r)
    for R in (1, 4):
        v = [r['img_s'] for r in res[R]]
        print('voc 416, R %d: median %.1f img/s (%.1f - %.1f)' % (R, np.median(v), min(v), max(v)), flush=True)
    print('R = 4 / R = 1 step time: %.3f' % (np.median([r['ms'] for r in res[4]]) / np.median([r['ms'] for r in res[1]])))
    line('voc 608, B 64, R 4', run(64, 20, 608, 4, a.steps, a.warmup))
    line('coco 416, B 64, 60 classes, R 4', run(64, 60, 416, 4, a.steps, a.warmup))
    print(card, flush=True)


if __name__ == '__main__':
    main()
