"""Achieved HBM bandwidth of the memory-bound kernels of one training step, from the ncu launch list
(profiles/launches_r01.csv: `--metrics gpu__time_duration.sum`, cold-cache, serialised) and the layer shapes of
configs[1] (64 query + 20 support images, 416x416).  Launches are matched to layers by kernel name, order and grid
size; only launches whose layer is unambiguous are listed.  Algorithmic bytes per element (DESIGN.md section 3):
  colstats           read z (4 B)
  bn_act_pool  fwd   read z (4 B) + write the pooled fp16 hi/lo planes (4 B per 4 elements)
  bwd reduce (<0>)   read z (4 B) + read dy at pooled resolution (1 B per element)
  bwd apply  (<1>)   read z (4 B) + read dy pooled (1 B) + write dz as fp16 hi/lo planes (4 B)
  sgd                20 B per parameter
Usage: python tools/hbm_table.py profiles/launches_r01.csv > profiles/hbm_kernels_r01.md"""
import csv
import json
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B, S = 64, 20
# pooled conv blocks: (name, images, H, C)
DET = [('det conv1', B, 416, 32), ('det conv2', B, 208, 64), ('det conv5', B, 104, 128), ('det conv8', B, 52, 256)]
SUP = [('sup conv1', S, 416, 32), ('sup conv2', S, 208, 64), ('sup conv3', S, 104, 128), ('sup conv4', S, 52, 256),
       ('sup conv5', S, 26, 512), ('sup conv6', S, 13, 1024)]


def short(n):
    n = re.sub(r'^void ', '', n)
    m = re.match(r'(?:fsdet::)?([A-Za-z0-9_]+(<[0-9, ]+>)?)', n)
    return m.group(1)


def main():
    path = sys.argv[1]
    lines = [l for l in open(path) if not l.startswith('==')]
    rows = [r for r in csv.DictReader(lines) if r['Metric Name'] == 'gpu__time_duration.sum']
    peak = json.load(open(os.path.join(ROOT, 'MEASURED_PEAKS.json')))['hbm_gbs'] if os.path.exists(os.path.join(ROOT, 'MEASURED_PEAKS.json')) else 3350.0   # H100 SXM HBM3 data sheet
    # one full step: from the first colstats of the support branch of the second step to the end, plus the tail of the first
    names = [short(r['Kernel Name']) for r in rows]
    us = [float(r['Metric Value']) / 1e3 for r in rows]
    half = len(rows) // 2

    def launches(kernel, lo=half, hi=None):
        return [(i, us[i]) for i in range(lo, hi or len(rows)) if names[i] == kernel]

    out = []

    def add(kernel, layer, elems, bpe, t_us):
        gb = elems * bpe / 1e9
        out.append((kernel, layer, elems / 1e6, gb, t_us, gb / (t_us * 1e-6) / 1e3, gb / (t_us * 1e-6) / peak))

    elems = lambda n, h, c: n * h * h * c
    # backward runs detector (deep -> shallow) then support (deep -> shallow); det conv13 feeds the passthrough and takes the general kernel
    for kernel, bpe in (('bn_act_bwd_pool_kernel<0>', 5.0), ('bn_act_bwd_pool_kernel<1>', 9.0)):
        ls = launches(kernel)
        # the step captured after `half` starts inside the previous step's support backward: keep the LAST 10 launches in order
        ls = ls[-10:]
        layers = list(reversed(DET)) + list(reversed(SUP))
        for (i, t), (nm, n, h, c) in zip(ls, layers):
            add(kernel, nm, elems(n, h, c), bpe, t)
    fw = launches('bn_act_pool_kernel<0>')[-10:]
    for (i, t), (nm, n, h, c) in zip(fw, SUP + DET):
        add('bn_act_pool_kernel<0>', nm, elems(n, h, c), 5.0, t)
    cs = launches('colstats_kernel')
    big = max(cs, key=lambda x: x[1])
    add('colstats_kernel', 'det conv1', elems(B, 416, 32), 4.0, big[1])
    sg = launches('sgd_multi_kernel', 0)
    per_step = sum(t for _, t in sg) / 2.0
    add('sgd_multi_kernel (all launches of a step)', '89 tensors', 66.29e6, 20.0, per_step)

    print('# Round 1 - achieved HBM bandwidth of the memory-bound kernels (from profiles/launches_r01.csv)\n')
    print(__doc__.split('Usage')[0].strip() + '\n')
    print('Peak = %.1f GB/s (MEASURED_PEAKS.json).  ncu per-launch times are cold-cache and serialised.\n' % peak)
    print('| kernel | layer | M elements | algorithmic GB | us | TB/s | of HBM peak |\n|---|---|---:|---:|---:|---:|---:|')
    for k, l, e, gb, t, tb, f in out:
        print('| `%s` | %s | %.1f | %.3f | %.1f | %.2f | %.0f %% |' % (k, l, e, gb, t, tb, 100 * f))
    tot_gb = sum(o[3] for o in out)
    tot_t = sum(o[4] for o in out)
    print('\nListed launches together: %.2f GB in %.2f ms = %.2f TB/s (%.0f %% of peak).'
          % (tot_gb, tot_t / 1e3, tot_gb / (tot_t * 1e-6) / 1e3, 100 * tot_gb / (tot_t * 1e-6) / peak))


if __name__ == '__main__':
    main()
