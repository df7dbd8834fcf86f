"""Per-layer time and algorithmic TFLOP/s of the detector's tensor-core convolutions (forward, input gradient, weight
gradient) in one training step, from the ncu launch list (profiles/launches_r01.csv; cold-cache, serialised launches)
and the layer table of cfg/darknet_dynamic.cfg at configs[1] (64 images, 20 classes).  Launches are matched to layers
by order: after the detector's first-layer kernel come conv2..conv22 and the fused head (22 conv_tc launches); the
backward pass then issues one (wgrad_tc, conv_tc = dgrad) pair per layer from the head down to conv2.
Ceiling = 1/3 of the measured bf16 tensor peak (three MMAs per fp32-equivalent MAC); the HBM floor counts the fp16
hi/lo operand planes (4 B per element) in and the fp32 result (4 B per element) out.
Usage: python tools/conv_table.py profiles/launches_r01.csv > profiles/conv_layers_r01.md"""
import csv
import json
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B, NCLS = 64, 20
LAYERS = [('conv2', 32, 64, 3, 208), ('conv3', 64, 128, 3, 104), ('conv4', 128, 64, 1, 104), ('conv5', 64, 128, 3, 104),
          ('conv6', 128, 256, 3, 52), ('conv7', 256, 128, 1, 52), ('conv8', 128, 256, 3, 52), ('conv9', 256, 512, 3, 26),
          ('conv10', 512, 256, 1, 26), ('conv11', 256, 512, 3, 26), ('conv12', 512, 256, 1, 26), ('conv13', 256, 512, 3, 26),
          ('conv14', 512, 1024, 3, 13), ('conv15', 1024, 512, 1, 13), ('conv16', 512, 1024, 3, 13), ('conv17', 1024, 512, 1, 13),
          ('conv18', 512, 1024, 3, 13), ('conv19', 1024, 1024, 3, 13), ('conv20', 1024, 1024, 3, 13), ('conv21', 512, 64, 1, 26),
          ('conv22', 1280, 1024, 3, 13), ('head (x20 classes)', 1024, 30 * NCLS, 1, 13)]


def short(n):
    n = re.sub(r'^void ', '', n)
    return re.match(r'(?:fsdet::)?([A-Za-z0-9_]+)', n).group(1)


def main():
    lines = [l for l in open(sys.argv[1]) if not l.startswith('==')]
    rows = [r for r in csv.DictReader(lines) if r['Metric Name'] == 'gpu__time_duration.sum']
    pk = json.load(open(os.path.join(ROOT, 'MEASURED_PEAKS.json'))) if os.path.exists(os.path.join(ROOT, 'MEASURED_PEAKS.json')) else {}
    peak_tf, peak_gb = pk.get('bf16_tflops_sustained', 989.4), pk.get('hbm_gbs', 3350.0)   # H100 SXM data sheet
    seq = [(short(r['Kernel Name']), float(r['Metric Value']) / 1e3) for r in rows]
    # the halo-tile flavour (conv_halo_kernel) is a conv_tc dispatch: same role in the sequence
    seq = [('conv_tc_kernel' if n == 'conv_halo_kernel' else n, t) for n, t in seq]
    firsts = [i for i, (n, _) in enumerate(seq) if n == 'conv_first_fwd_kernel']
    # the detector's first layer of the last COMPLETELY captured step (the support net runs before it)
    start = [f for f in firsts if sum(1 for n, _ in seq[f:] if n in ('conv_tc_kernel', 'wgrad_tc_kernel')) >= 66][-1]
    tc = [(i, n, t) for i, (n, t) in enumerate(seq) if i > start and n in ('conv_tc_kernel', 'wgrad_tc_kernel')]
    fwd = tc[:22]
    assert all(n == 'conv_tc_kernel' for _, n, _ in fwd)
    bwd = tc[22:22 + 44]
    assert [n for _, n, _ in bwd] == ['wgrad_tc_kernel', 'conv_tc_kernel'] * 22, 'unexpected backward launch order'
    print('# The detector\'s tensor-core convolutions layer by layer (from %s)\n' % os.path.relpath(sys.argv[1], ROOT))
    print(__doc__.split('Usage')[0].strip() + '\n')
    print('Ceiling %.0f TFLOP/s (= %.1f / 3), HBM peak %.1f GB/s.\n' % (peak_tf / 3, peak_tf, peak_gb))
    print('| layer | Cin→Cout k @H | GFLOP | fwd us | TF/s | dgrad us | TF/s | wgrad us | TF/s | HBM floor us (fwd) | fwd bound |')
    print('|---|---|---:|---:|---:|---:|---:|---:|---:|---:|---|')
    tot = [0.0, 0.0, 0.0, 0.0]
    for li, (name, cin, cout, k, h) in enumerate(LAYERS):
        gf = 2.0 * B * h * h * cin * cout * k * k / 1e9
        tf_ = fwd[li][2]
        tw_, td_ = bwd[2 * (21 - li)][2], bwd[2 * (21 - li) + 1][2]
        bytes_ = B * h * h * (cin + cout) * 4.0
        floor = bytes_ / (peak_gb * 1e9) * 1e6
        bound = 'HBM' if floor > gf * 1e9 / (peak_tf / 3 * 1e12) * 1e6 else 'tensor'
        print('| %s | %d→%d %dx%d @%d | %.1f | %.1f | %.0f | %.1f | %.0f | %.1f | %.0f | %.0f | %s |' % (
            name, cin, cout, k, k, h, gf, tf_, gf / (tf_ * 1e-6) / 1e3, td_, gf / (td_ * 1e-6) / 1e3,
            tw_, gf / (tw_ * 1e-6) / 1e3, floor, bound))
        tot[0] += gf
        tot[1] += tf_
        tot[2] += td_
        tot[3] += tw_
    print('| **all** | | %.0f | %.0f | %.0f | %.0f | %.0f | %.0f | %.0f | | |' % (
        tot[0], tot[1], tot[0] / (tot[1] * 1e-6) / 1e3, tot[2], tot[0] / (tot[2] * 1e-6) / 1e3, tot[3], tot[0] / (tot[3] * 1e-6) / 1e3))
    l2 = [fwd[0][2], bwd[43][2], bwd[42][2]]
    print('\nconv2 alone (32→64 channels at 208x208) takes %.2f ms of the step (forward %.0f + dgrad %.0f + wgrad %.0f us) for %.0f %% of '
          'these FLOPs (round 1: 2.77 ms; Cout = 64 means two ~100-clock MMAs per 96 clocks of tensor work, DESIGN.md section 3).'
          % (sum(l2) / 1e3, l2[0], l2[1], l2[2], 100 * 2.0 * B * 208 * 208 * 32 * 64 * 9 / 1e9 / tot[0]))

if __name__ == '__main__':
    main()
