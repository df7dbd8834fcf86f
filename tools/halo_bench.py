"""Developer tool: the halo-tile convolution kernel against the im2col kernel on the layer shapes of configs[1]
(B = 64 detector images, B = 20 support images), CUDA-event timed.  Usage: python tools/halo_bench.py [iters]"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from fewshot_detection_b200 import _lib as L

st = lambda: torch.cuda.current_stream().cuda_stream


def planes(rows, C, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    t = torch.randn(rows, C, device='cuda', generator=g)
    am = torch.zeros(1, device='cuda')
    L.call('fsdet_amax', t.data_ptr(), C, C, rows, am.data_ptr(), st())
    hi = torch.empty(rows, C, dtype=torch.float16, device='cuda')
    lo = torch.empty_like(hi)
    L.call('fsdet_split_f16', t.data_ptr(), C, C, C, rows, am.data_ptr(), hi.data_ptr(), lo.data_ptr(), st())
    return hi, lo, am


def main():
    iters = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    flag_list = [int(f) for f in sys.argv[2].split(',')] if len(sys.argv) > 2 else [0]
    ncu = len(sys.argv) > 3 and sys.argv[3] == 'ncu'      # one launch per (shape, flags), halo kernel only, no warm-up
    shapes = [
        # name, B, H, W, Cin, cpitch, Cout
        ('conv2 fwd', 64, 208, 208, 32, 64, 64), ('conv2 dgrad', 64, 208, 208, 64, 64, 32),
        ('conv3 fwd', 64, 104, 104, 64, 64, 128), ('conv3 dgrad', 64, 104, 104, 128, 128, 64),
        ('support conv2 fwd', 20, 208, 208, 32, 64, 64), ('support conv2 dgrad', 20, 208, 208, 64, 64, 32),
        ('support conv3 fwd', 20, 104, 104, 64, 64, 128), ('support conv3 dgrad', 20, 104, 104, 128, 128, 64),
    ]
    if ncu:
        shapes = shapes[:4]
    print('%-22s %10s  halo us by FSDET_HALO_FLAGS %s (1 / 2 = timing experiments: one halo copy / no stores)'
          % ('layer', 'im2col us', flag_list))
    for name, B, H, W, Cin, cp, Cout in shapes:
        npix = B * H * W
        xh, xl, xa = planes(npix, cp, 1)
        wh, wl, wa = planes(Cout * 9, cp, 2)
        z = torch.empty(npix, Cout, device='cuda')
        res = []
        for mode, fl in ([] if ncu else [(3 | 64, 0)]) + [(3, f) for f in flag_list]:
            os.environ['FSDET_HALO_FLAGS'] = str(fl)
            rows = L.lib.fsdet_conv_tc_stat_rows(B, H, W, Cin, Cout, 3, mode)
            part = torch.empty(rows, 4 * Cout, device='cuda')
            # statistics only for the forward shapes (the engine's input-gradient calls have none)
            args = (xh.data_ptr(), xl.data_ptr(), wh.data_ptr(), wl.data_ptr(), xa.data_ptr(), wa.data_ptr(), z.data_ptr(), Cout,
                    B, H, W, Cin, cp, Cout, 3, 0, mode, part.data_ptr() if 'fwd' in name else None, st())
            for _ in range(0 if ncu else 3):
                L.call('fsdet_conv_tc_fwd', *args)
            e0 = torch.cuda.Event(enable_timing=True)
            e1 = torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(iters):
                L.call('fsdet_conv_tc_fwd', *args)
            e1.record()
            torch.cuda.synchronize()
            res.append(e0.elapsed_time(e1) * 1e3 / iters)
        os.environ['FSDET_HALO_FLAGS'] = '0'
        fl = 2.0 * npix * Cin * Cout * 9
        print('%-22s ' % name + ' '.join('%10.1f' % r for r in res) + '   TF/s(first halo) %.1f' % (fl / res[0 if ncu else 1] / 1e6))


if __name__ == '__main__':
    main()
