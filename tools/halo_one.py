"""Developer tool: one halo-tile convolution launch (conv2 forward shape, B images) under FSDET_HALO_FLAGS, compared with
the im2col kernel - small enough for compute-sanitizer.  Usage: python tools/halo_one.py [B]"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from fewshot_detection_b200 import _lib as L
from halo_bench import planes, st

B = int(sys.argv[1]) if len(sys.argv) > 1 else 2
H = W = 208
Cin, cp, Cout = 32, 64, 64
npix = B * H * W
xh, xl, xa = planes(npix, cp, 1)
wh, wl, wa = planes(Cout * 9, cp, 2)
out = {}
for mode in (3 | 64, 3):
    z = torch.zeros(npix, Cout, device='cuda')
    L.call('fsdet_conv_tc_fwd', xh.data_ptr(), xl.data_ptr(), wh.data_ptr(), wl.data_ptr(), xa.data_ptr(), wa.data_ptr(), z.data_ptr(), Cout,
           B, H, W, Cin, cp, Cout, 3, 0, mode, None, st())
    torch.cuda.synchronize()
    out[mode] = z
print('flags', os.environ.get('FSDET_HALO_FLAGS'), 'halo vs im2col rel diff',
      ((out[3] - out[3 | 64]).norm() / out[3 | 64].norm()).item())
