"""Developer tool: measured precision of the 3xBF16 tensor-core convolution vs float64."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch, torch.nn.functional as F
from fewshot_detection_b200 import _lib as L
st = lambda: torch.cuda.current_stream().cuda_stream
rel = lambda a, b: ((a.double() - b.double()).norm() / b.double().norm()).item()
nhwc = lambda x: x.permute(0, 2, 3, 1).contiguous().view(-1, x.shape[1])


def split(t2d):
    rows, C = t2d.shape
    am = torch.zeros(1, device='cuda')
    L.call('fsdet_amax', t2d.data_ptr(), C, C, rows, am.data_ptr(), st())
    hi = torch.empty(rows, C, dtype=torch.float16, device='cuda'); lo = torch.empty_like(hi)
    L.call('fsdet_split_f16', t2d.data_ptr(), C, C, C, rows, am.data_ptr(), hi.data_ptr(), lo.data_ptr(), st())
    return hi, lo, am


for (B, H, W, Cin, Cout, k) in [(2, 13, 13, 64, 128, 3), (2, 13, 13, 1280, 1024, 3), (4, 26, 26, 128, 64, 1), (1, 52, 52, 64, 128, 3)]:
    for mode in ('random', 'f16-exact', 'positive'):
        g = torch.Generator(device='cuda').manual_seed(1)
        x = torch.randn(B, Cin, H, W, device='cuda', generator=g)
        w = torch.randn(Cout, Cin, k, k, device='cuda', generator=g) * 0.05
        if mode == 'f16-exact':
            x = x.to(torch.float16).float(); w = w.to(torch.float16).float()
        if mode == 'positive':
            x = x.abs()
        ref = F.conv2d(x.double(), w.double(), None, 1, (k - 1) // 2)
        xn = nhwc(x); wn = w.permute(0, 2, 3, 1).contiguous()
        xh, xl, xa = split(xn); wh, wl, wa = split(wn.view(Cout, -1))
        z = torch.zeros(B * H * W, Cout, device='cuda')
        L.call('fsdet_conv_tc_fwd', xh.data_ptr(), xl.data_ptr(), wh.data_ptr(), wl.data_ptr(), xa.data_ptr(), wa.data_ptr(), z.data_ptr(), Cout, B, H, W, Cin, Cin, Cout, k, 0, 3, None, st())
        got = z.view(B, H, W, Cout).permute(0, 3, 1, 2)
        z2 = torch.zeros(B * H * W, Cout, device='cuda')
        L.call('fsdet_conv_fwd', xn.data_ptr(), Cin, wn.data_ptr(), None, z2.data_ptr(), Cout, None, B, H, W, Cin, Cout, k, 0, st())
        got2 = z2.view(B, H, W, Cout).permute(0, 3, 1, 2)
        # ideal 3-term value in float64
        print('%-28s %-10s tc %.2e   simt-fp32 %.2e' % ((B, H, W, Cin, Cout, k), mode, rel(got, ref), rel(got2, ref)))
