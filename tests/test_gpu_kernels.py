"""Per-kernel parity of the C-ABI entry points against torch fp32 / the oracle.
All tests need an H100 (`-m gpu`)."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
TOL = 2e-5  # fp32 SIMT path: only the summation order differs


def rel(a, b):
    a = a.detach().double().cpu()
    b = b.detach().double().cpu()
    return ((a - b).norm() / max(b.norm().item(), 1e-30)).item()


@pytest.fixture(scope='module')
def L():
    from fewshot_detection_b200 import _lib
    assert torch.cuda.is_available()
    return _lib


def st():
    return torch.cuda.current_stream().cuda_stream


def nhwc(x):  # NCHW tensor -> [npix, C] contiguous
    return x.permute(0, 2, 3, 1).contiguous().view(-1, x.shape[1])


def nchw(buf, B, H, W):
    return buf.view(B, H, W, -1).permute(0, 3, 1, 2).contiguous()


def ohwi(w):
    return w.permute(0, 2, 3, 1).contiguous()


CONV_CASES = [
    # B, H, W, Cin, Cout, k
    (2, 13, 13, 64, 128, 3), (1, 6, 6, 32, 200, 3), (3, 8, 10, 4, 8, 3), (2, 26, 26, 128, 64, 1),
    (1, 19, 19, 36, 30, 1), (2, 16, 16, 16, 32, 3), (1, 5, 7, 260, 132, 3), (2, 13, 13, 1024, 480, 1),
]


@pytest.mark.parametrize('B,H,W,Cin,Cout,k', CONV_CASES)
def test_conv_fwd_stats_bias_accumulate(L, B, H, W, Cin, Cout, k):
    g = torch.Generator(device='cuda').manual_seed(B * 1000 + H + Cin + Cout)
    x = torch.randn(B, Cin, H, W, device='cuda', generator=g)
    w = torch.randn(Cout, Cin, k, k, device='cuda', generator=g) * 0.1
    bias = torch.randn(Cout, device='cuda', generator=g)
    ref = F.conv2d(x, w, None, 1, (k - 1) // 2)
    xb, wb = nhwc(x), ohwi(w)
    ld = Cout + 4  # exercise ld > C
    z = torch.zeros(B * H * W, ld, device='cuda')
    rows = L.lib.fsdet_conv_stat_rows(B * H * W)
    stat = torch.zeros(rows, 4 * Cout, device='cuda')
    L.call('fsdet_conv_fwd', xb.data_ptr(), Cin, wb.data_ptr(), None, z.data_ptr(), ld, stat.data_ptr(), B, H, W, Cin, Cout,
           k, 0, st())
    got = nchw(z[:, :Cout].contiguous(), B, H, W)
    assert rel(got, ref) < TOL
    assert (z[:, Cout:] == 0).all()
    s = stat.double().sum(0)
    assert rel(s[:Cout], ref.double().sum((0, 2, 3))) < 1e-4
    assert rel(s[Cout:2 * Cout], (ref.double() ** 2).sum((0, 2, 3))) < 1e-4
    assert torch.equal(stat[:, 2 * Cout:3 * Cout].min(0)[0], z[:, :Cout].min(0)[0])
    assert torch.equal(stat[:, 3 * Cout:].max(0)[0], z[:, :Cout].max(0)[0])
    # bias + accumulate
    z2 = z.clone()
    L.call('fsdet_conv_fwd', xb.data_ptr(), Cin, wb.data_ptr(), bias.data_ptr(), z2.data_ptr(), ld, None, B, H, W, Cin, Cout,
           k, 1, st())
    got2 = nchw(z2[:, :Cout].contiguous(), B, H, W)
    assert rel(got2, 2 * ref + bias.view(1, -1, 1, 1)) < TOL


@pytest.mark.parametrize('B,H,W,Cin,Cout,k', [c for c in CONV_CASES if c[4] % 4 == 0] + [(64, 52, 52, 8, 16, 3)])
def test_conv_wgrad_and_dgrad(L, B, H, W, Cin, Cout, k):
    g = torch.Generator(device='cuda').manual_seed(7 + Cin + Cout)
    x = torch.randn(B, Cin, H, W, device='cuda', generator=g, requires_grad=True)
    w = (torch.randn(Cout, Cin, k, k, device='cuda', generator=g) * 0.1).requires_grad_(True)
    dz = torch.randn(B, Cout, H, W, device='cuda', generator=g)
    F.conv2d(x, w, None, 1, (k - 1) // 2).backward(dz)
    xb, wb, dzb = nhwc(x.detach()), ohwi(w.detach()), nhwc(dz)
    nws = L.lib.fsdet_conv_wgrad_workspace_floats(B, H, W, Cin, Cout, k)
    ws = torch.empty(max(nws, 4), device='cuda')
    dw = torch.empty(Cout, k * k, Cin, device='cuda')
    L.call('fsdet_conv_wgrad', xb.data_ptr(), Cin, dzb.data_ptr(), Cout, dw.data_ptr(), ws.data_ptr(), nws, B, H, W, Cin,
           Cout, k, st())
    assert rel(dw.view(Cout, k, k, Cin).permute(0, 3, 1, 2), w.grad) < TOL * 5
    wt = torch.empty(Cin, k * k, Cout, device='cuda')
    L.call('fsdet_weight_flip_transpose', wb.data_ptr(), wt.data_ptr(), Cout, k * k, Cin, st())
    dx = torch.empty(B * H * W, Cin, device='cuda')
    L.call('fsdet_conv_fwd', dzb.data_ptr(), Cout, wt.data_ptr(), None, dx.data_ptr(), Cin, None, B, H, W, Cout, Cin, k, 0,
           st())
    assert rel(nchw(dx, B, H, W), x.grad) < TOL


@pytest.mark.parametrize('B,H,W,C,pool,full', [(2, 13, 13, 32, True, True), (3, 8, 8, 64, True, False),
                                               (2, 7, 9, 16, False, True), (1, 26, 26, 512, True, True),
                                               (4, 6, 6, 1024, False, True)])
def test_bn_act_pool_fwd_bwd(L, B, H, W, C, pool, full):
    g = torch.Generator(device='cuda').manual_seed(C + H)
    z = (torch.randn(B, C, H, W, device='cuda', generator=g) * 2 + 0.3).requires_grad_(True)
    gamma = (torch.rand(C, device='cuda', generator=g) + 0.5).requires_grad_(True)
    beta = (torch.randn(C, device='cuda', generator=g) * 0.1).requires_grad_(True)
    rm = torch.zeros(C, device='cuda')
    rv = torch.ones(C, device='cuda')
    y = F.leaky_relu(F.batch_norm(z, rm, rv, gamma, beta, True, 0.1, 1e-5), 0.1)
    outs, gouts = [], []
    if full:
        outs.append(y)
        gouts.append(torch.randn(y.shape, device='cuda', generator=g))
    if pool:
        yp = F.max_pool2d(y, 2, 2)
        outs.append(yp)
        gouts.append(torch.randn(yp.shape, device='cuda', generator=g))
    torch.autograd.backward(outs, gouts)
    # ours: column statistics of z (the same partial layout the conv epilogues write), finalize, activation
    zb = nhwc(z.detach())
    npix = B * H * W
    srows = L.lib.fsdet_colstats_rows(npix)
    stat = torch.zeros(srows + L.lib.fsdet_bn_stat_scratch_rows(), 4 * C, device='cuda')
    L.call('fsdet_colstats', zb.data_ptr(), C, npix, C, stat.data_ptr(), st())
    rm2, rv2 = torch.zeros(C, device='cuda'), torch.ones(C, device='cuda')
    vec = torch.empty(5, C, device='cuda')
    amax = torch.zeros(1, device='cuda')
    L.call('fsdet_bn_finalize', stat.data_ptr(), srows, float(npix), gamma.data_ptr(), beta.data_ptr(), rm2.data_ptr(),
           rv2.data_ptr(), 0.1, 1e-5, vec[0].data_ptr(), vec[1].data_ptr(), vec[2].data_ptr(), vec[3].data_ptr(), 0.1,
           amax.data_ptr(), vec[4].data_ptr(), C, 1, st())
    assert rel(rm2, rm) < 1e-5 and rel(rv2, rv) < 1e-5
    xh = (z.detach() - vec[0].view(1, C, 1, 1)) * vec[1].view(1, C, 1, 1)
    assert torch.equal(vec[4], xh.abs().amax(dim=(0, 2, 3)))
    assert abs(amax.item() - y.abs().max().item()) <= 1e-5 * y.abs().max().item()
    yf = torch.empty(npix, C, device='cuda') if full else None
    ypb = torch.empty(B * (H // 2) * (W // 2), C, device='cuda') if pool else None
    cp = (C + 63) // 64 * 64
    fh = torch.full((npix, cp), 7.0, dtype=torch.float16, device='cuda')
    fl = torch.full((npix, cp), 7.0, dtype=torch.float16, device='cuda')
    ph = torch.full((B * (H // 2) * (W // 2), cp), 7.0, dtype=torch.float16, device='cuda')
    pl = torch.full((B * (H // 2) * (W // 2), cp), 7.0, dtype=torch.float16, device='cuda')
    L.call('fsdet_bn_act_fwd', zb.data_ptr(), C, vec[2].data_ptr(), vec[3].data_ptr(), 0.1,
           yf.data_ptr() if full else None, C, ypb.data_ptr() if pool else None, C, fh.data_ptr(), fl.data_ptr(),
           ph.data_ptr() if pool else None, pl.data_ptr() if pool else None, cp, amax.data_ptr(), B, H, W, C, st())
    import math
    sc = 2.0 ** (10 - math.frexp(amax.item())[1])
    assert rel((fh.float() + fl.float())[:, :C] / sc, nhwc(y)) < 1e-5
    assert (fh[:, C:] == 0).all() and (fl[:, C:] == 0).all()
    if full:
        assert rel(nchw(yf, B, H, W), y) < 1e-5
    if pool:
        assert rel(nchw(ypb, B, H // 2, W // 2), yp) < 1e-5
        assert rel((ph.float() + pl.float())[:, :C] / sc, nhwc(yp)) < 1e-5
    gi = 0
    gf = gp = None
    if full:
        gf = nhwc(gouts[gi]); gi += 1
    if pool:
        gp = nhwc(gouts[gi])
    rows = L.lib.fsdet_bn_bwd_rows(B, H, W)
    part = torch.empty(rows + 1, 3 * C, dtype=torch.float64, device='cuda')
    coef = torch.empty(2, C, dtype=torch.float64, device='cuda')
    dgam, dbet = torch.empty(C, device='cuda'), torch.empty(C, device='cuda')
    a = (zb.data_ptr(), C, gf.data_ptr() if full else None, C, gp.data_ptr() if pool else None, C, vec[2].data_ptr(),
         vec[3].data_ptr(), vec[0].data_ptr(), vec[1].data_ptr())
    L.call('fsdet_bn_act_bwd_reduce', *a, 0.1, part.data_ptr(), B, H, W, C, 1, st())
    dzmax = torch.full((1,), 123.0, device='cuda')
    L.call('fsdet_bn_bwd_finalize', part.data_ptr(), rows, float(npix), gamma.data_ptr(), vec[1].data_ptr(), vec[4].data_ptr(),
           dgam.data_ptr(), dbet.data_ptr(), coef.data_ptr(), dzmax.data_ptr(), C, 1, st())
    dz = torch.empty(npix, C, device='cuda')
    dh = torch.full((npix, C), 7.0, dtype=torch.float16, device='cuda')
    dl = torch.full((npix, C), 7.0, dtype=torch.float16, device='cuda')
    L.call('fsdet_bn_act_bwd_apply', *a, coef.data_ptr(), 0.1, dz.data_ptr(), C, dh.data_ptr(), dl.data_ptr(), C,
           dzmax.data_ptr(), B, H, W, C, 1, st())
    # the plane scale comes from an upper bound of max|dz| (never below it, and not uselessly loose)
    true_max = dz.abs().max().item()
    assert true_max <= dzmax.item() <= 16 * true_max
    scd = 2.0 ** (10 - math.frexp(dzmax.item())[1])
    assert rel((dh.float() + dl.float()) / scd, dz) < 1e-5
    # planes only (no fp32 dz) gives the same planes
    dh2, dl2 = torch.empty_like(dh), torch.empty_like(dl)
    L.call('fsdet_bn_act_bwd_apply', *a, coef.data_ptr(), 0.1, None, 0, dh2.data_ptr(), dl2.data_ptr(), C,
           dzmax.data_ptr(), B, H, W, C, 1, st())
    assert torch.equal(dh, dh2) and torch.equal(dl, dl2)
    assert rel(dgam, gamma.grad) < 1e-4
    assert rel(dbet, beta.grad) < 1e-4
    assert rel(nchw(dz, B, H, W), z.grad) < 1e-4


def test_layers_vs_golden_and_torch(L):
    d = np.load(os.path.join(G, 'layers.npz'))
    from fewshot_detection_b200.pooling import Reorg, MaxPoolStride1, GlobalMaxPool2d
    x6 = torch.from_numpy(d['x']).cuda()
    assert torch.equal(MaxPoolStride1()(torch.cat([x6, x6[:, :2]], 1))[:, :6].cpu(), torch.from_numpy(d['maxpool_stride1']))
    assert torch.equal(GlobalMaxPool2d()(x6).cpu(), torch.from_numpy(d['globalmax']))
    x8 = torch.cat([x6, x6[:, :2]], 1)  # C = 8
    from oracle.darknet import Reorg as OReorg
    assert torch.equal(Reorg(2)(x8).cpu(), OReorg(2)(x8.cpu()))
    # maxpool backward, both strides, vs autograd
    for stride in (1, 2):
        for (B, H, W, C) in [(2, 13, 13, 8), (1, 6, 8, 4)]:
            x = torch.randn(B, C, H, W, device='cuda', requires_grad=True)
            if stride == 2:
                y = F.max_pool2d(x, 2, 2)
            else:
                y = F.max_pool2d(F.pad(x, (0, 1, 0, 1), mode='replicate'), 2, stride=1)
            gy = torch.randn_like(y)
            y.backward(gy)
            xb, gyb = nhwc(x.detach()), nhwc(gy)
            yb = torch.empty(gyb.shape, device='cuda')
            L.call('fsdet_maxpool_fwd', xb.data_ptr(), C, yb.data_ptr(), C, B, H, W, C, stride, st())
            assert torch.equal(nchw(yb, B, y.shape[2], y.shape[3]), y.detach())
            dx = torch.empty(B * H * W, C, device='cuda')
            L.call('fsdet_maxpool_bwd', xb.data_ptr(), C, gyb.data_ptr(), C, dx.data_ptr(), C, B, H, W, C, stride, st())
            assert rel(nchw(dx, B, H, W), x.grad) < 1e-6
    # reorg backward = inverse permutation
    x = torch.randn(2, 8, 6, 10, device='cuda')
    xb = nhwc(x)
    yb = torch.empty(2 * 3 * 5, 32, device='cuda')
    L.call('fsdet_reorg_fwd', xb.data_ptr(), 8, yb.data_ptr(), 32, 2, 6, 10, 8, st())
    back = torch.empty_like(xb)
    L.call('fsdet_reorg_bwd', yb.data_ptr(), 32, back.data_ptr(), 8, 2, 6, 10, 8, st())
    assert torch.equal(back, xb)


def test_nchw_nhwc_roundtrip_and_pad(L):
    a = torch.randn(3, 3, 7, 5, device='cuda')
    m = torch.randn(3, 1, 7, 5, device='cuda')
    buf = torch.full((3 * 35, 8), 7.0, device='cuda')
    L.call('fsdet_nchw_to_nhwc', a.data_ptr(), 3, m.data_ptr(), 1, buf.data_ptr(), 8, 8, 3, 35, st())
    exp = torch.cat([a, m, torch.zeros(3, 4, 7, 5, device='cuda')], 1)
    assert torch.equal(nchw(buf, 3, 7, 5), exp)
    out = torch.empty(3, 4, 7, 5, device='cuda')
    bias = torch.randn(4, device='cuda')
    L.call('fsdet_nhwc_to_nchw', buf.data_ptr(), 8, bias.data_ptr(), out.data_ptr(), 3, 4, 35, st())
    assert torch.allclose(out, exp[:, :4] + bias.view(1, -1, 1, 1))
    w = torch.randn(10, 3, device='cuda')
    wp = torch.empty(10, 4, device='cuda')
    L.call('fsdet_pad_channels', w.data_ptr(), 3, wp.data_ptr(), 4, 10, st())
    assert torch.equal(wp[:, :3], w) and (wp[:, 3] == 0).all()
    wc = torch.empty(10, 3, device='cuda')
    L.call('fsdet_pad_channels', wp.data_ptr(), 4, wc.data_ptr(), 3, 10, st())
    assert torch.equal(wc, w)


def test_fused_sgd_matches_torch(L):
    from fewshot_detection_b200.optim import FusedSGD
    torch.manual_seed(0)
    shapes = [(64, 32, 3, 3), (128,), (7,), (30, 1024, 1, 1), (1000001,)]
    ps = [torch.randn(s, device='cuda') for s in shapes]
    ps[0] = ps[0].contiguous(memory_format=torch.channels_last)
    a = [torch.nn.Parameter(p.clone()) for p in ps]
    b = [torch.nn.Parameter(p.clone()) for p in ps]
    oa = FusedSGD(a, lr=0.01, momentum=0.9, dampening=0, weight_decay=0.05)
    ob = torch.optim.SGD(b, lr=0.01, momentum=0.9, dampening=0, weight_decay=0.05)
    for it in range(3):
        for pa, pb in zip(a, b):
            gr = torch.randn_like(pb)
            pa.grad = gr.clone()
            pb.grad = gr.clone()
        oa.step()
        ob.step()
        for g_ in oa.param_groups:
            g_['lr'] *= 0.5
        for g_ in ob.param_groups:
            g_['lr'] *= 0.5
    for pa, pb in zip(a, b):
        assert rel(pa, pb) < 1e-6


@pytest.mark.parametrize('B,H,W,Cout,C0,C1', [(2, 13, 17, 32, 3, 0), (3, 64, 64, 16, 3, 1), (1, 5, 3, 8, 2, 1), (2, 416, 416, 32, 3, 1),
                                                (5, 200, 130, 32, 3, 1), (7, 100, 211, 24, 3, 0), (1, 40, 608, 32, 3, 0)])
def test_conv_first_layer_fwd_wgrad(L, B, H, W, Cout, C0, C1):
    g = torch.Generator(device='cuda').manual_seed(H + W)
    a = torch.rand(B, C0, H, W, device='cuda', generator=g)
    m = torch.rand(B, C1, H, W, device='cuda', generator=g) if C1 else None
    C = C0 + C1
    x = torch.cat([a, m], 1) if C1 else a
    w = (torch.randn(Cout, C, 3, 3, device='cuda', generator=g) * 0.2).double().requires_grad_(True)
    dz = torch.randn(B, Cout, H, W, device='cuda', generator=g)
    ref = F.conv2d(x.double(), w, None, 1, 1)
    ref.backward(dz.double())
    wp = torch.zeros(Cout, 9, 4, device='cuda')
    wp[:, :, :C] = w.detach().float().permute(0, 2, 3, 1).reshape(Cout, 9, C)
    z = torch.empty(B * H * W, Cout, device='cuda')
    L.call('fsdet_conv_first_fwd', a.data_ptr(), C0, m.data_ptr() if C1 else None, C1, wp.data_ptr(), z.data_ptr(), Cout, B, H, W,
           Cout, st())
    assert rel(nchw(z, B, H, W), ref) < 1e-5
    # the flavour that also emits the BatchNorm partial rows: same z bit for bit, statistics of exactly that z
    z2 = torch.empty(B * H * W, Cout + 4, device='cuda')
    rows = L.lib.fsdet_conv_first_stat_rows(B, H, W)
    part = torch.full((rows, 4 * Cout), 123.0, device='cuda')
    L.call('fsdet_conv_first_fwd_stats', a.data_ptr(), C0, m.data_ptr() if C1 else None, C1, wp.data_ptr(), z2.data_ptr(), Cout + 4,
           B, H, W, Cout, part.data_ptr(), st())
    assert torch.equal(z2[:, :Cout], z)
    sp = part.double().sum(0)
    assert rel(sp[:Cout], z.double().sum(0)) < 1e-5 or (sp[:Cout] - z.double().sum(0)).abs().max() < 1e-3
    assert rel(sp[Cout:2 * Cout], (z.double() ** 2).sum(0)) < 1e-5
    assert torch.equal(part[:, 2 * Cout:3 * Cout].min(0)[0], z.min(0)[0])
    assert torch.equal(part[:, 3 * Cout:].max(0)[0], z.max(0)[0])
    dzb = nhwc(dz)
    nws = L.lib.fsdet_conv_first_wgrad_workspace_floats(B, H, W, Cout)
    ws = torch.empty(nws, device='cuda')
    dw = torch.empty(Cout, 9, 4, device='cuda')
    L.call('fsdet_conv_first_wgrad', a.data_ptr(), C0, m.data_ptr() if C1 else None, C1, dzb.data_ptr(), Cout, dw.data_ptr(),
           ws.data_ptr(), nws, B, H, W, Cout, st())
    assert rel(dw.view(Cout, 3, 3, 4)[:, :, :, :C].permute(0, 3, 1, 2), w.grad) < 1e-5
    assert (dw.view(Cout, 9, 4)[:, :, C:] == 0).all()
