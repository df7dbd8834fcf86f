"""wgmma / TMA-im2col convolution path (csrc/conv_tc.cu) against torch fp32."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

TOL_TC = 1e-5  # vs float64: scaled fp16 hi/lo split (22 bits), hi*hi k-blocks added to an fp32 register total


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


def nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous().view(-1, x.shape[1])


class Planes(object):
    """scaled fp16 hi/lo planes + the device amax scalar (fsdet_amax + fsdet_split_f16)"""

    def __init__(self, L, t2d, cpad=None, scaled=True):
        rows, C = t2d.shape
        cpad = cpad or C
        self.src = t2d
        self.amax = torch.zeros(1, device='cuda')
        if scaled:
            L.call('fsdet_amax', t2d.data_ptr(), C, C, rows, self.amax.data_ptr(), st())
        self.hi = torch.empty(rows, cpad, dtype=torch.float16, device='cuda')
        self.lo = torch.empty(rows, cpad, dtype=torch.float16, device='cuda')
        L.call('fsdet_split_f16', t2d.data_ptr(), C, C, cpad, rows, self.amax.data_ptr() if scaled else None,
               self.hi.data_ptr(), self.lo.data_ptr(), st())
        self.a = self.amax.data_ptr() if scaled else None


def split(L, t2d, cpad=None):
    return Planes(L, t2d, cpad)


def test_amax_split_f16(L):
    x = torch.randn(1000, 64, device='cuda') * 3e-4
    p = Planes(L, x)
    assert p.amax.item() == x.abs().max().item()
    import math
    sc = 2.0 ** (10 - math.frexp(p.amax.item())[1])
    assert 512 <= p.amax.item() * sc < 1024
    assert torch.equal(p.hi, (x * sc).to(torch.float16))
    assert torch.equal(p.lo, (x * sc - p.hi.float()).to(torch.float16))
    assert rel((p.hi.float() + p.lo.float()) / sc, x) < 1e-6
    q = Planes(L, x * 1e4, scaled=False)
    assert torch.equal(q.hi, (x * 1e4).to(torch.float16))


@pytest.mark.parametrize('B,H,W,C,ks,m0,c0,tap', [
    (2, 13, 13, 64, 3, 0, 0, 0), (2, 13, 13, 128, 3, 128, 64, 4), (2, 13, 13, 64, 3, 256, 0, 8),
    (3, 26, 26, 64, 1, 640, 0, 0), (1, 52, 52, 64, 3, 2560, 0, 2), (5, 6, 6, 64, 3, 128, 0, 6), (1, 8, 8, 64, 3, 0, 0, 5)])
def test_tma_im2col_tile(L, B, H, W, C, ks, m0, c0, tap):
    g = torch.Generator(device='cuda').manual_seed(m0 + tap)
    x = torch.randn(B, H, W, C, device='cuda', generator=g).to(torch.float16)
    out = torch.zeros(128, 64, dtype=torch.float16, device='cuda')
    L.call('fsdet_debug_im2col_tile', x.data_ptr(), B, H, W, C, ks, m0, c0, tap, out.data_ptr(), st())
    torch.cuda.synchronize()
    pad = (ks - 1) // 2
    r, s = tap // ks, tap % ks
    exp = torch.zeros(128, 64, dtype=torch.float16, device='cuda')
    for i in range(128):
        m = m0 + i
        n, rem = divmod(m, H * W)
        p, q = divmod(rem, W)
        hh, ww = p + r - pad, q + s - pad
        if n < B and 0 <= hh < H and 0 <= ww < W:
            exp[i] = x[n, hh, ww, c0:c0 + 64]
    assert torch.equal(out, exp), (out.float() - exp.float()).abs().max().item()


TC_CASES = [
    # B, H, W, Cin, Cout, k
    (2, 13, 13, 64, 128, 3), (4, 26, 26, 128, 64, 1), (1, 52, 52, 64, 128, 3), (2, 13, 13, 1024, 480, 1),
    (2, 13, 13, 1280, 1024, 3), (3, 6, 6, 1024, 1024, 3), (2, 19, 19, 256, 512, 3), (1, 104, 104, 128, 256, 3),
    (3, 4, 4, 128, 256, 3), (3, 8, 8, 64, 128, 3), (3, 4, 4, 256, 256, 3), (1, 2, 2, 64, 64, 3), (3, 16, 16, 64, 64, 1),
    (2, 26, 26, 32, 64, 3), (2, 26, 26, 96, 128, 3), (2, 13, 13, 512, 1024, 3), (4, 26, 26, 512, 64, 1), (2, 52, 52, 256, 128, 1),
]


def plane_scale(P_):
    import math
    a = P_.amax.item()
    return 2.0 ** (10 - math.frexp(a)[1]) if a > 0 else 1.0


def planes_nchw(t, B, H, W, C):
    """[B*H*W][C] fp16 plane -> float64 NCHW"""
    return t[:, :C].double().view(B, H, W, C).permute(0, 3, 1, 2)


# mode = operand terms (bits 0-1) | 16 for the persistent tile loop (short-K layers only; ignored by the others)
#        | 32 for CTA pairs sharing the weight tile through TMA multicast (one-tile-per-CTA flavours)
#        | 128 for the unfused three-MMA form of mode 3 (default: x_hi * [w_hi | w_lo] as one MMA where one hi accumulator is kept)
MODES = [3, 3 | 16, 0, 0 | 16, 1, 2, 3 | 32, 0 | 32, 2 | 32, 3 | 128, 3 | 16 | 128]


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('B,H,W,Cin,Cout,k', TC_CASES)
def test_conv_tc_fwd(L, B, H, W, Cin, Cout, k, mode):
    """Every term mode multiplies exactly the planes it names (checked against a float64 convolution of those planes
    to 1e-5); mode 3 additionally reproduces the float64 convolution of the fp32 inputs to 1e-5.  The BatchNorm
    statistics that come out of the epilogue are those of the stored output."""
    g = torch.Generator(device='cuda').manual_seed(B + H + Cin + Cout)
    x = torch.randn(B, Cin, H, W, device='cuda', generator=g)
    w = torch.randn(Cout, Cin, k, k, device='cuda', generator=g) * 0.05
    X = split(L, nhwc(x))
    Wp = split(L, w.permute(0, 2, 3, 1).contiguous().view(Cout, -1))
    terms = mode & 3
    sx, sw = plane_scale(X), plane_scale(Wp)
    xh, xl = planes_nchw(X.hi, B, H, W, Cin), planes_nchw(X.lo, B, H, W, Cin)
    wh = Wp.hi.double().view(Cout, k, k, Cin).permute(0, 3, 1, 2)
    wl = Wp.lo.double().view(Cout, k, k, Cin).permute(0, 3, 1, 2)
    conv = lambda a, b: F.conv2d(a, b, None, 1, (k - 1) // 2)
    ref = conv(xh, wh)
    if terms & 1:
        ref = ref + conv(xl, wh)
    if terms & 2:
        ref = ref + conv(xh, wl)
    ref = ref / (sx * sw)
    assert L.lib.fsdet_conv_tc_supported(Cin, Cout, k)
    ld = Cout + 4
    z = torch.zeros(B * H * W, ld, device='cuda')
    rows = L.lib.fsdet_conv_tc_stat_rows(B, H, W, Cin, Cout, k, mode)
    part = torch.full((rows, 4 * Cout), 123.0, device='cuda')
    lo_x = X.lo.data_ptr() if terms & 1 else None      # planes a mode does not use may be NULL
    lo_w = Wp.lo.data_ptr() if terms & 2 else None
    L.call('fsdet_conv_tc_fwd', X.hi.data_ptr(), lo_x, Wp.hi.data_ptr(), lo_w, X.a, Wp.a, z.data_ptr(), ld,
           B, H, W, Cin, Cin, Cout, k, 0, mode, part.data_ptr(), st())
    torch.cuda.synchronize()
    got = z[:, :Cout].contiguous().view(B, H, W, Cout).permute(0, 3, 1, 2)
    # modes < 3 keep ONE fp32 accumulator for the hi*hi products (the tensor core's accumulation truncates: 3e-5)
    tol = TOL_TC if terms == 3 else 3e-5
    assert rel(got, ref) < tol
    if terms == 3:
        assert rel(got, conv(x.double(), w.double())) < TOL_TC
    assert (z[:, Cout:] == 0).all()
    zz = z[:, :Cout]
    s = part.double().sum(0)
    assert rel(s[:Cout], zz.double().sum(0)) < 1e-5 or (s[:Cout] - zz.double().sum(0)).abs().max() < 1e-3
    assert rel(s[Cout:2 * Cout], (zz.double() ** 2).sum(0)) < 1e-5
    assert torch.equal(part[:, 2 * Cout:3 * Cout].min(0)[0], zz.min(0)[0])
    assert torch.equal(part[:, 3 * Cout:].max(0)[0], zz.max(0)[0])
    L.call('fsdet_conv_tc_fwd', X.hi.data_ptr(), lo_x, Wp.hi.data_ptr(), lo_w, X.a, Wp.a, z.data_ptr(), ld,
           B, H, W, Cin, Cin, Cout, k, 1, mode, None, st())
    got2 = z[:, :Cout].contiguous().view(B, H, W, Cout).permute(0, 3, 1, 2)
    assert rel(got2, 2 * ref) < tol


HALO_CASES = [
    # B, H, W, Cin, cpitch, Cout     (3x3; every shape is one the plan sends to the halo-tile kernel)
    (4, 208, 208, 32, 32, 64),      # conv2 forward: weights resident in shared memory
    (4, 208, 208, 32, 64, 64),      # the engine's layout: 32 channels in 64-channel-pitched planes
    (4, 208, 208, 64, 64, 32),      # conv2 input gradient: N = 32, two chunks, resident
    (5, 104, 104, 64, 64, 128),     # conv3 / conv5 forward: streamed weights; 104 rows overhang the 16-row tiles
    (5, 104, 104, 128, 128, 64),    # conv3 / conv5 input gradient: four chunks
    (4, 104, 104, 128, 128, 128),
    (17, 46, 48, 32, 32, 48),       # Cout < BN and not a multiple of 32, H not a multiple of 16
    (11, 64, 56, 64, 64, 96),
]


@pytest.mark.parametrize('B,H,W,Cin,cpitch,Cout', HALO_CASES)
def test_conv_halo_fwd(L, B, H, W, Cin, cpitch, Cout):
    """The halo-tile kernel (8 x 16 pixel tiles, input tile + halo fetched once for all nine taps) against the float64
    convolution of the planes it multiplies and of the fp32 inputs (1e-5), against the im2col kernel on the same planes
    (mode | 64), with its fused BatchNorm statistics and in accumulate mode."""
    k = 3
    assert L.lib.fsdet_conv_tc_uses_halo(B, H, W, Cin, Cout, k, 3) == 1
    assert L.lib.fsdet_conv_tc_uses_halo(B, H, W, Cin, Cout, k, 3 | 64) == 0
    g = torch.Generator(device='cuda').manual_seed(B + H + Cin + Cout)
    x = torch.randn(B, Cin, H, W, device='cuda', generator=g)
    w = torch.randn(Cout, Cin, k, k, device='cuda', generator=g) * 0.05
    X = split(L, nhwc(x), cpitch)
    w2 = w.permute(0, 2, 3, 1).contiguous().view(Cout * k * k, Cin)
    Wp = split(L, w2, cpitch)                       # [Cout*9][cpitch]: k = tap * cpitch + c
    if cpitch > Cin:                                # poison the padding channels: they must never be multiplied
        for t in (X.hi, X.lo, Wp.hi, Wp.lo):
            t[:, Cin:] = 777.0
    sx, sw = plane_scale(X), plane_scale(Wp)
    xh, xl = planes_nchw(X.hi, B, H, W, Cin), planes_nchw(X.lo, B, H, W, Cin)
    wh = Wp.hi[:, :Cin].double().reshape(Cout, k, k, Cin).permute(0, 3, 1, 2)
    wl = Wp.lo[:, :Cin].double().reshape(Cout, k, k, Cin).permute(0, 3, 1, 2)
    conv = lambda a, b: F.conv2d(a, b, None, 1, 1)
    ref = (conv(xh, wh) + conv(xl, wh) + conv(xh, wl)) / (sx * sw)
    ld = Cout + 4
    outs = {}
    for mode in (3, 3 | 128, 3 | 64):
        z = torch.zeros(B * H * W, ld, device='cuda')
        rows = L.lib.fsdet_conv_tc_stat_rows(B, H, W, Cin, Cout, k, mode)
        part = torch.full((rows, 4 * Cout), 123.0, device='cuda')
        L.call('fsdet_conv_tc_fwd', X.hi.data_ptr(), X.lo.data_ptr(), Wp.hi.data_ptr(), Wp.lo.data_ptr(), X.a, Wp.a, z.data_ptr(), ld,
               B, H, W, Cin, cpitch, Cout, k, 0, mode, part.data_ptr(), st())
        torch.cuda.synchronize()
        got = z[:, :Cout].contiguous().view(B, H, W, Cout).permute(0, 3, 1, 2)
        assert rel(got, ref) < TOL_TC, mode
        assert rel(got, conv(x.double(), w.double())) < TOL_TC
        assert (z[:, Cout:] == 0).all()
        zz = z[:, :Cout]
        s = part.double().sum(0)
        assert rel(s[:Cout], zz.double().sum(0)) < 1e-5 or (s[:Cout] - zz.double().sum(0)).abs().max() < 1e-3
        assert rel(s[Cout:2 * Cout], (zz.double() ** 2).sum(0)) < 1e-5
        assert torch.equal(part[:, 2 * Cout:3 * Cout].min(0)[0], zz.min(0)[0])
        assert torch.equal(part[:, 3 * Cout:].max(0)[0], zz.max(0)[0])
        outs[mode] = got.clone()
        L.call('fsdet_conv_tc_fwd', X.hi.data_ptr(), X.lo.data_ptr(), Wp.hi.data_ptr(), Wp.lo.data_ptr(), X.a, Wp.a, z.data_ptr(), ld,
               B, H, W, Cin, cpitch, Cout, k, 1, mode, None, st())
        got2 = z[:, :Cout].contiguous().view(B, H, W, Cout).permute(0, 3, 1, 2)
        assert rel(got2, 2 * ref) < TOL_TC
    assert rel(outs[3], outs[3 | 64]) < 2e-6      # same products, different accumulation order
    assert rel(outs[3], outs[3 | 128]) < 2e-6


def test_conv_tc_term_modes_precision(L):
    """What each mode costs in accuracy on a long-K layer (printed; the bars are loose upper bounds)."""
    B, H, W, Cin, Cout, k = 2, 13, 13, 1024, 1024, 3
    g = torch.Generator(device='cuda').manual_seed(9)
    x = torch.randn(B, Cin, H, W, device='cuda', generator=g)
    w = torch.randn(Cout, Cin, k, k, device='cuda', generator=g) * 0.05
    ref = F.conv2d(x.double(), w.double(), None, 1, 1)
    X = split(L, nhwc(x))
    Wp = split(L, w.permute(0, 2, 3, 1).contiguous().view(Cout, -1))
    errs = {}
    for mode, bar in ((3, 1e-5), (1, 4e-4), (2, 4e-4), (0, 6e-4)):
        z = torch.zeros(B * H * W, Cout, device='cuda')
        L.call('fsdet_conv_tc_fwd', X.hi.data_ptr(), X.lo.data_ptr(), Wp.hi.data_ptr(), Wp.lo.data_ptr(), X.a, Wp.a,
               z.data_ptr(), Cout, B, H, W, Cin, Cin, Cout, k, 0, mode, None, st())
        errs[mode] = rel(z.view(B, H, W, Cout).permute(0, 3, 1, 2), ref)
        assert errs[mode] < bar, (mode, errs)
    print('conv_tc relative error by term mode:', errs)


def test_colstats(L):
    z = torch.randn(5000, 96, device='cuda') * 2 + 1
    buf = torch.zeros(5000, 100, device='cuda')
    buf[:, :96] = z
    rows = L.lib.fsdet_colstats_rows(5000)
    part = torch.zeros(rows, 4 * 96, device='cuda')
    L.call('fsdet_colstats', buf.data_ptr(), 100, 5000, 96, part.data_ptr(), st())
    s = part.double().sum(0)
    assert rel(s[:96], z.double().sum(0)) < 1e-5
    assert rel(s[96:192], (z.double() ** 2).sum(0)) < 1e-5
    assert torch.equal(part[:, 192:288].min(0)[0], z.min(0)[0])
    assert torch.equal(part[:, 288:].max(0)[0], z.max(0)[0])


WG_CASES = [
    # B, H, W, Cin, Cout, k
    (2, 13, 13, 64, 128, 3), (4, 26, 26, 128, 64, 1), (1, 52, 52, 64, 128, 3), (2, 13, 13, 1024, 640, 1),
    (2, 13, 13, 1280, 1024, 3), (3, 6, 6, 1024, 1024, 3), (2, 19, 19, 256, 512, 3), (8, 104, 104, 64, 128, 3),
    (1, 26, 26, 512, 64, 1), (3, 4, 4, 128, 256, 3), (3, 8, 8, 64, 128, 3), (3, 4, 4, 256, 256, 3), (1, 2, 2, 64, 64, 3),
]


@pytest.mark.parametrize('mode', [3, 0, 1, 2])
@pytest.mark.parametrize('B,H,W,Cin,Cout,k', WG_CASES)
def test_conv_tc_wgrad(L, B, H, W, Cin, Cout, k, mode):
    g = torch.Generator(device='cuda').manual_seed(B + H + Cin + Cout + 1)
    x = torch.randn(B, Cin, H, W, device='cuda', generator=g)
    dz = torch.randn(B, Cout, H, W, device='cuda', generator=g)
    X = split(L, nhwc(x))
    D = split(L, nhwc(dz))
    sx, sd = plane_scale(X), plane_scale(D)
    xh, xl = planes_nchw(X.hi, B, H, W, Cin), planes_nchw(X.lo, B, H, W, Cin)
    dh, dl = planes_nchw(D.hi, B, H, W, Cout), planes_nchw(D.lo, B, H, W, Cout)

    def wgrad64(xx, dd):
        w = torch.zeros(Cout, Cin, k, k, device='cuda', dtype=torch.float64, requires_grad=True)
        F.conv2d(xx, w, None, 1, (k - 1) // 2).backward(dd)
        return w.grad
    ref = wgrad64(xh, dh)
    if mode & 1:
        ref = ref + wgrad64(xh, dl)
    if mode & 2:
        ref = ref + wgrad64(xl, dh)
    ref = ref / (sx * sd)
    assert L.lib.fsdet_conv_tc_wgrad_supported(Cin, Cout, k)
    nws = L.lib.fsdet_conv_tc_wgrad_workspace_floats(B, H, W, Cin, Cout, k, mode)
    ws = torch.empty(max(nws, 4), device='cuda')
    dw = torch.full((Cout, k * k, Cin), 7.0, device='cuda')
    L.call('fsdet_conv_tc_wgrad', X.hi.data_ptr(), X.lo.data_ptr() if mode & 2 else None, D.hi.data_ptr(),
           D.lo.data_ptr() if mode & 1 else None, X.a, D.a, dw.data_ptr(), ws.data_ptr(), nws, B, H, W, Cin, Cout, k, mode, st())
    torch.cuda.synchronize()
    got = dw.view(Cout, k, k, Cin).permute(0, 3, 1, 2)
    assert rel(got, ref) < (TOL_TC if mode == 3 else 3e-5)
    if mode == 3:
        assert rel(got, wgrad64(x.double(), dz.double())) < TOL_TC


def test_conv_tc_padded_channels_and_small_cout(L):
    """32-channel layers: planes zero-padded to 64 channels; dgrad with 32 output channels (weight rows < tile)."""
    B, H, W, Cin, Cout, k = 2, 26, 26, 32, 64, 3
    g = torch.Generator(device='cuda').manual_seed(3)
    x = torch.randn(B, Cin, H, W, device='cuda', generator=g, requires_grad=True)
    w = (torch.randn(Cout, Cin, k, k, device='cuda', generator=g) * 0.05).requires_grad_(True)
    dz = torch.randn(B, Cout, H, W, device='cuda', generator=g) * 1e-5   # tiny gradients: exercises the scaling
    ref = F.conv2d(x, w, None, 1, 1)
    ref.backward(dz)
    X = split(L, nhwc(x.detach()), 64)
    Wp = split(L, w.detach().permute(0, 2, 3, 1).contiguous().view(Cout * k * k, Cin), 64)
    z = torch.zeros(B * H * W, Cout, device='cuda')
    L.call('fsdet_conv_tc_fwd', X.hi.data_ptr(), X.lo.data_ptr(), Wp.hi.data_ptr(), Wp.lo.data_ptr(), X.a, Wp.a, z.data_ptr(), Cout,
           B, H, W, 32, 64, Cout, k, 0, 3, None, st())
    assert rel(z.view(B, H, W, Cout).permute(0, 3, 1, 2), ref) < TOL_TC
    # dgrad: GEMM Cin = 64 (dz channels), Cout = 32
    wt = torch.empty(Cin, k * k, Cout, device='cuda')
    L.call('fsdet_weight_flip_transpose', w.detach().permute(0, 2, 3, 1).contiguous().data_ptr(), wt.data_ptr(), Cout, k * k, Cin, st())
    T = split(L, wt.view(Cin, k * k * Cout))
    D = split(L, nhwc(dz))
    dx = torch.zeros(B * H * W, Cin, device='cuda')
    L.call('fsdet_conv_tc_fwd', D.hi.data_ptr(), D.lo.data_ptr(), T.hi.data_ptr(), T.lo.data_ptr(), D.a, T.a, dx.data_ptr(), Cin,
           B, H, W, Cout, Cout, Cin, k, 0, 3, None, st())
    assert rel(dx.view(B, H, W, Cin).permute(0, 3, 1, 2), x.grad) < TOL_TC
    # wgrad with padded input channels: result [Cout][9][64], first 32 channels valid, rest zero
    nws = L.lib.fsdet_conv_tc_wgrad_workspace_floats(B, H, W, 64, Cout, k, 3)
    ws = torch.empty(max(nws, 4), device='cuda')
    dw = torch.full((Cout, k * k, 64), 7.0, device='cuda')
    L.call('fsdet_conv_tc_wgrad', X.hi.data_ptr(), X.lo.data_ptr(), D.hi.data_ptr(), D.lo.data_ptr(), X.a, D.a, dw.data_ptr(),
           ws.data_ptr(), nws, B, H, W, 64, Cout, k, 3, st())
    assert rel(dw[:, :, :32].reshape(Cout, k, k, Cin).permute(0, 3, 1, 2), w.grad) < TOL_TC
    assert (dw[:, :, 32:] == 0).all()
