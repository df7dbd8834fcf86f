"""Every tensor-core GEMM of a full-size eager training step against float64 of its own operands.

One step (Darknet forward, RegionLossV2, backward) runs through the public API with the shipped defaults, while every
convolution entry point the engine calls is intercepted: the device is synchronised, the call is made, and its output is
checked before the step goes on, while all operand buffers are still alive.  The call arguments (pointers and shapes)
define the operands completely; they are wrapped as tensors without copying.

  fsdet_conv_tc_fwd      forward, input gradient and head: float64 of exactly the products the mode multiplies
                         (mode 3: hi*hi + lo*hi + hi*lo), relative L2 < 1e-5 AND every element within
                         1e-4 * conv(|x|, |w|) of it - a norm over 10^8 elements dilutes one wrong tile edge, the
                         element-wise bound does not; columns past Cout untouched; fused BatchNorm partial rows
  fsdet_conv_tc_wgrad    float64 of the hi planes (mode 0), same two bars (the L2 bar allows for sums that cancel, see
                         ABS_L2); and the distance from the fp32-grade value (hi + lo planes), which is the precision
                         budget of engine._parse_terms (< 1e-3 per tensor)
  fsdet_conv_first_*     exact-fp32 SIMT first layer (3 + 1 channels on the support branch) and its statistics
  fsdet_weight_prep      every layer's forward / input-gradient planes equal fsdet_split_f16 of the weight (bit for bit)
  fsdet_conv_fwd / _wgrad  the SIMT fallbacks, should the step use them

A GEMM-like entry point the checker does not know fails the test, so coverage cannot shrink silently; each run also
asserts which kernel flavours (halo, short-K and long-K im2col, one- and two-tap weight-gradient tiles, split-K) it
reached.  The file name sorts last: the slowest GPU tests run last.
"""
import math
import re
import struct
import sys
import time

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

ELEM = 1e-4            # element-wise bar, as a fraction of the same GEMM over absolute values
SMALLK_MAX = 2304      # conv_tc.cu tc_plan: K = k*k*Cin above this (Cin % 64 == 0) runs the long-K (folded) flavour
# float64 references are built a few images at a time, at most this many elements per tensor (1 GB): at 608x608 and
# B = 64 the first layer's output alone is 7.6e8 elements
CHUNK = 1 << 27


def image_chunks(B, per_image):
    """[(b0, b1)] image ranges of at most CHUNK elements of `per_image` each (at least one image)"""
    step = max(1, CHUNK // max(1, per_image))
    return [(b, min(B, b + step)) for b in range(0, B, step)]


class _Dev(object):
    """A raw device pointer as a 1-D tensor (no copy)."""

    def __init__(self, p, n, typestr):
        self.__cuda_array_interface__ = {'shape': (int(n),), 'typestr': typestr, 'data': (int(p), False), 'version': 2}


def dev(p, n, dtype=torch.float32):
    typestr = {torch.float32: '<f4', torch.float16: '<f2', torch.int16: '<i2', torch.uint8: '|u1'}[dtype]
    return torch.as_tensor(_Dev(p, n, typestr), device='cuda')


def rows_view(p, rows, cols, ld):
    """[rows][cols] fp32 view of a row-major buffer with leading dimension ld (the last row may end the allocation)."""
    flat = dev(p, (rows - 1) * ld + cols)
    return flat.as_strided((rows, cols), (ld, 1))


def scale_from_amax(a):
    """conv_tc.cu: the power of two that maps the absolute maximum into [512, 1024)."""
    if not (a > 0) or not math.isfinite(a):
        return 1.0
    _, ex = math.frexp(a)
    return 2.0 ** max(-60, min(60, 10 - ex))


def nchw(t):          # [B,H,W,C] -> contiguous float64 NCHW
    return t.permute(0, 3, 1, 2).double().contiguous()


def rel(got, ref):
    return ((got - ref).norm() / ref.norm().clamp_min(1e-300)).item()


# A weight gradient sums dz * x over every pixel of the batch.  BatchNorm makes each dz channel sum to zero while x (a
# LeakyReLU / max-pool output, or the input images) has a large positive mean, so the signed sum cancels: for conv2 at
# B = 64 (2.77 M pixels), |dz| * |x| summed is 977 times the result (norms over the tensor).  The relative L2 error then
# measures the cancellation rather than the kernel: fp32 accumulation leaves 4.7e-5 of that gradient (element-wise
# ratio 0.001), which is 4.8e-8 of the absolute-value sum, below the fp32 epsilon; the first layer's weight gradient
# (images in [0, 1)) cancels 2171-fold and keeps 1.3e-4 of it.  Where the relative L2 bar is missed, the error norm is
# therefore taken against the GEMM of absolute values instead (measured <= 7.3e-8 over both configurations on an H100
# SXM 80 GB).  The element-wise bar is the same for every call.
ABS_L2 = 1e-6


def l2_ok(e, cancel, bar):
    """relative L2 e below bar, or - for a cancelling sum - below ABS_L2 of the absolute-value GEMM"""
    return e < bar or e / cancel < ABS_L2


def elem_ratio(got, ref, absref):
    """max |got - ref| / (ELEM * absref); a NaN or a difference where absref == 0 counts as infinite."""
    d = (got - ref).abs()
    r = d / (ELEM * absref)
    r = torch.where(d == 0, torch.zeros_like(r), r)
    return torch.nan_to_num(r, nan=math.inf, posinf=math.inf).max().item()


def fwd_refs(B, H, W, Cin, cpitch, Cout, k, terms, xh, xl, wh, wl, sx, sw, b0=0, b1=None):
    """(value, |value| bound) of the products mode `terms` multiplies (float64, unscaled): hi*hi (+ x_lo*w_hi)
    (+ x_hi*w_lo) of the fp16 planes; output rows of images [b0, b1)."""
    b1 = B if b1 is None else b1
    M = B * H * W
    X = lambda p: nchw(dev(p, M * cpitch, torch.float16).view(B, H, W, cpitch)[b0:b1, ..., :Cin])
    Wt = lambda p: nchw(dev(p, Cout * k * k * cpitch, torch.float16).view(Cout, k, k, cpitch)[..., :Cin])
    pad = (k - 1) // 2
    conv = lambda a, b: F.conv2d(a, b, None, 1, pad).permute(0, 2, 3, 1).reshape((b1 - b0) * H * W, Cout)
    inv = 1.0 / (sx * sw)
    Xh, Wh = X(xh), Wt(wh)
    Xa, Wa = Xh.abs(), Wh.abs()
    if terms & 1:
        Xl = X(xl)
        ref = conv(Xh + Xl, Wh)
        Xa = Xa + Xl.abs()
        del Xl
    else:
        ref = conv(Xh, Wh)
    if terms & 2:
        Wl = Wt(wl)
        ref += conv(Xh, Wl)
        Wa = Wa + Wl.abs()
    del Xh
    ref *= inv
    absref = conv(Xa, Wa) * inv
    return ref, absref


def check_stats(expect, S, z, what):
    """S [rows][4][C] partial rows (sum | sum of squares | min | max) against the stored z [M][C]."""
    s, q = S[:, 0].double().sum(0), S[:, 1].double().sum(0)
    s_ref, a_ref, q_ref = (torch.zeros(z.shape[1], dtype=torch.float64, device=z.device) for _ in range(3))
    for r0 in range(0, z.shape[0], CHUNK // z.shape[1]):
        zz = z[r0:r0 + CHUNK // z.shape[1]].double()
        s_ref += zz.sum(0)
        a_ref += zz.abs().sum(0)
        q_ref += (zz * zz).sum(0)
    del zz
    # column sums cancel (pre-BatchNorm values of both signs): bounded against the column's absolute sum
    expect(((s - s_ref).abs() <= 1e-5 * a_ref + 1e-30).all().item(), (what, 'partial sums'))
    expect(((q - q_ref).abs() <= 1e-5 * q_ref + 1e-30).all().item(), (what, 'partial sums of squares'))
    expect(torch.equal(S[:, 2].min(0).values, z.min(0).values), (what, 'partial minima'))
    expect(torch.equal(S[:, 3].max(0).values, z.max(0).values), (what, 'partial maxima'))


class StepChecker(object):
    """Wraps engine.call: GEMM entry points are run synchronously and checked against float64."""
    GEMM_LIKE = re.compile(r'conv|gemm|wgrad|weight_prep')

    def __init__(self, real_call, lib):
        self.real = real_call
        self.lib = lib
        self.log = []
        self.cov = set()
        self.unknown = []
        self.failures = []
        self.first_fwd = []     # (B, H, W) of every first-layer forward

    def expect(self, ok, what):
        """A failed check is recorded and raised when the step has finished, so that the whole table prints."""
        if not ok:
            self.failures.append(what)
            print('FAILED:', what)

    def __call__(self, fn, *a):
        handler = getattr(self, 'chk_' + fn[len('fsdet_'):], None)
        if handler is None:
            if self.GEMM_LIKE.search(fn):
                self.unknown.append(fn)
                raise AssertionError('GEMM-like entry point without a float64 check: %s' % fn)
            return self.real(fn, *a)
        torch.cuda.synchronize()
        t0 = time.time()
        rc = handler(fn, a)
        torch.cuda.synchronize()
        self.log[-1]['sec'] = time.time() - t0
        print('%-10s %-44s %-12s rel %.2e  elem %.3f%s' % (self.log[-1]['kind'], self.log[-1]['shape'], self.log[-1]['flavour'],
                                                          self.log[-1]['rel'], self.log[-1]['ratio'], self.log[-1].get('extra', '')))
        sys.stdout.flush()
        return rc

    @staticmethod
    def _kind():
        """Which GEMM of the network the current call is (read from the engine's call stack)."""
        frames = []
        f = sys._getframe(1)
        while f is not None and len(frames) < 16:
            frames.append(f)
            f = f.f_back
        head = any(f.f_code.co_name == '_head_bwd' for f in frames)
        for f in frames:
            if f.f_code.co_name == '_conv':
                n = f.f_locals.get('name')
                return 'head-dgrad' if (head and n == 'dgrad') else n
            if f.f_code.co_name == '_wgrad':
                return 'head-wgrad' if head else 'wgrad'
        return '?'

    # ---- tensor-core forward / input gradient / head
    def chk_conv_tc_fwd(self, fn, a):
        xh, xl, wh, wl, xa, wa, zp, ldz, B, H, W, Cin, cpitch, Cout, k, acc, mode, stat, st = a
        M = B * H * W
        terms = mode & 3
        kind = self._kind()
        z = rows_view(zp, M, Cout, ldz)
        tail = rows_view(zp + 4 * Cout, M - 1, ldz - Cout, ldz).clone() if ldz > Cout and M > 1 else None
        z0 = z.clone() if acc else None
        if not acc:
            z.fill_(float('nan'))            # every element must be stored
        rows = self.lib.fsdet_conv_tc_stat_rows(B, H, W, Cin, Cout, k, mode) if stat else 0
        S = dev(stat, rows * 4 * Cout).view(rows, 4, Cout) if stat else None
        if stat:
            S.fill_(float('nan'))
        rc = self.real(fn, *a)
        torch.cuda.synchronize()
        sx = scale_from_amax(dev(xa, 1).item())
        sw = scale_from_amax(dev(wa, 1).item())
        err2 = ref2 = r = 0.0
        for b0, b1 in image_chunks(B, H * W * max(cpitch, Cout)):
            ref, absref = fwd_refs(B, H, W, Cin, cpitch, Cout, k, terms, xh, xl, wh, wl, sx, sw, b0, b1)
            rs = slice(b0 * H * W, b1 * H * W)
            got = z[rs].double()
            if acc:
                got -= z0[rs].double()
                # the stored sum z0 + conv is rounded to fp32 once: half an ulp of the stored value on top of the bar
                absref += (0.5 * 2.0 ** -23 / ELEM) * z[rs].double().abs()
            err2 += (got - ref).norm().item() ** 2
            ref2 += ref.norm().item() ** 2
            r = max(r, elem_ratio(got, ref, absref))
            del got, ref, absref
        e = math.sqrt(err2) / max(math.sqrt(ref2), 1e-300)      # rel() over the whole output
        halo = self.lib.fsdet_conv_tc_uses_halo(B, H, W, Cin, Cout, k, mode) == 1
        fold = not halo and Cin % 64 == 0 and k * k * Cin > SMALLK_MAX
        flav = 'halo' if halo else ('im2col-long' if fold else 'im2col-short')
        self.cov.add(flav)
        self.cov.add(kind)
        if kind == 'fwd':
            # the epilogue with or without BatchNorm statistics rows: a replica step (and evaluation) runs every forward
            # without them, its segmented BatchNorm pass reads z once more instead
            self.cov.add('fwd-stats' if stat else 'fwd-nostats')
        if acc:
            self.cov.add('accumulate')
        self._record(kind, '%dx%dx%dx%d->%d k%d m%d%s' % (B, H, W, Cin, Cout, k, mode, ' acc' if acc else ''), flav, e, r)
        self.expect(e < 1e-5, (kind, flav, B, H, W, Cin, Cout, k, 'relative L2', e))
        self.expect(r <= 1.0, (kind, flav, B, H, W, Cin, Cout, k, 'element-wise', r))
        if tail is not None:
            self.expect(torch.equal(rows_view(zp + 4 * Cout, M - 1, ldz - Cout, ldz), tail), (kind, 'columns past Cout written'))
        if stat:
            check_stats(self.expect, S, z, (kind, flav, B, H, W, Cin, Cout))
        return rc

    # ---- tensor-core weight gradient
    def chk_conv_tc_wgrad(self, fn, a):
        xh, xl, dh, dl, xa, da, dw, ws, nws, B, H, W, Cin, Cout, k, mode, st = a
        M = B * H * W
        terms = mode & 3
        kind = self._kind()
        out = dev(dw, Cout * k * k * Cin)
        out.fill_(float('nan'))
        rc = self.real(fn, *a)
        torch.cuda.synchronize()
        inv = 1.0 / (scale_from_amax(dev(da, 1).item()) * scale_from_amax(dev(xa, 1).item()))
        X = lambda p, b0, b1: nchw(dev(p, M * Cin, torch.float16).view(B, H, W, Cin)[b0:b1])
        D = lambda p, b0, b1: nchw(dev(p, M * Cout, torch.float16).view(B, H, W, Cout)[b0:b1])
        wg = lambda x, d: torch.nn.grad.conv2d_weight(x, (Cout, Cin, k, k), d, 1, (k - 1) // 2).permute(0, 2, 3, 1).reshape(-1)
        ref = absref = full = 0.0
        for b0, b1 in image_chunks(B, H * W * max(Cin, Cout)):     # a sum over images: accumulated chunk by chunk
            Xh, Dh = X(xh, b0, b1), D(dh, b0, b1)
            Xl, Dl = X(xl, b0, b1), D(dl, b0, b1)
            # what the mode multiplies: dz_hi*x_hi (+ dz_lo*x_hi) (+ dz_hi*x_lo)
            ref = ref + wg(Xh, Dh + Dl if terms & 1 else Dh)
            if terms & 2:
                ref = ref + wg(Xl, Dh)
            absref = absref + wg(Xh.abs() + (Xl.abs() if terms & 2 else 0), Dh.abs() + (Dl.abs() if terms & 1 else 0))
            full = full + wg(Xh + Xl, Dh + Dl)      # fp32-grade operands: the value the budget is measured against
            del Xh, Xl, Dh, Dl
        got = out.double()
        e, r = rel(got, ref * inv), elem_ratio(got, ref * inv, absref * inv)
        cancel = (absref.norm() / ref.norm()).item()       # how much the sum cancels: |x|*|dz| over x*dz
        del ref, absref
        ef = rel(got, full * inv)
        del full, got
        taps = 1 if Cin >= 128 else 2
        splits = 0
        if self.lib.fsdet_conv_tc_wgrad_workspace_floats(B, H, W, Cin, Cout, k, mode) > 0:
            splits = self.lib.fsdet_conv_tc_wgrad_workspace_floats(B, H, W, Cin, Cout, k, mode) // (Cout * k * k * Cin)
        flav = 'taps%d split%d' % (taps, max(splits, 1))
        self.cov.update({'wgrad-taps%d' % taps, 'wgrad-splitk' if splits > 1 else 'wgrad-nosplit', kind})
        self._record(kind, '%dx%dx%dx%d->%d k%d m%d' % (B, H, W, Cin, Cout, k, mode), flav, e, r,
                     extra='  vs fp32-grade %.2e  cancellation %.0f' % (ef, cancel), full=ef)
        bar = 3e-5 if terms == 0 else 1e-5
        self.expect(l2_ok(e, cancel, bar), (kind, B, H, W, Cin, Cout, k, 'relative L2', e, 'cancellation', cancel))
        self.expect(r <= 1.0, (kind, B, H, W, Cin, Cout, k, 'element-wise', r))
        self.expect(ef < 1e-3, (kind, B, H, W, Cin, Cout, k, 'distance from the fp32-grade weight gradient', ef))
        return rc

    # ---- exact-fp32 first layer
    def _first_input(self, in0, c0, in1, c1, B, H, W, b0=0, b1=None):
        """float64 NCHW input of images [b0, b1)"""
        x = dev(in0, B * c0 * H * W).view(B, c0, H, W)[b0:b1]
        if c1:
            x = torch.cat([x, dev(in1, B * c1 * H * W).view(B, c1, H, W)[b0:b1]], 1)
        return x.double()

    def chk_conv_first_fwd_stats(self, fn, a):
        in0, c0, in1, c1, w, zp, ldz, B, H, W, Cout, stat, st = a
        return self._first_fwd(fn, a, in0, c0, in1, c1, w, zp, ldz, B, H, W, Cout, stat)

    def chk_conv_first_fwd(self, fn, a):
        in0, c0, in1, c1, w, zp, ldz, B, H, W, Cout, st = a
        return self._first_fwd(fn, a, in0, c0, in1, c1, w, zp, ldz, B, H, W, Cout, None)

    def _first_fwd(self, fn, a, in0, c0, in1, c1, w, zp, ldz, B, H, W, Cout, stat):
        M = B * H * W
        z = rows_view(zp, M, Cout, ldz)
        z.fill_(float('nan'))
        rows = self.lib.fsdet_conv_first_stat_rows(B, H, W) if stat else 0
        S = dev(stat, rows * 4 * Cout).view(rows, 4, Cout) if stat else None
        if stat:
            S.fill_(float('nan'))
        rc = self.real(fn, *a)
        torch.cuda.synchronize()
        self.first_fwd.append((B, H, W))
        wt = dev(w, Cout * 36).view(Cout, 3, 3, 4)[..., :c0 + c1].permute(0, 3, 1, 2).double()
        err2 = ref2 = r = 0.0
        for b0, b1 in image_chunks(B, H * W * Cout):
            x = self._first_input(in0, c0, in1, c1, B, H, W, b0, b1)
            ref = F.conv2d(x, wt, None, 1, 1).permute(0, 2, 3, 1).reshape(-1, Cout)
            absref = F.conv2d(x.abs(), wt.abs(), None, 1, 1).permute(0, 2, 3, 1).reshape(-1, Cout)
            got = z[b0 * H * W:b1 * H * W].double()
            err2 += (got - ref).norm().item() ** 2
            ref2 += ref.norm().item() ** 2
            r = max(r, elem_ratio(got, ref, absref))
            del x, ref, absref, got
        e = math.sqrt(err2) / max(math.sqrt(ref2), 1e-300)
        self.cov.add('first-fwd')
        self._record('first-fwd', '%dx%dx%dx%d->%d k3' % (B, H, W, c0 + c1, Cout), 'simt', e, r)
        self.expect(e < 1e-5 and r <= 1.0, ('first-layer forward', B, H, W, c0, c1, e, r))
        if stat:
            check_stats(self.expect, S, z, ('first-layer forward', B, H, W))
        return rc

    def chk_conv_first_wgrad(self, fn, a):
        in0, c0, in1, c1, dz, lddz, dw, ws, nws, B, H, W, Cout, st = a
        M = B * H * W
        out = dev(dw, Cout * 36)
        out.fill_(float('nan'))
        rc = self.real(fn, *a)
        torch.cuda.synchronize()
        wg = lambda xx, dd: torch.nn.grad.conv2d_weight(xx, (Cout, 4, 3, 3), dd, 1, 1).permute(0, 2, 3, 1).reshape(-1)
        ref = absref = 0.0
        for b0, b1 in image_chunks(B, H * W * Cout):
            x = torch.zeros(b1 - b0, 4, H, W, dtype=torch.float64, device='cuda')
            x[:, :c0 + c1] = self._first_input(in0, c0, in1, c1, B, H, W, b0, b1)
            d = nchw(rows_view(dz, M, Cout, lddz).view(B, H, W, Cout)[b0:b1])
            ref = ref + wg(x, d)
            absref = absref + wg(x.abs(), d.abs())
            del x, d
        got = out.double()
        e, r = rel(got, ref), elem_ratio(got, ref, absref)
        cancel = (absref.norm() / ref.norm()).item()
        self.cov.add('first-wgrad')
        self._record('first-wgrad', '%dx%dx%dx%d->%d k3' % (B, H, W, c0 + c1, Cout), 'simt', e, r,
                     extra='  cancellation %.0f' % cancel)
        self.expect(l2_ok(e, cancel, 1e-5) and r <= 1.0, ('first-layer weight gradient', B, H, W, c0, c1, e, r, cancel))
        return rc

    # ---- SIMT fallbacks (not expected in the shipped configuration, checked if they run)
    def chk_conv_fwd(self, fn, a):
        x, ldx, w, bias, zp, ldz, stat, B, H, W, Cin, Cout, k, acc, st = a
        M = B * H * W
        z = rows_view(zp, M, Cout, ldz)
        z0 = z.clone() if acc else None
        rows = self.lib.fsdet_conv_stat_rows(M) if stat else 0
        rc = self.real(fn, *a)
        torch.cuda.synchronize()
        X = nchw(rows_view(x, M, Cin, ldx).view(B, H, W, Cin))
        Wt = nchw(dev(w, Cout * k * k * Cin).view(Cout, k, k, Cin))
        b = dev(bias, Cout).double() if bias else None
        ref = F.conv2d(X, Wt, b, 1, (k - 1) // 2).permute(0, 2, 3, 1).reshape(M, Cout)
        absref = F.conv2d(X.abs(), Wt.abs(), b.abs() if b is not None else None, 1, (k - 1) // 2).permute(0, 2, 3, 1).reshape(M, Cout)
        got = z.double() - (z0.double() if acc else 0)
        if acc:
            absref += (0.5 * 2.0 ** -23 / ELEM) * z.double().abs()
        e, r = rel(got, ref), elem_ratio(got, ref, absref)
        kind = self._kind()
        self.cov.add('simt-fwd')
        self._record(kind, '%dx%dx%dx%d->%d k%d' % (B, H, W, Cin, Cout, k), 'simt', e, r)
        self.expect(e < 1e-5 and r <= 1.0, ('SIMT convolution', kind, B, H, W, Cin, Cout, k, e, r))
        if stat:
            check_stats(self.expect, dev(stat, rows * 4 * Cout).view(rows, 4, Cout), z, ('SIMT convolution', B, H, W, Cin, Cout))
        return rc

    def chk_conv_wgrad(self, fn, a):
        x, ldx, dz, lddz, dw, ws, nws, B, H, W, Cin, Cout, k, st = a
        M = B * H * W
        rc = self.real(fn, *a)
        torch.cuda.synchronize()
        X = nchw(rows_view(x, M, Cin, ldx).view(B, H, W, Cin))
        D = nchw(rows_view(dz, M, Cout, lddz).view(B, H, W, Cout))
        wg = lambda xx, dd: torch.nn.grad.conv2d_weight(xx, (Cout, Cin, k, k), dd, 1, (k - 1) // 2).permute(0, 2, 3, 1).reshape(-1)
        ref, absref = wg(X, D), wg(X.abs(), D.abs())
        got = dev(dw, Cout * k * k * Cin).double()
        e, r = rel(got, ref), elem_ratio(got, ref, absref)
        self.cov.add('simt-wgrad')
        self._record(self._kind(), '%dx%dx%dx%d->%d k%d' % (B, H, W, Cin, Cout, k), 'simt', e, r)
        self.expect(e < 1e-5 and r <= 1.0, ('SIMT weight gradient', B, H, W, Cin, Cout, k, e, r))
        return rc

    # ---- weight planes of all tensor-core layers
    def chk_weight_prep(self, fn, a):
        descs, tiles, n_tiles, amax_all, n, st = a
        rc = self.real(fn, *a)
        torch.cuda.synchronize()
        raw = bytes(dev(descs, 80 * n, torch.uint8).cpu().numpy())
        for i in range(n):
            w, fh, fl, bh, bl, am, Cout, kk, Cin, fp, bp, _, _, _ = struct.unpack_from('<6Q8i', raw, 80 * i)
            wt = dev(w, Cout * kk * Cin)
            amax = dev(am, 1)
            self.expect(amax.item() == wt.abs().max().item(), ('weight amax', i))
            for hi, lo, C, pitch, rows, src in ((fh, fl, Cin, fp, Cout * kk, wt), (bh, bl, Cout, bp, Cin * kk, None)):
                if not hi:
                    continue
                if src is None:       # input-gradient operand: wt[ci][kk-1-tap][co] = w[co][tap][ci]
                    src = torch.empty(Cin * kk * Cout, device='cuda')
                    self.real('fsdet_weight_flip_transpose', w, src.data_ptr(), Cout, kk, Cin, st)
                eh = torch.empty(rows, pitch, dtype=torch.float16, device='cuda')
                el = torch.empty_like(eh)
                self.real('fsdet_split_f16', src.data_ptr(), C, C, pitch, rows, am, eh.data_ptr(), el.data_ptr(), st)
                torch.cuda.synchronize()
                gh = dev(hi, rows * pitch, torch.int16).view(rows, pitch)
                gl = dev(lo, rows * pitch, torch.int16).view(rows, pitch)
                self.expect(torch.equal(gh, eh.view(torch.int16)) and torch.equal(gl, el.view(torch.int16)), ('weight planes', i, C, pitch))
                self.expect(not gh[:, C:].any() and not gl[:, C:].any(), ('weight plane padding', i))
        self.cov.add('weight-prep')
        self._record('wprep', '%d layers' % n, 'split', 0.0, 0.0)
        return rc

    def _record(self, kind, shape, flav, e, r, extra='', full=None):
        self.log.append(dict(kind=kind, shape=shape, flavour=flav, rel=e, ratio=r, extra=extra, full=full))


def run_step(side, bs, cs, seed, wrap, replicas=1):
    """One eager step (forward, RegionLossV2, backward) of the full network with `bs` query images of side x side and
    `cs` classes (support images at 416x416), while engine.call is replaced by wrap(engine.call).  With replicas = R
    the model is Darknet(..., replicas=R) and the support batch R * cs images (R support sets).  Returns the head
    output (detached), the region loss module, the label tensor and the seconds the step took."""
    from fewshot_detection_b200 import engine
    from test_gpu_zz_configs import _batch
    from fewshot_detection_b200 import netcfg
    from fewshot_detection_b200.darknet_meta import Darknet
    from seeding import seeded_init
    m = Darknet(netcfg.darknet_dynamic_blocks(side, side), netcfg.reweighting_net_blocks(), replicas=replicas)
    seeded_init(m, seed)
    m = m.cuda().train()
    x, metax, mask, tgt = _batch(bs, cs, side, seed + 1, replicas=replicas)
    L = m.models[len(m.models) - 1]
    L.seen = 20000
    L.verbose = False
    real = engine.call
    engine.call = wrap(real)
    t0 = time.time()
    try:
        out = m(x.cuda(), metax.cuda(), mask.cuda())
        loss = L(out, tgt)
        loss.backward()
        torch.cuda.synchronize()
    finally:
        engine.call = real
    secs = time.time() - t0
    assert torch.isfinite(loss).item()
    return out.detach(), L, tgt, secs


def _run_step(side, bs, cs, seed):
    from fewshot_detection_b200 import _lib
    chk = []
    secs = run_step(side, bs, cs, seed, lambda real: chk.append(StepChecker(real, _lib.lib)) or chk[0])[3]
    return report(chk[0], secs)


def report(chk, secs):
    """Prints the worst ratio per GEMM class of one checked step and fails if any check failed."""
    assert not chk.unknown, chk.unknown
    tc = [l for l in chk.log if l['flavour'] not in ('split',)]
    worst = {}
    for l in tc:
        k = (l['kind'], l['flavour'].split()[0] if l['kind'].endswith('wgrad') else l['flavour'])
        w = worst.setdefault(k, [0.0, 0.0, 0, 0.0])
        w[0] = max(w[0], l['rel'])
        w[1] = max(w[1], l['ratio'])
        w[2] += 1
        if l['full'] is not None:
            w[3] = max(w[3], l['full'])
    print('\n%d checked calls, %.1f s (step + float64 references); worst per class:' % (len(chk.log), secs))
    for k, w in sorted(worst.items()):
        print('  %-12s %-14s n=%3d  rel %.2e  elem %.3f%s' % (k[0], k[1], w[2], w[0], w[1],
                                                              '  vs fp32-grade %.2e' % w[3] if w[3] else ''))
    print('coverage:', sorted(chk.cov))
    assert not chk.failures, chk.failures
    return chk


# the flavours a full-size step must reach (the accumulating GEMM is optional: see below)
COVERAGE = {'halo', 'im2col-short', 'im2col-long', 'fwd', 'dgrad', 'head', 'head-dgrad', 'head-wgrad', 'wgrad',
            'wgrad-taps1', 'wgrad-taps2', 'wgrad-splitk', 'wgrad-nosplit', 'first-fwd', 'first-wgrad', 'weight-prep'}


def test_configs1_step_gemms_vs_float64():
    """configs[1]: B = 64 query images + 20 support images at 416x416, 20 classes (head N = 600 -> 640)."""
    chk = _run_step(416, 64, 20, 61)
    assert COVERAGE <= chk.cov, sorted(COVERAGE - chk.cov)
    # an input gradient accumulates into an existing gradient through a GEMM only when the GEMM is not the first writer
    # (the route after conv13 is summed by fsdet_copy_channels); the accumulate path is covered by test_gpu_tc.py
    print('accumulating GEMM in the step:', 'accumulate' in chk.cov)


def test_configs4_step_gemms_vs_float64():
    """configs[4]: 608x608 (G = 19), 80 classes (head N = 2400 -> 2432), B = 2."""
    chk = _run_step(608, 2, 80, 71)
    assert {'halo', 'im2col-short', 'im2col-long', 'head', 'head-dgrad', 'head-wgrad', 'wgrad-taps1',
            'wgrad-taps2'} <= chk.cov, sorted(chk.cov)
    print('accumulating GEMM in the step:', 'accumulate' in chk.cov)


def test_checker_reports_one_corrupted_element():
    """The element-wise bar has teeth: one element of a real fsdet_conv_tc_fwd output moved by four times its bar is
    reported, although the relative L2 over the whole tensor stays below 1e-5."""
    from fewshot_detection_b200 import _lib
    st = torch.cuda.current_stream().cuda_stream
    B, H, W, Ci, Co = 16, 52, 52, 64, 256
    g = torch.Generator(device='cuda').manual_seed(3)
    x = torch.randn(B * H * W, Ci, device='cuda', generator=g)
    w = torch.randn(Co * 9, Ci, device='cuda', generator=g) * 0.03

    def planes(t):
        am = torch.zeros(1, device='cuda')
        _lib.call('fsdet_amax', t.data_ptr(), t.shape[1], t.shape[1], t.shape[0], am.data_ptr(), st)
        hi = torch.empty(t.shape, dtype=torch.float16, device='cuda')
        lo = torch.empty_like(hi)
        _lib.call('fsdet_split_f16', t.data_ptr(), t.shape[1], t.shape[1], t.shape[1], t.shape[0], am.data_ptr(), hi.data_ptr(),
                  lo.data_ptr(), st)
        return hi, lo, am
    (xh, xl, xa), (wh, wl, wa) = planes(x), planes(w)
    z = torch.empty(B * H * W, Co, device='cuda')
    _lib.call('fsdet_conv_tc_fwd', xh.data_ptr(), xl.data_ptr(), wh.data_ptr(), wl.data_ptr(), xa.data_ptr(), wa.data_ptr(),
              z.data_ptr(), Co, B, H, W, Ci, Ci, Co, 3, 0, 3, None, st)
    torch.cuda.synchronize()
    ref, absref = fwd_refs(B, H, W, Ci, Ci, Co, 3, 3, xh.data_ptr(), xl.data_ptr(), wh.data_ptr(), wl.data_ptr(),
                           scale_from_amax(xa.item()), scale_from_amax(wa.item()))
    got = z.double()
    assert rel(got, ref) < 1e-5 and elem_ratio(got, ref, absref) <= 1.0
    i, j = 12345, 77
    got[i, j] += 4 * ELEM * absref[i, j]
    assert rel(got, ref) < 1e-5                         # invisible to the norm ...
    assert elem_ratio(got, ref, absref) > 3.0          # ... reported by the element-wise bar
    got[i, j] = float('nan')
    assert elem_ratio(got, ref, absref) == math.inf
