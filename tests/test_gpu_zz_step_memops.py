"""Every non-GEMM kernel of a full-size eager training step against float64 of its own operands.

The twin of test_gpu_zz_step_gemms.py for the rest of the step: one step (Darknet forward, RegionLossV2, backward) runs
through the public API with the shipped defaults while engine.call is intercepted.  Before each call the device is
synchronised and every output is filled with NaN (an element left unwritten is caught); after it, the output is checked
against its own operands while the buffers are alive.  GEMM entry points pass through (test_gpu_zz_step_gemms owns
them); the ones that fill BatchNorm partial rows are remembered, so that fsdet_bn_finalize is checked against the z that
produced its rows.  An entry point that is neither checked nor on PASS fails the test, so coverage cannot shrink
silently.

  fsdet_bn_finalize        mean / invstd against float64 of z (|d| <= 1e-5 std, 1e-5 invstd), scale and shift within
                           an ulp, running statistics, amax_y within an ulp of max|leaky(z*scale+shift)|, xhat_absmax
                           bit-equal to the fp32 max|(z - mean)*invstd|; max |mean|/std per layer is reported.
                           Eval mode: the running statistics as mean / 1 / sqrtf(var + eps), scale and shift within an
                           ulp, running statistics bit-unchanged, xhat_absmax and amax_y 0 when given and untouched
                           when not
  fsdet_bn_act_fwd         fp32 outputs bit-equal to the fp32 arithmetic (one fma, one multiply by the slope) and within
                           two roundings of float64; pooled = max of its window; fp16 planes bit-equal to the split;
                           padding zero; amax_y >= every value written
  fsdet_bn_act_bwd_reduce  (checked through the finalize that consumes the rows)
  + fsdet_bn_bwd_finalize  dbeta, dgamma, c1, c2 within 1e-6 of the sum of absolute terms (du in float64: dy_pool to the
                           first maximum, strict >, + dy_full, through leaky' of the fp32 pre-activation)
  fsdet_bn_act_bwd_apply   dz within 1e-6 |scale| (|du| + |c1| + |xhat c2|) of float64 with the kernel's coefficients, and
                           within 1e-5 of the same bound of a from-scratch float64 BatchNorm backward, on top of the
                           first-order propagation of the fp32 statistics' measured error and of the sums' bar;
                           planes bit-equal to
                           the split of fp32 dz; amax_bound >= max|dz|; conv + bias (has_bn = 0) dz bit-exact
  segmented passes         (a replica step: [nseg][C] vectors, [nseg][2C] coefficients, segment k = images
  (fsdet_*_seg)            [k B/nseg, (k+1) B/nseg)) the plain checks above applied per segment: colstats partial rows
                           per segment (sums to 1e-5 of the absolute sums, minima and maxima exact); each segment's mean
                           and invstd against float64 of that segment alone, running statistics from segment 0
                           (unbiased over its pixels, and bit-unchanged when the other segments' rows change), one
                           amax_y over all segments, max |mean|/std per segment reported; segment k's scale and shift on
                           segment k's images; per-segment c1 / c2, dgamma / dbeta summed over segments, dz per segment
                           including the from-scratch backward over the segment's statistics; one amax_bound >= max|dz|
  data movement            maxpool, reorg, copy_channels, layout conversions, pad_channels, weight_flip_transpose, amax,
                           split_f16, head_weff, globalmax (first maximum in pixel order): bit-exact
  head_param_grads / head_bias_grad   float64, within 1e-6 of the sum of absolute terms
"""
import math
import re
import sys
import time

import pytest
import torch

from test_gpu_zz_step_gemms import check_stats, run_step, scale_from_amax

pytestmark = pytest.mark.gpu

EPS = 1e-5
STAT_BAR = 1e-5          # finalize: |d mean| / std and |d invstd| / invstd
SUM_BAR = 1e-6           # backward sums and dz, as a fraction of the sum of absolute terms
SCRATCH_BAR = 1e-5       # dz against a from-scratch float64 BatchNorm backward
CHUNK = 1 << 25          # elements per float64 chunk (the first layer's z is 64 * 416^2 * 32 = 3.5e8 elements)

GEMM = re.compile(r'conv|gemm|wgrad|weight_prep')
# entry points that fill BatchNorm partial rows: their z is what fsdet_bn_finalize is checked against
STAT_WRITERS = {'fsdet_conv_tc_fwd': (6, 7, 8, 9, 10, 13, 17), 'fsdet_conv_first_fwd_stats': (5, 6, 7, 8, 9, 10, 11),
                'fsdet_conv_fwd': (4, 5, 7, 8, 9, 11, 6)}   # (z, ldz, B, H, W, Cout, stat) argument positions
PASS = set()             # checked elsewhere or pure queries: none in the step so far

_TYPES = {torch.float32: '<f4', torch.float64: '<f8', torch.float16: '<f2', torch.int16: '<i2', torch.int32: '<i4',
          torch.uint8: '|u1'}


class _Dev(object):
    def __init__(self, p, n, typestr):
        self.__cuda_array_interface__ = {'shape': (int(n),), 'typestr': typestr, 'data': (int(p), False), 'version': 2}


def dev(p, n, dtype=torch.float32):
    """a raw device pointer as a 1-D tensor (no copy)"""
    return torch.as_tensor(_Dev(p, n, _TYPES[dtype]), device='cuda')


def rows(p, n, C, ld, dtype=torch.float32):
    """[n][C] view of a row-major buffer with leading dimension ld"""
    return dev(p, (n - 1) * ld + C, dtype).as_strided((n, C), (ld, 1))


def act(p, B, H, W, C, ld):
    """[B][H][W][C] view of an NHWC activation with pitch ld"""
    return dev(p, (B * H * W - 1) * ld + C).as_strided((B, H, W, C), (H * W * ld, W * ld, ld, 1))


def chunks(B, H, W, C):
    step = max(1, CHUNK // max(1, H * W * C))
    return [(b, min(B, b + step)) for b in range(0, B, step)]


def seg_chunks(B, H, W, C, nseg):
    """[(segment, b0, b1)]: chunks() of each of nseg segments of B / nseg whole images, none straddling two"""
    nb = B // nseg
    return [(k, k * nb + b0, k * nb + b1) for k in range(nseg) for b0, b1 in chunks(nb, H, W, C)]


def rows_of_segment(p, ld, seg_pix, k, C):
    """[seg_pix][C] view of segment k's pixel rows of a buffer with leading dimension ld"""
    return rows(p + 4 * k * seg_pix * ld, seg_pix, C, ld)


def bits(t):
    """int view with -0 == +0 (fmaxf of two zeros may return either)"""
    t = t + 0.0
    return t.view(torch.int16 if t.dtype == torch.float16 else torch.int32)


def pre_act(z, sc, sh):
    """fp32 fma(z, scale, shift): the product of two floats is exact in float64"""
    return (z.double() * sc.double() + sh.double()).float()


def leaky(y, slope):
    return torch.where(y > 0, y, y * slope)


def windows(a):
    """[B,H,W,C] -> [4,B,Hp,Wp,C], the whole 2x2 windows in scan order"""
    Hp, Wp = a.shape[1] // 2, a.shape[2] // 2
    a = a[:, :2 * Hp, :2 * Wp]
    return torch.stack([a[:, 0::2, 0::2], a[:, 0::2, 1::2], a[:, 1::2, 0::2], a[:, 1::2, 1::2]])


def first_max(w):
    """index of the first maximum over dim 0 in scan order with strict > (torch's tie order is not specified)"""
    best = torch.zeros(w.shape[1:], dtype=torch.int64, device=w.device)
    bv = w[0]
    for q in range(1, w.shape[0]):
        m = w[q] > bv
        best[m] = q
        bv = torch.where(m, w[q], bv)
    return best


def split16(v, s):
    f = v * s
    hi = f.half()
    return hi, (f - hi.float()).half()


def ulps(got, ref):
    """|got - ref| in float32 spacings at ref (float64 ref)"""
    r = ref.abs().float().clamp_min(torch.finfo(torch.float32).tiny)
    sp = (torch.nextafter(r, torch.tensor(math.inf, device=r.device)) - r).double()
    return ((got.double() - ref).abs() / sp)


def route(y32, a32, dyf, dyp, slope):
    """float64 du: dy_pool to the first maximum of the activated fp32 values, + dy_full, times leaky'(y) on the fp32
    pre-activation; and the fp32 du the kernel forms (dy_full + dy_pool in fp32, times the slope in fp32)"""
    du = torch.zeros(y32.shape, dtype=torch.float64, device=y32.device)
    routed = torch.zeros_like(y32)
    if dyp is not None and dyp.numel():
        Hp, Wp = dyp.shape[1], dyp.shape[2]
        best = first_max(windows(a32))
        for q in range(4):
            routed[:, q >> 1:2 * Hp:2, q & 1:2 * Wp:2] = torch.where(best == q, dyp, torch.zeros_like(dyp))
    du += routed.double()
    d32 = routed
    if dyf is not None:
        du += dyf.double()
        d32 = dyf + routed
    fac = torch.where(y32 > 0, 1.0, float(slope))
    return du * fac.double(), d32 * fac.float()


class MemChecker(object):
    def __init__(self, real_call, lib):
        self.real = real_call
        self.lib = lib
        self.log = []
        self.cov = set()
        self.unknown = []
        self.failures = []
        self.stat_src = {}      # stat pointer -> (z, ldz, B, H, W, C) of the convolution that filled it
        self.seg_src = {}       # stat pointer -> (z, ld, seg_pix, nseg, C, rows) of the segmented colstats that filled it
        self.seg_meanstd = {}   # segment -> worst |mean|/std of its layers (segmented passes only)
        self.running_before = (None, None)
        self.amax_of = {}       # scale pointer -> amax_y pointer of the same finalize
        self.reduce = {}        # partial pointer -> arguments of the reduce pass
        self.stats = {}         # (mean pointer) -> [(mean64, var64)] of z per segment, for the from-scratch backward
        self.meanstd = []
        self.cancel = []
        self.bound_ratio = []

    def expect(self, ok, what):
        if not ok:
            self.failures.append(what)
            print('FAILED:', what)

    def _record(self, kind, shape, flav, ratio, extra=''):
        self.log.append(dict(kind=kind, shape=shape, flavour=flav, ratio=ratio, extra=extra))

    def __call__(self, fn, *a):
        if fn in STAT_WRITERS:
            z, ldz, B, H, W, C, stat = (a[i] for i in STAT_WRITERS[fn])
            if stat:
                self.stat_src[stat] = (z, ldz, B, H, W, C)
            return self.real(fn, *a)
        handler = getattr(self, 'chk_' + fn[len('fsdet_'):], None)
        if handler is None:
            if GEMM.search(fn) or fn in PASS:
                return self.real(fn, *a)
            self.unknown.append(fn)
            raise AssertionError('entry point without a check: %s' % fn)
        torch.cuda.synchronize()
        t0 = time.time()
        n = len(self.log)
        rc = handler(fn, a)
        torch.cuda.synchronize()
        for l in self.log[n:]:
            l['sec'] = time.time() - t0
            print('%-18s %-30s %-22s ratio %.3f%s' % (l['kind'], l['shape'], l['flavour'], l['ratio'], l['extra']))
        sys.stdout.flush()
        return rc

    # ---------------------------------------------------------------- finalize
    def chk_bn_finalize(self, fn, a):
        stat, nparts, count, gamma, beta, rm, rv, mom, eps, mean, invstd, scale, shift, slope, amax_y, xhat, C, training, st = a
        if training:
            zp, ldz, B, H, W, zc = self.stat_src[stat]
            assert zc == C, (zc, C)
            return self._finalize_train(fn, a, [act(zp, B, H, W, C, ldz)], gamma, beta, rm, rv, mom, eps, mean, invstd,
                                        scale, shift, slope, amax_y, xhat, C)
        outs = [dev(p, C) for p in (mean, invstd, scale, shift, xhat) if p]
        for o in outs:
            o.fill_(float('nan'))
        rm0 = dev(rm, C).clone() if rm else None
        rv0 = dev(rv, C).clone() if rv else None
        rc = self.real(fn, *a)
        torch.cuda.synchronize()
        m, inv, sc, sh = dev(mean, C), dev(invstd, C), dev(scale, C), dev(shift, C)
        g = dev(gamma, C).double() if gamma else torch.ones(C, dtype=torch.float64, device='cuda')
        b = dev(beta, C).double() if beta else torch.zeros(C, dtype=torch.float64, device='cuda')
        self.amax_of[scale] = amax_y
        return self._finalize_eval(fn, a, rc, m, inv, sc, sh, g, b, rm0, rv0)

    def chk_bn_seg_colstats(self, fn, a):
        """partial rows of each segment against float64 of that segment alone (sums to 1e-5 of the absolute sums, minima
        and maxima exact): a strip that straddled two segments moves both segments' minima or maxima"""
        zp, ld, seg_pix, nseg, C, part, st = a
        rows = self.lib.fsdet_bn_seg_colstats_rows(seg_pix, nseg)
        S = dev(part, nseg * rows * 4 * C).view(nseg, rows, 4, C)
        S.fill_(float('nan'))
        rc = self.real(fn, *a)
        torch.cuda.synchronize()
        for k in range(nseg):
            check_stats(self.expect, S[k], rows_of_segment(zp, ld, seg_pix, k, C), ('seg_colstats', seg_pix, nseg, C, k))
        self.seg_src[part] = (zp, ld, seg_pix, nseg, C, rows)
        self.cov.add('seg-colstats')
        self._record('bn_seg_colstats', '%dx%dx%d' % (nseg, seg_pix, C), 'seg', 0.0)
        return rc

    def chk_bn_seg_finalize(self, fn, a):
        stat, nparts, nseg, seg_pix, gamma, beta, rm, rv, mom, eps, mean, invstd, scale, shift, slope, amax_y, xhat, C, st = a
        zp, ld, sp, ns, zc, rows = self.seg_src[stat]
        assert (sp, ns, zc, rows) == (seg_pix, nseg, C, nparts), ((sp, ns, zc, rows), (seg_pix, nseg, C, nparts))
        zs = [rows_of_segment(zp, ld, seg_pix, k, C).view(seg_pix, 1, 1, C) for k in range(nseg)]
        rc = self._finalize_train(fn, a, zs, gamma, beta, rm, rv, mom, eps, mean, invstd, scale, shift, slope, amax_y, xhat, C)
        if rm:
            # the running statistics come from segment 0 alone: the same finalize with every other segment's partial rows
            # doubled leaves them bit-unchanged (the reduction order is fixed, so a rerun is bit-reproducible)
            rm1, rv1 = dev(rm, C).clone(), dev(rv, C).clone()
            dev(rm, C).copy_(self.running_before[0])
            dev(rv, C).copy_(self.running_before[1])
            other = dev(stat, nseg * nparts * 4 * C)[nparts * 4 * C:]
            keep = other.clone()
            other.mul_(2.0)
            probe = torch.full((5 * nseg * C + 1,), float('nan'), device='cuda')
            P = lambda i: probe.data_ptr() + 4 * i * nseg * C
            self.real(fn, stat, nparts, nseg, seg_pix, gamma, beta, rm, rv, mom, eps, P(0), P(1), P(2), P(3), slope,
                      probe.data_ptr() + 4 * 5 * nseg * C, P(4), C, st)
            torch.cuda.synchronize()
            same = torch.equal(bits(dev(rm, C)), bits(rm1)) and torch.equal(bits(dev(rv, C)), bits(rv1))
            moved = not torch.equal(bits(probe[nseg * C:2 * nseg * C]), bits(dev(invstd, nseg * C)))
            self.expect(same and moved, ('seg_finalize: running statistics depend on segments 1..', C, same, moved))
            other.copy_(keep)
            dev(rm, C).copy_(rm1)
            dev(rv, C).copy_(rv1)
        self.cov.add('seg-finalize')
        return rc

    def _finalize_train(self, fn, a, zs, gamma, beta, rm, rv, mom, eps, mean, invstd, scale, shift, slope, amax_y, xhat, C):
        """Train-mode finalize of len(zs) segments ([nseg][C] vectors, segment k normalised by the statistics of zs[k]):
        each segment's mean / invstd against float64 of its own z, scale / shift within an ulp, xhat_absmax per segment,
        running statistics from segment 0 (unbiased over its pixels), one amax_y over every segment."""
        nseg = len(zs)
        V = lambda p, k: dev(p + 4 * k * C, C)
        for p in (mean, invstd, scale, shift, xhat):
            if p:
                dev(p, nseg * C).fill_(float('nan'))
        rm0 = dev(rm, C).clone() if rm else None
        rv0 = dev(rv, C).clone() if rv else None
        self.running_before = (rm0, rv0)
        rc = self.real(fn, *a)
        torch.cuda.synchronize()
        g = dev(gamma, C).double() if gamma else torch.ones(C, dtype=torch.float64, device='cuda')
        b = dev(beta, C).double() if beta else torch.zeros(C, dtype=torch.float64, device='cuda')
        self.amax_of[scale] = amax_y
        pos = torch.zeros(1, dtype=torch.float64, device='cuda')
        neg = torch.zeros(1, dtype=torch.float64, device='cuda')
        stats = []
        for k, z in enumerate(zs):
            m, inv, sc, sh = V(mean, k), V(invstd, k), V(scale, k), V(shift, k)
            B, H, W = z.shape[:3]
            N = B * H * W
            s = torch.zeros(C, dtype=torch.float64, device='cuda')
            for b0, b1 in chunks(B, H, W, C):
                s += z[b0:b1].double().sum((0, 1, 2))
            mu = s / N
            v = torch.zeros_like(s)
            xmax = torch.zeros(C, device='cuda')
            for b0, b1 in chunks(B, H, W, C):
                zz = z[b0:b1]
                v += ((zz.double() - mu) ** 2).sum((0, 1, 2))
                y32 = pre_act(zz, sc, sh)
                u64 = zz.double() * sc.double() + sh.double()
                pos = torch.maximum(pos, torch.where(y32 > 0, u64, 0.0).max())
                neg = torch.maximum(neg, torch.where(y32 > 0, 0.0, -u64 * float(slope)).max())
                xmax = torch.maximum(xmax, ((zz - m) * inv).abs().amax((0, 1, 2)))
            var = v / N
            std = torch.sqrt(var + eps)
            rmean = ((m.double() - mu).abs() / (STAT_BAR * std)).max().item()
            rinv = ((inv.double() - 1 / std).abs() * std / STAT_BAR).max().item()
            ms = (mu.abs() / var.sqrt().clamp_min(1e-30)).max().item()
            self.meanstd.append(ms)
            if nseg > 1:
                self.seg_meanstd[k] = max(self.seg_meanstd.get(k, 0.0), ms)
            self.expect(rmean <= 1 and rinv <= 1, ('bn_finalize mean / invstd', B, H, W, C, k, rmean, rinv, ms))
            self.expect((ulps(sc, g * inv.double()) <= 1).all().item(), ('bn_finalize scale', C, k))
            self.expect((ulps(sh, b - m.double() * sc.double()) <= 1).all().item(), ('bn_finalize shift', C, k))
            if xhat:
                self.expect(torch.equal(V(xhat, k), xmax), ('bn_finalize xhat_absmax', C, k))
            if rm and k == 0:
                want_m = (1 - mom) * rm0.double() + mom * m.double()
                want_v = (1 - mom) * rv0.double() + mom * var * N / max(N - 1, 1)
                self.expect(((dev(rm, C).double() - want_m).abs() <= 2.0 ** -22 * (want_m.abs() + m.double().abs())).all().item(),
                            ('running mean', C))
                self.expect(((dev(rv, C).double() - want_v).abs() <= 2 * STAT_BAR * mom * var * N / max(N - 1, 1) +
                             2.0 ** -22 * want_v.abs()).all().item(), ('running var', C))
            stats.append((mu, var))
            shape = '%dx%dx%dx%d' % (B, H, W, C) if nseg == 1 else '%d/%dx%dx%d' % (k, nseg, N, C)
            self._record('bn_finalize', shape, 'train' if nseg == 1 else 'train seg', max(rmean, rinv),
                         '  |mean|/std %.2f' % ms)
        if amax_y:
            ref = torch.maximum(pos, neg)
            # the negative side is rounded twice (fma, then the slope)
            self.expect(ulps(dev(amax_y, 1), ref).item() <= (1 if pos.item() >= neg.item() else 2), ('bn_finalize amax_y', C))
        self.stats[mean] = stats
        self.cov.add('finalize-train')
        return rc

    def _finalize_eval(self, fn, a, rc, m, inv, sc, sh, g, b, rm0, rv0):
        """Eval mode: mean and invstd are the running statistics (invstd = 1 / sqrtf(running_var + eps), three fp32
        roundings), scale and shift within an ulp as in training, the running statistics untouched, and nothing
        derived from a batch range: xhat_absmax (when given) is 0, amax_y (when given) is 0.  Then the same finalize is
        run once more into a NaN-filled [5][C] buffer with both optional outputs left out: the four coefficient rows must
        equal the first call's and the fifth row, where xhat_absmax would go, must keep its NaN bits."""
        stat, nparts, count, gamma, beta, rm, rv, mom, eps, mean, invstd, scale, shift, slope, amax_y, xhat, C, training, st = a
        ok_stats = torch.equal(m, rm0) and torch.equal(inv, 1 / torch.sqrt(rv0 + eps))
        self.expect(ok_stats, ('eval finalize mean / invstd', C))
        r_sc = ulps(sc, g * inv.double()).max().item()
        r_sh = ulps(sh, b - m.double() * sc.double()).max().item()
        self.expect(r_sc <= 1, ('eval finalize scale', C, r_sc))
        self.expect(r_sh <= 1, ('eval finalize shift', C, r_sh))
        self.expect(torch.equal(bits(dev(rm, C)), bits(rm0)) and torch.equal(bits(dev(rv, C)), bits(rv0)),
                    ('eval finalize wrote the running statistics', C))
        if xhat:
            self.expect(torch.equal(bits(dev(xhat, C)), torch.zeros(C, dtype=torch.int32, device='cuda')),
                        ('eval finalize xhat_absmax', C))
        if amax_y:
            self.expect(dev(amax_y, 1).item() == 0.0, ('eval finalize amax_y', C))
        probe = torch.full((5 * C + 1,), float('nan'), device='cuda')
        P = lambda i: probe.data_ptr() + 4 * i * C
        self.real(fn, stat, nparts, count, gamma, beta, rm, rv, mom, eps, P(0), P(1), P(2), P(3), slope, None, None, C,
                  training, st)
        torch.cuda.synchronize()
        same = all(torch.equal(bits(probe[i * C:(i + 1) * C]), bits(t)) for i, t in enumerate((m, inv, sc, sh)))
        self.expect(same, ('eval finalize: a second call gives other coefficients', C))
        self.expect(torch.isnan(probe[4 * C:]).all().item(), ('eval finalize wrote an output it was not given', C))
        self.expect(torch.equal(bits(dev(rm, C)), bits(rm0)) and torch.equal(bits(dev(rv, C)), bits(rv0)),
                    ('eval finalize wrote the running statistics', C))
        self.cov.add('finalize-eval')
        self._record('bn_finalize', 'eval C%d' % C, 'eval', max(r_sc, r_sh) if ok_stats else math.inf,
                     '  scale / shift in ulps')
        return rc

    # ----------------------------------------------------------------- forward
    def chk_bn_act_fwd(self, fn, a):
        return self._act_fwd(fn, a, 1)

    def chk_bn_act_fwd_seg(self, fn, a):
        B, H, W, C, nseg, seg_pix = a[15:21]
        assert seg_pix * nseg == B * H * W, (B, H, W, nseg, seg_pix)
        return self._act_fwd(fn, a, nseg)

    def _act_fwd(self, fn, a, nseg):
        """the forward check, segment k's scale and shift ([nseg][C]) on segment k's images"""
        zp, ldz, scale, shift, slope, yf, ldf, yp, ldp, fh, fl, ph, pl, Cpad, amax, B, H, W, C = a[:19]
        Hp, Wp = H // 2, W // 2
        M, Mp = B * H * W, B * Hp * Wp
        YF = act(yf, B, H, W, C, ldf) if yf else None
        YP = act(yp, B, Hp, Wp, C, ldp) if (yp and Mp) else None
        FH, FL = [dev(p, M * Cpad, torch.int16).view(B, H, W, Cpad) if p else None for p in (fh, fl)]
        PH, PL = [dev(p, Mp * Cpad, torch.int16).view(B, Hp, Wp, Cpad) if (p and Mp) else None for p in (ph, pl)]
        for t in (YF, YP):
            if t is not None:
                t.fill_(float('nan'))
        for t in (FH, FL, PH, PL):
            if t is not None:
                t.fill_(0x7e01)
        rc = self.real(fn, *a)
        torch.cuda.synchronize()
        z = act(zp, B, H, W, C, ldz)
        s = scale_from_amax(dev(amax, 1).item()) if amax else 1.0
        am = self.amax_of.get(scale)
        am = dev(am, 1).item() if am else None
        ok = True
        worst = 0.0
        for k, b0, b1 in seg_chunks(B, H, W, C, nseg):
            sc, sh = dev(scale + 4 * k * C, C), dev(shift + 4 * k * C, C)
            zz = z[b0:b1]
            y32 = leaky(pre_act(zz, sc, sh), slope)
            u64 = zz.double() * sc.double() + sh.double()
            y64 = torch.where(y32 > 0, u64, u64 * float(slope))
            worst = max(worst, ((y32.double() - y64).abs() / (2.0 ** -23 * y64.abs()).clamp_min(1e-300)).max().item())
            pooled = windows(y32).max(0).values
            if YF is not None:
                ok &= torch.equal(bits(YF[b0:b1]), bits(y32))
            if YP is not None:
                ok &= torch.equal(bits(YP[b0:b1]), bits(pooled))
            for hi, lo, ref in ((FH, FL, y32), (PH, PL, pooled)):
                if hi is None:
                    continue
                h, l = split16(ref, s)
                ok &= torch.equal(bits(hi[b0:b1, ..., :C].view(torch.float16)), bits(h))
                ok &= torch.equal(bits(lo[b0:b1, ..., :C].view(torch.float16)), bits(l))
                ok &= not hi[b0:b1, ..., C:].any().item() and not lo[b0:b1, ..., C:].any().item()
            if am is not None:
                ok &= y32.abs().max().item() <= am
        self.expect(ok, ('bn_act_fwd', B, H, W, C, Cpad, nseg, bool(yf), bool(yp), bool(fh), bool(ph)))
        self.expect(worst <= 1.0, ('bn_act_fwd: more than two roundings from float64', B, H, W, C, nseg, worst))
        pool = bool(yp or ph)
        full = bool(yf or fh)
        flav = 'pool+full' if (pool and full) else ('pool' if pool else 'full')
        pre = 'seg-' if nseg > 1 else ''
        self.cov.add(pre + 'fwd-' + flav)
        if yf or yp:
            self.cov.add(pre + 'fwd-f32')
        if fh or ph:
            self.cov.add(pre + 'fwd-planes')
        if pool and (H % 2 or W % 2):
            self.cov.add(pre + 'fwd-odd')
        self._record('bn_act_fwd', '%dx%dx%dx%d pad%d' % (B, H, W, C, Cpad) + (' /%d' % nseg if nseg > 1 else ''),
                     flav + (' planes' if (fh or ph) else '') + (' seg' if nseg > 1 else ''), worst, '' if ok else '  MISMATCH')
        return rc

    # ---------------------------------------------------------------- backward
    def _du(self, r, b0, b1, k=0):
        """float64 du, fp32 du, xhat (segment k's kernel statistics) and the fp32 pre-activation of images [b0, b1)"""
        zp, ldz, dyf, ldf, dyp, ldp, scale, shift, mean, invstd, slope, B, H, W, C, has_bn = r[:16]
        Hp, Wp = H // 2, W // 2
        V = lambda p: dev(p + 4 * k * C, C)
        sc, sh = V(scale), V(shift)
        zz = act(zp, B, H, W, C, ldz)[b0:b1]
        y32 = pre_act(zz, sc, sh)
        a32 = leaky(y32, slope)
        gf = act(dyf, B, H, W, C, ldf)[b0:b1] if dyf else None
        gp = act(dyp, B, Hp, Wp, C, ldp)[b0:b1] if (dyp and Hp * Wp) else None
        du, d32 = route(y32, a32, gf, gp, slope)
        xh = (zz.double() - V(mean).double()) * V(invstd).double() if has_bn else torch.zeros_like(du)
        return du, d32, xh, zz

    def chk_bn_act_bwd_reduce(self, fn, a):
        zp, ldz, dyf, ldf, dyp, ldp, scale, shift, mean, invstd, slope, part, B, H, W, C, has_bn, st = a
        nrows = self.lib.fsdet_bn_bwd_rows(B, H, W)
        dev(part, (nrows + 1) * 3 * C, torch.float64).fill_(float('nan'))
        rc = self.real(fn, *a)
        self.reduce[part] = (zp, ldz, dyf, ldf, dyp, ldp, scale, shift, mean, invstd, slope, B, H, W, C, has_bn, 1)
        return rc

    def chk_bn_act_bwd_reduce_seg(self, fn, a):
        zp, ldz, dyf, ldf, dyp, ldp, scale, shift, mean, invstd, slope, part, B, H, W, C, nseg, seg_pix, st = a
        assert seg_pix * nseg == B * H * W, (B, H, W, nseg, seg_pix)
        nrows = self.lib.fsdet_bn_seg_bwd_rows(B, H, W, nseg)
        dev(part, nseg * (nrows + 1) * 3 * C, torch.float64).fill_(float('nan'))
        rc = self.real(fn, *a)
        self.reduce[part] = (zp, ldz, dyf, ldf, dyp, ldp, scale, shift, mean, invstd, slope, B, H, W, C, 1, nseg)
        return rc

    def _sums(self, r):
        """per segment: float64 sum du, sum du xhat, sum |du|, sum |du xhat| over the segment's images"""
        B, H, W, C = r[11:15]
        acc = [[torch.zeros(C, dtype=torch.float64, device='cuda') for _ in range(4)] for _ in range(r[16])]
        for k, b0, b1 in seg_chunks(B, H, W, C, r[16]):
            du, _, xh, _ = self._du(r, b0, b1, k)
            for i, t in enumerate((du, du * xh, du.abs(), (du * xh).abs())):
                acc[k][i] += t.sum((0, 1, 2))
        return acc

    def chk_bn_bwd_finalize(self, fn, a):
        part, nrows, count, gamma, invstd, xabs, dgamma, dbeta, coef, amax, C, has_bn, st = a
        return self._bwd_finalize(fn, a, part, dgamma, dbeta, coef, C, has_bn)

    def chk_bn_bwd_finalize_seg(self, fn, a):
        part, nrows, nseg, seg_pix, gamma, invstd, xabs, dgamma, dbeta, coef, amax, C, st = a
        assert self.reduce[part][16] == nseg, (self.reduce[part][16], nseg)
        return self._bwd_finalize(fn, a, part, dgamma, dbeta, coef, C, 1)

    def _bwd_finalize(self, fn, a, part, dgamma, dbeta, coef, C, has_bn):
        """per segment k: c1 = sum du / N_k and c2 = sum du xhat / N_k within 1e-6 of the segment's absolute sums;
        dgamma, dbeta: the sums over every segment, within 1e-6 of the absolute sums over every segment"""
        r = self.reduce[part]
        nseg = r[16]
        for p, n, t in ((dgamma, C, torch.float32), (dbeta, C, torch.float32), (coef, 2 * C * nseg, torch.float64)):
            if p:
                dev(p, n, t).fill_(float('nan'))
        rc = self.real(fn, *a)
        torch.cuda.synchronize()
        B, H, W = r[11:14]
        N = B * H * W // nseg
        acc = self._sums(r)
        s1, s2, a1, a2 = (sum(acc[k][i] for k in range(nseg)) for i in range(4))
        worst = 0.0
        if dbeta:
            e = ((dev(dbeta, C).double() - s1).abs() / (SUM_BAR * a1).clamp_min(1e-300)).max().item()
            worst = max(worst, e)
        if has_bn:
            e2 = ((dev(dgamma, C).double() - s2).abs() / (SUM_BAR * a2).clamp_min(1e-300)).max().item() if dgamma else 0.0
            worst = max(worst, e2)
            for k in range(nseg):
                k1, k2, b1, b2 = acc[k]
                cf = dev(coef + 8 * 2 * C * k, 2 * C, torch.float64)
                e3 = ((cf[:C] - k1 / N).abs() / (SUM_BAR * b1 / N).clamp_min(1e-300)).max().item()
                e4 = ((cf[C:] - k2 / N).abs() / (SUM_BAR * b2 / N).clamp_min(1e-300)).max().item()
                worst = max(worst, e3, e4)
        cancel = (a1 / s1.abs().clamp_min(1e-300)).max().item()
        self.cancel.append(cancel)
        self.expect(worst <= 1.0, ('bn_bwd_finalize sums', B, H, W, C, has_bn, nseg, worst))
        if nseg > 1:
            self.cov.add('seg-bwd-finalize')
        self._record('bn_bwd_finalize', '%dx%dx%dx%d' % (B, H, W, C) + (' /%d' % nseg if nseg > 1 else ''),
                     ('bn' if has_bn else 'bias') + (' seg' if nseg > 1 else ''), worst, '  cancellation %.0f' % cancel)
        return rc

    def chk_bn_act_bwd_apply(self, fn, a):
        return self._bwd_apply(fn, a, a[22], 1)

    def chk_bn_act_bwd_apply_seg(self, fn, a):
        B, H, W, C, nseg, seg_pix = a[18:24]
        assert seg_pix * nseg == B * H * W, (B, H, W, nseg, seg_pix)
        return self._bwd_apply(fn, a, 1, nseg)

    def _bwd_apply(self, fn, a, has_bn, nseg):
        """the apply check, segment k's vectors ([nseg][C]) and coefficients ([nseg][2C]) on segment k's images and the
        from-scratch float64 backward over segment k's statistics; one amax_bound over every segment"""
        zp, ldz, dyf, ldf, dyp, ldp, scale, shift, mean, invstd, coef, slope, dzp, lddz, dh, dl, cpad, amax, B, H, W, C = a[:22]
        tail = a[22:-1]         # (has_bn,) or (nseg, seg_pix)
        st = a[-1]
        M = B * H * W
        DZ = act(dzp, B, H, W, C, lddz) if dzp else None
        DH, DL = [dev(p, M * C, torch.int16).view(B, H, W, C) if p else None for p in (dh, dl)]
        if DZ is not None:
            DZ.fill_(float('nan'))
        for t in (DH, DL):
            if t is not None:
                t.fill_(0x7e01)
        rc = self.real(fn, *a)
        torch.cuda.synchronize()
        if DZ is None:      # planes only: the fp32 dz they were split from (the apply pass only reads its inputs)
            tmp = torch.full((M, C), float('nan'), device='cuda')
            self.real(fn, zp, ldz, dyf, ldf, dyp, ldp, scale, shift, mean, invstd, coef, slope, tmp.data_ptr(), C, None,
                      None, cpad, amax, B, H, W, C, *tail, st)
            torch.cuda.synchronize()
            DZ = tmp.view(B, H, W, C)
        r = (zp, ldz, dyf, ldf, dyp, ldp, scale, shift, mean, invstd, slope, B, H, W, C, has_bn, nseg)
        Ms = M // nseg
        ok = True
        worst = scratch = 0.0
        dzmax = 0.0
        prop = 0.0
        seg = []
        if has_bn:
            # from scratch, per segment: float64 statistics of the segment's z, float64 xhat, the float64 sums
            acc = [[torch.zeros(C, dtype=torch.float64, device='cuda') for _ in range(4)] for _ in range(nseg)]
            for k, b0, b1 in seg_chunks(B, H, W, C, nseg):
                mu, var = self.stats[mean][k]
                du, _, _, zz = self._du(r, b0, b1, k)
                xs = (zz.double() - mu) / torch.sqrt(var + EPS)
                for i, t in enumerate((du, du * xs, du.abs(), (du * xs).abs())):
                    acc[k][i] += t.sum((0, 1, 2))
            for k in range(nseg):
                V = lambda p: dev(p + 4 * k * C, C).double()
                mu, var = self.stats[mean][k]
                cf = dev(coef + 8 * 2 * C * k, 2 * C, torch.float64)
                # the kernel's fp32 statistics differ from float64 (within the finalize bars): to first order, a mean
                # error kappa = (mu - mean) * invstd and an invstd error delta move dz by
                # |scale| (|delta| |dz| + 2 |delta| |xhat c2| + |kappa| (|c2| + |xhat c1|)); and c1, c2 are exact only to
                # the backward sums' bar (1e-6 of sum|du| / N and sum|du xhat| / N: c2 cancels, and its products are
                # fp32), which moves dz by |scale| 1e-6 (sum|du| + |xhat| sum|du xhat|) / N.  That propagation is
                # allowed on top.
                seg.append(dict(sc=V(scale), c1=cf[:C], c2=cf[C:], mu=mu, var=var, g=V(scale) / V(invstd),
                                c1s=acc[k][0] / Ms, c2s=acc[k][1] / Ms, e1=SUM_BAR * acc[k][2] / Ms,
                                e2=SUM_BAR * acc[k][3] / Ms, kappa=((mu - V(mean)) * V(invstd)).abs(),
                                delta=(V(invstd) * torch.sqrt(var + EPS) - 1).abs()))
        s = scale_from_amax(dev(amax, 1).item()) if amax else 1.0
        for k, b0, b1 in seg_chunks(B, H, W, C, nseg):
            du, d32, xh, zz = self._du(r, b0, b1, k)
            got = DZ[b0:b1]
            ok &= not torch.isnan(got).any().item()
            dzmax = max(dzmax, got.abs().max().item())
            if has_bn:
                q = seg[k]
                sc, c1, c2, c1s, c2s = q['sc'], q['c1'], q['c2'], q['c1s'], q['c2s']
                ref = sc * (du - c1 - xh * c2)
                bar = sc.abs() * (du.abs() + c1.abs() + (xh * c2).abs())
                d = (got.double() - ref).abs()
                worst = max(worst, torch.where(d == 0, 0.0, d / (SUM_BAR * bar)).max().item())
                xs = (zz.double() - q['mu']) / torch.sqrt(q['var'] + EPS)
                ref_s = q['g'] / torch.sqrt(q['var'] + EPS) * (du - c1s - xs * c2s)
                p = 1.1 * sc.abs() * (q['delta'] * ref_s.abs() / sc.abs() + 2 * q['delta'] * (xs * c2s).abs() +
                                      q['kappa'] * (c2s.abs() + (xs * c1s).abs()) + q['e1'] + xs.abs() * q['e2'])
                prop = max(prop, (p / bar).max().item())
                d = (got.double() - ref_s).abs()
                rr = torch.where(d == 0, 0.0, d / (SCRATCH_BAR * bar + p))
                if rr.max().item() > scratch:
                    scratch = rr.max().item()
                    i = rr.flatten().argmax().item()
                    at = lambda t: t.expand(rr.shape).flatten()[i].item()
                    c = i % C
                    worst_at = dict(segment=k, du=at(du), c1=c1s[c].item(), xs=at(xs), c2=c2s[c].item(),
                                    kappa=q['kappa'][c].item(), delta=q['delta'][c].item(), got=at(got), ref=at(ref),
                                    ref_s=at(ref_s), bar=at(bar), p=at(p))
            else:
                ok &= torch.equal(bits(got), bits(d32))
                d = (got.double() - du).abs()
                worst = max(worst, torch.where(d == 0, 0.0, d / (SUM_BAR * du.abs())).max().item())
            if DH is not None:
                h, l = split16(got.contiguous(), s)
                ok &= torch.equal(bits(DH[b0:b1].view(torch.float16)), bits(h))
                ok &= torch.equal(bits(DL[b0:b1].view(torch.float16)), bits(l))
        extra = ''
        if amax and has_bn:
            bound = dev(amax, 1).item()
            self.expect(bound > dzmax, ('amax_bound below max|dz|', B, H, W, C, nseg, bound, dzmax))
            self.bound_ratio.append(bound / max(dzmax, 1e-300))
            extra = '  bound/max|dz| %.2f  statistics propagation %.1e of the bound' % (bound / max(dzmax, 1e-300), prop)
        self.expect(ok, ('bn_act_bwd_apply', B, H, W, C, has_bn, nseg, bool(dzp), bool(dh)))
        if has_bn and scratch > 1.0:
            k = worst_at['segment']
            nb = B // nseg
            z = act(zp, B, H, W, C, ldz)[k * nb:(k + 1) * nb]
            mu2 = sum(z[b0:b1].double().sum((0, 1, 2)) for b0, b1 in chunks(nb, H, W, C)) / Ms
            print('  scratch worst element:', worst_at, ' z changed since the forward:', not torch.equal(mu2, seg[k]['mu']))
        self.expect(worst <= 1.0 and scratch <= 1.0, ('bn_act_bwd_apply dz', B, H, W, C, has_bn, nseg, worst, scratch))
        pool_only = not dyf and dyp and has_bn and 0.0 <= slope <= 1.0
        flav = 'pool-only' if pool_only else ('general ' + '+'.join(n for n, p in (('full', dyf), ('pool', dyp)) if p))
        pre = 'seg-' if nseg > 1 else ''
        self.cov.add(pre + 'bwd-' + flav.replace(' ', '-'))
        if not has_bn:
            self.cov.add('bwd-bias')
        if (H % 2 or W % 2) and dyp:
            self.cov.add(pre + 'bwd-odd')
        self._record('bn_act_bwd_apply', '%dx%dx%dx%d' % (B, H, W, C) + (' /%d' % nseg if nseg > 1 else ''),
                     flav + ('' if has_bn else ' bias') + (' seg' if nseg > 1 else ''), max(worst, scratch),
                     '  scratch %.3f%s%s' % (scratch, extra, '' if ok else '  MISMATCH'))
        return rc

    # -------------------------------------------------------- data movement
    def _exact(self, kind, shape, ok, flav='exact'):
        self.cov.add(kind)
        self.expect(ok, (kind, shape))
        self._record(kind, shape, flav, 0.0 if ok else math.inf)

    def chk_maxpool_fwd(self, fn, a):
        x, ldx, y, ldy, B, H, W, C, stride, st = a
        Ho, Wo = (H // 2, W // 2) if stride == 2 else (H, W)
        Y = act(y, B, Ho, Wo, C, ldy)
        Y.fill_(float('nan'))
        rc = self.real(fn, *a)
        torch.cuda.synchronize()
        X = act(x, B, H, W, C, ldx)
        if stride == 1:       # MaxPoolStride1: replicate the last row and column
            X = torch.cat([X, X[:, -1:]], 1)
            X = torch.cat([X, X[:, :, -1:]], 2)
            ref = torch.stack([X[:, :H, :W], X[:, :H, 1:], X[:, 1:, :W], X[:, 1:, 1:]]).max(0).values
        else:
            ref = windows(X).max(0).values
        self._exact('maxpool', '%dx%dx%dx%d s%d' % (B, H, W, C, stride), torch.equal(bits(Y), bits(ref)))
        return rc

    def chk_maxpool_bwd(self, fn, a):
        x, ldx, dy, lddy, dx, lddx, B, H, W, C, stride, st = a
        DX = act(dx, B, H, W, C, lddx)
        DX.fill_(float('nan'))
        rc = self.real(fn, *a)
        torch.cuda.synchronize()
        X = act(x, B, H, W, C, ldx)
        if stride == 2:
            Hp, Wp = H // 2, W // 2
            G = act(dy, B, Hp, Wp, C, lddy)
            best = first_max(windows(X))
            ref = torch.zeros(B, H, W, C, device='cuda')
            for q in range(4):
                ref[:, q >> 1:2 * Hp:2, q & 1:2 * Wp:2] = torch.where(best == q, G, torch.zeros_like(G))
            self._exact('maxpool-bwd', '%dx%dx%dx%d s2' % (B, H, W, C), torch.equal(bits(DX), bits(ref)))
            return rc
        # stride 1: each pixel collects the gradient of up to four windows (replicated taps fold back onto the last row
        # and column): float64 sums, within three fp32 roundings of their absolute sum
        Xp = torch.cat([X, X[:, -1:]], 1)
        Xp = torch.cat([Xp, Xp[:, :, -1:]], 2)
        best = first_max(torch.stack([Xp[:, :H, :W], Xp[:, :H, 1:], Xp[:, 1:, :W], Xp[:, 1:, 1:]]))
        G = act(dy, B, H, W, C, lddy).double()
        ref = torch.zeros(B, H + 1, W + 1, C, dtype=torch.float64, device='cuda')
        absref = torch.zeros_like(ref)
        for q in range(4):
            t = torch.where(best == q, G, torch.zeros_like(G))
            ref[:, q >> 1:(q >> 1) + H, q & 1:(q & 1) + W] += t
            absref[:, q >> 1:(q >> 1) + H, q & 1:(q & 1) + W] += t.abs()
        for r_ in (ref, absref):
            r_[:, H - 1] += r_[:, H]
            r_[:, :, W - 1] += r_[:, :, W]
        ref, absref = ref[:, :H, :W], absref[:, :H, :W]
        ok = bool(((DX.double() - ref).abs() <= 3 * 2.0 ** -24 * absref).all().item())
        self._exact('maxpool-bwd-s1', '%dx%dx%dx%d s1' % (B, H, W, C), ok, 'float64')
        return rc

    def chk_reorg_fwd(self, fn, a):
        x, ldx, y, ldy, B, H, W, C, st = a
        Y = act(y, B, H // 2, W // 2, 4 * C, ldy)
        Y.fill_(float('nan'))
        rc = self.real(fn, *a)
        torch.cuda.synchronize()
        X = act(x, B, H, W, C, ldx)
        ref = torch.cat([X[:, i::2, j::2] for i in range(2) for j in range(2)], 3)    # channel (i*2+j)*C + c
        self._exact('reorg', '%dx%dx%dx%d' % (B, H, W, C), torch.equal(bits(Y), bits(ref)))
        return rc

    def chk_reorg_bwd(self, fn, a):
        dy, lddy, dx, lddx, B, H, W, C, st = a
        DX = act(dx, B, H, W, C, lddx)
        DX.fill_(float('nan'))
        rc = self.real(fn, *a)
        torch.cuda.synchronize()
        G = act(dy, B, H // 2, W // 2, 4 * C, lddy)
        ref = torch.empty(B, H, W, C, device='cuda')
        for i in range(2):
            for j in range(2):
                ref[:, i::2, j::2] = G[..., (i * 2 + j) * C:(i * 2 + j + 1) * C]
        self._exact('reorg-bwd', '%dx%dx%dx%d' % (B, H, W, C), torch.equal(bits(DX), bits(ref)))
        return rc

    def chk_copy_channels(self, fn, a):
        src, lds, dst, ldd, npix, C, accumulate, st = a
        D = rows(dst, npix, C, ldd)
        d0 = D.clone() if accumulate else None
        if not accumulate:
            D.fill_(float('nan'))
        rc = self.real(fn, *a)
        torch.cuda.synchronize()
        S = rows(src, npix, C, lds)
        ref = d0 + S if accumulate else S
        self._exact('copy-acc' if accumulate else 'copy', '%dx%d' % (npix, C), torch.equal(bits(D), bits(ref)))
        return rc

    def chk_nchw_to_nhwc(self, fn, a):
        in0, C0, in1, C1, out, ld, Cpad, B, HW, st = a
        O = rows(out, B * HW, Cpad, ld)
        O.fill_(float('nan'))
        rc = self.real(fn, *a)
        torch.cuda.synchronize()
        parts = [dev(in0, B * C0 * HW).view(B, C0, HW)]
        if C1:
            parts.append(dev(in1, B * C1 * HW).view(B, C1, HW))
        ref = torch.cat(parts, 1).permute(0, 2, 1).reshape(B * HW, C0 + C1)
        ok = torch.equal(bits(O[:, :C0 + C1]), bits(ref)) and not O[:, C0 + C1:].any().item()
        self._exact('nchw-to-nhwc', '%dx%dx%d->%d' % (B, HW, C0 + C1, Cpad), ok)
        return rc

    def chk_nhwc_to_nchw(self, fn, a):
        x, ld, bias, out, B, C, HW, st = a
        O = dev(out, B * C * HW).view(B, C, HW)
        O.fill_(float('nan'))
        rc = self.real(fn, *a)
        torch.cuda.synchronize()
        ref = rows(x, B * HW, C, ld).view(B, HW, C).permute(0, 2, 1)
        if bias:
            ref = ref + dev(bias, C).view(1, C, 1)
        self._exact('nhwc-to-nchw' + ('-bias' if bias else ''), '%dx%dx%d' % (B, HW, C), torch.equal(bits(O), bits(ref)))
        return rc

    def chk_pad_channels(self, fn, a):
        src, cin, out, cout, n, st = a
        O = dev(out, n * cout).view(n, cout)
        O.fill_(float('nan'))
        rc = self.real(fn, *a)
        torch.cuda.synchronize()
        m = min(cin, cout)
        ok = torch.equal(bits(O[:, :m]), bits(dev(src, n * cin).view(n, cin)[:, :m])) and not O[:, m:].any().item()
        self._exact('pad-channels', '%dx%d->%d' % (n, cin, cout), ok)
        return rc

    def chk_weight_flip_transpose(self, fn, a):
        w, wt, Cout, kk, Cin, st = a
        O = dev(wt, Cin * kk * Cout).view(Cin, kk, Cout)
        O.fill_(float('nan'))
        rc = self.real(fn, *a)
        torch.cuda.synchronize()
        ref = dev(w, Cout * kk * Cin).view(Cout, kk, Cin).flip(1).permute(2, 1, 0)
        self._exact('flip-transpose', '%dx%dx%d' % (Cout, kk, Cin), torch.equal(bits(O), bits(ref)))
        return rc

    def chk_amax(self, fn, a):
        src, ld, C, n, out, st = a
        dev(out, 1).fill_(float('nan'))
        rc = self.real(fn, *a)
        torch.cuda.synchronize()
        ref = rows(src, n, C, ld).abs().max()
        self._exact('amax', '%dx%d' % (n, C), torch.equal(dev(out, 1)[0], ref))
        return rc

    def chk_split_f16(self, fn, a):
        src, ld, C, Cpad, n, amax, hi, lo, st = a
        H_, L_ = dev(hi, n * Cpad, torch.int16).view(n, Cpad), dev(lo, n * Cpad, torch.int16).view(n, Cpad)
        H_.fill_(0x7e01)
        L_.fill_(0x7e01)
        rc = self.real(fn, *a)
        torch.cuda.synchronize()
        h, l = split16(rows(src, n, C, ld), scale_from_amax(dev(amax, 1).item()) if amax else 1.0)
        ok = (torch.equal(bits(H_[:, :C].view(torch.float16)), bits(h)) and torch.equal(bits(L_[:, :C].view(torch.float16)), bits(l))
              and not H_[:, C:].any().item() and not L_[:, C:].any().item())
        self._exact('split-f16', '%dx%d->%d' % (n, C, Cpad), ok)
        return rc

    # ------------------------------------------------------------------ head
    def chk_head_weff(self, fn, a):
        Wp, bias, rw, weff, beff, n_cls, O, K, Npad, st = a
        E, BE = dev(weff, Npad * K).view(Npad, K), dev(beff, Npad)
        E.fill_(float('nan'))
        BE.fill_(float('nan'))
        rc = self.real(fn, *a)
        torch.cuda.synchronize()
        N = n_cls * O
        ref = (dev(Wp, O * K).view(1, O, K) * dev(rw, n_cls * K).view(n_cls, 1, K)).reshape(N, K)
        bref = dev(bias, O).repeat(n_cls) if bias else torch.zeros(N, device='cuda')
        ok = (torch.equal(bits(E[:N]), bits(ref)) and not E[N:].any().item() and torch.equal(bits(BE[:N]), bits(bref))
              and not BE[N:].any().item())
        self._exact('head-weff', '%dx%d->%d' % (N, K, Npad), ok)
        return rc

    def chk_head_param_grads(self, fn, a):
        dweff, Wp, rw, dW, drw, n_cls, O, K, st = a
        GW, GR = dev(dW, O * K).view(O, K), dev(drw, n_cls * K).view(n_cls, K)
        GW.fill_(float('nan'))
        GR.fill_(float('nan'))
        rc = self.real(fn, *a)
        torch.cuda.synchronize()
        D = dev(dweff, n_cls * O * K).view(n_cls, O, K).double()
        Wt, R = dev(Wp, O * K).view(1, O, K).double(), dev(rw, n_cls * K).view(n_cls, 1, K).double()
        worst = 0.0
        for got, ref, absref in ((GW, (D * R).sum(0), (D * R).abs().sum(0)), (GR, (D * Wt).sum(1), (D * Wt).abs().sum(1))):
            d = (got.double() - ref).abs()
            worst = max(worst, torch.nan_to_num(torch.where(d == 0, 0.0, d / (SUM_BAR * absref)), nan=math.inf).max().item())
        self.cov.add('head-param-grads')
        self.expect(worst <= 1.0, ('head_param_grads', n_cls, O, K, worst))
        self._record('head-param-grads', '%dx%dx%d' % (n_cls, O, K), 'float64', worst)
        return rc

    def chk_head_bias_grad(self, fn, a):
        d, ld, dbias, ws, npix, n_cls, O, st = a
        G = dev(dbias, O)
        G.fill_(float('nan'))
        rc = self.real(fn, *a)
        torch.cuda.synchronize()
        D = rows(d, npix, n_cls * O, ld).double()
        ref = D.sum(0).view(n_cls, O).sum(0)
        absref = D.abs().sum(0).view(n_cls, O).sum(0)
        dd = (G.double() - ref).abs()
        worst = torch.nan_to_num(torch.where(dd == 0, 0.0, dd / (SUM_BAR * absref)), nan=math.inf).max().item()
        cancel = (absref / ref.abs().clamp_min(1e-300)).max().item()
        self.cov.add('head-bias-grad')
        self.expect(worst <= 1.0, ('head_bias_grad', npix, n_cls, O, worst))
        self._record('head-bias-grad', '%dx%dx%d' % (npix, n_cls, O), 'float64', worst, '  cancellation %.0f' % cancel)
        return rc

    def chk_globalmax_fwd(self, fn, a):
        x, ldx, y, arg, N, HW, C, st = a
        Y, A = dev(y, N * C).view(N, C), dev(arg, N * C, torch.int32).view(N, C)
        Y.fill_(float('nan'))
        A.fill_(-1)
        rc = self.real(fn, *a)
        torch.cuda.synchronize()
        X = rows(x, N * HW, C, ldx).view(N, HW, C)
        m = X.max(1).values
        idx = torch.arange(HW, device='cuda', dtype=torch.int32).view(1, HW, 1)
        first = torch.where(X == m.unsqueeze(1), idx, HW).min(1).values     # the first maximum in pixel order
        self._exact('globalmax', '%dx%dx%d' % (N, HW, C), torch.equal(bits(Y), bits(m)) and torch.equal(A, first))
        return rc

    def chk_globalmax_bwd(self, fn, a):
        dy, arg, dx, lddx, N, HW, C, st = a
        DX = rows(dx, N * HW, C, lddx).view(N, HW, C)
        DX.fill_(float('nan'))
        rc = self.real(fn, *a)
        torch.cuda.synchronize()
        A = dev(arg, N * C, torch.int32).view(N, 1, C).long()
        G = dev(dy, N * C).view(N, 1, C)
        idx = torch.arange(HW, device='cuda').view(1, HW, 1)
        ref = torch.where(idx == A, G, torch.zeros_like(G))
        self._exact('globalmax-bwd', '%dx%dx%d' % (N, HW, C), torch.equal(bits(DX), bits(ref)))
        return rc


def _run_step(side, bs, cs, seed):
    from fewshot_detection_b200 import _lib
    chk = []
    secs = run_step(side, bs, cs, seed, lambda real: chk.append(MemChecker(real, _lib.lib)) or chk[0])[3]
    return report(chk[0], secs)


def report(chk, secs):
    """Prints the worst ratio per kernel class of one checked step and fails if any check failed."""
    assert not chk.unknown, chk.unknown
    worst = {}
    for l in chk.log:
        w = worst.setdefault((l['kind'], l['flavour']), [0.0, 0])
        w[0] = max(w[0], l['ratio'])
        w[1] += 1
    print('\n%d checked calls, %.1f s (step + float64 references); worst ratio to the bar per class:' % (len(chk.log), secs))
    for k, w in sorted(worst.items()):
        print('  %-18s %-22s n=%3d  %.3f' % (k[0], k[1], w[1], w[0]))
    if chk.meanstd:         # a training step (an evaluation pass has no batch statistics and no backward)
        print('worst |mean|/std %.2f, worst cancellation sum|du|/|sum du| %.0f, amax_bound / max|dz| in [%.2f, %.2f]' % (
            max(chk.meanstd), max(chk.cancel), min(chk.bound_ratio), max(chk.bound_ratio)))
    if chk.seg_meanstd:
        print('worst |mean|/std per segment:', ', '.join('%d: %.2f' % kv for kv in sorted(chk.seg_meanstd.items())))
    print('coverage:', sorted(chk.cov))
    assert not chk.failures, chk.failures
    return chk


# what both configurations reach.  Neither has a conv + bias block (has_bn = 0: tests/test_bn_act_host_emul.py) or a
# copied route (the routes are written in place), so fsdet_copy_channels and the accumulating copy do not run.
COVERAGE = {'finalize-train', 'fwd-full', 'fwd-pool', 'fwd-pool+full', 'fwd-f32', 'fwd-planes', 'fwd-odd', 'bwd-pool-only',
            'bwd-general-full', 'bwd-general-full+pool', 'bwd-odd', 'reorg', 'reorg-bwd', 'globalmax', 'globalmax-bwd',
            'head-weff', 'head-param-grads', 'head-bias-grad', 'nchw-to-nhwc', 'nhwc-to-nchw-bias', 'pad-channels',
            'flip-transpose', 'amax', 'split-f16'}


def test_configs1_step_memops_vs_float64():
    """configs[1]: B = 64 query images + 20 support images at 416x416, 20 classes."""
    chk = _run_step(416, 64, 20, 61)
    assert COVERAGE <= chk.cov, sorted(COVERAGE - chk.cov)


def test_configs4_step_memops_vs_float64():
    """configs[4]: 608x608 (G = 19), 80 classes, B = 2."""
    chk = _run_step(608, 2, 80, 71)
    assert COVERAGE <= chk.cov, sorted(COVERAGE - chk.cov)


def test_checker_reports_one_wrong_dz_element_and_a_flipped_window():
    """The element-wise bar of the apply pass has teeth: on a real fsdet_bn_act_bwd_apply output, one dz element moved by
    four times its bar is reported although the relative L2 does not move, and so is a pooled window whose gradient went
    to another pixel."""
    from fewshot_detection_b200 import _lib
    st = torch.cuda.current_stream().cuda_stream
    B, H, W, C = 8, 26, 26, 64
    g = torch.Generator(device='cuda').manual_seed(5)
    z = torch.randn(B, H, W, C, device='cuda', generator=g) * 2 + 0.5
    mean = z.double().mean((0, 1, 2)).float()
    invstd = (1 / torch.sqrt(z.double().var((0, 1, 2), unbiased=False) + EPS)).float()
    scale = invstd * 1.3
    shift = -mean * scale + 0.1
    gp = torch.randn(B, H // 2, W // 2, C, device='cuda', generator=g)
    nrows = _lib.lib.fsdet_bn_bwd_rows(B, H, W)
    part = torch.empty(nrows + 1, 3 * C, dtype=torch.float64, device='cuda')
    coef = torch.empty(2 * C, dtype=torch.float64, device='cuda')
    dgamma, dbeta = torch.empty(C, device='cuda'), torch.empty(C, device='cuda')
    dz = torch.empty(B, H, W, C, device='cuda')
    P = lambda t: t.data_ptr()
    _lib.call('fsdet_bn_act_bwd_reduce', P(z), C, None, 0, P(gp), C, P(scale), P(shift), P(mean), P(invstd), 0.1, P(part),
              B, H, W, C, 1, st)
    gamma = scale / invstd
    _lib.call('fsdet_bn_bwd_finalize', P(part), nrows, float(B * H * W), P(gamma), P(invstd), None, P(dgamma),
              P(dbeta), P(coef), None, C, 1, st)
    _lib.call('fsdet_bn_act_bwd_apply', P(z), C, None, 0, P(gp), C, P(scale), P(shift), P(mean), P(invstd), P(coef), 0.1,
              P(dz), C, None, None, 0, None, B, H, W, C, 1, st)
    torch.cuda.synchronize()
    y32 = pre_act(z, scale, shift)
    du, _ = route(y32, leaky(y32, 0.1), None, gp, 0.1)
    xh = (z.double() - mean.double()) * invstd.double()
    c1, c2 = coef[:C], coef[C:]
    sc = scale.double()
    ref = sc * (du - c1 - xh * c2)
    bar = SUM_BAR * sc.abs() * (du.abs() + c1.abs() + (xh * c2).abs())

    def ratio(got):
        d = (got.double() - ref).abs()
        return torch.where(d == 0, 0.0, d / bar).max().item()

    def rel(got):
        return ((got.double() - ref).norm() / ref.norm()).item()
    assert ratio(dz) <= 1.0
    bad = dz.clone()
    bad[3, 7, 11, 5] += 4 * bar[3, 7, 11, 5].item()
    assert rel(bad) < 1e-6 and ratio(bad) > 3.0              # invisible to a norm bar, reported by the element-wise bar
    # one pooled window whose gradient went to another pixel of the window
    best = first_max(windows(leaky(y32, 0.1)))
    b, h2, w2, c = 2, 4, 9, 17
    q = best[b, h2, w2, c].item()
    o = (q + 1) % 4
    moved = (sc[c] * du[b, 2 * h2 + (q >> 1), 2 * w2 + (q & 1), c]).item()
    flip = dz.clone()
    flip[b, 2 * h2 + (q >> 1), 2 * w2 + (q & 1), c] -= moved
    flip[b, 2 * h2 + (o >> 1), 2 * w2 + (o & 1), c] += moved
    assert ratio(flip) > 3.0
