"""The segmented BatchNorm passes of csrc/bn_act.cu (per-replica statistics: one launch, `nseg` segments of whole images)
without a GPU (tools/host_emul/bn_act_emul.cpp), at shapes where segments cut through the CTA rows of the plain passes:
13x13 and 26x26 maps with 16 images per segment and 19x19 with 4.

- statistics: each segment's mean / invstd within the step bars of float64 over that segment alone, running statistics
  from segment 0 only (unbiased over its pixels), amax_y over every segment;
- forward: bit-equal to the plain pass run on each segment with that segment's scale / shift;
- backward: per-segment sums within 1e-6 of the sum of absolute terms, dgamma / dbeta the sum over segments, dz
  bit-equal to the plain apply pass run on each segment with that segment's coefficients;
- one segment: every segmented entry point is bit-equal to the plain one."""
import ctypes

import numpy as np
import pytest

from emul_util import build_emul
from test_bn_act_host_emul import EPS, P, f32, bwd_ref, plane_scale

SCRATCH_ROWS = 128
SHAPES = [(64, 13, 13, 8, 4), (32, 26, 26, 8, 2), (16, 19, 19, 12, 4)]   # B, H, W, C, segments (16, 16, 4 images each)
D, F = ctypes.c_double, ctypes.c_float


@pytest.fixture(scope='module')
def emul():
    return build_emul('bn_act', 'bn_act.cu')


def segmented_z(rs, B, H, W, C, nseg):
    """z whose segments have visibly different statistics"""
    z = rs.randn(nseg, B // nseg, H, W, C) * rs.uniform(0.3, 3, (nseg, 1, 1, 1, C)) + rs.uniform(-2, 2, (nseg, 1, 1, 1, C))
    return f32(z.reshape(B, H, W, C))


def seg_stats(emul, z, nseg, gamma, beta, rm, rv, momentum=0.1):
    B, H, W, C = z.shape
    seg_pix = B * H * W // nseg
    rows = emul.emul_bn_seg_colstats_rows(ctypes.c_size_t(seg_pix), nseg)
    part = np.full((nseg * (rows + SCRATCH_ROWS), 4 * C), np.nan, np.float32)
    assert emul.emul_bn_seg_colstats(P(z), C, ctypes.c_size_t(seg_pix), nseg, C, P(part)) == 0
    o = {k: np.full((nseg, C), np.nan, np.float32) for k in ('mean', 'invstd', 'scale', 'shift', 'xhat')}
    o['amax'] = np.full(1, np.nan, np.float32)
    assert emul.emul_bn_seg_finalize(P(part), rows, nseg, ctypes.c_size_t(seg_pix), P(gamma), P(beta), P(rm), P(rv),
                                     F(momentum), F(EPS), P(o['mean']), P(o['invstd']), P(o['scale']), P(o['shift']),
                                     F(0.1), P(o['amax']), P(o['xhat']), C) == 0
    o['rows'] = rows
    return o


@pytest.mark.parametrize('shape', SHAPES)
def test_segmented_statistics_against_float64(emul, shape):
    B, H, W, C, nseg = shape
    rs = np.random.RandomState(B + H)
    z = segmented_z(rs, B, H, W, C, nseg)
    gamma, beta = f32(rs.uniform(0.5, 1.5, C)), f32(rs.randn(C) * 0.3)
    rm0, rv0 = f32(rs.randn(C)), f32(rs.uniform(0.5, 2, C))
    rm, rv = rm0.copy(), rv0.copy()
    o = seg_stats(emul, z, nseg, gamma, beta, rm, rv)
    zs = z.reshape(nseg, -1, C).astype(np.float64)
    ymax = 0.0
    for g in range(nseg):
        mu, var = zs[g].mean(0), zs[g].var(0)
        std = np.sqrt(var + EPS)
        assert np.all(np.abs(o['mean'][g] - mu) <= 1e-5 * std), g
        assert np.all(np.abs(o['invstd'][g] - 1 / std) * std <= 1e-5), g
        assert np.array_equal(o['scale'][g], (gamma * o['invstd'][g]).astype(np.float32))
        xh = ((zs[g].astype(np.float32) - o['mean'][g]).astype(np.float32) * o['invstd'][g]).astype(np.float32)
        assert np.array_equal(o['xhat'][g], np.abs(xh).max(0))
        u = zs[g].astype(np.float32) * np.float64(1) * o['scale'][g] + o['shift'][g]
        ymax = max(ymax, np.abs(np.where(u > 0, u, 0.1 * u)).max())
    assert abs(o['amax'][0] - ymax) <= 2 * np.spacing(np.float32(ymax))      # one amax over every segment
    # running statistics: replica 0 only, unbiased over its own pixels
    n0 = zs.shape[1]
    np.testing.assert_allclose(rm, 0.9 * rm0 + 0.1 * o['mean'][0].astype(np.float64), rtol=0, atol=1e-6)
    np.testing.assert_allclose(rv, 0.9 * rv0 + 0.1 * zs[0].var(0) * n0 / (n0 - 1), rtol=1e-5)


@pytest.mark.parametrize('shape', SHAPES)
def test_segmented_forward_is_the_plain_pass_per_segment(emul, shape):
    B, H, W, C, nseg = shape
    rs = np.random.RandomState(B * H)
    z = segmented_z(rs, B, H, W, C, nseg)
    sc, sh = f32(rs.uniform(-1.5, 1.5, (nseg, C))), f32(rs.randn(nseg, C) * 0.5)
    Cpad = C + 4
    amax = f32([np.abs(z).max() * 2 + 2])
    M, Mp, nb = B * H * W, B * (H // 2) * (W // 2), B // nseg

    def run(fn, zz, s, t, nbat, *extra):
        m, mp = nbat * H * W, nbat * (H // 2) * (W // 2)
        o = [np.full((m, C), np.nan, np.float32), np.full((mp, C), np.nan, np.float32),
             np.zeros((m, Cpad), np.uint16), np.zeros((m, Cpad), np.uint16), np.zeros((mp, Cpad), np.uint16),
             np.zeros((mp, Cpad), np.uint16)]
        assert fn(P(zz), C, P(s), P(t), F(0.1), P(o[0]), C, P(o[1]), C, P(o[2]), P(o[3]), P(o[4]), P(o[5]), Cpad, P(amax),
                  nbat, H, W, C, *extra) == 0
        return o

    def run_flat(fn, zz, s, t, nbat, *extra):
        y = np.full((nbat * H * W, C), np.nan, np.float32)
        assert fn(P(zz), C, P(s), P(t), F(0.1), P(y), C, None, 0, None, None, None, None, C, None, nbat, H, W, C, *extra) == 0
        return y

    got = run(emul.emul_bn_act_fwd_seg, z, sc, sh, B, nseg, ctypes.c_size_t(M // nseg))
    got_flat = run_flat(emul.emul_bn_act_fwd_seg, z, sc, sh, B, nseg, ctypes.c_size_t(M // nseg))
    for g in range(nseg):
        zg = np.ascontiguousarray(z[g * nb:(g + 1) * nb])
        want = run(emul.emul_bn_act_fwd, zg, sc[g], sh[g], nb)
        for a, b, rows in zip(got, want, [nb * H * W, nb * (H // 2) * (W // 2)] * 1 + [nb * H * W] * 2 + [nb * (H // 2) * (W // 2)] * 2):
            k = a.shape[0] // nseg
            assert np.array_equal(a[g * k:(g + 1) * k].view(np.uint8), b.view(np.uint8)), g
        wf = run_flat(emul.emul_bn_act_fwd, zg, sc[g], sh[g], nb)
        assert np.array_equal(got_flat[g * nb * H * W:(g + 1) * nb * H * W].view(np.uint32), wf.view(np.uint32))


@pytest.mark.parametrize('shape', SHAPES)
@pytest.mark.parametrize('pooled', [True, False])
def test_segmented_backward(emul, shape, pooled):
    B, H, W, C, nseg = shape
    rs = np.random.RandomState(B + W + pooled)
    z = segmented_z(rs, B, H, W, C, nseg)
    gamma, beta = f32(rs.uniform(0.5, 1.5, C)), f32(rs.randn(C) * 0.3)
    o = seg_stats(emul, z, nseg, gamma, beta, None, None)
    Hp, Wp = H // 2, W // 2
    dyp = f32(rs.randn(B, Hp, Wp, C) + 0.5) if pooled else None
    dyf = None if pooled else f32(rs.randn(B, H, W, C) * 0.2 + 0.3)
    seg_pix = ctypes.c_size_t(B * H * W // nseg)
    rows = emul.emul_bn_seg_bwd_rows(B, H, W, nseg)
    part = np.full((nseg * (rows + 1), 3 * C), np.nan)
    assert emul.emul_bn_act_bwd_reduce_seg(P(z), C, P(dyf), C, P(dyp), C, P(o['scale']), P(o['shift']), P(o['mean']),
                                           P(o['invstd']), F(0.1), P(part), B, H, W, C, nseg, seg_pix) >= 0
    dg, db = np.full(C, np.nan, np.float32), np.full(C, np.nan, np.float32)
    coef = np.full((nseg, 2 * C), np.nan)
    amax = np.full(1, np.nan, np.float32)
    assert emul.emul_bn_bwd_finalize_seg(P(part), rows, nseg, seg_pix, P(gamma), P(o['invstd']), P(o['xhat']), P(dg), P(db),
                                         P(coef), P(amax), C) == 0
    dz = np.full((B * H * W, C), np.nan, np.float32)
    hi, lo = np.zeros((B * H * W, C), np.uint16), np.zeros((B * H * W, C), np.uint16)
    assert emul.emul_bn_act_bwd_apply_seg(P(z), C, P(dyf), C, P(dyp), C, P(o['scale']), P(o['shift']), P(o['mean']),
                                          P(o['invstd']), P(coef), F(0.1), P(dz), C, P(hi), P(lo), C, P(amax), B, H, W, C,
                                          nseg, seg_pix) >= 0
    nb = B // nseg
    s1_all = s2_all = 0.0
    for g in range(nseg):
        sl = slice(g * nb, (g + 1) * nb)
        zg = np.ascontiguousarray(z[sl])
        r = bwd_ref(zg, None if dyf is None else dyf[sl], None if dyp is None else dyp[sl], o['scale'][g], o['shift'][g],
                    o['mean'][g].astype(np.float64), o['invstd'][g].astype(np.float64), 0.1, 1)
        n = nb * H * W
        assert np.all(np.abs(coef[g, :C] * n - r['s1']) <= 1e-6 * r['a1'] + 1e-300), g
        assert np.all(np.abs(coef[g, C:] * n - r['s2']) <= 1e-6 * r['a2'] + 1e-300), g
        s1_all, s2_all = s1_all + r['s1'], s2_all + r['s2']
        # dz of the segment: the plain apply pass over that segment with its own coefficients and the shared plane scale
        want = np.full((n, C), np.nan, np.float32)
        wh, wl = np.zeros((n, C), np.uint16), np.zeros((n, C), np.uint16)
        assert emul.emul_bn_act_bwd_apply(P(zg), C, P(None if dyf is None else np.ascontiguousarray(dyf[sl])), C,
                                          P(None if dyp is None else np.ascontiguousarray(dyp[sl])), C, P(o['scale'][g]),
                                          P(o['shift'][g]), P(o['mean'][g]), P(o['invstd'][g]), P(np.ascontiguousarray(coef[g])),
                                          F(0.1), P(want), C, P(wh), P(wl), C, P(amax), nb, H, W, C, 1) >= 0
        assert np.array_equal(dz[g * n:(g + 1) * n].view(np.uint32), want.view(np.uint32)), g
        assert np.array_equal(hi[g * n:(g + 1) * n], wh) and np.array_equal(lo[g * n:(g + 1) * n], wl), g
        assert np.all(np.abs(dz[g * n:(g + 1) * n].astype(np.float64) - r['dz'].reshape(-1, C)) <= 1e-6 * r['bar'].reshape(-1, C) + 1e-30)
        assert amax[0] >= np.abs(want).max()                       # one plane scale bounds every segment's dz
    a1 = np.abs(s1_all) + 1e-30
    assert np.all(np.abs(db - s1_all) <= 1e-6 * a1 + np.spacing(np.abs(db)))
    assert np.all(np.abs(dg - s2_all) <= 1e-6 * (np.abs(s2_all) + 1) + np.spacing(np.abs(dg)))


def test_one_segment_is_the_plain_pass_bit_for_bit(emul):
    B, H, W, C = 3, 13, 13, 20
    rs = np.random.RandomState(9)
    z = f32(rs.randn(B, H, W, C) * 2 + 1)
    M = B * H * W
    # column statistics
    rows = emul.emul_colstats_rows(ctypes.c_size_t(M))
    assert emul.emul_bn_seg_colstats_rows(ctypes.c_size_t(M), 1) == rows
    a = np.full((rows + SCRATCH_ROWS, 4 * C), np.nan, np.float32)
    b = a.copy()
    assert emul.emul_colstats(P(z), C, ctypes.c_size_t(M), C, P(a)) == 0
    assert emul.emul_bn_seg_colstats(P(z), C, ctypes.c_size_t(M), 1, C, P(b)) == 0
    assert np.array_equal(a[:rows].view(np.uint32), b[:rows].view(np.uint32))
    # finalize
    gamma, beta = f32(rs.uniform(0.5, 1.5, C)), f32(rs.randn(C))
    outs = []
    for seg in (False, True):
        part = a.copy()
        rm, rv = f32(np.zeros(C)), f32(np.ones(C))
        o = [np.full(C, np.nan, np.float32) for _ in range(5)] + [np.full(1, np.nan, np.float32)]
        common = (P(gamma), P(beta), P(rm), P(rv), F(0.1), F(EPS), P(o[0]), P(o[1]), P(o[2]), P(o[3]), F(0.1), P(o[5]), P(o[4]), C)
        if seg:
            assert emul.emul_bn_seg_finalize(P(part), rows, 1, ctypes.c_size_t(M), *common) == 0
        else:
            assert emul.emul_bn_finalize(P(part), rows, D(M), *common, 1) == 0
        outs.append([rm, rv] + o)
    for x, y in zip(*outs):
        assert np.array_equal(x.view(np.uint32), y.view(np.uint32))
    mean, invstd, sc, sh, xabs = outs[0][2:7]
    # forward, every output
    Cpad = C + 12
    am = f32([10.0])
    res = []
    for seg in (False, True):
        o = [np.zeros((M, C), np.float32), np.zeros((B * 36, C), np.float32)] + [np.zeros((n, Cpad), np.uint16) for n in (M, M, B * 36, B * 36)]
        args = (P(z), C, P(sc), P(sh), F(0.1), P(o[0]), C, P(o[1]), C, P(o[2]), P(o[3]), P(o[4]), P(o[5]), Cpad, P(am), B, H, W, C)
        assert (emul.emul_bn_act_fwd_seg(*args, 1, ctypes.c_size_t(M)) if seg else emul.emul_bn_act_fwd(*args)) == 0
        res.append(o)
    for x, y in zip(*res):
        assert np.array_equal(x.view(np.uint8), y.view(np.uint8))
    # backward: reduce, finalize, apply
    dyp = f32(rs.randn(B, 6, 6, C))
    res = []
    for seg in (False, True):
        nrow = emul.emul_bn_seg_bwd_rows(B, H, W, 1) if seg else emul.emul_bn_bwd_rows(B, H, W)
        part = np.full((nrow + 1, 3 * C), np.nan)
        base = (P(z), C, None, C, P(dyp), C, P(sc), P(sh), P(mean), P(invstd), F(0.1), P(part), B, H, W, C)
        assert (emul.emul_bn_act_bwd_reduce_seg(*base, 1, ctypes.c_size_t(M)) if seg else emul.emul_bn_act_bwd_reduce(*base, 1)) >= 0
        dg, db, coef, amax = np.zeros(C, np.float32), np.zeros(C, np.float32), np.zeros(2 * C), np.zeros(1, np.float32)
        fin = (P(gamma), P(invstd), P(xabs), P(dg), P(db), P(coef), P(amax), C)
        assert (emul.emul_bn_bwd_finalize_seg(P(part), nrow, 1, ctypes.c_size_t(M), *fin) if seg else
                emul.emul_bn_bwd_finalize(P(part), nrow, D(M), *fin, 1)) == 0
        dz, hi, lo = np.zeros((M, C), np.float32), np.zeros((M, C), np.uint16), np.zeros((M, C), np.uint16)
        app = (P(z), C, None, C, P(dyp), C, P(sc), P(sh), P(mean), P(invstd), P(coef), F(0.1), P(dz), C, P(hi), P(lo), C, P(amax),
               B, H, W, C)
        assert (emul.emul_bn_act_bwd_apply_seg(*app, 1, ctypes.c_size_t(M)) if seg else emul.emul_bn_act_bwd_apply(*app, 1)) >= 0
        res.append([part, dg, db, coef, amax, dz, hi, lo])
    for x, y in zip(*res):
        assert np.array_equal(x.view(np.uint8), y.view(np.uint8))


def test_segments_must_be_whole_images(emul):
    z = f32(np.zeros((4 * 5 * 5, 4)))
    s = f32(np.ones(8))
    y = np.zeros((100, 4), np.float32)
    ok = emul.emul_bn_act_fwd_seg(P(z), 4, P(s), P(s), F(0.1), P(y), 4, None, 0, None, None, None, None, 4, None, 4, 5, 5, 4, 2,
                                  ctypes.c_size_t(50))
    assert ok == 0
    for nseg, seg_pix in ((3, 33), (2, 49), (8, 12)):
        assert emul.emul_bn_act_fwd_seg(P(z), 4, P(s), P(s), F(0.1), P(y), 4, None, 0, None, None, None, None, 4, None, 4, 5, 5, 4,
                                        nseg, ctypes.c_size_t(seg_pix)) == -1
