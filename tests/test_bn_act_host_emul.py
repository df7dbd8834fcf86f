"""csrc/bn_act.cu's BatchNorm / LeakyReLU / max-pool passes without a GPU (tools/host_emul/bn_act_emul.cpp: the kernel
source compiled by g++, CUDA threads = OS threads, launched on the device's own grids) against float64 references in
numpy, at the edges the step never reaches: channel counts whose C/4 is not a multiple of the lane count, H or W of 1,
odd maps whose cut windows have no pooled output, ties after the LeakyReLU, count = 1, zero variance, more stage-1 rows
than the finalize split takes at once, gradients dominated by their mean, and a grid-stride loop that wraps.

Bars: finalize |d mean| <= 1e-5 std and |d invstd| <= 1e-5 invstd (std of the float64 z), scale / shift within an ulp;
forward bit-exact against the fp32 arithmetic the kernel performs and within two roundings of float64; backward sums
within 1e-6 of the sum of absolute terms, dz within 1e-6 * |scale| * (|du| + |c1| + |xhat * c2|) of float64."""
import ctypes

import numpy as np
import pytest

from emul_util import build_emul

SCRATCH_ROWS = 128          # fsdet_bn_stat_scratch_rows(): the stage-1 result lives behind the partial rows
EPS = 1e-5


@pytest.fixture(scope='module')
def emul():
    return build_emul('bn_act', 'bn_act.cu')


def P(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def fma32(a, b, c):
    """float32 fma(a, b, c): the product of two floats is exact in float64"""
    return (np.float64(1) * a * b + c).astype(np.float32)


def leaky32(y, slope):
    return np.where(y > 0, y, y * np.float32(slope)).astype(np.float32)


def ulps(got, ref64):
    """distance of float32 `got` from float64 `ref64` in units of the float32 spacing at ref64"""
    r = np.abs(ref64).astype(np.float32)
    sp = np.spacing(np.maximum(r, np.float32(np.finfo(np.float32).tiny))).astype(np.float64)
    return np.abs(got.astype(np.float64) - ref64) / sp


def plane_scale(a):
    """bn_act.cu plane_scale: the power of two that maps the absolute maximum into [512, 1024)"""
    a = float(a)
    if not (a > 0) or not np.isfinite(a):
        return 1.0
    return 2.0 ** max(-60, min(60, 10 - np.frexp(a)[1]))


def split16(v, s):
    f = (v * np.float32(s)).astype(np.float32)
    hi = f.astype(np.float16)
    lo = (f - hi.astype(np.float32)).astype(np.float16)
    return hi, lo


def same_value(a, b):
    """bit equality with -0 == +0 (fmaxf of two zeros may return either)"""
    return np.array_equal((a + np.float32(0)).view(np.uint32), (b + np.float32(0)).view(np.uint32))


# ------------------------------------------------------------------ finalize
def stat_rows(z, nparts):
    """the conv epilogue's partial rows [nparts + scratch][4C] (sum | sum of squares | min | max) of z [M][C]"""
    M, C = z.shape
    part = np.full((nparts + SCRATCH_ROWS, 4 * C), np.nan, dtype=np.float32)
    for r, rows in enumerate(np.array_split(np.arange(M), nparts)):
        zz = z[rows].astype(np.float64)
        part[r] = np.concatenate([zz.sum(0), (zz * zz).sum(0), zz.min(0), zz.max(0)]).astype(np.float32)
    return part


def finalize(emul, z, nparts, gamma, beta, slope=0.1, training=1, rm=None, rv=None, momentum=0.1, count=None):
    C = gamma.shape[0]
    part = stat_rows(z, nparts) if training else None
    o = {k: np.full(C, np.nan, dtype=np.float32) for k in ('mean', 'invstd', 'scale', 'shift', 'xhat')}
    o['amax'] = np.full(1, np.nan, dtype=np.float32)
    o['rm'], o['rv'] = rm, rv
    rc = emul.emul_bn_finalize(P(part), nparts, ctypes.c_double(z.shape[0] if count is None else count), P(gamma), P(beta),
                               P(rm), P(rv), ctypes.c_float(momentum), ctypes.c_float(EPS), P(o['mean']), P(o['invstd']),
                               P(o['scale']), P(o['shift']), ctypes.c_float(slope), P(o['amax']), P(o['xhat']), C, training)
    assert rc == 0
    return o


def check_finalize(z, o, gamma, beta, slope, bar=1e-5):
    """returns (mean ratio, invstd ratio) to the step bars"""
    z64 = z.astype(np.float64)
    mu, var = z64.mean(0), z64.var(0)
    std = np.sqrt(var + EPS)
    rm = np.abs(o['mean'] - mu) / (bar * std)
    ri = np.abs(o['invstd'] - 1 / std) * std / bar
    assert np.all(ulps(o['scale'], gamma.astype(np.float64) * o['invstd']) <= 1)
    prod = o['mean'].astype(np.float64) * o['scale']
    sh64 = beta.astype(np.float64) - prod
    # one rounding of the result, plus half an ulp of mean * scale where the multiply is not fused
    assert np.all(np.abs(o['shift'] - sh64) <= np.spacing(np.abs(sh64).astype(np.float32)) +
                  0.5 * np.spacing(np.abs(prod).astype(np.float32)))
    y = leaky32(fma32(z, o['scale'], o['shift']), slope)
    ymax64 = np.abs(np.where(fma32(z, o['scale'], o['shift']) > 0, 1.0, slope) *
                    (z64 * o['scale'] + o['shift'])).max()
    assert ulps(o['amax'], np.float64(ymax64)).item() <= 1
    assert o['amax'][0] >= np.abs(y).max()                       # a valid plane scale for every element written
    xh = ((z - o['mean']).astype(np.float32) * o['invstd']).astype(np.float32)
    assert np.array_equal(o['xhat'], np.abs(xh).max(0))
    return rm.max(), ri.max()


@pytest.mark.parametrize('gsign', [1, -1])
def test_finalize_training(emul, gsign):
    rs = np.random.RandomState(1)
    M, C = 3000, 20
    z = f32(rs.randn(M, C) * rs.uniform(0.1, 3, C) + rs.uniform(-2, 2, C))
    gamma = f32(gsign * rs.uniform(0.5, 1.5, C))
    beta = f32(rs.randn(C) * 0.3)
    rm0, rv0 = f32(rs.randn(C)), f32(rs.uniform(0.5, 2, C))
    rm, rv = rm0.copy(), rv0.copy()
    o = finalize(emul, z, 37, gamma, beta, rm=rm, rv=rv, momentum=0.1)
    r = check_finalize(z, o, gamma, beta, 0.1)
    assert max(r) <= 1.0, r
    z64 = z.astype(np.float64)
    want_m = 0.9 * rm0.astype(np.float64) + 0.1 * o['mean']
    want_v = 0.9 * rv0.astype(np.float64) + 0.1 * z64.var(0, ddof=1)
    np.testing.assert_allclose(rm, want_m, rtol=0, atol=1e-6 * (np.abs(want_m).max() + 1))
    np.testing.assert_allclose(rv, want_v, rtol=1e-5)
    if gsign < 0:   # y is decreasing in z: the absolute maximum comes from the minimum end
        s, t = o['scale'], o['shift']
        lo = np.abs(leaky32(fma32(z.min(0), s, t), 0.1))
        assert o['amax'][0] == lo.max() and lo.max() > np.abs(leaky32(fma32(z.max(0), s, t), 0.1)).max()


def test_finalize_eval(emul):
    rs = np.random.RandomState(2)
    C = 12
    rm, rv = f32(rs.randn(C)), f32(rs.uniform(0.1, 2, C))
    gamma, beta = f32(rs.uniform(0.5, 1.5, C)), f32(rs.randn(C))
    rm0, rv0 = rm.copy(), rv.copy()
    o = finalize(emul, np.zeros((1, C), np.float32), 0, gamma, beta, training=0, rm=rm, rv=rv)
    assert np.array_equal(rm, rm0) and np.array_equal(rv, rv0)        # eval leaves the running statistics alone
    assert np.array_equal(o['mean'], rm)
    assert np.array_equal(o['invstd'], (np.float32(1) / np.sqrt(rv + np.float32(EPS))).astype(np.float32))
    # three fp32 roundings (add, sqrt, divide), as torch's eval BatchNorm in fp32
    assert np.all(ulps(o['invstd'], 1 / np.sqrt(rv.astype(np.float64) + np.float32(EPS))) <= 2)
    assert np.array_equal(o['scale'], gamma * o['invstd'])
    assert o['amax'][0] == 0 and not o['xhat'].any()                    # no batch range: nothing derived from it


def test_finalize_count_one_and_constant_channel(emul):
    C = 8
    gamma, beta = f32(np.linspace(0.5, 2, C)), f32(np.linspace(-1, 1, C))
    z = f32(np.full((1, C), 0.75))                                       # squares exact in fp32: var == 0
    rm, rv = f32(np.ones(C)), f32(np.full(C, 2.0))
    o = finalize(emul, z, 1, gamma, beta, rm=rm, rv=rv, momentum=0.5)
    assert np.all(o['mean'] == 0.75)
    assert np.array_equal(o['invstd'], np.full(C, 1 / np.sqrt(np.float64(np.float32(EPS))), dtype=np.float32))
    assert np.all(rv == 1.0)                                               # unbiased guard: var * 1 / 0 never formed
    assert np.all(rm == 0.875)
    # a constant channel in a larger batch: var = 0, invstd = 1/sqrt(eps), xhat = 0
    z = f32(np.tile(np.float32([0.5, -1.25, 3.0, 0.0, 2.5, -4.0, 1.0, 0.25]), (500, 1)))
    o = finalize(emul, z, 9, gamma, beta)
    assert np.array_equal(o['mean'], z[0])
    assert np.all(o['invstd'] == np.float32(1 / np.sqrt(np.float64(np.float32(EPS)))))
    assert not o['xhat'].any()
    check_finalize(z, o, gamma, beta, 0.1)


def test_finalize_more_rows_than_one_split(emul):
    """more than 64 x 64 partial rows: the stage-1 split is capped at 64 blocks and every row must still count"""
    nparts = 64 * 64 + 37
    assert emul.emul_bn_stat_splits(nparts) == 64
    rs = np.random.RandomState(4)
    C = 8
    z = f32(rs.randn(2 * nparts, C) + 0.5)
    z[-1] += 40.0                                   # the last row carries the maximum: dropping it moves amax and mean
    gamma, beta = f32(np.ones(C)), f32(np.zeros(C))
    o = finalize(emul, z, nparts, gamma, beta)
    r = check_finalize(z, o, gamma, beta, 0.1)
    assert max(r) <= 1.0, r


@pytest.mark.parametrize('ratio', [1, 10, 100])
def test_finalize_one_pass_variance_vs_shift(emul, ratio):
    """var = q/N - mean^2 from fp32 partial rows loses about (1 + (mean/std)^2) * 2^-24 of var: the step bars hold up to
    |mean|/std = 10; at 100 the analytical bound of the formula is what holds."""
    rs = np.random.RandomState(5)
    M, C = 20000, 12
    std = rs.uniform(0.5, 2, C)
    z = f32(rs.randn(M, C) * std + ratio * std)
    gamma, beta = f32(np.ones(C)), f32(np.zeros(C))
    rv = f32(np.zeros(C))
    o = finalize(emul, z, 200, gamma, beta, rm=f32(np.zeros(C)), rv=rv, momentum=1.0)
    z64 = z.astype(np.float64)
    var, r = z64.var(0), np.abs(z64.mean(0)) / z64.std(0)
    got_var = rv.astype(np.float64) * (M - 1) / M          # momentum 1: the unbiased batch variance, rounded once
    # fp32 rounding of every partial sum and sum of squares: 2^-24 (var + mean^2) + 2^-23 |mean| E|z| <= 4 (1 + r^2) 2^-24
    rel = np.abs(got_var - var) / var
    assert np.all(rel <= 4 * (1 + r * r) * 2.0 ** -24 + 2.0 ** -23), (rel, r)
    ratios = check_finalize(z, o, gamma, beta, 0.1, bar=1e-5)
    print('mean/std %d: worst ratio to the step bars %.3f %.3f; var error %.2e (bound %.2e)'
          % (ratio, ratios[0], ratios[1], rel.max(), (4 * (1 + r * r) * 2.0 ** -24).max()))
    if ratio <= 10:
        assert max(ratios) <= 1.0, ratios


# ------------------------------------------------------------------- forward
def windows(a):
    """[B,H,W,C] -> [4,B,Hp,Wp,C]: the whole 2x2 windows in scan order (0,0), (0,1), (1,0), (1,1)"""
    Hp, Wp = a.shape[1] // 2, a.shape[2] // 2
    a = a[:, :2 * Hp, :2 * Wp]
    return np.stack([a[:, 0::2, 0::2], a[:, 0::2, 1::2], a[:, 1::2, 0::2], a[:, 1::2, 1::2]])


GUARD = 8        # sentinel rows behind every output buffer: a store past the end (a cut window's row: W/2 + 1) is caught


def run_fwd(emul, z, sc, sh, slope, full, pool, fplanes, pplanes, Cpad, amax):
    B, H, W, C = z.shape
    Hp, Wp = H // 2, W // 2
    M, Mp = B * H * W, B * Hp * Wp
    o = {}
    o['yf'] = np.full((M + GUARD, C), np.nan, np.float32) if full else None
    o['yp'] = np.full((Mp + GUARD, C), np.nan, np.float32) if pool else None
    sent = np.uint16(0x7e01)
    o['fh'], o['fl'] = [np.full((M + GUARD, Cpad), sent, np.uint16) if fplanes else None for _ in range(2)]
    o['ph'], o['pl'] = [np.full((Mp + GUARD, Cpad), sent, np.uint16) if pplanes else None for _ in range(2)]
    am = f32([amax])
    rc = emul.emul_bn_act_fwd(P(z), C, P(sc), P(sh), ctypes.c_float(slope), P(o['yf']), C, P(o['yp']), C, P(o['fh']),
                              P(o['fl']), P(o['ph']), P(o['pl']), Cpad, P(am), B, H, W, C)
    assert rc == 0
    for k in ('yf', 'yp'):
        if o[k] is not None:
            assert np.all(np.isnan(o[k][-GUARD:])), k + ' written past the end'
            o[k] = o[k][:-GUARD]
    for k in ('fh', 'fl', 'ph', 'pl'):
        if o[k] is not None:
            assert np.all(o[k][-GUARD:] == sent), k + ' written past the end'
            o[k] = o[k][:-GUARD]
    return o


def check_fwd(z, sc, sh, slope, o, Cpad, amax):
    B, H, W, C = z.shape
    y = leaky32(fma32(z, sc, sh), slope)                      # the fp32 arithmetic of the kernel
    u64 = z.astype(np.float64) * sc + sh
    y64 = np.where(y > 0, u64, u64 * np.float64(np.float32(slope)))
    assert np.all(np.abs(y - y64) <= 2.0 ** -23 * np.abs(y64)), 'more than two roundings from float64'
    pooled = windows(y).max(0).reshape(-1, C)
    s = plane_scale(amax)
    if o['yf'] is not None:
        assert np.array_equal(o['yf'].view(np.uint32), y.reshape(-1, C).view(np.uint32))
    if o['yp'] is not None:
        assert same_value(o['yp'], pooled)
    for hk, lk, ref in (('fh', 'fl', y.reshape(-1, C)), ('ph', 'pl', pooled)):
        if o[hk] is None:
            continue
        hi, lo = split16(ref, s)
        h16 = lambda a: (a + np.float16(0)).view(np.uint16)          # bit equality with -0 == +0
        assert np.array_equal(h16(o[hk][:, :C].view(np.float16)), h16(hi)), hk
        assert np.array_equal(h16(o[lk][:, :C].view(np.float16)), h16(lo)), lk
        assert not o[hk][:, C:].any() and not o[lk][:, C:].any(), 'plane padding [C, Cpad) not zero'


COMBOS = [  # full, pool, full planes, pool planes
    (1, 0, 0, 0), (0, 1, 0, 0), (1, 1, 0, 0), (0, 0, 1, 0), (0, 0, 0, 1), (1, 0, 1, 0), (0, 1, 0, 1), (1, 1, 1, 1), (0, 1, 1, 0)]


@pytest.mark.parametrize('shape', [(2, 13, 13, 12), (1, 6, 7, 20), (1, 7, 6, 4), (2, 1, 5, 36), (1, 5, 1, 12), (1, 1, 1, 8),
                                   (1, 8, 8, 132), (1, 3, 3, 4)])
@pytest.mark.parametrize('slope', [0.1, 1.0])
def test_forward_every_output_combination(emul, shape, slope):
    B, H, W, C = shape
    rs = np.random.RandomState(H * 100 + W + C)
    z = f32(rs.randn(B, H, W, C) * 2)
    sc, sh = f32(rs.uniform(-1.5, 1.5, C)), f32(rs.randn(C) * 0.5)
    amax = float(np.abs(leaky32(fma32(z, sc, sh), slope)).max())
    for full, pool, fpl, ppl in COMBOS:
        for Cpad in ((C, C + 4, C + 60) if (fpl or ppl) else (C,)):
            o = run_fwd(emul, z, sc, sh, slope, full, pool, fpl, ppl, Cpad, amax)
            check_fwd(z, sc, sh, slope, o, Cpad, amax)


# ------------------------------------------------------------------ backward
def bwd_ref(z, dyf, dyp, sc, sh, mu, istd, slope, has_bn):
    """float64 du (dy_pool to the first maximum of the fp32 activation, strict >, + dy_full, through the LeakyReLU on
    the fp32 pre-activation), xhat from the kernel's fp32 statistics, the sums, c1, c2 and dz"""
    B, H, W, C = z.shape
    y = fma32(z, sc, sh)
    du = np.zeros(z.shape) if dyf is None else dyf.astype(np.float64).copy()
    if dyp is not None:
        Hp, Wp = H // 2, W // 2
        best = windows(leaky32(y, slope)).argmax(0)             # first index of the maximum; -0 == +0 as in the scan
        for q in range(4):
            du[:, q >> 1:2 * Hp:2, q & 1:2 * Wp:2] += np.where(best == q, dyp.astype(np.float64), 0.0)
    du *= np.where(y > 0, 1.0, np.float64(np.float32(slope)))
    N = B * H * W
    xh = (z.astype(np.float64) - mu) * istd if has_bn else np.zeros(z.shape)
    s1, s2 = du.reshape(-1, C).sum(0), (du * xh).reshape(-1, C).sum(0)
    a1, a2 = np.abs(du).reshape(-1, C).sum(0), np.abs(du * xh).reshape(-1, C).sum(0)
    c1, c2 = s1 / N, s2 / N
    if has_bn:
        dz = sc.astype(np.float64) * (du - c1 - xh * c2)
        bar = np.abs(sc).astype(np.float64) * (np.abs(du) + np.abs(c1) + np.abs(xh * c2))
    else:
        dz, bar = du, np.abs(du)
    return dict(du=du, xh=xh, s1=s1, s2=s2, a1=a1, a2=a2, c1=c1, c2=c2, dz=dz, bar=bar)


def run_bwd(emul, z, dyf, dyp, sc, sh, mu, istd, slope, has_bn, planes=False):
    B, H, W, C = z.shape
    rows = emul.emul_bn_bwd_rows(B, H, W)
    part = np.full((rows + 1, 3 * C), np.nan)
    kern = emul.emul_bn_act_bwd_reduce(P(z), C, P(dyf), C, P(dyp), C, P(sc), P(sh), P(mu), P(istd), ctypes.c_float(slope),
                                       P(part), B, H, W, C, has_bn)
    assert kern in (0, 1)
    o = dict(kernel='pool' if kern == 1 else 'general', rows=rows)
    gamma = f32(sc / istd) if has_bn else None
    xabs = f32(np.abs(((z - mu).astype(np.float32) * istd).astype(np.float32)).reshape(-1, C).max(0)) if has_bn else None
    o['dgamma'], o['dbeta'] = np.full(C, np.nan, np.float32), np.full(C, np.nan, np.float32)
    o['coef'] = np.full(2 * C, np.nan)
    o['amax'] = np.full(1, np.nan, np.float32)
    rc = emul.emul_bn_bwd_finalize(P(part), rows, ctypes.c_double(B * H * W), P(gamma), P(istd if has_bn else None), P(xabs),
                                   P(o['dgamma'] if has_bn else None), P(o['dbeta']), P(o['coef'] if has_bn else None),
                                   P(o['amax']), C, has_bn)
    assert rc == 0
    o['dz'] = np.full(z.shape, np.nan, np.float32)
    o['dh'] = np.full(z.shape, 0x7e01, np.uint16) if planes else None
    o['dl'] = np.full(z.shape, 0x7e01, np.uint16) if planes else None
    k2 = emul.emul_bn_act_bwd_apply(P(z), C, P(dyf), C, P(dyp), C, P(sc), P(sh), P(mu), P(istd),
                                    P(o['coef'] if has_bn else None), ctypes.c_float(slope), P(o['dz']), C, P(o['dh']),
                                    P(o['dl']), C, P(o['amax']), B, H, W, C, has_bn)
    assert k2 == kern
    return o


def check_bwd(o, r, has_bn, bar=1e-6):
    """returns the worst ratio of dz to its bar"""
    C = r['s1'].shape[0]
    assert np.all(np.abs(o['dbeta'] - r['s1']) <= bar * r['a1'] + 1e-30)
    if has_bn:
        assert np.all(np.abs(o['dgamma'] - r['s2']) <= bar * r['a2'] + 1e-30)
        N = r['du'].size // C
        assert np.all(np.abs(o['coef'][:C] - r['c1']) <= bar * r['a1'] / N + 1e-300)
        assert np.all(np.abs(o['coef'][C:] - r['c2']) <= bar * r['a2'] / N + 1e-300)
    d = np.abs(o['dz'] - r['dz'])
    ratio = np.where(d == 0, 0.0, d / (bar * r['bar']))
    assert not np.isnan(o['dz']).any()
    if has_bn:
        assert o['amax'][0] >= np.abs(o['dz']).max(), 'plane scale bound below max|dz|'
    if o['dh'] is not None:
        hi, lo = split16(o['dz'], plane_scale(o['amax'][0]))
        assert np.array_equal(o['dh'].view(np.float16), hi) and np.array_equal(o['dl'].view(np.float16), lo)
    return np.nan_to_num(ratio, nan=np.inf).max()


def bwd_inputs(rs, B, H, W, C, dyf=False, dyp=True, mean_shift=0.0):
    z = f32(rs.randn(B, H, W, C) * rs.uniform(0.5, 2, C) + rs.randn(C))
    z64 = z.astype(np.float64).reshape(-1, C)
    mu, istd = f32(z64.mean(0)), f32(1 / np.sqrt(z64.var(0) + EPS))
    gamma = f32(rs.uniform(0.5, 1.5, C) * rs.choice([-1, 1], C))
    sc = f32(gamma * istd)
    sh = f32(rs.randn(C) * 0.3 - mu * sc)
    gf = f32(rs.randn(B, H, W, C) + mean_shift) if dyf else None
    gp = f32(rs.randn(B, H // 2, W // 2, C) + mean_shift) if dyp else None
    return z, gf, gp, sc, sh, mu, istd


@pytest.mark.parametrize('shape', [(2, 13, 13, 12), (1, 7, 6, 20), (1, 6, 9, 36), (3, 1, 5, 4), (1, 5, 1, 132), (2, 8, 8, 8)])
def test_backward_pool_only_vs_general_and_float64(emul, shape):
    """dy_pool only: the pool-only specialisation, and the general kernel on the same inputs (a dy_full of zeros); cut
    windows of an odd edge get dz = scale * (-c1 - xhat * c2), not zero"""
    B, H, W, C = shape
    rs = np.random.RandomState(sum(shape))
    z, _, gp, sc, sh, mu, istd = bwd_inputs(rs, B, H, W, C)
    r = bwd_ref(z, None, gp, sc, sh, mu, istd, 0.1, 1)
    o = run_bwd(emul, z, None, gp, sc, sh, mu, istd, 0.1, 1, planes=True)
    assert o['kernel'] == 'pool'
    assert check_bwd(o, r, 1) <= 1.0
    zero = np.zeros_like(z)
    og = run_bwd(emul, z, zero, gp, sc, sh, mu, istd, 0.1, 1, planes=True)
    assert og['kernel'] == 'general'
    assert check_bwd(og, bwd_ref(z, zero, gp, sc, sh, mu, istd, 0.1, 1), 1) <= 1.0
    if (H % 2 or W % 2) and H > 1 and W > 1:         # (H or W of 1: no whole window, no gradient at all)
        cut = np.concatenate([o['dz'][:, 2 * (H // 2):].ravel(), o['dz'][:, :, 2 * (W // 2):].ravel()])
        assert cut.size and np.all(cut != 0)


@pytest.mark.parametrize('slope', [-0.5, 1.5])
def test_backward_dispatch_slope_outside_unit_interval(emul, slope):
    """the pool-only kernel's fmaxf(y, y * slope) is leaky only for 0 <= slope <= 1: other slopes take the general
    kernel, and the result is still right"""
    rs = np.random.RandomState(7)
    z, _, gp, sc, sh, mu, istd = bwd_inputs(rs, 2, 7, 7, 12)
    o = run_bwd(emul, z, None, gp, sc, sh, mu, istd, slope, 1)
    assert o['kernel'] == 'general'
    assert check_bwd(o, bwd_ref(z, None, gp, sc, sh, mu, istd, slope, 1), 1) <= 1.0


@pytest.mark.parametrize('has_bn', [1, 0])
def test_backward_full_and_pooled_gradient(emul, has_bn):
    rs = np.random.RandomState(8 + has_bn)
    B, H, W, C = 2, 9, 11, 20
    z, gf, gp, sc, sh, mu, istd = bwd_inputs(rs, B, H, W, C, dyf=True)
    if not has_bn:          # conv + bias: scale 1, shift 0, no statistics
        sc, sh, mu, istd = f32(np.ones(C)), f32(np.zeros(C)), None, None
    r = bwd_ref(z, gf, gp, sc, sh, mu, istd, 0.1, has_bn)
    o = run_bwd(emul, z, gf, gp, sc, sh, mu, istd, 0.1, has_bn)
    assert o['kernel'] == 'general'
    assert check_bwd(o, r, has_bn) <= 1.0
    if not has_bn:          # dz = (dy_full + routed dy_pool) * leaky'(y) in fp32: exact
        y = fma32(z, sc, sh)
        du = np.zeros_like(z)
        best = windows(leaky32(y, 0.1)).argmax(0)
        for q in range(4):
            du[:, q >> 1:2 * (H // 2):2, q & 1:2 * (W // 2):2] += np.where(best == q, gp, np.float32(0))
        want = ((gf + du).astype(np.float32) * np.where(y > 0, np.float32(1), np.float32(0.1))).astype(np.float32)
        assert np.array_equal(o['dz'], want)


def test_backward_has_bn0_pool_only_takes_general_kernel(emul):
    rs = np.random.RandomState(10)
    B, H, W, C = 1, 7, 7, 12
    z, _, gp, _, _, _, _ = bwd_inputs(rs, B, H, W, C)
    sc, sh = f32(np.ones(C)), f32(np.zeros(C))
    o = run_bwd(emul, z, None, gp, sc, sh, None, None, 1.0, 0)
    assert o['kernel'] == 'general'
    assert check_bwd(o, bwd_ref(z, None, gp, sc, sh, None, None, 1.0, 0), 0) <= 1.0


def test_backward_grid_stride_wraps(emul):
    """more windows than bwd_rows * TY: every thread row visits several windows"""
    B, H, W, C = 1, 902, 902, 4
    rows, tc = emul.emul_bn_bwd_rows(B, H, W), emul.emul_bn_chan_lanes(C)
    assert B * (H // 2) * (W // 2) > rows * (256 // tc)
    rs = np.random.RandomState(11)
    z, _, gp, sc, sh, mu, istd = bwd_inputs(rs, B, H, W, C)
    o = run_bwd(emul, z, None, gp, sc, sh, mu, istd, 0.1, 1)
    assert check_bwd(o, bwd_ref(z, None, gp, sc, sh, mu, istd, 0.1, 1), 1) <= 1.0


def test_backward_mean_dominated_gradient(emul):
    """dy = 1 + ~1e-4 * noise: du - mean(du) keeps only 1e-4 of du.  Subtracting c1 as a (hi, lo) float pair loses
    nothing to that cancellation: dz stays within 1e-6 of the cancelled result |du - c1| + |xhat * c2|.  A reference
    that rounds c1 to one float misses that bar, so the case measures what the pair is for.  Every other term is made
    exact, so that only c1 can move dz: du is a multiple of 2^-12, xhat = z (mean 0, invstd 1) lies on a grid of 1/8
    and is symmetric per channel (c2 stays small), and N = 450 is not a power of two (c1 does not fit one float)."""
    rs = np.random.RandomState(12)
    B, H, W, C = 2, 15, 15, 8
    N = B * H * W
    half = rs.randint(1, 33, (N // 2, C)) / 8.0
    z = f32(np.stack([rs.permutation(np.concatenate([half[:, c], -half[:, c]])) for c in range(C)], 1).reshape(B, H, W, C))
    mu, istd = f32(np.zeros(C)), f32(np.ones(C))
    sc, sh = f32(rs.uniform(0.5, 2, C)), f32(np.zeros(C))
    gf = f32(1 + rs.randint(-2, 3, (B, H, W, C)) * 2.0 ** -12)
    slope = 1.0                              # linear: du = dy exactly
    r = bwd_ref(z, gf, None, sc, sh, mu, istd, slope, 1)
    o = run_bwd(emul, z, gf, None, sc, sh, mu, istd, slope, 1, planes=True)
    assert check_bwd(o, r, 1) <= 1.0
    du, xh = r['du'], r['xh']
    tight = 1e-6 * np.abs(sc) * (np.abs(du - r['c1']) + np.abs(xh * r['c2']))
    assert np.all(np.abs(o['dz'] - r['dz']) <= tight)
    c1f = r['c1'].astype(np.float32).astype(np.float64)
    rounded = sc.astype(np.float64) * (du - c1f - xh * r['c2'])
    assert np.any(np.abs(rounded - r['dz']) > 10 * tight)
    print('cancellation %.0f; kernel %.3f of the tight bar, single-float c1 %.0f' % (
        np.abs(du).max() / np.abs(du - r['c1']).max(), (np.abs(o['dz'] - r['dz']) / tight).max(),
        (np.abs(rounded - r['dz']) / tight).max()))


def test_backward_plane_bound_with_coinciding_maxima(emul):
    """max|du| and max|xhat| on the same pixel, with signs that add in dz: amax_bound >= max|dz| still"""
    rs = np.random.RandomState(13)
    B, H, W, C = 1, 8, 8, 8
    z, gf, _, sc, sh, mu, istd = bwd_inputs(rs, B, H, W, C, dyf=True, dyp=False)
    z[0, 3, 5] = z.max() + 6.0                       # the largest xhat of every channel ...
    gf[0, 3, 5] = -8.0                               # ... carries the largest |du|
    gf = gf * np.where(fma32(z, sc, sh) > 0, 1, 10).astype(np.float32)
    z64 = z.astype(np.float64).reshape(-1, C)
    mu, istd = f32(z64.mean(0)), f32(1 / np.sqrt(z64.var(0) + EPS))
    sc = f32(np.abs(sc))
    sh = f32(-mu * sc)
    r = bwd_ref(z, gf, None, sc, sh, mu, istd, 0.1, 1)
    o = run_bwd(emul, z, gf, None, sc, sh, mu, istd, 0.1, 1, planes=True)
    assert check_bwd(o, r, 1) <= 1.0
    i = np.unravel_index(np.abs(o['dz']).argmax(), o['dz'].shape)
    assert i[1:3] == (3, 5)


# --------------------------------------------------------------------- ties
def tie_pair(slope=0.1):
    """two distinct negative floats y0 < y1 whose y * slope round to the same float (y * 0.1 in [0.125, 0.2): the
    product's spacing is wider than 0.1 times y's)"""
    y = -np.float32(1.5) - np.arange(1, 4000, dtype=np.float32) * np.spacing(np.float32(1.5))
    p = (y * np.float32(slope)).astype(np.float32)
    i = np.nonzero(p[:-1] == p[1:])[0][0]
    return y[i + 1], y[i]            # y0 < y1 < 0, same activation


@pytest.mark.parametrize('case', ['equal', 'rounded-negative', 'all-negative', 'signed-zero'])
def test_ties_route_to_the_first_maximum(emul, case):
    """dy_pool reaches the first maximum in scan order (torch's strict >) in both backward kernels; the forward's
    pooled value is that maximum"""
    B, H, W, C = 1, 4, 4, 4
    z = f32(np.full((B, H, W, C), -3.0))
    y0, y1 = tie_pair()
    w = {'equal': [2.0, 2.0, 1.0, 2.0], 'rounded-negative': [-5.0, y0, -4.0, y1], 'all-negative': [-2.0, -0.5, -0.5, -1.0],
         'signed-zero': [-1.0, -0.0, 0.0, -0.0]}[case]
    for q in range(4):                   # the first window of every channel, and the last window shifted by a pixel
        z[0, q >> 1, q & 1] = w[q]
        z[0, 2 + (q >> 1), 2 + (q & 1)] = w[(q + 1) % 4]
    sc, sh = f32(np.ones(C)), f32(np.zeros(C))
    mu, istd = f32(np.full(C, -1.0)), f32(np.full(C, 0.7))
    gp = f32(np.arange(1, 1 + B * 2 * 2 * C).reshape(B, 2, 2, C))
    o = run_fwd(emul, z, sc, sh, 0.1, 1, 1, 0, 0, C, 1.0)
    check_fwd(z, sc, sh, 0.1, o, C, 1.0)
    r = bwd_ref(z, None, gp, sc, sh, mu, istd, 0.1, 1)
    first = [next(q for q in range(4) if leaky32(f32(w[q]), 0.1) == leaky32(f32(w), 0.1).max()),
             next(q for q in range(4) if leaky32(f32(w[(q + 1) % 4]), 0.1) == leaky32(f32(w), 0.1).max())]
    for (h0, w0), q in zip(((0, 0), (2, 2)), first):
        assert r['du'][0, h0 + (q >> 1), w0 + (q & 1), 0] != 0       # the reference routes as specified
    for dyf in (None, np.zeros_like(z)):
        o = run_bwd(emul, z, dyf, gp, sc, sh, mu, istd, 0.1, 1)
        assert check_bwd(o, bwd_ref(z, dyf, gp, sc, sh, mu, istd, 0.1, 1), 1) <= 1.0, (case, o['kernel'])
