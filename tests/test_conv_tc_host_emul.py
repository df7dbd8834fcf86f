"""Control flow of the wgmma convolution kernel (csrc/conv_tc_kernels.cuh) on the CPU: the kernel source is compiled
against functional models of its PTX wrappers (tools/host_emul/conv_tc_emul.cpp: mbarrier phases and transaction counts,
im2col / tiled TMA loads into swizzled shared memory, wgmma with the device descriptor encoding, named barriers) and
must reproduce the convolution - for one-tile-per-CTA grids and for persistent grids smaller than, equal to and larger
than the tile count, for every operand-term mode (which planes are loaded and multiplied), with and without the fused
BatchNorm statistics.  A wrong barrier phase deadlocks (reported as -100 after a timeout) or corrupts the result.
The shared-memory descriptors and swizzle modes are checked too: the modelled TMA stores its boxes swizzled and the wgmma
model reads them back through the device descriptor encoding (tools/host_emul/wgmma_emul.h)."""
import ctypes

import numpy as np
import pytest

from emul_util import build_emul


@pytest.fixture(scope='module')
def emul():
    return build_emul('conv_tc', 'conv_tc_kernels.cuh')


def P(a):
    return a.ctypes.data_as(ctypes.c_void_p) if a is not None else None


def scale_from_amax(a):
    """conv_tc.cu: the power of two that maps the absolute maximum into [512, 1024)."""
    if not (a > 0) or not np.isfinite(a):
        return 1.0
    m, ex = np.frexp(np.float32(a))          # a = m * 2^ex, m in [0.5, 1)
    return float(2.0 ** (10 - int(ex)))


def split_planes(x):
    """fp32 tensor -> (hi, lo) fp16 planes of s*x as uint16 bit patterns, amax, and the exactly representable values."""
    amax = np.float32(np.abs(x).max())
    s = np.float32(scale_from_amax(amax))
    f = (x.astype(np.float32) * s).astype(np.float32)
    hi = f.astype(np.float16)
    lo = (f - hi.astype(np.float32)).astype(np.float16)
    exact = (hi.astype(np.float64) + lo.astype(np.float64)) / float(s)
    return hi.view(np.uint16), lo.view(np.uint16), np.array([amax], dtype=np.float32), exact


def conv_ref(x, w, k):
    """x [B,H,W,Cin], w [Cout,k*k,Cin] (float64) -> [B*H*W, Cout], stride 1, same padding."""
    B, H, W, Cin = x.shape
    pad = (k - 1) // 2
    xp = np.zeros((B, H + 2 * pad, W + 2 * pad, Cin))
    xp[:, pad:pad + H, pad:pad + W] = x
    out = np.zeros((B, H, W, w.shape[0]))
    for r in range(k):
        for s in range(k):
            out += np.einsum('bhwc,oc->bhwo', xp[:, r:r + H, s:s + W], w[:, r * k + s])
    return out.reshape(B * H * W, -1)


def expected(xh, xl, wh, wl, ax, aw, k, terms):
    """float64 value of the terms the kernel multiplies: hi*hi (+ x_lo*w_hi) (+ x_hi*w_lo), unscaled."""
    sx, sw = scale_from_amax(ax[0]), scale_from_amax(aw[0])
    f = lambda u: u.view(np.float16).astype(np.float64)
    out = conv_ref(f(xh), f(wh), k)
    if terms & 1:
        out += conv_ref(f(xl), f(wh), k)
    if terms & 2:
        out += conv_ref(f(xh), f(wl), k)
    return out / (sx * sw)


CASES = [
    # B, H, W, Cin, Cout, k, bn, bk, terms, persist, ctas, accumulate, stats
    (2, 16, 16, 32, 64, 3, 64, 32, 3, 1, 3, 0, 1),      # conv2-like: 4 tiles over 3 CTAs (uneven), 9 k-blocks per tile
    (2, 16, 16, 32, 64, 3, 64, 32, 3, 1, 1, 0, 1),      # one CTA walks all tiles: accumulator sets alternate 4 times
    (2, 16, 16, 32, 64, 3, 64, 32, 3, 1, 4, 0, 1),      # as many CTAs as tiles
    (1, 13, 13, 64, 32, 3, 64, 32, 3, 1, 2, 0, 1),      # dgrad-like: Cout < BN, M = 169 not a multiple of 128 (clipped rows)
    (2, 12, 12, 64, 200, 1, 128, 32, 3, 1, 2, 0, 1),    # 1x1, BN = 128, two N tiles (the second one partial), 2 k-blocks per tile
    (1, 20, 20, 32, 64, 3, 64, 32, 3, 1, 2, 1, 0),      # accumulate into z (TMA reduce-add)
    (3, 8, 8, 96, 64, 3, 64, 32, 3, 1, 2, 0, 1),        # 27 k-blocks per tile, 3 channel chunks per tap
    (2, 16, 16, 32, 64, 3, 64, 32, 3, 0, 0, 0, 1),      # one tile per CTA
    (1, 13, 13, 64, 136, 3, 128, 32, 3, 0, 0, 0, 1),    # two N tiles, partial second one, clipped rows, statistics per M tile
    (1, 20, 20, 32, 64, 3, 64, 32, 3, 0, 0, 1, 0),      # accumulate, one tile per CTA
    (2, 10, 10, 128, 128, 3, 128, 64, 3, 0, 0, 0, 1),   # long-K flavour: hi*hi k-blocks folded into a register total + lo accumulator
    (2, 10, 10, 128, 64, 3, 64, 64, 3, 0, 0, 0, 1),     # long-K, BN = 64
    (2, 16, 16, 32, 64, 3, 64, 32, 0, 1, 2, 0, 1),      # terms = 0: only the hi planes exist (lo maps are poisoned)
    (2, 16, 16, 32, 64, 3, 64, 32, 1, 1, 2, 0, 1),      # terms = 1: x_lo * w_hi added
    (2, 16, 16, 32, 64, 3, 64, 32, 2, 0, 0, 0, 1),      # terms = 2: x_hi * w_lo added
    (2, 10, 10, 128, 128, 3, 128, 64, 0, 0, 0, 0, 1),   # long-K, terms = 0 (single accumulator, deeper pipeline)
    (2, 10, 10, 128, 128, 3, 128, 64, 1, 0, 0, 1, 0),   # long-K, terms = 1, accumulate
]


@pytest.mark.parametrize('B,H,W,Cin,Cout,k,bn,bk,terms,persist,ctas,acc,stats', CASES)
def test_kernel_control_flow(emul, B, H, W, Cin, Cout, k, bn, bk, terms, persist, ctas, acc, stats):
    rs = np.random.RandomState(B * 100 + H + Cin + Cout + ctas + terms)
    x = rs.randn(B, H, W, Cin).astype(np.float32)
    w = (rs.randn(Cout, k * k, Cin) * 0.1).astype(np.float32)
    xh, xl, ax, xe = split_planes(x)
    wh, wl, aw, we = split_planes(w)
    M = B * H * W
    ld = Cout + 4
    z0 = rs.randn(M, ld).astype(np.float32) if acc else np.full((M, ld), 7.0, dtype=np.float32)
    z = z0.copy()
    tiles_n = -(-Cout // bn)
    rows = (ctas // tiles_n) if persist else -(-M // 128)
    st = np.full((rows, 4 * Cout), 123.0, dtype=np.float32) if stats else None
    rc = emul.emul_conv_tc(P(xh), P(xl), P(wh), P(wl), P(ax), P(aw), P(z), ld, B, H, W, Cin, Cin, Cout, k, acc, bn, bk, terms,
                           persist, ctas, P(st))
    assert rc == 0, 'barrier deadlock in the kernel' if rc == -100 else rc
    ref = expected(xh, xl, wh, wl, ax, aw, k, terms)
    got = z[:, :Cout].astype(np.float64) - (z0[:, :Cout] if acc else 0)
    err = np.linalg.norm(got - ref) / np.linalg.norm(ref)
    assert err < 2e-6, err
    assert np.array_equal(z[:, Cout:], z0[:, Cout:])      # columns beyond Cout are never written (clipped stores)
    if stats:
        zz = z[:, :Cout].astype(np.float64)
        assert np.allclose(st[:, :Cout].astype(np.float64).sum(0), zz.sum(0), rtol=1e-5, atol=1e-4)
        assert np.allclose(st[:, Cout:2 * Cout].astype(np.float64).sum(0), (zz * zz).sum(0), rtol=1e-5, atol=1e-4)
        assert np.array_equal(st[:, 2 * Cout:3 * Cout].min(0), z[:, :Cout].min(0))
        assert np.array_equal(st[:, 3 * Cout:].max(0), z[:, :Cout].max(0))
        if not persist:   # one row per 128-pixel tile: row r holds exactly the statistics of its pixels
            for r in range(rows):
                blk = zz[r * 128:(r + 1) * 128]
                assert np.allclose(st[r, :Cout], blk.sum(0), rtol=1e-5, atol=1e-4)


def test_slow_epilogue_does_not_lose_accumulators(emul):
    """With slow MMA warpgroups the producer runs ahead across tile boundaries: it must wait until every MMA warp has
    released a stage before refilling it - one CTA, four tiles."""
    emul.emul_set_ld_delay_us(30000)
    try:
        test_kernel_control_flow(emul, *CASES[1])
    finally:
        emul.emul_set_ld_delay_us(0)
