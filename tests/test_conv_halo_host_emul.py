"""Control flow of the halo-tile wgmma convolution (csrc/conv_halo_kernels.cuh) on the CPU: the kernel source compiled
against functional models of its PTX wrappers (tools/host_emul/conv_halo_emul.cpp) must reproduce the 3x3 convolution of
the operand planes - persistent grids smaller than / equal to the tile count, resident and streamed weight operands
(both producer warps), one to four 32-channel chunks, tiles that overhang the image (clipped stores, masked statistics),
zero fill at the border, channel pitches larger than the channel count, accumulation into z.  A wrong barrier phase
deadlocks (-100) or corrupts the result.  Swizzle modes and descriptors are the im2col kernel's and are exercised on
the GPU (tests/test_gpu_tc.py)."""
import numpy as np
import pytest

from emul_util import build_emul
from test_conv_tc_host_emul import P, split_planes, expected


@pytest.fixture(scope='module')
def emul():
    return build_emul('conv_halo', 'conv_halo_kernels.cuh')


CASES = [
    # B, H, W, Cin, cpitch, Cout, ctas, accumulate, stats
    (2, 32, 16, 32, 32, 64, 3, 0, 1),     # conv2 forward: resident weights, 8 tiles over 3 CTAs (uneven)
    (1, 32, 16, 32, 64, 64, 4, 0, 1),     # channel pitch 64 with 32 channels (the engine's plane layout), one tile per CTA
    (1, 24, 16, 64, 64, 32, 2, 1, 0),     # conv2 input gradient: N = 32, two chunks, resident; H overhangs the 16-row tiles; accumulate
    (1, 24, 16, 64, 64, 32, 1, 0, 1),     # same shape, one CTA walks all tiles: both accumulator sets reused, masked statistics
    (1, 16, 16, 64, 64, 128, 2, 0, 1),    # conv3 forward: streamed weights (ring of 4), two chunks
    (1, 20, 8, 128, 128, 64, 1, 0, 1),    # conv3 input gradient: four chunks, ring of 8, overhang
    (1, 16, 8, 32, 32, 48, 1, 0, 1),      # Cout < BN: clipped channels (weight rows zero-filled, statistics / stores only below Cout)
    (2, 16, 8, 32, 32, 128, 2, 0, 1),     # N = 128 with one chunk (streamed)
]


@pytest.mark.parametrize('B,H,W,Cin,cpitch,Cout,ctas,acc,stats', CASES)
def test_halo_kernel_control_flow(emul, B, H, W, Cin, cpitch, Cout, ctas, acc, stats, flags=0):
    rs = np.random.RandomState(B * 100 + H + Cin + Cout + ctas)
    x = rs.randn(B, H, W, Cin).astype(np.float32)
    w = (rs.randn(Cout, 9, Cin) * 0.1).astype(np.float32)
    xh, xl, ax, _ = split_planes(x)
    wh, wl, aw, _ = split_planes(w)

    def pitched(a, n):      # [.., Cin] -> [.., cpitch], the padding channels poisoned (they must never be multiplied)
        out = np.full(a.shape[:-1] + (n,), np.float16(777.0).view(np.uint16), dtype=np.uint16)
        out[..., :a.shape[-1]] = a
        return np.ascontiguousarray(out)
    xhp, xlp, whp, wlp = pitched(xh, cpitch), pitched(xl, cpitch), pitched(wh, cpitch), pitched(wl, cpitch)
    M = B * H * W
    ld = Cout + 4
    z0 = rs.randn(M, ld).astype(np.float32) if acc else np.full((M, ld), 7.0, dtype=np.float32)
    z = z0.copy()
    st = np.full((ctas, 4 * Cout), 123.0, dtype=np.float32) if stats else None
    rc = emul.emul_conv_halo(P(xhp), P(xlp), P(whp), P(wlp), P(ax), P(aw), P(z), ld, B, H, W, Cin, cpitch, Cout, acc, ctas, P(st), flags)
    assert rc == 0, 'barrier deadlock in the kernel' if rc == -100 else rc
    ref = expected(xh, xl, wh, wl, ax, aw, 3, 3)
    got = z[:, :Cout].astype(np.float64) - (z0[:, :Cout] if acc else 0)
    err = np.linalg.norm(got - ref) / np.linalg.norm(ref)
    assert err < 2e-6, err
    assert np.array_equal(z[:, Cout:], z0[:, Cout:])      # columns beyond Cout are never written
    if stats:
        zz = z[:, :Cout].astype(np.float64)
        assert np.allclose(st[:, :Cout].astype(np.float64).sum(0), zz.sum(0), rtol=1e-5, atol=1e-4)
        assert np.allclose(st[:, Cout:2 * Cout].astype(np.float64).sum(0), (zz * zz).sum(0), rtol=1e-5, atol=1e-4)
        assert np.array_equal(st[:, 2 * Cout:3 * Cout].min(0), z[:, :Cout].min(0))
        assert np.array_equal(st[:, 3 * Cout:].max(0), z[:, :Cout].max(0))


def test_slow_epilogue(emul):
    """The producers run ahead of slow MMA warpgroups: they must wait for every MMA warp to release a stage."""
    emul.emul_set_ld_delay_us(20000)
    try:
        test_halo_kernel_control_flow(emul, *CASES[3])
    finally:
        emul.emul_set_ld_delay_us(0)


@pytest.mark.parametrize('case', [0, 2, 4, 5])
def test_three_mma_form(emul, case):
    """flags bit 2: the three separate MMAs per K step instead of the default pair A_hi * [B_hi | B_lo] (ONE MMA of width
    2*BN into the adjacent hi / lo accumulators) + A_lo * B_hi - same products."""
    test_halo_kernel_control_flow(emul, *CASES[case], flags=4)
