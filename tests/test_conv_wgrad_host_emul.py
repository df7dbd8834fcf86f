"""Control flow of the wgmma weight-gradient kernel (csrc/conv_wgrad_kernels.cuh) on the CPU: the kernel source is
compiled against functional models of its PTX wrappers (tools/host_emul/conv_wgrad_emul.cpp and tc_models_emul.h:
mbarrier phases and transaction counts, the 2-D tiled dz map and the 64-pixel im2col x map landing 128-byte swizzled,
wgmma reading both operands MN-major through the device descriptor encoding) and must reproduce every split-K slice of
the weight gradient on its own - two filter taps per N tile (with the clamped tail tap of an odd tap count, and the
duplicate of a 1x1 layer's only tap) and one, channel tiles half outside Cin, output-channel tiles half outside Cout,
64-pixel stages that straddle images, slices past the last pixel, and every operand-term mode.  A wrong barrier phase
deadlocks (-100 after a timeout); a filter offset outside the im2col window is reported as -101."""
import ctypes

import numpy as np
import pytest

from emul_util import build_emul
from test_conv_tc_host_emul import P, split_planes, scale_from_amax

WG_BP = 64


@pytest.fixture(scope='module')
def emul():
    return build_emul('conv_wgrad', 'conv_wgrad_kernels.cuh')


def pix_per_split(M, splits):
    """fsdet_conv_tc_wgrad: ceil(M / splits) rounded up to whole 64-pixel stages."""
    pps = -(-M // splits)
    return -(-pps // WG_BP) * WG_BP


def im2col(x, k):
    """x [B,H,W,C] -> [k*k, B*H*W, C]: tap t = (r, s) holds x[b, h + r - pad, w + s - pad] (zero outside)."""
    B, H, W, C = x.shape
    pad = (k - 1) // 2
    xp = np.zeros((B, H + 2 * pad, W + 2 * pad, C), dtype=x.dtype)
    xp[:, pad:pad + H, pad:pad + W] = x
    return np.stack([xp[:, r:r + H, s:s + W].reshape(B * H * W, C) for r in range(k) for s in range(k)])


def wgrad_ref(dz, cols, lo, hi):
    """float64 dw [Cout][k*k*Cin] over pixels lo..hi-1: dw[co][tap][ci] = sum_p dz[p][co] * cols[tap][p][ci]."""
    out = np.einsum('po,tpc->otc', dz[lo:hi], cols[:, lo:hi])
    return out.reshape(dz.shape[1], -1)


def expected_slices(xh, xl, dh, dl, ax, ad, B, H, W, k, terms, splits):
    """float64 of exactly the planes each term multiplies (bit 0 = dz_lo * x_hi, bit 1 = dz_hi * x_lo), unscaled, per
    split slice; and the whole-tensor value of the same terms."""
    Cin = xh.shape[-1]
    f = lambda u: u.view(np.float16).astype(np.float64)
    cxh = im2col(f(xh).reshape(B, H, W, Cin), k)
    cxl = im2col(f(xl).reshape(B, H, W, Cin), k) if terms & 2 else None
    Dh, Dl = f(dh), (f(dl) if terms & 1 else None)
    M = B * H * W
    inv = 1.0 / (scale_from_amax(ad[0]) * scale_from_amax(ax[0]))

    def ref(lo, hi):
        r = wgrad_ref(Dh, cxh, lo, hi)
        if terms & 1:
            r = r + wgrad_ref(Dl, cxh, lo, hi)
        if terms & 2:
            r = r + wgrad_ref(Dh, cxl, lo, hi)
        return r * inv
    pps = pix_per_split(M, splits)
    return [ref(min(z * pps, M), min((z + 1) * pps, M)) for z in range(splits)], ref(0, M)


CASES = [
    # B, H, W, Cin, Cout, k, terms, splits
    (2, 13, 13, 64, 128, 3, 3, 1),      # two taps per tile, 9 taps: tail tile = tap 8 + clamped duplicate; 169-pixel images
    (2, 13, 13, 64, 64, 1, 3, 3),       # 1x1: the only tap and its duplicate; three slices of 128, 128 and 82 pixels
    (2, 13, 13, 64, 128, 3, 2, 5),      # 128-pixel slices: the last two start past M = 338 (zero output)
    (1, 12, 12, 128, 192, 3, 0, 2),     # one tap per tile (Cin = 128), second co tile half outside Cout
    (1, 10, 10, 192, 64, 1, 1, 1),      # second channel tile half outside Cin: zero-filled loads, stores skipped
    (1, 9, 9, 192, 128, 3, 3, 2),       # 3x3 over a partial channel tile, M = 81: two slices of 64 and 17 pixels
    (3, 7, 7, 64, 192, 3, 1, 2),        # 49-pixel images: every stage straddles images; partial co tile, odd taps
    (2, 8, 8, 128, 64, 3, 2, 1),        # M = 128 (whole stages), terms 2: x_lo accumulates from the first stage
]


def run_case(emul, B, H, W, Cin, Cout, k, terms, splits):
    rs = np.random.RandomState(B * 1000 + H * 10 + Cin + Cout + k + terms + splits)
    M = B * H * W
    x = rs.randn(B, H, W, Cin).astype(np.float32)
    dz = (rs.randn(M, Cout) * 1e-3).astype(np.float32)
    xh, xl, ax, _ = split_planes(x)
    dh, dl, ad, _ = split_planes(dz)
    K = k * k * Cin
    out = np.full((splits, Cout, K), np.nan, dtype=np.float32)       # every element of every slice must be stored
    pps = pix_per_split(M, splits)
    rc = emul.emul_conv_wgrad(P(xh), P(xl), P(dh), P(dl), P(ax), P(ad), P(out), B, H, W, Cin, Cout, k, terms, splits,
                              ctypes.c_longlong(pps))
    assert rc == 0, {-100: 'barrier deadlock in the kernel', -101: 'im2col load outside the filter window'}.get(rc, rc)
    assert not np.isnan(out).any(), 'elements of the output never stored'
    refs, whole = expected_slices(xh, xl.copy(), dh, dl, ax, ad, B, H, W, k, terms, splits)
    for z in range(splits):
        got = out[z].astype(np.float64)
        if z * pps >= M:
            assert np.array_equal(out[z], np.zeros_like(out[z])), ('slice past the last pixel not zero', z)
            continue
        err = np.linalg.norm(got - refs[z]) / np.linalg.norm(refs[z])
        assert err < 2e-6, ('slice', z, err)
    tot = out.astype(np.float64).sum(0)
    assert np.linalg.norm(tot - whole) / np.linalg.norm(whole) < 2e-6


@pytest.mark.parametrize('B,H,W,Cin,Cout,k,terms,splits', CASES)
def test_wgrad_kernel_control_flow(emul, B, H, W, Cin, Cout, k, terms, splits):
    run_case(emul, B, H, W, Cin, Cout, k, terms, splits)


def test_split_counts_cover_empty_slices():
    """The split counts above include slices that start past the last pixel (the kernel's nk = 0 path)."""
    assert any(s * pix_per_split(B * H * W, s) - pix_per_split(B * H * W, s) >= B * H * W
               for B, H, W, _, _, _, _, s in CASES)


def test_slow_mma_does_not_lose_stages(emul):
    """With slow MMA warpgroups the producer laps them (six stages per CTA through a three-stage ring at terms = 3): it
    must wait until all eight MMA warps have released a stage before refilling it."""
    emul.emul_set_ld_delay_us(20000)
    try:
        run_case(emul, *CASES[0])
    finally:
        emul.emul_set_ld_delay_us(0)
