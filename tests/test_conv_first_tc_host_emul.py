"""The recomputing first-layer kernels (csrc/conv_first_tc.cuh: conv 3x3 + BatchNorm + LeakyReLU + max-pool in four
passes that never store the pre-BN tensor) on the CPU: the kernel source compiled against functional models of its
PTX wrappers (tools/host_emul/conv_first_tc_emul.cpp; the wgmma model reads the 128-byte-swizzled operand tiles the
kernel itself writes, K-major for the forward GEMM and MN-major for the weight-gradient GEMM) against numpy."""
import ctypes

import numpy as np
import pytest

from emul_util import build_emul


@pytest.fixture(scope='module')
def emul():
    return build_emul('conv_first_tc', 'conv_first_tc.cuh')


def P(a):
    return a.ctypes.data_as(ctypes.c_void_p) if a is not None else None


F = ctypes.c_float


def conv_ref(x, w):
    """x [B, C, H, W] float64, w [Cout, 9, 4] -> z [B, H, W, Cout] (3x3, pad 1)"""
    B, C, H, W = x.shape
    xp = np.zeros((B, 4, H + 2, W + 2))
    xp[:, :C, 1:-1, 1:-1] = x
    z = np.zeros((B, H, W, w.shape[0]))
    for t in range(9):
        r, s = divmod(t, 3)
        z += np.einsum('bchw,oc->bhwo', xp[:, :, r:r + H, s:s + W], w[:, t, :])
    return z


def leaky(v, slope):
    return np.where(v > 0, v, v * slope)


def scale_from_amax(a):
    m, ex = np.frexp(np.float32(a))
    return float(2.0 ** (10 - int(ex)))


def problem(B, C0, C1, H, W, Cout, seed):
    rs = np.random.RandomState(seed)
    x0 = rs.rand(B, C0, H, W).astype(np.float32)
    x1 = (rs.rand(B, C1, H, W) > 0.5).astype(np.float32) if C1 else None
    w = np.zeros((Cout, 9, 4), dtype=np.float32)
    w[:, :, :C0 + C1] = (rs.randn(Cout, 9, C0 + C1) * 0.3).astype(np.float32)
    x = np.concatenate([x0, x1], 1) if C1 else x0
    amax = np.array([np.abs(x).max()], dtype=np.float32)
    return x0, x1, x, w, amax


def call(emul, mode, ctas, x0, x1, w, amax, Cout, **kw):
    B, C0, H, W = x0.shape
    C1 = x1.shape[1] if x1 is not None else 0
    g = lambda k: kw.get(k)
    rc = emul.emul_conv_first_tc(mode, ctas, P(x0), C0, P(x1), C1, P(w), P(amax), B, H, W, Cout, P(g('stats')), P(g('scale')),
                                 P(g('shift')), F(kw.get('slope', 0.1)), P(g('ph')), P(g('pl')), kw.get('cpad', 0), P(g('amax_y')),
                                 P(g('yp')), kw.get('ldp', 0), P(g('dyp')), kw.get('ld_dyp', 0), P(g('mean')), P(g('invstd')),
                                 P(g('partial')), P(g('coef')), P(g('amax_dz')), P(g('dw_partial')))
    assert rc == 0, 'barrier deadlock / descriptor mismatch' if rc == -100 else rc


CASES = [(2, 3, 0, 16, 32, 32, 3), (1, 3, 1, 16, 16, 32, 2), (2, 3, 1, 8, 32, 8, 5), (1, 3, 0, 24, 16, 32, 1)]


@pytest.mark.parametrize('B,C0,C1,H,W,Cout,ctas', CASES)
def test_first_layer_passes(emul, B, C0, C1, H, W, Cout, ctas):
    x0, x1, x, w, amax = problem(B, C0, C1, H, W, Cout, B + H + Cout)
    z = conv_ref(x.astype(np.float64), w.astype(np.float64))                   # [B, H, W, Cout]
    # ---- pass 0: statistics
    stats = np.full((ctas, 4 * Cout), 77.0, dtype=np.float32)
    call(emul, 0, ctas, x0, x1, w, amax, Cout, stats=stats)
    zz = z.reshape(-1, Cout)
    assert np.allclose(stats[:, :Cout].astype(np.float64).sum(0), zz.sum(0), rtol=2e-5, atol=2e-4)
    assert np.allclose(stats[:, Cout:2 * Cout].astype(np.float64).sum(0), (zz * zz).sum(0), rtol=2e-5, atol=2e-4)
    assert np.allclose(stats[:, 2 * Cout:3 * Cout].min(0), zz.min(0), rtol=1e-5, atol=1e-5)
    assert np.allclose(stats[:, 3 * Cout:].max(0), zz.max(0), rtol=1e-5, atol=1e-5)
    # ---- pass 1: BN + leaky + pool -> fp32 and planes
    rs = np.random.RandomState(9)
    mean, var = zz.mean(0), zz.var(0)
    invstd = 1.0 / np.sqrt(var + 1e-5)
    gamma, beta = rs.rand(Cout) + 0.5, rs.randn(Cout) * 0.1
    scale = (gamma * invstd).astype(np.float32)
    shift = (beta - mean * gamma * invstd).astype(np.float32)
    y = leaky(z * scale.astype(np.float64) + shift.astype(np.float64), 0.1)
    Hp, Wp = H // 2, W // 2
    yp_ref = y.reshape(B, Hp, 2, Wp, 2, Cout).max(axis=(2, 4)).reshape(-1, Cout)
    amax_y = np.array([np.abs(y).max() * 1.0001], dtype=np.float32)
    cpad, ldp = 64, Cout + 4 if Cout % 8 else 36
    ldp = 36 if Cout == 32 else 12
    yp = np.full((B * Hp * Wp, ldp), 7.0, dtype=np.float32)
    ph = np.full((B * Hp * Wp, cpad), 0x7e00, dtype=np.uint16)
    pl = np.full((B * Hp * Wp, cpad), 0x7e00, dtype=np.uint16)
    call(emul, 1, ctas, x0, x1, w, amax, Cout, scale=scale, shift=shift, yp=yp, ldp=ldp, ph=ph, pl=pl, cpad=cpad, amax_y=amax_y)
    assert np.allclose(yp[:, :Cout], yp_ref, rtol=1e-5, atol=1e-5)
    assert np.all(yp[:, 32 if Cout == 32 else 8 * ((Cout + 7) // 8):] == 7.0)
    s = scale_from_amax(amax_y[0])
    planes = (ph.view(np.float16).astype(np.float64) + pl.view(np.float16).astype(np.float64)) / s
    assert np.allclose(planes[:, :Cout], yp_ref, rtol=2e-6, atol=1e-6)
    assert np.all(planes[:, 32:] == 0)                                       # padding channels zero filled
    assert np.array_equal(ph.view(np.float16)[:, :Cout], (yp[:, :Cout] * np.float32(s)).astype(np.float16))
    # ---- pass 2: backward reduce (du routed to the FIRST arg-max in scan order, times leaky')
    dyp = rs.randn(B * Hp * Wp, Cout).astype(np.float32)
    v = leaky(z * scale.astype(np.float64) + shift.astype(np.float64), 0.1).astype(np.float32)   # the kernel compares float32 values
    yv = (z * scale.astype(np.float64) + shift.astype(np.float64))
    win = v.reshape(B, Hp, 2, Wp, 2, Cout).transpose(0, 1, 3, 2, 4, 5).reshape(B, Hp, Wp, 4, Cout)
    arg = win.argmax(3)                                                      # first maximum
    du = np.zeros((B, Hp, Wp, 4, Cout))
    np.put_along_axis(du, arg[:, :, :, None, :], dyp.reshape(B, Hp, Wp, 1, Cout).astype(np.float64), 3)
    du = du.reshape(B, Hp, Wp, 2, 2, Cout).transpose(0, 1, 3, 2, 4, 5).reshape(B, H, W, Cout)
    du = du * np.where(yv > 0, 1.0, 0.1)
    xhat = (z - mean) * invstd
    partial = np.full((ctas, 3 * Cout), 5.0, dtype=np.float64)
    mean32, invstd32 = mean.astype(np.float32), invstd.astype(np.float32)
    call(emul, 2, ctas, x0, x1, w, amax, Cout, scale=scale, shift=shift, mean=mean32, invstd=invstd32, dyp=dyp, ld_dyp=Cout,
         partial=partial)
    assert np.allclose(partial[:, :Cout].sum(0), du.reshape(-1, Cout).sum(0), rtol=1e-4, atol=1e-4)
    assert np.allclose(partial[:, Cout:2 * Cout].sum(0), (du * xhat).reshape(-1, Cout).sum(0), rtol=1e-4, atol=2e-4)
    assert np.allclose(partial[:, 2 * Cout:].max(0), np.abs(du).reshape(-1, Cout).max(), rtol=1e-5) or \
        np.allclose(partial[:, 2 * Cout:].max(), np.abs(du).max(), rtol=1e-5)
    # ---- pass 3: weight gradient from dz formed on the fly
    n = B * H * W
    c1, c2 = du.reshape(-1, Cout).sum(0) / n, (du * xhat).reshape(-1, Cout).sum(0) / n
    dz = scale.astype(np.float64) * (du - c1 - xhat * c2)
    coef = np.concatenate([c1, c2]).astype(np.float64)
    amax_dz = np.array([np.abs(dz).max() * 1.3], dtype=np.float32)
    ws = np.full((ctas, 36, 32), 3.0, dtype=np.float32)
    call(emul, 3, ctas, x0, x1, w, amax, Cout, scale=scale, shift=shift, mean=mean32, invstd=invstd32, dyp=dyp, ld_dyp=Cout, coef=coef,
         amax_dz=amax_dz, dw_partial=ws)
    dw = ws.astype(np.float64).sum(0).T[:Cout] / (scale_from_amax(amax[0]) * scale_from_amax(amax_dz[0]))     # [Cout][36]
    xp = np.zeros((B, 4, H + 2, W + 2))
    xp[:, :x.shape[1], 1:-1, 1:-1] = x
    ref = np.zeros((Cout, 9, 4))
    for t in range(9):
        r, s_ = divmod(t, 3)
        ref[:, t, :] = np.einsum('bhwo,bchw->oc', dz, xp[:, :, r:r + H, s_:s_ + W])
    err = np.linalg.norm(dw - ref.reshape(Cout, 36)) / np.linalg.norm(ref)
    assert err < 1e-3, err            # x exact (hi + lo planes), dz rounded to fp16: the 2-term weight-gradient mode
