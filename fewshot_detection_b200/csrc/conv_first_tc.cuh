// First convolution block (3 or 3+1 input channels -> Cout <= 32, 3x3, BatchNorm, LeakyReLU, 2x2 max-pool) on the
// tensor cores WITHOUT ever storing its pre-BN output - included by conv_first_tc.cu after the PTX wrappers and by
// tools/host_emul/conv_first_tc_emul.cpp after functional models of them.
//
// Why: at 416x416 the first layer's pre-BN tensor z is the largest tensor of the network (64 x 173056 x 32 fp32 =
// 1.4 GB) while its input is 12 B per pixel.  Round 1 wrote z once and read it four more times (statistics, BN-apply,
// BN-backward reduce, BN-backward apply) plus a 1.4 GB dz round trip into the weight-gradient kernel: 4.5 ms of a
// 27 ms step for 1.6 % of its FLOPs.  Here every pass RECOMPUTES z from the input images with one small wgmma GEMM
// per 128-pixel tile (K = 9 taps x 4 channels = 36, padded to 48) and consumes it in the same kernel:
//   MODE 0  statistics   : per-channel sum / sum of squares / min / max of z           -> fsdet_bn_finalize
//   MODE 1  apply        : y = leaky(z*scale+shift), 2x2 max-pool -> pooled fp16 planes (and/or fp32) of the next layer
//   MODE 2  bwd reduce   : du = dy_pool routed to the arg-max pixel x leaky'; sum(du), sum(du*xhat), max|du|
//   MODE 3  bwd wgrad    : dz = scale*(du - c1 - xhat*c2) written to SHARED memory only and contracted with the same
//                          im2col tile by a second wgmma GEMM (pixels = K) into register accumulators that live for
//                          the whole CTA: dW partials per CTA, no dz in HBM at all.
// The recomputed z is bit-identical in all four passes (same tiles, same MMAs), so arg-max decisions agree.
//
// Tile: 8 rows x 16 columns = 128 pixels = 128 GEMM rows; warp q (0..3) owns the 4 x 8 sub-block of rows 32q..32q+31
// (lane l -> row l>>3, column l&7), so the four pixels of a pooling window are lanes l, l^1, l^8, l^9 of one warp.
// The accumulators come out of wgmma in its fragment layout and pass through a shared-memory tile to the thread that
// owns the pixel.
// Operand layout: A = im2col rows [pixel][64 halves] (128 B, 128-byte swizzle) as TWO fp16 planes (hi, lo) of the
// input scaled by a power of two; the forward GEMM reads them K-major, the weight-gradient GEMM reads the very same
// bytes MN-major with M = 128 = [hi plane | lo plane] (so the input stays exact to 22 bits and only dz is rounded to
// fp16 - the "x exact, dz rounded" weight-gradient mode).  B = weights [32][64] hi/lo.  Three forward terms
// (hi*hi + lo*hi + hi*lo) as everywhere else in the forward chain.
// Threads: warps 0-3 = one warpgroup, one thread per pixel (builds its im2col row, issues the wgmma GEMMs, owns its
// pixel's accumulator row), warp 4 = input staging (cp.async, one tile ahead).  Persistent CTAs walk the tile list.
// Registers: two CTAs per SM (launch bounds 160, 2) cap a thread at 168 registers.  Modes 0 and 1 fit (96 / 126); the
// backward modes hold z and du (32 channels each) and, in mode 3, the two 64 x 64 dW fragments (64 more) across the
// tile loop, and spill 58 (mode 2) / 64 (mode 3) bytes to the stack - L1-resident, and on an opt-in path.  One CTA per
// SM would remove the spill but halve the warps that hide the per-tile barriers.
#pragma once

constexpr int FT_TH = 8, FT_TW = 16;                        // tile rows x columns (128 pixels)
constexpr int FT_HW = FT_TW + 2, FT_HH = FT_TH + 2;         // with halo
constexpr int FT_HALO = FT_HH * FT_HW;                      // 180 pixels (float4 each)
constexpr int FT_PLANE = 128 * 128;                         // one A plane: 128 rows x 128 B
constexpr int FT_BPLANE = 32 * 128;                         // one B plane: 32 rows x 128 B
constexpr int FT_THREADS = 160;
constexpr int FT_ZLD = 33;                                  // row pitch (floats) of the z tile: conflict-free row reads

enum { FT_STATS = 0, FT_APPLY = 1, FT_BWD_REDUCE = 2, FT_BWD_WGRAD = 3 };

struct FtArgs {
    const float* in0; const float* in1;     // NCHW inputs [B][C0][H][W] (+ optional [B][C1][H][W]), C0 + C1 <= 4
    const float* w;                         // [Cout][9][4] fp32 (input channels zero padded to 4)
    const float* amax_x;                    // device scalar >= max |input|
    int C0, C1, B, H, W, Cout;
    // MODE 0
    float* stats;                           // [gridDim.x][4*Cout] = (sum | sum of squares | min | max)
    // MODE 1..3
    const float* scale; const float* shift; float slope;
    // MODE 1
    void* ph; void* pl; int cpad; const float* amax_y;   // pooled fp16 planes [B*Hp*Wp][cpad] (optional)
    float* yp; int ldp;                                  // pooled fp32 output (optional)
    // MODE 2, 3
    const float* dyp; int ld_dyp;           // gradient of the pooled output, fp32 [B*Hp*Wp][ld]
    const float* mean; const float* invstd;
    double* partial;                        // MODE 2: [gridDim.x][3*Cout] = (sum du | sum du*xhat | max |du|)
    const double* coef;                     // MODE 3: [2*Cout] = (c1 | c2)
    const float* amax_dz;                   // MODE 3: device scalar >= max |dz| (bound from fsdet_bn_bwd_finalize)
    float* dw_partial;                      // MODE 3: [gridDim.x][36 k][32 co] raw accumulator sums (operand scales not removed)
    int tiles_h, tiles_w, tiles;
};

template <int MODE>
struct FtCfg {
    static constexpr int OFF_AHI = 0;
    static constexpr int OFF_ALO = FT_PLANE;
    static constexpr int OFF_BHI = 2 * FT_PLANE;
    static constexpr int OFF_BLO = OFF_BHI + FT_BPLANE;
    static constexpr int OFF_DZ = OFF_BLO + FT_BPLANE;                              // MODE 3: [128 px][64 co] fp16
    static constexpr int OFF_EPI = OFF_DZ + (MODE == FT_BWD_WGRAD ? FT_PLANE : 0);  // 4 warps x 4 KB transposition tiles
    static constexpr int EPI_BYTES = (MODE == FT_STATS || MODE == FT_BWD_REDUCE) ? 4 * 4096 : 0;
    static constexpr int OFF_ZT = OFF_EPI + EPI_BYTES;                              // z tile [128 px][FT_ZLD] fp32
    static constexpr int OFF_HALO = OFF_ZT + 128 * FT_ZLD * 4;                      // [2][180] float4
    static constexpr int OFF_CONST = OFF_HALO + 2 * FT_HALO * 16;                   // 7 x 32 floats
    static constexpr int OFF_COMB = OFF_CONST + 7 * 32 * 4;                         // cross-warp combine: 4 x 32 x 32 B
    static constexpr int OFF_BAR = OFF_COMB + 4 * 32 * 32;
    static constexpr int SMEM_BYTES = OFF_BAR + 64 + 1024 /*align*/;
};

__device__ __forceinline__ float ft_leaky(float u, float slope) { return u > 0.f ? u : u * slope; }

__device__ __forceinline__ uint32_t ft_pack_h2(__half a, __half b) {
    return (uint32_t)__half_as_ushort(a) | ((uint32_t)__half_as_ushort(b) << 16);
}

// one 16-byte chunk of an im2col row: 8 values -> (hi, lo) fp16
__device__ __forceinline__ void ft_split8(const float (&f)[8], float sc, uint4& hi, uint4& lo) {
    uint32_t h[4], l[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float a = f[2 * i] * sc, b = f[2 * i + 1] * sc;
        const __half ha = __float2half_rn(a), hb = __float2half_rn(b);
        h[i] = ft_pack_h2(ha, hb);
        l[i] = ft_pack_h2(__float2half_rn(a - __half2float(ha)), __float2half_rn(b - __half2float(hb)));
    }
    hi = make_uint4(h[0], h[1], h[2], h[3]);
    lo = make_uint4(l[0], l[1], l[2], l[3]);
}

template <int MODE>
__global__ void __launch_bounds__(FT_THREADS, 2) conv_first_tc_kernel(const FtArgs p) {
    using Cfg = FtCfg<MODE>;
    FSDET_TC_DYN_SMEM(smem_raw);
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    float4* halo = reinterpret_cast<float4*>(smem + Cfg::OFF_HALO);
    float* cst = reinterpret_cast<float*>(smem + Cfg::OFF_CONST);     // x32: scale, shift, mean, invstd, c1 (hi), c2, c1 (lo)
    float* zt = reinterpret_cast<float*>(smem + Cfg::OFF_ZT);
    float* red = reinterpret_cast<float*>(smem + Cfg::OFF_BAR);       // small block reductions

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int HW = p.H * p.W;
    const int Hp = p.H >> 1, Wp = p.W >> 1;

    // ---- one-time set-up: zero the operand tiles (their padding chunks are never written again), weights, constants
    for (int i = tid; i < (Cfg::OFF_EPI) / 16; i += FT_THREADS) reinterpret_cast<uint4*>(smem)[i] = make_uint4(0, 0, 0, 0);
    float wmax = 0.f;
    for (int i = tid; i < p.Cout * 36; i += FT_THREADS) wmax = fmaxf(wmax, fabsf(ldg_f32(p.w + i)));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) wmax = fmaxf(wmax, __shfl_xor_sync(0xffffffffu, wmax, o));
    if (lane == 0) red[warp] = wmax;
    __syncthreads();
    wmax = fmaxf(fmaxf(red[0], red[1]), fmaxf(fmaxf(red[2], red[3]), red[4]));
    const float sw = scale_from_amax(wmax);
    const float sx = scale_from_amax(p.amax_x ? ldg_f32(p.amax_x) : 0.f);
    const float inv = 1.f / (sx * sw);
    // weights: row = output channel, chunk j = taps 2j, 2j+1 (4 channels each); k = tap*4 + c
    for (int i = tid; i < 32 * 5; i += FT_THREADS) {
        const int co = i / 5, j = i - co * 5;
        float f[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            const int k = j * 8 + e;
            f[e] = (co < p.Cout && k < 36) ? ldg_f32(p.w + co * 36 + k) : 0.f;
        }
        uint4 hi, lo;
        ft_split8(f, sw, hi, lo);
        const int off = co * 128 + ((j ^ (co & 7)) << 4);
        *reinterpret_cast<uint4*>(smem + Cfg::OFF_BHI + off) = hi;
        *reinterpret_cast<uint4*>(smem + Cfg::OFF_BLO + off) = lo;
    }
    if (MODE != FT_STATS) {
        for (int c = tid; c < 32; c += FT_THREADS) {
            const bool ok = c < p.Cout;
            cst[c] = ok ? ldg_f32(p.scale + c) : 0.f;
            cst[32 + c] = ok ? ldg_f32(p.shift + c) : 0.f;
            if (MODE >= FT_BWD_REDUCE) {
                cst[64 + c] = ok ? ldg_f32(p.mean + c) : 0.f;
                cst[96 + c] = ok ? ldg_f32(p.invstd + c) : 0.f;
            }
            if (MODE == FT_BWD_WGRAD) {
                // c1 = mean(du) as a (hi, lo) float pair: du - c1 cancels heavily when du is dominated by its mean
                const double c1 = ok ? p.coef[c] : 0.0;
                cst[128 + c] = (float)c1;
                cst[192 + c] = (float)(c1 - (double)(float)c1);
                cst[160 + c] = ok ? (float)p.coef[p.Cout + c] : 0.f;
            }
        }
    }

    // input tile (+halo) of tile t: 4-byte asynchronous copies, zero fill outside the image / beyond the channels
    auto stage = [&](int t, int buf) {
        const int tw = t % p.tiles_w;
        const int rest = t / p.tiles_w;
        const int th = rest % p.tiles_h;
        const int b = rest / p.tiles_h;
        const int h0 = th * FT_TH - 1, w0 = tw * FT_TW - 1;
        float* dst = reinterpret_cast<float*>(halo + buf * FT_HALO);
        for (int i = lane; i < FT_HALO * 4; i += 32) {
            const int ch = i & 3, px = i >> 2;
            const int hy = px / FT_HW, hx = px - hy * FT_HW;
            const int h = h0 + hy, w = w0 + hx;
            const float* plane = ch < p.C0 ? p.in0 + ((long long)b * p.C0 + ch) * HW
                                           : (ch < p.C0 + p.C1 ? p.in1 + ((long long)b * p.C1 + (ch - p.C0)) * HW : nullptr);
            const bool ok = plane != nullptr && h >= 0 && h < p.H && w >= 0 && w < p.W;
            cp_async4_zfill(dst + i, ok ? plane + (long long)h * p.W + w : p.in0, ok);
        }
    };

    // per-lane persistent accumulators of the reduction modes (lane = channel after the transposition)
    float s1 = 0.f, e1 = 0.f, s2 = 0.f, e2 = 0.f, vmin = INFINITY, vmax = -INFINITY;
    // MODE 3: dW^T accumulators [hi plane k 0..63 | lo plane k 0..63] x 64 co, one 64 x 64 wgmma fragment each
    float dwh[32], dwl[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) dwh[i] = dwl[i] = 0.f;
    const uint32_t sa = smem_u32(smem);

    if (warp == 4 && (int)blockIdx.x < p.tiles) stage(blockIdx.x, 0);
    unsigned it = 0;
    int buf = 0;
    for (int t = blockIdx.x; t < p.tiles; t += gridDim.x, ++it, buf ^= 1) {
        if (warp == 4) cp_async_wait_all();
        __syncthreads();                                   // S1: halo(t) landed; everyone is done with the previous tile
        const int tw = t % p.tiles_w;
        const int rest = t / p.tiles_w;
        const int th = rest % p.tiles_h;
        const int b = rest / p.tiles_h;
        int Y = 0, X = 0;                                  // this thread's pixel (warps 0-3)
        if (warp == 4) {
            if (t + (int)gridDim.x < p.tiles) stage(t + gridDim.x, buf ^ 1);
        } else {
            // ---- im2col row of this thread's pixel
            const int m = tid;
            const int ty = ((warp >> 1) << 2) + (lane >> 3), tx = ((warp & 1) << 3) + (lane & 7);
            Y = th * FT_TH + ty; X = tw * FT_TW + tx;
            const float4* hb = halo + buf * FT_HALO + ty * FT_HW + tx;
#pragma unroll
            for (int j = 0; j < 5; ++j) {
                float f[8];
                const int t0 = 2 * j, t1 = 2 * j + 1;
                const float4 a = hb[(t0 / 3) * FT_HW + (t0 % 3)];
                f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w;
                if (t1 < 9) {
                    const float4 c = hb[(t1 / 3) * FT_HW + (t1 % 3)];
                    f[4] = c.x; f[5] = c.y; f[6] = c.z; f[7] = c.w;
                } else {
                    f[4] = f[5] = f[6] = f[7] = 0.f;
                }
                uint4 hi, lo;
                ft_split8(f, sx, hi, lo);
                const int off = m * 128 + ((j ^ (m & 7)) << 4);
                *reinterpret_cast<uint4*>(smem + Cfg::OFF_AHI + off) = hi;
                *reinterpret_cast<uint4*>(smem + Cfg::OFF_ALO + off) = lo;
            }
            fence_proxy_async();
        }
        __syncthreads();                                   // S2: the A tile is complete
        if (warp < 4) {
            {
                // z = A * B^T: M = 128 (two 64-row halves), N = 32, K = 48 >= 36; both operands K-major, 128-byte swizzle
                float dh[2][16], dl[2][16];
                const uint64_t bhi = gmma_desc(sa + Cfg::OFF_BHI, 0, 1024, GMMA_SW128), blo = gmma_desc(sa + Cfg::OFF_BLO, 0, 1024, GMMA_SW128);
                wgmma_fence();
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const uint64_t ahi = gmma_desc(sa + Cfg::OFF_AHI + h * 64 * 128, 0, 1024, GMMA_SW128);
                    const uint64_t alo = gmma_desc(sa + Cfg::OFF_ALO + h * 64 * 128, 0, 1024, GMMA_SW128);
#pragma unroll
                    for (int k = 0; k < 3; ++k) {
                        const uint64_t adv = (uint64_t)(k * 32 >> 4);
                        wgmma<32>(dh[h], ahi + adv, bhi + adv, k > 0 ? 1u : 0u);
                        wgmma<32>(dl[h], alo + adv, bhi + adv, k > 0 ? 1u : 0u);
                        wgmma<32>(dl[h], ahi + adv, blo + adv, 1u);
                    }
                }
                wgmma_commit();
                wgmma_wait<0>();
                wgmma_use<16>(dh[0]); wgmma_use<16>(dh[1]); wgmma_use<16>(dl[0]); wgmma_use<16>(dl[1]);
                // fragment -> z tile (row = pixel): lo terms first, as (lo + hi) * inv
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int r0 = 64 * h + 16 * warp + (lane >> 2);
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const int c = 8 * j + 2 * (lane & 3);
                        zt[r0 * FT_ZLD + c] = (dl[h][4 * j] + dh[h][4 * j]) * inv;
                        zt[r0 * FT_ZLD + c + 1] = (dl[h][4 * j + 1] + dh[h][4 * j + 1]) * inv;
                        zt[(r0 + 8) * FT_ZLD + c] = (dl[h][4 * j + 2] + dh[h][4 * j + 2]) * inv;
                        zt[(r0 + 8) * FT_ZLD + c + 1] = (dl[h][4 * j + 3] + dh[h][4 * j + 3]) * inv;
                    }
                }
            }
            named_bar_sync(1, 128);
            float z[32];
#pragma unroll
            for (int c = 0; c < 32; ++c) z[c] = zt[tid * FT_ZLD + c];
            uint8_t* tb = smem + Cfg::OFF_EPI + warp * 4096;      // this warp's 32 x 32 transposition tile (modes 0, 2)

            if (MODE == FT_STATS) {
                __syncwarp();
#pragma unroll
                for (int j = 0; j < 8; ++j)
                    *reinterpret_cast<float4*>(tb + lane * 128 + ((j ^ (lane & 7)) << 4)) = make_float4(z[4 * j], z[4 * j + 1], z[4 * j + 2], z[4 * j + 3]);
                __syncwarp();
                float s = 0.f, q = 0.f;
#pragma unroll 8
                for (int rr = 0; rr < 32; ++rr) {
                    const float v = *reinterpret_cast<const float*>(tb + rr * 128 + ((((lane >> 2) ^ (rr & 7))) << 4) + (lane & 3) * 4);
                    s += v; q += v * v; vmin = fminf(vmin, v); vmax = fmaxf(vmax, v);
                }
                tc_kahan_add(s1, e1, s);
                tc_kahan_add(s2, e2, q);
            } else {
                // activation y and (modes 2, 3) the gradient du routed through leaky + max-pool
                const long long pp = ((long long)b * Hp + (Y >> 1)) * Wp + (X >> 1);
                const int wq = ((Y & 1) << 1) | (X & 1);       // position in the window, scan order
                float du[32];
                float dmax = 0.f;
#pragma unroll
                for (int c4 = 0; c4 < 8; ++c4) {
                    float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (MODE >= FT_BWD_REDUCE && 4 * c4 < p.Cout) g = ldg4(p.dyp + pp * p.ld_dyp + 4 * c4);
                    const float gv[4] = {g.x, g.y, g.z, g.w};
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const int c = 4 * c4 + e;
                        const float y = fmaf(z[c], cst[c], cst[32 + c]);
                        const float v = ft_leaky(y, p.slope);
                        const float v1 = __shfl_xor_sync(0xffffffffu, v, 1), v8 = __shfl_xor_sync(0xffffffffu, v, 8),
                                    v9 = __shfl_xor_sync(0xffffffffu, v, 9);
                        if (MODE == FT_APPLY) {
                            z[c] = fmaxf(fmaxf(v, v1), fmaxf(v8, v9));          // pooled activation (all four lanes hold it)
                        } else {
                            // first maximum in scan order (torch max_pool2d: strict >): earlier positions must be
                            // strictly smaller, later ones smaller or equal
                            const float o1 = v1, o2 = v8, o3 = v9;             // partners at wq^1, wq^2, wq^3
                            const bool b1 = ((wq ^ 1) < wq) ? (v > o1) : (v >= o1);
                            const bool b2 = ((wq ^ 2) < wq) ? (v > o2) : (v >= o2);
                            const bool b3 = ((wq ^ 3) < wq) ? (v > o3) : (v >= o3);
                            const float d = (b1 && b2 && b3) ? gv[e] * (y > 0.f ? 1.f : p.slope) : 0.f;
                            du[c] = d;
                            dmax = fmaxf(dmax, fabsf(d));
                        }
                    }
                }
                if (MODE == FT_APPLY) {
                    // the four lanes of a window share the stores: lane at window position wq writes channels [8wq, 8wq+8)
                    const float psc = p.ph ? scale_from_amax(ldg_f32(p.amax_y)) : 1.f;
                    float o[8];
#pragma unroll
                    for (int c = 0; c < 32; ++c)                      // select with constant indices (no local memory)
                        if ((c >> 3) == wq) o[c & 7] = z[c];
                    const int c0 = 8 * wq;
                    if (p.yp && c0 < p.Cout) {          // Cout % 4 == 0
                        *reinterpret_cast<float4*>(p.yp + pp * p.ldp + c0) = make_float4(o[0], o[1], o[2], o[3]);
                        if (c0 + 4 < p.Cout) *reinterpret_cast<float4*>(p.yp + pp * p.ldp + c0 + 4) = make_float4(o[4], o[5], o[6], o[7]);
                    }
                    if (p.ph) {
                        uint4 hi, lo;
                        ft_split8(o, psc, hi, lo);
                        __half* ph = reinterpret_cast<__half*>(p.ph) + pp * p.cpad;
                        __half* pl = reinterpret_cast<__half*>(p.pl) + pp * p.cpad;
                        *reinterpret_cast<uint4*>(ph + c0) = hi;      // channels >= Cout are exact zeros (zero weights / scale)
                        *reinterpret_cast<uint4*>(pl + c0) = lo;
                        for (int cz = 32 + c0; cz < p.cpad; cz += 32) {   // zero padding channels of the planes
                            *reinterpret_cast<uint4*>(ph + cz) = make_uint4(0, 0, 0, 0);
                            *reinterpret_cast<uint4*>(pl + cz) = make_uint4(0, 0, 0, 0);
                        }
                    }
                } else if (MODE == FT_BWD_REDUCE) {
                    // column sums of du and du*xhat over this warp's 32 pixels (two transpositions through shared memory)
                    float s = 0.f, q = 0.f;
#pragma unroll
                    for (int pass = 0; pass < 2; ++pass) {
                        __syncwarp();
#pragma unroll
                        for (int j = 0; j < 8; ++j) {
                            float4 v;
                            if (pass == 0) v = make_float4(du[4 * j], du[4 * j + 1], du[4 * j + 2], du[4 * j + 3]);
                            else v = make_float4(du[4 * j] * ((z[4 * j] - cst[64 + 4 * j]) * cst[96 + 4 * j]),
                                                 du[4 * j + 1] * ((z[4 * j + 1] - cst[64 + 4 * j + 1]) * cst[96 + 4 * j + 1]),
                                                 du[4 * j + 2] * ((z[4 * j + 2] - cst[64 + 4 * j + 2]) * cst[96 + 4 * j + 2]),
                                                 du[4 * j + 3] * ((z[4 * j + 3] - cst[64 + 4 * j + 3]) * cst[96 + 4 * j + 3]));
                            *reinterpret_cast<float4*>(tb + lane * 128 + ((j ^ (lane & 7)) << 4)) = v;
                        }
                        __syncwarp();
                        float acc = 0.f;
#pragma unroll 8
                        for (int rr = 0; rr < 32; ++rr)
                            acc += *reinterpret_cast<const float*>(tb + rr * 128 + ((((lane >> 2) ^ (rr & 7))) << 4) + (lane & 3) * 4);
                        if (pass == 0) s = acc; else q = acc;
                    }
                    tc_kahan_add(s1, e1, s);
                    tc_kahan_add(s2, e2, q);
                    vmax = fmaxf(vmax, dmax);      // max |du| over everything this lane saw (folded across lanes at the end)
                } else {                           // FT_BWD_WGRAD
                    const float dsc = scale_from_amax(ldg_f32(p.amax_dz));
                    const int m = tid;
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        float f[8];
#pragma unroll
                        for (int e = 0; e < 8; ++e) {
                            const int c = 8 * j + e;
                            const float xh = (z[c] - cst[64 + c]) * cst[96 + c];
                            f[e] = cst[c] * fmaf(-xh, cst[160 + c], (du[c] - cst[128 + c]) - cst[192 + c]);
                        }
                        uint4 hi, lo;
                        ft_split8(f, dsc, hi, lo);
                        *reinterpret_cast<uint4*>(smem + Cfg::OFF_DZ + m * 128 + ((j ^ (m & 7)) << 4)) = hi;
                    }
                    fence_proxy_async();
                    named_bar_sync(1, 128);                // the dz tile is complete
                    // dW^T[k][co] += sum_p A[p][k] * dz[p][co]: both operands MN-major (pixel = K), M = 64 per plane, N = 64
                    const uint64_t ah = gmma_desc(sa + Cfg::OFF_AHI, FT_PLANE, 1024, GMMA_SW128);
                    const uint64_t al = gmma_desc(sa + Cfg::OFF_ALO, FT_PLANE, 1024, GMMA_SW128);
                    const uint64_t bd = gmma_desc(sa + Cfg::OFF_DZ, FT_PLANE, 1024, GMMA_SW128);
                    wgmma_fence();
#pragma unroll
                    for (int k = 0; k < 8; ++k) {             // 8 x 16 pixels
                        const uint64_t adv = (uint64_t)(k * 2048 >> 4);
                        wgmma<64, 1, 1>(dwh, ah + adv, bd + adv, 1u);
                        wgmma<64, 1, 1>(dwl, al + adv, bd + adv, 1u);
                    }
                    wgmma_commit();
                    wgmma_wait<0>();                       // the A / dz tiles are rewritten by the next tile
                    wgmma_use<32>(dwh); wgmma_use<32>(dwl);
                }
            }
        }
    }

    // ---- CTA epilogue
    if (MODE == FT_STATS || MODE == FT_BWD_REDUCE) {
        float4* comb = reinterpret_cast<float4*>(smem + Cfg::OFF_COMB);     // [4 warps][32 channels]
        if (MODE == FT_BWD_REDUCE) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) vmax = fmaxf(vmax, __shfl_xor_sync(0xffffffffu, vmax, o));
        }
        __syncthreads();
        if (warp < 4) comb[warp * 32 + lane] = make_float4(s1 - e1, s2 - e2, vmin, vmax);
        __syncthreads();
        if (tid < 32 && tid < p.Cout) {
            float4 a = comb[tid];
            double ds = a.x, dq = a.y;
#pragma unroll
            for (int w = 1; w < 4; ++w) {
                const float4 o = comb[w * 32 + tid];
                ds += o.x; dq += o.y; a.z = fminf(a.z, o.z); a.w = fmaxf(a.w, o.w);
            }
            if (MODE == FT_STATS) {
                float* dst = p.stats + (long long)blockIdx.x * 4 * p.Cout + tid;
                dst[0] = (float)ds; dst[p.Cout] = (float)dq; dst[2 * p.Cout] = a.z; dst[3 * p.Cout] = a.w;
            } else {
                double* dst = p.partial + (long long)blockIdx.x * 3 * p.Cout + tid;
                dst[0] = ds; dst[p.Cout] = dq; dst[2 * p.Cout] = (double)fmaxf(a.w, 0.f);
            }
        }
    }
    if (MODE == FT_BWD_WGRAD && warp < 4) {
        // dW fragments: row = k (hi and lo plane rows of the same k sit in the same thread), column = co.  This CTA's
        // partial [k < 36][co < 32] (unscaled: the reduce kernel divides by the operand scales).
#pragma unroll
        for (int j = 0; j < 4; ++j) {                      // columns 0..31 = the output channels
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int k = 16 * warp + (lane >> 2) + 8 * h;
                const int co = 8 * j + 2 * (lane & 3);
                if (k < 36) {
                    float* dst = p.dw_partial + ((long long)blockIdx.x * 36 + k) * 32 + co;
                    *reinterpret_cast<float2*>(dst) = make_float2(dwh[4 * j + 2 * h] + dwl[4 * j + 2 * h],
                                                                  dwh[4 * j + 2 * h + 1] + dwl[4 * j + 2 * h + 1]);
                }
            }
        }
    }
}

// dw[co][k] = sum over CTAs (fixed order) of partial[cta][k][co] / (scale_x * scale_dz);  dw is [Cout][9][4]
__global__ void conv_first_tc_wgrad_reduce_kernel(const float* __restrict__ partial, int nparts, const float* __restrict__ amax_x,
                                                  const float* __restrict__ amax_dz, float* __restrict__ dw, int Cout) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= Cout * 36) return;
    const int co = i / 36, k = i - co * 36;
    double s = 0.0;
    for (int c = 0; c < nparts; ++c) s += (double)partial[((long long)c * 36 + k) * 32 + co];
    const float inv = 1.f / (scale_from_amax(amax_x ? ldg_f32(amax_x) : 0.f) * scale_from_amax(ldg_f32(amax_dz)));
    dw[i] = (float)(s * (double)inv);
}
