// wgmma implicit-GEMM convolution for sm_90a (forward, input gradient and weight gradient).
//
//   z[p][n] = sum_{tap,ci} x[p+tap][ci] * w[n][tap][ci]      (stride 1, "same" padding, k in {1,3})
//
// Tensor-core path of nn.Conv2d (darknet_meta.py:236-252) for every layer with Cin % 32 == 0.
//
// Precision: the reference is fp32 end to end and the parity bar is 1e-3 relative through a 23-layer
// train-mode-BN stack with max-pool / LeakyReLU kinks (every rounding error also flips arg-max decisions), which
// single-pass bf16/tf32 operands do not meet.  Operands are therefore split into two fp16 planes of the tensor
// scaled by a power of two so that its max lies in [512, 1024)  (hi = fp16(s*x), lo = fp16(s*x - hi): 22 mantissa
// bits in the same 4 B/element as fp32) and each K step issues three MMAs  Ahi*Bhi + Alo*Bhi + Ahi*Blo  into fp32
// register accumulators; on long K the hi*hi sums of every k-block are added to a register total with
// round-to-nearest, because the tensor core's fp32 accumulation truncates and its error grows with the number of
// accumulation steps.
//
// Structure (conv_tc_kernels.cuh): a producer warp fills a ring of shared-memory stages with TMA - A tiles straight
// from the NHWC activation planes through an *im2col* tensor map (128 consecutive output pixels x BK channels of one
// filter tap, zero-filled halo), B tiles from the [Cout][K] weight planes - in the swizzled K-major layout wgmma
// consumes; two MMA warpgroups (64 tile rows each) issue wgmma and run the epilogue from their registers.
#include <cuda.h>
#include <cuda_fp16.h>
#include <stdlib.h>

#include "common.cuh"

namespace fsdet {

#include "tc_ptx.cuh"   // scale_from_amax + the PTX wrappers

__global__ void __launch_bounds__(256) amax_kernel(const float* __restrict__ src, int ld, int C4, long long rows, float* __restrict__ out) {
    float m = 0.f;
    const unsigned n = (unsigned)rows * (unsigned)C4;   // host guarantees < 2^31
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const unsigned ru = i / (unsigned)C4;
        const long long r = ru;
        const int c = (int)(i - ru * (unsigned)C4) * 4;
        float4 v = ldg4(src + r * ld + c);
        m = fmaxf(m, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    __shared__ float red[8];
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < 8; ++w) m = fmaxf(m, red[w]);
        if (isfinite(m)) atomicMax(reinterpret_cast<int*>(out), __float_as_int(m));  // non-negative floats order as ints
    }
}

__global__ void __launch_bounds__(256) split_f16_kernel(const float* __restrict__ src, int ld, int C, int Cpad4, long long rows,
                                                        const float* __restrict__ amax, __half* __restrict__ hi,
                                                        __half* __restrict__ lo) {
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;   // host guarantees rows * Cpad4 < 2^31
    if (i >= (unsigned)rows * (unsigned)Cpad4) return;
    const float sc = amax ? scale_from_amax(__ldg(amax)) : 1.f;
    const unsigned ru = i / (unsigned)Cpad4;
    const long long r = ru;
    const int c = (int)(i - ru * (unsigned)Cpad4) * 4;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c < C) v = ldg4(src + r * ld + c);  // C % 4 == 0; channels C..Cpad-1 are zero filled
    float f[4] = {v.x * sc, v.y * sc, v.z * sc, v.w * sc};
    __half h[4], l[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        h[k] = __float2half_rn(f[k]);
        l[k] = __float2half_rn(f[k] - __half2float(h[k]));
    }
    long long o = r * (long long)(Cpad4 * 4) + c;
    *reinterpret_cast<uint2*>(hi + o) = *reinterpret_cast<uint2*>(h);
    *reinterpret_cast<uint2*>(lo + o) = *reinterpret_cast<uint2*>(l);
}

constexpr int TC_BK = 64;                       // halves per 128-byte row (im2col debug tile, weight-gradient tiles)
constexpr int TC_A_BYTES = 128 * TC_BK * 2;     // 16 KB per plane

#include "conv_tc_kernels.cuh"   // inside namespace fsdet
#include "conv_halo_kernels.cuh" // halo-tile flavour of the high-resolution 3x3 layers
#include "conv_wgrad_kernels.cuh" // weight gradient: TcWgArgs, WgCfg, wgrad_tc_kernel

__global__ void splitk_reduce4_kernel(const float4* __restrict__ ws, float4* __restrict__ out, long long n4, int splits) {
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n4) return;
    float4 s = ws[i];
    for (int k = 1; k < splits; ++k) {
        float4 v = ws[(long long)k * n4 + i];
        s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
    }
    out[i] = s;
}

// debug: dump one im2col A tile (un-swizzled) to global memory
__global__ void __launch_bounds__(128) debug_im2col_kernel(const __grid_constant__ CUtensorMap tmA, int H, int W, int pad, long long m0,
                                                           int c0, int tap, int ks, uint16_t* __restrict__ out) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint64_t* bar = reinterpret_cast<uint64_t*>(smem + TC_A_BYTES);
    if (threadIdx.x == 0) {
        mbar_init(bar, 1);
        fence_barrier_init();
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const int HW = H * W;
        const int img = (int)(m0 / HW);
        const int rem = (int)(m0 - (long long)img * HW);
        const int ph = rem / W, pw = rem - ph * W;
        mbar_expect_tx(bar, TC_A_BYTES);
        const int r = tap / ks, sx = tap - r * ks;
        tma_load_im2col_4d(smem, &tmA, bar, c0, pw - pad, ph - pad, img, (uint16_t)sx, (uint16_t)r);
    }
    mbar_wait(bar, 0);
    // row = threadIdx.x; un-swizzle: 16-byte chunk j of row r is stored at chunk (j ^ (r & 7))
    const int row = threadIdx.x;
    for (int j = 0; j < 8; ++j) {
        const uint4 v = *reinterpret_cast<const uint4*>(smem + row * 128 + ((j ^ (row & 7)) << 4));
        *reinterpret_cast<uint4*>(out + row * 64 + j * 8) = v;
    }
}

// ------------------------------------------------------------------ host side: tensor maps
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
typedef CUresult (*PFN_encodeIm2col)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                     const int*, const int*, cuuint32_t, cuuint32_t, const cuuint32_t*, CUtensorMapInterleave,
                                     CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// driver entry points, resolved once (thread-safe static initialisation, immutable afterwards)
struct DriverFns {
    PFN_encodeTiled encodeTiled = nullptr;
    PFN_encodeIm2col encodeIm2col = nullptr;
    bool ok = false;
};

static const DriverFns& driver_fns() {
    static const DriverFns fns = [] {
        DriverFns f;
        void* f1 = nullptr;
        void* f2 = nullptr;
        cudaDriverEntryPointQueryResult q;
        cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f1, cudaEnableDefault, &q);
        if (e != cudaSuccess || q != cudaDriverEntryPointSuccess || !f1) return f;
        e = cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &f2, cudaEnableDefault, &q);
        if (e != cudaSuccess || q != cudaDriverEntryPointSuccess || !f2) return f;
        f.encodeTiled = (PFN_encodeTiled)f1;
        f.encodeIm2col = (PFN_encodeIm2col)f2;
        f.ok = true;
        return f;
    }();
    return fns;
}

static int load_driver_fns() {
    if (!driver_fns().ok) {
        set_error("cuTensorMapEncodeTiled / cuTensorMapEncodeIm2col entry points unavailable");
        return -2;
    }
    return 0;
}

// activation plane [B][H][W][cpitch] fp16 (first C channels used) -> im2col map: `pixels` x `bk` channels per load
static int make_im2col_map(CUtensorMap* map, const void* base, int B, int H, int W, int C, int ks, int pixels, int cpitch = 0,
                           int bk = TC_BK) {
    if (cpitch == 0) cpitch = C;
    cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
    cuuint64_t strides[3] = {(cuuint64_t)cpitch * 2, (cuuint64_t)W * cpitch * 2, (cuuint64_t)H * W * cpitch * 2};
    const int pad = (ks - 1) / 2;
    int lower[2] = {-pad, -pad};
    int upper[2] = {pad - (ks - 1), pad - (ks - 1)};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = driver_fns().encodeIm2col(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(base), dims, strides, lower, upper,
                                (cuuint32_t)bk, (cuuint32_t)pixels, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                bk == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                                CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeIm2col failed (%d) for B=%d H=%d W=%d C=%d ks=%d", (int)r, B, H, W, C, ks);
        return -3;
    }
    // Driver quirk handled the same way by CUTLASS (copy_traits_sm90_im2col.hpp): for tensors smaller than
    // 128 KiB, drivers <= 13.1 set a bit that must be cleared.
    int drv = 0;
    cudaDriverGetVersion(&drv);
    if (drv <= 13010 && (size_t)B * H * W * cpitch * 2 < 131072) reinterpret_cast<uint64_t*>(map)[1] &= ~(1ull << 21);
    return 0;
}

// weight plane [rows][K] fp16 -> 2-D tiled map with box bk x box_rows
static int make_tiled_map(CUtensorMap* map, const void* base, long long rows, long long K, int box_rows, int bk = TC_BK) {
    cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)K * 2};
    cuuint32_t box[2] = {(cuuint32_t)bk, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = driver_fns().encodeTiled(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                               CU_TENSOR_MAP_INTERLEAVE_NONE, bk == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                               CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled failed (%d) rows=%lld K=%lld", (int)r, rows, K);
        return -3;
    }
    return 0;
}

// ---- tile plan of one convolution: which kernel flavour runs, its grid and the number of statistics rows
//   mode bits 0-1 = TERMS (operand precision, see conv_tc_kernels.cuh), bit 4 = persistent tile loop (short-K only)
struct TcPlan {
    int bn, bk, terms;
    bool fold;                       // long K: hi*hi k-blocks added to a register total (conv_tc_kernels.cuh)
    bool persist, cluster;
    int tiles_n, tiles_m, grid;      // tiles_m counts the padding tile of an odd tile count in cluster mode
    bool halo;                       // halo-tile kernel (conv_halo_kernels.cuh): 8 x 16 pixel tiles, persistent grid
    int tiles_x, tiles_y;
};

// The halo-tile kernel takes the 3x3 layers whose input tile is worth keeping in shared memory: 3-term arithmetic, at most
// 128 input and output channels (short K: the im2col kernel is L2-bound there), a width that tiles by 8, little padding
// waste in the 16-row direction and enough tiles to fill the persistent grid.  mode bit 6 switches it off.
static bool halo_ok(int B, int H, int W, int Cin, int Cout, int ksize, int mode) {
    if (ksize != 3 || (mode & 3) != 3 || (mode & 0x70)) return false;
    if (!(Cin == 32 || Cin == 64 || Cin == 128) || Cout > 128) return false;
    if (W % HALO_TW != 0) return false;
    const int ty = ceil_div(H, HALO_TH);
    if ((long long)ty * HALO_TH * 10 > (long long)H * 11) return false;          // more than 10 % of the MMA rows would be padding
    return (long long)B * ty * (W / HALO_TW) >= 2LL * kNumSMs;
}

static TcPlan tc_plan(long long M, int Cin, int Cout, int ksize, int mode, int B = 0, int H = 0, int W = 0) {
    TcPlan pl;
    pl.terms = mode & 3;
    pl.halo = B > 0 && halo_ok(B, H, W, Cin, Cout, ksize, mode);
    pl.tiles_x = pl.tiles_y = 0;
    if (pl.halo) {
        pl.bn = Cout <= 32 ? 32 : (Cout <= 64 ? 64 : 128);
        pl.bk = 32; pl.fold = false; pl.persist = true; pl.cluster = false;
        pl.tiles_n = 1;
        pl.tiles_x = W / HALO_TW;
        pl.tiles_y = ceil_div(H, HALO_TH);
        const long long total = (long long)B * pl.tiles_x * pl.tiles_y;
        pl.tiles_m = (int)total;
        pl.grid = (int)(total < kNumSMs ? total : kNumSMs);
        return pl;
    }
    // layers up to this K run the short-K flavour (64-byte rows, one accumulation chain).  FSDET_TC_SMALLK_MAX: developer knob for A/B runs
    static const int small_k_max = [] { const char* e = getenv("FSDET_TC_SMALLK_MAX"); return e ? atoi(e) : 2304; }();
    const bool small_k = (Cin % 64 != 0) || (ksize * ksize * Cin <= small_k_max);
    pl.bn = Cout >= 128 ? 128 : 64;
    pl.bk = small_k ? 32 : 64;
    pl.fold = !small_k;
    pl.persist = small_k && (mode & 16);
    pl.tiles_n = ceil_div(Cout, pl.bn);
    pl.tiles_m = ceil_div(M, TC_BM);
    pl.cluster = (mode & 32) && !pl.persist && pl.tiles_m >= 2;
    if (pl.cluster) pl.tiles_m = (pl.tiles_m + 1) / 2 * 2;      // CTA pairs: an odd tail gets an all-padding partner
    const long long total = (long long)pl.tiles_n * pl.tiles_m;
    if (pl.persist) {
        long long g = total < kNumSMs ? total : kNumSMs;
        g = g / pl.tiles_n * pl.tiles_n;          // every CTA keeps one channel range (statistics in registers)
        pl.grid = (int)(g < pl.tiles_n ? pl.tiles_n : g);
    } else {
        pl.grid = (int)total;
    }
    return pl;
}

template <int BN, int BK, int TERMS, bool PERSIST, bool FOLD>
static int launch_tc(const CUtensorMap& a_hi, const CUtensorMap& a_lo, const CUtensorMap& b_hi, const CUtensorMap& b_lo,
                     const TcArgs& a, int grid, bool cluster, cudaStream_t s) {
    using Cfg = TcCfg<BN, BK, TERMS, PERSIST>;
    if constexpr (!PERSIST) {
        if (cluster) {      // CTA pairs sharing the weight tile (TMA multicast)
            auto kern = conv_tc_kernel<BN, BK, TERMS, false, FOLD, 2>;
            cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES);
            if (e != cudaSuccess) {
                set_error("conv_tc(cluster): cudaFuncSetAttribute(%d bytes): %s", Cfg::SMEM_BYTES, cudaGetErrorString(e));
                return (int)e;
            }
            cudaLaunchConfig_t cfg = {};
            cfg.gridDim = dim3((unsigned)grid);
            cfg.blockDim = dim3(TC_THREADS);
            cfg.dynamicSmemBytes = Cfg::SMEM_BYTES;
            cfg.stream = s;
            cudaLaunchAttribute attr[1];
            attr[0].id = cudaLaunchAttributeClusterDimension;
            attr[0].val.clusterDim.x = 2;
            attr[0].val.clusterDim.y = 1;
            attr[0].val.clusterDim.z = 1;
            cfg.attrs = attr;
            cfg.numAttrs = 1;
            e = cudaLaunchKernelEx(&cfg, kern, a_hi, a_lo, b_hi, b_lo, a);
            if (e != cudaSuccess) {
                set_error("conv_tc(cluster): launch: %s", cudaGetErrorString(e));
                return (int)e;
            }
            return launch_status("conv_tc(cluster)");
        }
    }
    auto kern = conv_tc_kernel<BN, BK, TERMS, PERSIST, FOLD>;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES);
    if (e != cudaSuccess) {
        set_error("conv_tc: cudaFuncSetAttribute(%d bytes): %s", Cfg::SMEM_BYTES, cudaGetErrorString(e));
        return (int)e;
    }
    kern<<<grid, TC_THREADS, Cfg::SMEM_BYTES, s>>>(a_hi, a_lo, b_hi, b_lo, a);
    return launch_status(PERSIST ? "conv_tc(persistent)" : "conv_tc");
}

template <int BN, int BK, bool PERSIST, bool FOLD>
static int launch_tc_terms(int terms, const CUtensorMap& a_hi, const CUtensorMap& a_lo, const CUtensorMap& b_hi,
                           const CUtensorMap& b_lo, const TcArgs& a, int grid, bool cluster, cudaStream_t s) {
    switch (terms) {
        case 0: return launch_tc<BN, BK, 0, PERSIST, FOLD>(a_hi, a_lo, b_hi, b_lo, a, grid, cluster, s);
        case 1: return launch_tc<BN, BK, 1, PERSIST, FOLD>(a_hi, a_lo, b_hi, b_lo, a, grid, cluster, s);
        case 2: return launch_tc<BN, BK, 2, PERSIST, FOLD>(a_hi, a_lo, b_hi, b_lo, a, grid, cluster, s);
        default: return launch_tc<BN, BK, 3, PERSIST, FOLD>(a_hi, a_lo, b_hi, b_lo, a, grid, cluster, s);
    }
}

// ---- halo-tile flavour: tensor maps and launch
// activation plane [B][H][W][cpitch] fp16 -> tiled 4-D map, box = (32 channels, 8 x, 18 y) with zero fill outside
static int make_halo_act_map(CUtensorMap* map, const void* base, int B, int H, int W, int C, int cpitch) {
    cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
    cuuint64_t strides[3] = {(cuuint64_t)cpitch * 2, (cuuint64_t)W * cpitch * 2, (cuuint64_t)H * W * cpitch * 2};
    cuuint32_t box[4] = {32, (cuuint32_t)HALO_TW, (cuuint32_t)(HALO_TH + 2), 1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = driver_fns().encodeTiled(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(base), dims, strides, box, estr,
                                          CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("conv_halo: activation tensor map failed (%d) B=%d H=%d W=%d C=%d pitch=%d", (int)r, B, H, W, C, cpitch);
        return -3;
    }
    return 0;
}

template <int BN, int NCH>
static int launch_halo(const CUtensorMap& a_hi, const CUtensorMap& a_lo, const CUtensorMap& b_hi, const CUtensorMap& b_lo,
                       const HaloArgs& a, int grid, cudaStream_t s) {
    constexpr bool BRES = NCH * BN <= 64;          // the whole weight operand (9 * NCH blocks of BN x 64 B x 2 planes) stays in shared memory
    using Cfg = HaloCfg<BN, NCH, BRES>;
    auto kern = conv_halo_kernel<BN, NCH, BRES>;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES);
    if (e != cudaSuccess) {
        set_error("conv_halo: cudaFuncSetAttribute(%d bytes): %s", Cfg::SMEM_BYTES, cudaGetErrorString(e));
        return (int)e;
    }
    kern<<<grid, HALO_THREADS, Cfg::SMEM_BYTES, s>>>(a_hi, a_lo, b_hi, b_lo, a);
    return launch_status("conv_halo");
}

template <int BN>
static int launch_halo_nch(int nch, const CUtensorMap& a_hi, const CUtensorMap& a_lo, const CUtensorMap& b_hi, const CUtensorMap& b_lo,
                           const HaloArgs& a, int grid, cudaStream_t s) {
    switch (nch) {
        case 1: return launch_halo<BN, 1>(a_hi, a_lo, b_hi, b_lo, a, grid, s);
        case 2: return launch_halo<BN, 2>(a_hi, a_lo, b_hi, b_lo, a, grid, s);
        default: return launch_halo<BN, 4>(a_hi, a_lo, b_hi, b_lo, a, grid, s);
    }
}

static int run_halo(const void* x_hi, const void* x_lo, const void* w_hi, const void* w_lo, int B, const TcArgs& a, const TcPlan& pl,
                    cudaStream_t s) {
    CUtensorMap a_hi, a_lo, b_hi, b_lo;
    int rc = make_halo_act_map(&a_hi, x_hi, B, a.H, a.W, a.Cin, a.cpitch);
    if (rc) return rc;
    rc = make_halo_act_map(&a_lo, x_lo, B, a.H, a.W, a.Cin, a.cpitch);
    if (rc) return rc;
    const long long K = 9LL * a.cpitch;
    rc = make_tiled_map(&b_hi, w_hi, a.Cout, K, pl.bn, 32);
    if (rc) return rc;
    rc = make_tiled_map(&b_lo, w_lo, a.Cout, K, pl.bn, 32);
    if (rc) return rc;
    HaloArgs h;
    h.amax_a = a.amax_a; h.amax_b = a.amax_b; h.z = a.z; h.ldz = a.ldz; h.stats = a.stats; h.H = a.H; h.W = a.W; h.Cout = a.Cout; h.cpitch = a.cpitch;
    h.tiles_x = pl.tiles_x; h.tiles_y = pl.tiles_y; h.tiles_total = pl.tiles_m; h.accumulate = a.accumulate;
    const char* dbg = getenv("FSDET_HALO_FLAGS");      // developer knob (tools/halo_bench.py): see HaloArgs::flags
    h.flags = dbg ? atoi(dbg) : 0;
    const int nch = a.Cin / 32;
    if (pl.bn == 32) return launch_halo_nch<32>(nch, a_hi, a_lo, b_hi, b_lo, h, pl.grid, s);
    if (pl.bn == 64) return launch_halo_nch<64>(nch, a_hi, a_lo, b_hi, b_lo, h, pl.grid, s);
    return launch_halo_nch<128>(nch, a_hi, a_lo, b_hi, b_lo, h, pl.grid, s);
}

static int run_tc(const void* x_hi, const void* x_lo, const void* w_hi, const void* w_lo, int B, TcArgs a, int mode, cudaStream_t s) {
    const TcPlan pl = tc_plan(a.M, a.Cin, a.Cout, a.ks, mode, B, a.H, a.W);
    if (pl.halo) return run_halo(x_hi, x_lo, w_hi, w_lo, B, a, pl, s);
    CUtensorMap a_hi, a_lo, b_hi, b_lo;
    int rc = make_im2col_map(&a_hi, x_hi, B, a.H, a.W, a.Cin, a.ks, TC_BM, a.cpitch, pl.bk);
    if (rc) return rc;
    a_lo = a_hi;
    if (pl.terms & 1) {
        rc = make_im2col_map(&a_lo, x_lo, B, a.H, a.W, a.Cin, a.ks, TC_BM, a.cpitch, pl.bk);
        if (rc) return rc;
    }
    const long long K = (long long)a.ks * a.ks * a.cpitch;
    const int b_rows = pl.cluster ? pl.bn / 2 : pl.bn;      // cluster mode: each CTA of a pair loads half of the weight rows
    rc = make_tiled_map(&b_hi, w_hi, a.Cout, K, b_rows, pl.bk);
    if (rc) return rc;
    b_lo = b_hi;
    if (pl.terms & 2) {
        rc = make_tiled_map(&b_lo, w_lo, a.Cout, K, b_rows, pl.bk);
        if (rc) return rc;
    }
    a.tiles_n = pl.tiles_n;
    a.tiles_total = pl.tiles_n * pl.tiles_m;
    const int t = pl.terms;
    const bool cl = pl.cluster;
    if (pl.bk == 32) {
        if (pl.persist) {
            if (pl.bn == 128) return launch_tc_terms<128, 32, true, false>(t, a_hi, a_lo, b_hi, b_lo, a, pl.grid, false, s);
            return launch_tc_terms<64, 32, true, false>(t, a_hi, a_lo, b_hi, b_lo, a, pl.grid, false, s);
        }
        if (pl.bn == 128) return launch_tc_terms<128, 32, false, false>(t, a_hi, a_lo, b_hi, b_lo, a, pl.grid, cl, s);
        return launch_tc_terms<64, 32, false, false>(t, a_hi, a_lo, b_hi, b_lo, a, pl.grid, cl, s);
    }
    if (pl.bn == 128) return launch_tc_terms<128, 64, false, true>(t, a_hi, a_lo, b_hi, b_lo, a, pl.grid, cl, s);
    return launch_tc_terms<64, 64, false, true>(t, a_hi, a_lo, b_hi, b_lo, a, pl.grid, cl, s);
}

}  // namespace fsdet

using namespace fsdet;

extern "C" int fsdet_amax(const float* src, int ld, int C, size_t rows, float* amax_out, void* stream) {
    FSDET_CHECK_ARG(src && amax_out && C % 4 == 0 && ld % 4 == 0 && ld >= C && aligned16(src), "amax: C=%d ld=%d", C, ld);
    cudaStream_t s = (cudaStream_t)stream;
    cudaError_t e = cudaMemsetAsync(amax_out, 0, sizeof(float), s);
    if (e != cudaSuccess) { set_error("amax: memset: %s", cudaGetErrorString(e)); return (int)e; }
    long long n = (long long)rows * (C / 4);
    if (n == 0) return 0;
    FSDET_CHECK_ARG(n < (1ll << 31), "amax: tensor too large for 32-bit indexing");
    int blocks = ceil_div(n, 256 * 8);
    if (blocks > 4 * kNumSMs) blocks = 4 * kNumSMs;
    amax_kernel<<<blocks, 256, 0, s>>>(src, ld, C / 4, (long long)rows, amax_out);
    return launch_status("amax");
}

extern "C" int fsdet_split_f16(const float* src, int ld, int C, int Cpad, size_t rows, const float* amax, void* hi, void* lo,
                               void* stream) {
    FSDET_CHECK_ARG(src && hi && lo && C % 4 == 0 && ld % 4 == 0 && ld >= C && Cpad >= C && Cpad % 4 == 0,
                    "split_f16: C=%d Cpad=%d ld=%d", C, Cpad, ld);
    FSDET_CHECK_ARG(aligned16(src) && ((uintptr_t)hi % 8 == 0) && ((uintptr_t)lo % 8 == 0), "split_f16: alignment");
    long long n = (long long)rows * (Cpad / 4);
    if (n == 0) return 0;
    FSDET_CHECK_ARG(n < (1ll << 31), "split_f16: tensor too large for 32-bit indexing");
    split_f16_kernel<<<ceil_div(n, 256), 256, 0, (cudaStream_t)stream>>>(src, ld, C, Cpad / 4, (long long)rows, amax, (__half*)hi,
                                                                         (__half*)lo);
    return launch_status("split_f16");
}

extern "C" int fsdet_conv_tc_supported(int Cin, int Cout, int ksize) {
    return (Cin % 32 == 0) && (Cout >= 8) && (Cout % 4 == 0) && (ksize == 1 || ksize == 3);
}

extern "C" int fsdet_conv_tc_stat_rows(int B, int H, int W, int Cin, int Cout, int ksize, int mode) {
    const TcPlan pl = tc_plan((long long)B * H * W, Cin, Cout, ksize, mode, B, H, W);
    return pl.persist ? pl.grid / pl.tiles_n : pl.tiles_m;
}

extern "C" int fsdet_conv_tc_uses_halo(int B, int H, int W, int Cin, int Cout, int ksize, int mode) {
    return halo_ok(B, H, W, Cin, Cout, ksize, mode) ? 1 : 0;
}

extern "C" int fsdet_conv_tc_fwd(const void* x_hi, const void* x_lo, const void* w_hi, const void* w_lo, const float* amax_x,
                                 const float* amax_w, float* z, int ldz, int B, int H, int W, int Cin, int cpitch, int Cout,
                                 int ksize, int accumulate, int mode, float* stat_partial, void* stream) {
    const int terms = mode & 3;
    // bit 7 asks for three MMAs per K step, which every kernel issues: accepted so that callers setting it keep working
    FSDET_CHECK_ARG((mode & ~0xf3) == 0, "conv_tc_fwd: unknown mode bits 0x%x", mode);
    FSDET_CHECK_ARG(x_hi && w_hi && z && (!(terms & 1) || x_lo) && (!(terms & 2) || w_lo), "conv_tc_fwd: null pointer (mode %d)", mode);
    FSDET_CHECK_ARG(fsdet_conv_tc_supported(Cin, Cout, ksize) && cpitch >= Cin && cpitch % 8 == 0,
                    "conv_tc_fwd: unsupported Cin=%d (pitch %d) Cout=%d k=%d", Cin, cpitch, Cout, ksize);
    FSDET_CHECK_ARG(ldz % 4 == 0 && aligned16(z) && aligned16(x_hi) && aligned16(x_lo) && aligned16(w_hi) && aligned16(w_lo),
                    "conv_tc_fwd: alignment");
    FSDET_CHECK_ARG(!(stat_partial && accumulate), "conv_tc_fwd: statistics of an accumulated output are not defined");
    int rc = load_driver_fns();
    if (rc) return rc;
    TcArgs a;
    a.z = z; a.amax_a = amax_x; a.amax_b = amax_w; a.stats = stat_partial; a.ldz = ldz; a.H = H; a.W = W; a.Cin = Cin;
    a.Cout = Cout; a.ks = ksize; a.pad = (ksize - 1) / 2; a.cpitch = cpitch; a.M = (long long)B * H * W;
    a.accumulate = accumulate; a.tiles_n = a.tiles_total = 0;
    if (a.M == 0) return 0;
    FSDET_CHECK_ARG(a.M < (1ll << 31) - 256, "conv_tc_fwd: too many pixels");
    return run_tc(x_hi, x_lo, w_hi, w_lo, B, a, mode, (cudaStream_t)stream);
}

// tile shape of the weight-gradient kernel: 128-wide N tiles (two MMA warpgroups of 64 co x 128 keep a [hi | lo]
// accumulator and the hi total in registers); Cin <= 64 packs two filter taps into one tile
static inline int wg_taps(int Cin) { return Cin >= 128 ? 1 : 2; }
static inline int wg_cib(int Cin) { return WG_BN / wg_taps(Cin); }

// split-K factor of the weight gradient: every CTA is the same size (one CTA per SM), so the kernel takes
// ceil(tiles * splits / SMs) rounds of 1 / splits of the pixels each - pick the smallest split count within 3 % of the best
// rounds / splits ratio (265 CTAs on 132 SMs are three rounds, 264 are two; fewer splits = fewer partials to reduce)
static int wg_splits(long long M, int Cin, int Cout, int ks, int terms) {
    (void)terms;
    const int cib = wg_cib(Cin), taps = wg_taps(Cin);
    const long long tiles = (long long)((Cin + cib - 1) / cib) * ((ks * ks + taps - 1) / taps) * ((Cout + 127) / 128);
    long long maxs = (M + 511) / 512;  // at least 512 pixels (8 stages) per split
    if (maxs < 1) maxs = 1;
    if (maxs > 512) maxs = 512;
    const long long cap = (4LL * kNumSMs + tiles - 1) / tiles;      // beyond four rounds nothing is gained
    if (maxs > cap) maxs = cap;
    double best = 1e30;
    for (long long sp = 1; sp <= maxs; ++sp) {
        const double c = (double)((tiles * sp + kNumSMs - 1) / kNumSMs) / (double)sp;
        if (c < best) best = c;
    }
    for (long long sp = 1; sp <= maxs; ++sp) {
        const double c = (double)((tiles * sp + kNumSMs - 1) / kNumSMs) / (double)sp;
        if (c <= best * 1.03) return (int)sp;
    }
    return 1;
}

extern "C" int fsdet_conv_tc_wgrad_supported(int Cin, int Cout, int ksize) {
    return (Cin % 64 == 0) && (Cout % 64 == 0) && (ksize == 1 || ksize == 3);
}

extern "C" size_t fsdet_conv_tc_wgrad_workspace_floats(int B, int H, int W, int Cin, int Cout, int ksize, int mode) {
    int splits = wg_splits((long long)B * H * W, Cin, Cout, ksize, mode & 3);
    return splits > 1 ? (size_t)splits * Cout * ksize * ksize * Cin : 0;
}

template <int TAPS, int TERMS>
static int launch_wg(const CUtensorMap& dhi, const CUtensorMap& dlo, const CUtensorMap& xhi, const CUtensorMap& xlo,
                     const TcWgArgs& a, int splits, cudaStream_t s) {
    using Cfg = WgCfg<TERMS>;
    auto kern = wgrad_tc_kernel<TAPS, TERMS>;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES);
    if (e != cudaSuccess) {
        set_error("conv_tc_wgrad: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
        return (int)e;
    }
    constexpr int CIB = WG_BN / TAPS;
    dim3 grid(((a.Cin + CIB - 1) / CIB) * ((a.ks * a.ks + TAPS - 1) / TAPS), (a.Cout + 127) / 128, splits);
    kern<<<grid, 384, Cfg::SMEM_BYTES, s>>>(dhi, dlo, xhi, xlo, a);
    return launch_status("conv_tc_wgrad");
}

template <int TAPS>
static int launch_wg_terms(int terms, const CUtensorMap& dhi, const CUtensorMap& dlo, const CUtensorMap& xhi,
                           const CUtensorMap& xlo, const TcWgArgs& a, int splits, cudaStream_t s) {
    switch (terms) {
        case 0: return launch_wg<TAPS, 0>(dhi, dlo, xhi, xlo, a, splits, s);
        case 1: return launch_wg<TAPS, 1>(dhi, dlo, xhi, xlo, a, splits, s);
        case 2: return launch_wg<TAPS, 2>(dhi, dlo, xhi, xlo, a, splits, s);
        default: return launch_wg<TAPS, 3>(dhi, dlo, xhi, xlo, a, splits, s);
    }
}

extern "C" int fsdet_conv_tc_wgrad(const void* x_hi, const void* x_lo, const void* dz_hi, const void* dz_lo, const float* amax_x,
                                   const float* amax_dz, float* dw, float* workspace, size_t workspace_floats, int B, int H,
                                   int W, int Cin, int Cout, int ksize, int mode, void* stream) {
    const int terms = mode & 3;
    FSDET_CHECK_ARG((mode & ~3) == 0, "conv_tc_wgrad: unknown mode bits 0x%x", mode);
    FSDET_CHECK_ARG(x_hi && dz_hi && dw && (!(terms & 1) || dz_lo) && (!(terms & 2) || x_lo), "conv_tc_wgrad: null pointer (mode %d)", mode);
    FSDET_CHECK_ARG(fsdet_conv_tc_wgrad_supported(Cin, Cout, ksize), "conv_tc_wgrad: unsupported Cin=%d Cout=%d k=%d", Cin, Cout, ksize);
    FSDET_CHECK_ARG(aligned16(dw) && aligned16(x_hi) && aligned16(x_lo) && aligned16(dz_hi) && aligned16(dz_lo), "conv_tc_wgrad: alignment");
    int rc = load_driver_fns();
    if (rc) return rc;
    const long long M = (long long)B * H * W;
    FSDET_CHECK_ARG(M < (1ll << 31) - 256, "conv_tc_wgrad: too many pixels");
    const int splits = wg_splits(M, Cin, Cout, ksize, terms);
    const size_t need = splits > 1 ? (size_t)splits * Cout * ksize * ksize * Cin : 0;
    FSDET_CHECK_ARG(workspace_floats >= need && (need == 0 || (workspace && aligned16(workspace))),
                    "conv_tc_wgrad: workspace too small (%zu < %zu floats)", workspace_floats, need);
    TcWgArgs a;
    a.out = splits > 1 ? workspace : dw;
    a.amax_a = amax_dz; a.amax_b = amax_x;
    a.H = H; a.W = W; a.Cin = Cin; a.Cout = Cout; a.ks = ksize; a.pad = (ksize - 1) / 2; a.M = M;
    long long pps = (M + splits - 1) / splits;
    a.pix_per_split = (pps + WG_BP - 1) / WG_BP * WG_BP;
    CUtensorMap dhi, dlo, xhi, xlo;
    // dz planes [M][Cout] fp16: 2-D tiled map, box = 64 channels x 64 pixels
    {
        cuuint64_t dims[2] = {(cuuint64_t)Cout, (cuuint64_t)M};
        cuuint64_t strides[1] = {(cuuint64_t)Cout * 2};
        cuuint32_t box[2] = {64, (cuuint32_t)WG_BP};
        cuuint32_t estr[2] = {1, 1};
        for (int t = 0; t < 2; ++t) {
            if (t == 1 && !(terms & 1)) { dlo = dhi; break; }
            CUresult r = driver_fns().encodeTiled(t ? &dlo : &dhi, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2,
                                                  const_cast<void*>(t ? dz_lo : dz_hi), dims, strides, box, estr,
                                                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                                                  CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            if (r != CUDA_SUCCESS) {
                set_error("conv_tc_wgrad: cuTensorMapEncodeTiled failed (%d)", (int)r);
                return -3;
            }
        }
    }
    rc = make_im2col_map(&xhi, x_hi, B, H, W, Cin, ksize, WG_BP);
    if (rc) return rc;
    xlo = xhi;
    if (terms & 2) {
        rc = make_im2col_map(&xlo, x_lo, B, H, W, Cin, ksize, WG_BP);
        if (rc) return rc;
    }
    cudaStream_t s = (cudaStream_t)stream;
    if (wg_taps(Cin) == 2) {
        rc = launch_wg_terms<2>(terms, dhi, dlo, xhi, xlo, a, splits, s);
    } else {
        rc = launch_wg_terms<1>(terms, dhi, dlo, xhi, xlo, a, splits, s);
    }
    if (rc) return rc;
    if (splits > 1) {
        long long n4 = (long long)Cout * ksize * ksize * Cin / 4;
        splitk_reduce4_kernel<<<ceil_div(n4, 256), 256, 0, s>>>(reinterpret_cast<const float4*>(workspace),
                                                               reinterpret_cast<float4*>(dw), n4, splits);
        rc = launch_status("conv_tc_wgrad_reduce");
    }
    return rc;
}

extern "C" int fsdet_debug_im2col_tile(const void* x_plane, int B, int H, int W, int C, int ksize, long long m0, int c0, int tap,
                                       void* out_tile, void* stream) {
    int rc = load_driver_fns();
    if (rc) return rc;
    CUtensorMap m;
    rc = make_im2col_map(&m, x_plane, B, H, W, C, ksize, TC_BM);
    if (rc) return rc;
    debug_im2col_kernel<<<1, 128, TC_A_BYTES + 1024 + 64, (cudaStream_t)stream>>>(m, H, W, (ksize - 1) / 2, m0, c0, tap, ksize,
                                                                                 (uint16_t*)out_tile);
    return launch_status("debug_im2col_tile");
}
