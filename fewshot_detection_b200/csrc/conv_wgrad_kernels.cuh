// The wgmma weight-gradient kernel - included by conv_tc.cu after the PTX wrappers and conv_tc_kernels.cuh, and by
// tools/host_emul/conv_wgrad_emul.cpp after FUNCTIONAL MODELS of the same wrappers, which is how its control flow - split-K
// pixel ranges, tap pairs and the clamped tail tap, stage phases, the accumulate flags of the hi/lo terms and the fold
// into the register total - is tested on the CPU (tests/test_conv_wgrad_host_emul.py).
//
//   dw[co][tap][ci] = sum_p dz[p][co] * x[p + tap][ci]
// GEMM with the pixel index as K: both operands are "MN-major" in shared memory (a row = one pixel, 64 channels
// = 128 B), A = dz tile via a 2-D tiled map, B = x tile of ONE filter tap via the im2col map (zero-filled halo).
// One CTA = 128 co x BN ci x one tap over a range of pixels (split-K across blockIdx.z): a producer warp and two MMA
// warpgroups of 64 co each.  The hi*hi products of every 64-pixel stage are summed in a fresh accumulator and added to
// a register total (round-to-nearest: the tensor core's fp32 accumulation truncates, see conv_tc.cu).  That addition
// overlaps MMAs still in flight: TERMS = 0 alternates two hi accumulators (stage kb + 1 is issued before stage kb is
// added), the other modes issue the lo terms as a second wgmma group after the hi*hi group.  A stage is released one
// k-block late, once every group that read it is complete.
#pragma once

struct TcWgArgs {
    float* out;  // [splits][Cout][K]
    const float* amax_a;  // of dz
    const float* amax_b;  // of x
    int H, W, Cin, Cout, ks, pad;
    long long M;              // pixels
    long long pix_per_split;  // multiple of 64
};

constexpr int WG_BP = 64;                      // pixels per stage
constexpr int WG_BLK = WG_BP * 128;            // one [64 pixels][64 channels] fp16 block = 8 KB
constexpr int WG_BN = 128;                     // N tile: 1 or 2 filter taps x 128 or 64 input channels

// TERMS as in conv_tc_kernel (A = dz, B = x): bit 0 adds dz_lo * x_hi, bit 1 adds dz_hi * x_lo
template <int TERMS>
struct WgCfg {
    static constexpr int A_BYTES = 2 * WG_BLK;            // 128 co
    static constexpr int B_BYTES = (WG_BN / 64) * WG_BLK;
    static constexpr int NA = 1 + (TERMS & 1);
    static constexpr int NBP = 1 + ((TERMS >> 1) & 1);
    static constexpr int STAGE_BYTES = NA * A_BYTES + NBP * B_BYTES;
    static constexpr int OFF_ALO = A_BYTES;
    static constexpr int OFF_BHI = NA * A_BYTES;
    static constexpr int OFF_BLO = OFF_BHI + B_BYTES;
    static constexpr int BUDGET = 227 * 1024 - 1024 - 256;
    static constexpr int STAGES = (BUDGET / STAGE_BYTES) > 6 ? 6 : (BUDGET / STAGE_BYTES);
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 + 256;
    static_assert(STAGES >= 2, "at least two pipeline stages");
};

template <int TAPS, int TERMS>   // N tile = TAPS filter taps x (WG_BN / TAPS) input channels
__global__ void __launch_bounds__(384, 1)
wgrad_tc_kernel(const __grid_constant__ CUtensorMap tmDhi, const __grid_constant__ CUtensorMap tmDlo,
                const __grid_constant__ CUtensorMap tmXhi, const __grid_constant__ CUtensorMap tmXlo, const TcWgArgs p) {
    using Cfg = WgCfg<TERMS>;
    constexpr int STAGES = Cfg::STAGES;
    constexpr int BN = WG_BN;
    FSDET_TC_DYN_SMEM(smem_raw);
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * Cfg::STAGE_BYTES);
    uint64_t* empty_bar = full_bar + STAGES;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    constexpr int CIB = BN / TAPS;                      // input channels per tap in this tile (64 or 128)
    const int kk = p.ks * p.ks;
    const int ci_tiles = (p.Cin + CIB - 1) / CIB;
    const int tap0 = (blockIdx.x / ci_tiles) * TAPS;
    const int ci0 = (blockIdx.x - (blockIdx.x / ci_tiles) * ci_tiles) * CIB;
    const int co0 = blockIdx.y * 128;
    const long long pbeg = (long long)blockIdx.z * p.pix_per_split;
    long long pend = pbeg + p.pix_per_split;
    if (pend > p.M) pend = p.M;
    const int nk = pend > pbeg ? (int)((pend - pbeg + WG_BP - 1) / WG_BP) : 0;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmDhi);
        if (TERMS & 1) tma_prefetch_desc(&tmDlo);
        tma_prefetch_desc(&tmXhi);
        if (TERMS & 2) tma_prefetch_desc(&tmXlo);
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], 8);                // the 8 MMA warps
        }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp < 4) {
        regs_dec<40>();
        if (warp == 0) {                                // producer: whole warp converged, instructions under elect_one()
            const int HW = p.H * p.W;
#pragma unroll 1
            for (int kb = 0; kb < nk; ++kb) {
                const int s = kb % STAGES;
                mbar_wait_warp(&empty_bar[s], ((kb / STAGES) & 1) ^ 1);
                if (elect_one()) {
                    uint8_t* st = smem + s * Cfg::STAGE_BYTES;
                    mbar_expect_tx(&full_bar[s], Cfg::STAGE_BYTES);
                    const long long p0 = pbeg + (long long)kb * WG_BP;
                    const int img = (int)(p0 / HW);
                    const int rem = (int)(p0 - (long long)img * HW);
                    const int ph = rem / p.W, pw = rem - ph * p.W;
#pragma unroll
                    for (int j = 0; j < 2; ++j) {
                        tma_load_2d(st + j * WG_BLK, &tmDhi, &full_bar[s], co0 + 64 * j, (int)p0);
                        if (TERMS & 1) tma_load_2d(st + Cfg::OFF_ALO + j * WG_BLK, &tmDlo, &full_bar[s], co0 + 64 * j, (int)p0);
                    }
#pragma unroll
                    for (int j = 0; j < BN / 64; ++j) {
                        int tap = tap0 + (j * 64) / CIB;
                        if (tap >= kk) tap = kk - 1;      // tail group: duplicate load, its columns are not stored
                        const int r = tap / p.ks, sx = tap - r * p.ks;
                        const int ci = ci0 + (j * 64) % CIB;
                        tma_load_im2col_4d(st + Cfg::OFF_BHI + j * WG_BLK, &tmXhi, &full_bar[s], ci, pw - p.pad, ph - p.pad, img,
                                           (uint16_t)sx, (uint16_t)r);
                        if (TERMS & 2)
                            tma_load_im2col_4d(st + Cfg::OFF_BLO + j * WG_BLK, &tmXlo, &full_bar[s], ci, pw - p.pad, ph - p.pad, img,
                                               (uint16_t)sx, (uint16_t)r);
                    }
                }
                __syncwarp();
            }
        }
    } else {
        regs_inc<232>();
        const int cw = (warp >> 2) - 1;                 // MMA warpgroup: output channels co0 + 64 cw .. + 63
        const int wq = warp & 3;
        constexpr int NR = BN / 2;
        // TERMS != 0: [hi | lo].  TERMS = 0: two hi accumulators used in turn, so that k-block kb + 1 is in flight while
        // the sum of k-block kb is added to the total
        float acc[2 * NR];
        float tot[NR];
#pragma unroll
        for (int i = 0; i < NR; ++i) tot[i] = 0.f;
#pragma unroll
        for (int i = 0; i < 2 * NR; ++i) acc[i] = 0.f;
        const uint32_t smem_base = smem_u32(smem);
        // k-block kb: its hi*hi products into the fresh accumulator `hi` as one wgmma group, then (TERMS != 0) the lo terms
        // into acc[NR..] as a second group
        auto issue = [&](int kb, float* hi) {
            const int s = kb % STAGES;
            mbar_wait(&full_bar[s], (kb / STAGES) & 1);
            const uint32_t st = smem_base + s * Cfg::STAGE_BYTES;
            // MN-major, 128-byte swizzle: LBO = next 64-channel block, SBO = next group of 8 pixels
            const uint64_t ah = gmma_desc(st + cw * WG_BLK, WG_BLK, 1024, GMMA_SW128);
            const uint64_t al = ah + (uint64_t)(Cfg::OFF_ALO >> 4);
            const uint64_t bh = gmma_desc(st + Cfg::OFF_BHI, WG_BLK, 1024, GMMA_SW128);
            const uint64_t bl = bh + (uint64_t)(Cfg::B_BYTES >> 4);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < WG_BP / 16; ++k)        // 16 pixels = two 8-row groups of 1024 B
                wgmma<BN, 1, 1>(hi, ah + k * (2048 >> 4), bh + k * (2048 >> 4), k > 0 ? 1u : 0u);
            wgmma_commit();
            if (TERMS) {
#pragma unroll
                for (int k = 0; k < WG_BP / 16; ++k) {
                    const uint64_t adv = (uint64_t)(k * (2048 >> 4));
                    const uint32_t first_lo = (kb > 0 || k > 0) ? 1u : 0u;
                    if (TERMS & 1) wgmma<BN, 1, 1>(acc + NR, al + adv, bh + adv, first_lo);
                    if (TERMS & 2) wgmma<BN, 1, 1>(acc + NR, ah + adv, bl + adv, (TERMS & 1) ? 1u : first_lo);
                }
                wgmma_commit();
            }
        };
        auto fold = [&](float* hi) {                    // `hi` holds a completed k-block sum
            wgmma_use<NR>(hi);
#pragma unroll
            for (int i = 0; i < NR; ++i) tot[i] += hi[i];
        };
        auto release = [&](int kb) {                    // every group that read k-block kb's stage is complete
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[kb % STAGES]);
        };
        if (TERMS) {
#pragma unroll 1
            for (int kb = 0; kb < nk; ++kb) {
                issue(kb, acc);
                wgmma_wait<1>();                        // only this k-block's lo group may still run
                fold(acc);
                if (kb > 0) release(kb - 1);
            }
        } else {
#pragma unroll 1
            for (int kb = 0; kb < nk; kb += 2) {
                issue(kb, acc);
                if (kb > 0) {
                    wgmma_wait<1>();                    // k-block kb - 1 is complete
                    fold(acc + NR);
                    release(kb - 1);
                }
                if (kb + 1 < nk) {
                    issue(kb + 1, acc + NR);
                    wgmma_wait<1>();                    // k-block kb is complete
                    fold(acc);
                    release(kb);
                }
            }
        }
        wgmma_wait<0>();
        wgmma_use<2 * NR>(acc);
        if (nk > 0) {
            if (!TERMS) {                               // the last k-block's sum (even k-blocks use acc, odd ones acc + NR)
                if (nk & 1) fold(acc);
                else fold(acc + NR);
            }
            release(nk - 1);
        }
        const float inv = 1.f / (scale_from_amax(p.amax_a ? __ldg(p.amax_a) : 0.f) * scale_from_amax(p.amax_b ? __ldg(p.amax_b) : 0.f));
        const long long K = (long long)p.ks * p.ks * p.Cin;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int co = co0 + 64 * cw + 16 * wq + (lane >> 2) + 8 * h;
            if (co >= p.Cout) continue;
            float* orow = p.out + ((long long)blockIdx.z * p.Cout + co) * K;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
                const int n = 8 * j + 2 * (lane & 3);
                const int tap = tap0 + n / CIB;
                const int c = ci0 + n % CIB;
                if (tap < kk && c < p.Cin) {            // Cin % 64 == 0: c + 1 < Cin as well
                    const int e = 4 * j + 2 * h;
                    const float v0 = TERMS ? (acc[NR + e] + tot[e]) * inv : tot[e] * inv;
                    const float v1 = TERMS ? (acc[NR + e + 1] + tot[e + 1]) * inv : tot[e + 1] * inv;
                    *reinterpret_cast<float2*>(orow + (long long)tap * p.Cin + c) = make_float2(v0, v1);
                }
            }
        }
    }
}
