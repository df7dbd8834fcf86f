// The wgmma implicit-GEMM convolution kernel (forward and input gradient) - included by conv_tc.cu after the PTX
// wrappers, and by tools/host_emul/conv_tc_emul.cpp after FUNCTIONAL MODELS of the same wrappers (mbarrier, TMA,
// wgmma, named barriers as host code), which is how its control flow - barrier phases, tile sequencing, operand-term
// selection, the epilogue and the fused BatchNorm statistics - is tested on the CPU (tests/test_conv_tc_host_emul.py).
//
//   z[p][n] = sum_{tap,ci} x[p+tap][ci] * w[n][tap][ci]      (stride 1, "same" padding, k in {1,3})
//
// One CTA = three warpgroups (384 threads):
//   warpgroup 0   : TMA producer (one warp).  A tiles (128 output pixels x BK channels of one filter tap, zero-filled
//                   halo) come straight from the NHWC activation planes through an im2col tensor map, B tiles (BN output
//                   channels x BK) from the [Cout][K] weight planes; both land swizzled K-major in shared memory.
//   warpgroups 1-2: MMA + epilogue, 64 tile rows each.  wgmma reads both operands from shared memory and accumulates in
//                   registers; the epilogue scales the accumulators, stores z rows (adds to them when accumulating) and -
//                   for BatchNorm layers - folds the per-channel sum / sum of squares / min / max of z into one partial
//                   row per CTA (fsdet_bn_finalize reads them), so that no separate statistics pass over z exists.
//   Producer registers are handed to the MMA warpgroups (setmaxnreg).
//
// Operand precision (template parameter TERMS): every operand exists as two fp16 planes (hi, lo) of the tensor
// scaled by a power of two; hi*hi is always issued, bit 0 of TERMS adds A_lo*B_hi, bit 1 adds A_hi*B_lo.  TERMS = 3
// is fp32-grade (22 mantissa bits per operand), TERMS = 1 / 2 keep one operand exact and round the other to fp16
// (relative rounding 2^-12 per element), TERMS = 0 is plain fp16 x fp16 -> fp32.  Only the planes that are used are
// loaded.  FOLD (long K): the tensor core's fp32 accumulation truncates, so the hi*hi products of every k-block are
// summed in a fresh accumulator and added to a register total with round-to-nearest; the small lo terms accumulate
// over the whole K.
//
// Every MMA of a K step has the width BN and writes registers no other MMA of the same group writes at the same time
// (a wider A_hi * [B_hi | B_lo] followed by A_lo * B_hi into half of its registers makes ptxas serialise every wgmma of
// the kernel).  One wgmma group stays in flight across k-blocks: the short-K flavour issues one group per k-block and
// waits for the previous one; the FOLD flavour issues the hi*hi group and then the lo group of a k-block, so that
// wait<1> completes the hi group and its sum is added to the total while the lo MMAs still run.  A stage is released
// once every group that read it is complete, i.e. one k-block late.
//
// PERSIST = false: one output tile per CTA (grid = number of tiles).
// PERSIST = true : CTAs walk tiles blockIdx.x, blockIdx.x + gridDim.x, ...; the producer runs ahead across tile
//              boundaries.  gridDim.x must be a multiple of tiles_n (then every CTA keeps one channel range: the
//              statistics are carried in registers across its tiles and written once).
#pragma once

#ifdef FSDET_HOST_EMULATION
#define FSDET_TC_DYN_SMEM(name) uint8_t* name = emul::g_dyn_smem
#else
#define FSDET_TC_DYN_SMEM(name) extern __shared__ uint8_t name[]
#endif

struct TcArgs {
    float* z;
    const float* amax_a;
    const float* amax_b;
    float* stats;     // optional [rows][4*Cout] = (sum | sum of squares | min | max), row = blockIdx.x / tiles_n
    int ldz;
    int H, W, Cin, Cout, ks, pad;
    int cpitch;       // channel pitch of the weight planes' K axis: k = tap * cpitch + c
    long long M;      // B*H*W
    int accumulate;
    int tiles_n, tiles_total;
};

constexpr int TC_BM = 128;
constexpr int TC_THREADS = 384;   // producer warpgroup + two MMA warpgroups

constexpr int tc_max(int a, int b) { return a > b ? a : b; }

template <int BN, int BK, int TERMS, bool PERSIST>
struct TcCfg {
    static constexpr int ROW_BYTES = BK * 2;
    static constexpr int A_BYTES = TC_BM * ROW_BYTES;
    static constexpr int B_BYTES = BN * ROW_BYTES;
    static constexpr int NA = 1 + (TERMS & 1);
    static constexpr int NBP = 1 + ((TERMS >> 1) & 1);
    static constexpr int STAGE_BYTES = NA * A_BYTES + NBP * B_BYTES;
    static constexpr int OFF_ALO = A_BYTES;
    static constexpr int OFF_BHI = NA * A_BYTES;
    static constexpr int OFF_BLO = OFF_BHI + B_BYTES;
    static constexpr int STAT_BYTES = 8 * BN * 16;                  // 8 MMA warps x BN channels x float4
    static constexpr int BUDGET = 227 * 1024 - 1024 /*align*/ - 256 /*barriers*/;
    static constexpr int STAGES = ((BUDGET - STAT_BYTES) / STAGE_BYTES) > 8 ? 8 : ((BUDGET - STAT_BYTES) / STAGE_BYTES);
    static constexpr int STAT_OFF = STAGES * STAGE_BYTES;
    static constexpr int BAR_OFF = STAT_OFF + STAT_BYTES;
    static constexpr int SMEM_BYTES = BAR_OFF + 1024 + 256;
    static_assert(STAGES >= 2, "at least two pipeline stages");
    static_assert(STAGE_BYTES % 1024 == 0 && A_BYTES % 1024 == 0 && B_BYTES % 1024 == 0, "swizzle atoms need 1 KB alignment");
};

// compensated fp32 accumulation (the statistics of a persistent CTA run over thousands of pixels)
__device__ __forceinline__ void tc_kahan_add(float& s, float& e, float x) {
    const float y = x - e;
    const float t = s + y;
    e = (t - s) - y;
    s = t;
}

// dynamic shared memory aligned to 1 KB WITHOUT leaving the shared address space (a round trip through uintptr_t makes
// every later access a generic LD / ST)
__device__ __forceinline__ uint8_t* tc_align_smem(uint8_t* raw) { return raw + ((1024u - (smem_u32(raw) & 1023u)) & 1023u); }

// ---- epilogue (shared with conv_halo_kernels.cuh).  One MMA warp holds 16 rows x N columns of the accumulator in the
// wgmma fragment layout: lane l has rows l / 4 and l / 4 + 8, columns 8j + 2 (l % 4) + {0, 1}.  z0 / z1 point at the
// output rows of those two rows (nullptr: the row lies outside the tensor), cvalid = output channels left in this tile.
// The values are scaled, stored as float2 (added to z when accumulating) and - with `wstat` - the column statistics of
// the warp's valid rows go to wstat[0..N) (lanes with the same l % 4 combined by shuffles).
template <int N, bool HAS_LO>
__device__ __forceinline__ void epi_tile(const float* hi, const float* lo, float inv, float* z0, float* z1, int cvalid, int accumulate,
                                         float4* wstat) {
    const int lane = threadIdx.x & 31;
    const bool ok0 = z0 != nullptr, ok1 = z1 != nullptr;
#pragma unroll
    for (int j = 0; j < N / 8; ++j) {
        const int c = 8 * j + 2 * (lane & 3);
        float v[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) v[e] = HAS_LO ? (lo[4 * j + e] + hi[4 * j + e]) * inv : hi[4 * j + e] * inv;
        if (c < cvalid) {
            if (ok0) {
                float2* o = reinterpret_cast<float2*>(z0 + c);
                float2 w = make_float2(v[0], v[1]);
                if (accumulate) { const float2 u = *o; w.x += u.x; w.y += u.y; }
                *o = w;
            }
            if (ok1) {
                float2* o = reinterpret_cast<float2*>(z1 + c);
                float2 w = make_float2(v[2], v[3]);
                if (accumulate) { const float2 u = *o; w.x += u.x; w.y += u.y; }
                *o = w;
            }
        }
        if (wstat) {
            float t[8];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const float a = v[e], b = v[2 + e];
                t[4 * e + 0] = (ok0 ? a : 0.f) + (ok1 ? b : 0.f);
                t[4 * e + 1] = (ok0 ? a * a : 0.f) + (ok1 ? b * b : 0.f);
                t[4 * e + 2] = fminf(ok0 ? a : INFINITY, ok1 ? b : INFINITY);
                t[4 * e + 3] = fmaxf(ok0 ? a : -INFINITY, ok1 ? b : -INFINITY);
            }
#pragma unroll
            for (int o = 4; o < 32; o <<= 1) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    t[4 * e + 0] += __shfl_xor_sync(0xffffffffu, t[4 * e + 0], o);
                    t[4 * e + 1] += __shfl_xor_sync(0xffffffffu, t[4 * e + 1], o);
                    t[4 * e + 2] = fminf(t[4 * e + 2], __shfl_xor_sync(0xffffffffu, t[4 * e + 2], o));
                    t[4 * e + 3] = fmaxf(t[4 * e + 3], __shfl_xor_sync(0xffffffffu, t[4 * e + 3], o));
                }
            }
            if (lane < 4) {
                wstat[c] = make_float4(t[0], t[1], t[2], t[3]);
                wstat[c + 1] = make_float4(t[4], t[5], t[6], t[7]);
            }
        }
    }
}

// statistics of one tile: the 8 MMA warps' column partials (sstat[warp][BN], written by epi_tile) folded in a fixed order
// by consumer thread `ct` (< BN) into its compensated running sums; barrier 1 spans the 256 MMA threads
template <int BN>
__device__ __forceinline__ void epi_fold_stats(const float4* sstat, int ct, float& ssum, float& esum, float& ssq, float& esq,
                                               float& smin, float& smax) {
    named_bar_sync(1, 256);
    if (ct < BN) {
        float4 tt = sstat[ct];
#pragma unroll
        for (int w = 1; w < 8; ++w) {
            const float4 o = sstat[w * BN + ct];
            tt.x += o.x; tt.y += o.y; tt.z = fminf(tt.z, o.z); tt.w = fmaxf(tt.w, o.w);
        }
        tc_kahan_add(ssum, esum, tt.x);
        tc_kahan_add(ssq, esq, tt.y);
        smin = fminf(smin, tt.z);
        smax = fmaxf(smax, tt.w);
    }
    named_bar_sync(1, 256);     // sstat is rewritten by the next tile
}

// CLUSTER = 2 (one-tile-per-CTA flavours only): two CTAs of a thread-block cluster work on two M tiles of the SAME
// channel range; each loads its own activation tiles and only HALF of the weight tile, multicast into both CTAs'
// shared memory - the weight operand crosses the L2 -> SM fabric once per pair instead of once per CTA.  A stage may be
// refilled once BOTH CTAs' MMA warps have consumed it (its empty barrier counts the arrivals of both CTAs).
template <int BN, int BK, int TERMS, bool PERSIST, bool FOLD, int CLUSTER = 1>
__global__ void __launch_bounds__(TC_THREADS, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap tmAhi, const __grid_constant__ CUtensorMap tmAlo,
               const __grid_constant__ CUtensorMap tmBhi, const __grid_constant__ CUtensorMap tmBlo, const TcArgs p) {
    using Cfg = TcCfg<BN, BK, TERMS, PERSIST>;
    constexpr int STAGES = Cfg::STAGES;
    FSDET_TC_DYN_SMEM(smem_raw);
    uint8_t* smem = tc_align_smem(smem_raw);
    float4* sstat = reinterpret_cast<float4*>(smem + Cfg::STAT_OFF);   // [8 MMA warps][BN]
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + Cfg::BAR_OFF);
    uint64_t* empty_bar = full_bar + STAGES;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int kchunks = p.Cin / BK;
    const int nk = p.ks * p.ks * kchunks;
    static_assert(CLUSTER == 1 || (CLUSTER == 2 && !PERSIST), "the cluster flavour is one tile per CTA");
    const int tiles_n = p.tiles_n;
    const int tiles_total = p.tiles_total;
    const int tile_step = PERSIST ? (int)gridDim.x : tiles_total;   // non-persistent: exactly one tile per CTA
    // CLUSTER == 2: CTAs 2c and 2c+1 take M tiles 2m and 2m+1 of channel range n (gridDim.x = 2 * tiles_n * ceil(tiles_m / 2))
    const uint32_t crank = CLUSTER == 2 ? cluster_ctarank() : 0u;
    const int first_tile = CLUSTER == 2 ? (((int)(blockIdx.x >> 1) / tiles_n) * 2 + (int)crank) * tiles_n + (int)(blockIdx.x >> 1) % tiles_n
                                        : (int)blockIdx.x;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmAhi);
        if (TERMS & 1) tma_prefetch_desc(&tmAlo);
        tma_prefetch_desc(&tmBhi);
        if (TERMS & 2) tma_prefetch_desc(&tmBlo);
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], 8 * CLUSTER);     // every MMA warp of every CTA that reads the stage
        }
        fence_barrier_init();
    }
    __syncthreads();
    if (CLUSTER == 2) cluster_sync_all();                      // the peer's barriers exist before anything remote touches them

    if (warp < 4) {
        regs_dec<40>();
        if (warp == 0) {
            // the producer warp runs converged and issues under elect_one() (tc_ptx.cuh)
            const int HW = p.H * p.W;
            unsigned it = 0;                                   // k-blocks issued so far (all tiles)
            for (int tile = first_tile; tile < tiles_total; tile += tile_step) {
                const int n_tile = tile % tiles_n;
                const long long m0 = (long long)(tile / tiles_n) * TC_BM;
                const int img = (int)(m0 / HW);
                const int rem = (int)(m0 - (long long)img * HW);
                const int ph = rem / p.W, pw = rem - ph * p.W;
#pragma unroll 1
                for (int kb = 0; kb < nk; ++kb, ++it) {
                    const int s = it % STAGES;
                    mbar_wait_warp(&empty_bar[s], ((it / STAGES) & 1) ^ 1);
                    if (elect_one()) {
                        uint8_t* st = smem + s * Cfg::STAGE_BYTES;
                        mbar_expect_tx(&full_bar[s], Cfg::STAGE_BYTES);
                        const int tap = kb / kchunks;
                        const int c0 = (kb - tap * kchunks) * BK;
                        const int r = tap / p.ks, sx = tap - r * p.ks;
                        tma_load_im2col_4d(st, &tmAhi, &full_bar[s], c0, pw - p.pad, ph - p.pad, img, (uint16_t)sx, (uint16_t)r);
                        if (TERMS & 1)
                            tma_load_im2col_4d(st + Cfg::OFF_ALO, &tmAlo, &full_bar[s], c0, pw - p.pad, ph - p.pad, img, (uint16_t)sx,
                                               (uint16_t)r);
                        if (CLUSTER == 2) {       // my half of the weight rows, delivered to both CTAs of the pair
                            const int half = (int)crank * (BN / 2);
                            tma_load_2d_mc(st + Cfg::OFF_BHI + half * Cfg::ROW_BYTES, &tmBhi, &full_bar[s], tap * p.cpitch + c0,
                                           n_tile * BN + half, (uint16_t)3);
                            if (TERMS & 2)
                                tma_load_2d_mc(st + Cfg::OFF_BLO + half * Cfg::ROW_BYTES, &tmBlo, &full_bar[s], tap * p.cpitch + c0,
                                               n_tile * BN + half, (uint16_t)3);
                        } else {
                            tma_load_2d(st + Cfg::OFF_BHI, &tmBhi, &full_bar[s], tap * p.cpitch + c0, n_tile * BN);
                            if (TERMS & 2) tma_load_2d(st + Cfg::OFF_BLO, &tmBlo, &full_bar[s], tap * p.cpitch + c0, n_tile * BN);
                        }
                    }
                    __syncwarp();
                }
            }
        }
    } else {
        regs_inc<232>();
        const int cw = (warp >> 2) - 1;                        // MMA warpgroup: tile rows 64 cw .. 64 cw + 63
        const int wq = warp & 3;
        const int ct = (int)threadIdx.x - 128;                 // 0 .. 255
        constexpr int NR = BN / 2;                             // accumulator registers per thread and term
        constexpr uint32_t SWZ = BK == 64 ? GMMA_SW128 : GMMA_SW64;
        constexpr uint32_t SBO = 8 * Cfg::ROW_BYTES;
        const float inv = 1.f / (scale_from_amax(p.amax_a ? ldg_f32(p.amax_a) : 0.f) * scale_from_amax(p.amax_b ? ldg_f32(p.amax_b) : 0.f));
        const bool want_stats = p.stats != nullptr;
        float ssum = 0.f, esum = 0.f, ssq = 0.f, esq = 0.f, smin = INFINITY, smax = -INFINITY;
        float acc[TERMS ? 2 * NR : NR];                        // [hi | lo]
        float tot[FOLD ? NR : 1];                              // FOLD: round-to-nearest total of the hi*hi k-blocks
        const uint32_t smem_base = smem_u32(smem);
        // this warp has read stage `st` (its wgmma group is complete): one arrival per MMA warp of every CTA that reads it
        auto release = [&](int st) {
            __syncwarp();
            if (lane == 0) {
                if (CLUSTER == 2) {
                    mbar_arrive_cluster(&empty_bar[st], 0u);
                    mbar_arrive_cluster(&empty_bar[st], 1u);
                } else {
                    mbar_arrive(&empty_bar[st]);
                }
            }
        };
        int pend = -1;                                         // stage whose k-block group may still be in flight
        unsigned it = 0;
        for (int tile = first_tile; tile < tiles_total; tile += tile_step) {
            const int n_tile = tile % tiles_n;
            const long long m0 = (long long)(tile / tiles_n) * TC_BM;
            if (FOLD) {
#pragma unroll
                for (int i = 0; i < NR; ++i) tot[i] = 0.f;
            }
#pragma unroll 1
            for (int kb = 0; kb < nk; ++kb, ++it) {
                const int s = it % STAGES;
                mbar_wait(&full_bar[s], (it / STAGES) & 1);
                const uint32_t st = smem_base + s * Cfg::STAGE_BYTES;
                const uint64_t ah = gmma_desc(st + cw * 64 * Cfg::ROW_BYTES, 0, SBO, SWZ);
                const uint64_t al = ah + (uint64_t)(Cfg::OFF_ALO >> 4);
                const uint64_t bh = gmma_desc(st + Cfg::OFF_BHI, 0, SBO, SWZ);
                const uint64_t bl = bh + (uint64_t)(Cfg::B_BYTES >> 4);
                // 16 halves = 32 B along K inside the swizzle atom: + 2 in the descriptor
                wgmma_fence();
                if (FOLD) {
#pragma unroll
                    for (int k = 0; k < BK / 16; ++k) wgmma<BN>(acc, ah + 2 * k, bh + 2 * k, k > 0 ? 1u : 0u);
                    if (TERMS) {                               // the lo terms as a second group
                        wgmma_commit();
#pragma unroll
                        for (int k = 0; k < BK / 16; ++k) {
                            const uint32_t first_lo = (kb > 0 || k > 0) ? 1u : 0u;
                            if (TERMS & 1) wgmma<BN>(acc + NR, al + 2 * k, bh + 2 * k, first_lo);
                            if (TERMS & 2) wgmma<BN>(acc + NR, ah + 2 * k, bl + 2 * k, (TERMS & 1) ? 1u : first_lo);
                        }
                    }
                } else {
#pragma unroll
                    for (int k = 0; k < BK / 16; ++k) {
                        const uint32_t first = (kb > 0 || k > 0) ? 1u : 0u;
                        wgmma<BN>(acc, ah + 2 * k, bh + 2 * k, first);
                        if (TERMS & 2) wgmma<BN>(acc + NR, ah + 2 * k, bl + 2 * k, first);
                        if (TERMS & 1) wgmma<BN>(acc + NR, al + 2 * k, bh + 2 * k, (TERMS & 2) ? 1u : first);
                    }
                }
                wgmma_commit();
                // short K: the previous k-block is complete.  FOLD: so is this k-block's hi group (TERMS = 0 has no lo group)
                if (FOLD && TERMS == 0) wgmma_wait<0>();
                else wgmma_wait<1>();
                if (FOLD) {
                    wgmma_use<NR>(acc);
#pragma unroll
                    for (int i = 0; i < NR; ++i) tot[i] += acc[i];
                }
                if (pend >= 0) release(pend);
                pend = s;
            }
            wgmma_wait<0>();
            wgmma_use<TERMS ? 2 * NR : NR>(acc);
            if (pend >= 0) release(pend);
            pend = -1;
            if (nk == 0) {
#pragma unroll
                for (int i = 0; i < (TERMS ? 2 * NR : NR); ++i) acc[i] = 0.f;
            }
            const long long r0 = m0 + 64 * cw + 16 * wq + (lane >> 2), r1 = r0 + 8;
            float* z0 = r0 < p.M ? p.z + r0 * p.ldz + n_tile * BN : nullptr;
            float* z1 = r1 < p.M ? p.z + r1 * p.ldz + n_tile * BN : nullptr;
            epi_tile<BN, TERMS != 0>(FOLD ? tot : acc, acc + NR, inv, z0, z1, p.Cout - n_tile * BN, p.accumulate,
                                     want_stats ? sstat + (warp - 4) * BN : nullptr);
            if (want_stats) epi_fold_stats<BN>(sstat, ct, ssum, esum, ssq, esq, smin, smax);
        }
        if (want_stats && ct < BN) {
            // this CTA's partial row (one channel range: persistent grids are a multiple of tiles_n)
            const int n = (first_tile % tiles_n) * BN + ct;
            const long long row = PERSIST ? (long long)(blockIdx.x / (unsigned)tiles_n) : (long long)(first_tile / tiles_n);
            if (n < p.Cout) {
                float* dst = p.stats + row * 4 * p.Cout + n;
                dst[0] = ssum - esum; dst[p.Cout] = ssq - esq; dst[2 * p.Cout] = smin; dst[3 * p.Cout] = smax;
            }
        }
    }
    if (CLUSTER == 2) cluster_sync_all();                      // no CTA leaves while its peer may still signal its barriers
}
