// Halo-tile wgmma convolution (3x3, stride 1, "same" padding) for the HIGH-RESOLUTION layers - included by conv_tc.cu
// after the PTX wrappers and by tools/host_emul/conv_halo_emul.cpp after functional models of the same wrappers.
//
// Why: the im2col kernel (conv_tc_kernels.cuh) fetches the activation tile once PER FILTER TAP (9 x) and the weight tile
// once per 128-pixel tile.  With 3-term operands (two fp16 planes each) the short-K, high-resolution layers (conv2 at
// 208 x 208, conv3/5 at 104 x 104, forward and input gradient) ask the L2 for more operand bytes per MMA than it
// delivers.  Here the activation tile is fetched with its halo ONCE per 128 output pixels and all nine taps are served
// from shared memory:
//
//   * tile = 8 x 16 output pixels (x fastest): GEMM row m = py * 8 + px, so every 8-row swizzle atom of the K-major
//     operand is one spatial row of 8 pixels;
//   * the halo tile is stored as three x-shifted copies [dx][18 rows][8 px][32 channels] (64-byte rows, 64-byte swizzle,
//     a plain tiled TMA box of (32 c, 8 w, 18 h) at x0 + dx - 1, y0 - 1 with zero fill outside the image);
//     filter tap (dy, dx) is then the ordinary K-major tile that starts dy atoms (dy * 512 B) into copy dx - the
//     shared-memory descriptor and swizzle are those of the im2col kernel, only the start address moves by whole atoms;
//   * activation traffic per tile: 3 x 18/16 = 3.4 tile-equivalents instead of 9;
//   * persistent CTAs (one per SM); where the whole weight operand fits (Cin/32 * BN <= 64: conv2 forward and input
//     gradient, 72 KB) it is loaded ONCE per CTA and stays resident, otherwise it streams through a ring of (tap, chunk)
//     stages filled by a second producer warp.
//
// Arithmetic: 3-term fp16 hi/lo scheme (conv_tc_kernels.cuh, TERMS = 3) - D_hi += A_hi * B_hi, D_lo += A_hi * B_lo +
// A_lo * B_hi (three MMAs of width BN per K step), summed in the epilogue.  K <= 1152 here, so one hi accumulator (the
// im2col short-K flavour's choice).
//
// Warps (384 threads): 0 = activation producer (+ resident weights), 1 = weight-ring producer (idle when the weights
// are resident), 2-3 idle (the producer warpgroup hands its registers to the MMA warpgroups); warpgroups 1 and 2 =
// MMA + epilogue for tile rows 0-63 (pixel rows 0-7) and 64-127 (pixel rows 8-15).
#pragma once

struct HaloArgs {
    const float* amax_a;
    const float* amax_b;
    float* z;            // fp32 output [B][H][W][ldz] (first Cout channels)
    float* stats;        // optional [gridDim.x][4*Cout] = (sum | sum of squares | min | max), row = blockIdx.x
    int ldz;
    int H, W, Cout;
    int cpitch;          // channel pitch of the weight planes' K axis: k = tap * cpitch + c
    int tiles_x, tiles_y;
    int tiles_total;     // B * tiles_x * tiles_y
    int accumulate;
    int flags;           // developer knob FSDET_HALO_FLAGS, timing experiments only (results invalid): bit 0 = fetch one
                         // halo copy instead of three, bit 1 = no output stores.  Other bits are ignored.
};

constexpr int HALO_TW = 8, HALO_TH = 16;
constexpr int HALO_ROWS = (HALO_TH + 2) * HALO_TW;          // 144 rows of 64 B per (plane, dx) copy
constexpr int HALO_COPY_BYTES = HALO_ROWS * 64;             // 9216
constexpr int HALO_ASTAGE_BYTES = 2 * 3 * HALO_COPY_BYTES;  // hi + lo planes, three x-shifts: 55296
constexpr int HALO_THREADS = 384;

template <int BN, int NCH, bool BRES>
struct HaloCfg {
    static constexpr int SA = 2;                                   // activation stages (one = one tile x 32 channels)
    static constexpr int BBLK = BN * 64;                           // one (tap, chunk) weight block of one plane
    static constexpr int BSTAGE = 2 * BBLK;                        // hi + lo
    static constexpr int NKB = 9 * NCH;                            // k-blocks (tap, chunk) per tile
    static constexpr int STAT_BYTES = 8 * BN * 16;                 // 8 MMA warps x BN channels x float4
    static constexpr int BUDGET = 227 * 1024 - 1024 - 256;
    static constexpr int FREE_FOR_B = BUDGET - SA * HALO_ASTAGE_BYTES - STAT_BYTES;
    static constexpr int SB = BRES ? NKB : ((FREE_FOR_B / BSTAGE) > 8 ? 8 : (FREE_FOR_B / BSTAGE));
    static constexpr int OFF_B = SA * HALO_ASTAGE_BYTES;
    static constexpr int OFF_STAT = OFF_B + SB * BSTAGE;
    static constexpr int OFF_BAR = OFF_STAT + STAT_BYTES;
    static constexpr int SMEM_BYTES = OFF_BAR + 1024 + 256;
    static_assert(SB >= 3, "weight ring too small");
    static_assert(!BRES || NKB * BSTAGE <= FREE_FOR_B, "resident weights do not fit");
    static_assert(BSTAGE % 1024 == 0 || BN == 32, "swizzle atoms need 512-byte alignment");
};

template <int BN, int NCH, bool BRES>
__global__ void __launch_bounds__(HALO_THREADS, 1)
conv_halo_kernel(const __grid_constant__ CUtensorMap tmAhi, const __grid_constant__ CUtensorMap tmAlo,
                 const __grid_constant__ CUtensorMap tmBhi, const __grid_constant__ CUtensorMap tmBlo, const HaloArgs p) {
    using Cfg = HaloCfg<BN, NCH, BRES>;
    constexpr int SA = Cfg::SA, SB = Cfg::SB;
    FSDET_TC_DYN_SMEM(smem_raw);
    uint8_t* smem = tc_align_smem(smem_raw);
    float4* sstat = reinterpret_cast<float4*>(smem + Cfg::OFF_STAT);   // [8 MMA warps][BN]
    uint64_t* a_full = reinterpret_cast<uint64_t*>(smem + Cfg::OFF_BAR);
    uint64_t* a_empty = a_full + SA;
    uint64_t* b_full = a_empty + SA;              // [SB] ring, or [0] only when the weights are resident
    uint64_t* b_empty = b_full + 8;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int tiles_total = p.tiles_total;
    const int tiles_img = p.tiles_x * p.tiles_y;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmAhi);
        tma_prefetch_desc(&tmAlo);
        tma_prefetch_desc(&tmBhi);
        tma_prefetch_desc(&tmBlo);
        for (int s = 0; s < SA; ++s) {
            mbar_init(&a_full[s], 1);
            mbar_init(&a_empty[s], 8);                 // the 8 MMA warps
        }
        for (int s = 0; s < 8; ++s) {
            mbar_init(&b_full[s], 1);
            mbar_init(&b_empty[s], 8);
        }
        fence_barrier_init();
    }
    __syncthreads();

    // The producer warps run converged and issue under elect_one() (see tc_ptx.cuh).
    if (warp < 4) {
        regs_dec<40>();
        if (warp == 0) {
            if (BRES) {          // the whole weight operand, once
                if (elect_one()) {
                    mbar_expect_tx(&b_full[0], (uint32_t)(Cfg::NKB * Cfg::BSTAGE));
#pragma unroll 1
                    for (int kb = 0; kb < Cfg::NKB; ++kb) {
                        const int chunk = kb / 9, tap = kb - chunk * 9;
                        uint8_t* st = smem + Cfg::OFF_B + kb * Cfg::BSTAGE;
                        tma_load_2d(st, &tmBhi, &b_full[0], tap * p.cpitch + chunk * 32, 0);
                        tma_load_2d(st + Cfg::BBLK, &tmBlo, &b_full[0], tap * p.cpitch + chunk * 32, 0);
                    }
                }
                __syncwarp();
            }
            unsigned it = 0;                                   // activation stages issued so far
            for (int tile = (int)blockIdx.x; tile < tiles_total; tile += (int)gridDim.x) {
                const int img = tile / tiles_img;
                const int r = tile - img * tiles_img;
                const int ty = r / p.tiles_x, tx = r - ty * p.tiles_x;
                const int x0 = tx * HALO_TW - 1, y0 = ty * HALO_TH - 1;
#pragma unroll 1
                for (int chunk = 0; chunk < NCH; ++chunk, ++it) {
                    const int s = it % SA;
                    mbar_wait_warp(&a_empty[s], ((it / SA) & 1) ^ 1);
                    if (elect_one()) {
                        uint8_t* st = smem + s * HALO_ASTAGE_BYTES;
                        const int ncopy = (p.flags & 1) ? 1 : 3;
                        mbar_expect_tx(&a_full[s], (uint32_t)(ncopy * 2 * HALO_COPY_BYTES));
                        for (int dx = 0; dx < ncopy; ++dx) {
                            tma_load_tiled_4d(st + dx * HALO_COPY_BYTES, &tmAhi, &a_full[s], chunk * 32, x0 + dx, y0, img);
                            tma_load_tiled_4d(st + (3 + dx) * HALO_COPY_BYTES, &tmAlo, &a_full[s], chunk * 32, x0 + dx, y0, img);
                        }
                    }
                    __syncwarp();
                }
            }
        } else if (warp == 1 && !BRES) {
            unsigned it = 0;                                   // weight stages issued so far
            for (int tile = (int)blockIdx.x; tile < tiles_total; tile += (int)gridDim.x) {
#pragma unroll 1
                for (int kb = 0; kb < Cfg::NKB; ++kb, ++it) {
                    const int chunk = kb / 9, tap = kb - chunk * 9;
                    const int s = it % SB;
                    mbar_wait_warp(&b_empty[s], ((it / SB) & 1) ^ 1);
                    if (elect_one()) {
                        uint8_t* st = smem + Cfg::OFF_B + s * Cfg::BSTAGE;
                        mbar_expect_tx(&b_full[s], (uint32_t)Cfg::BSTAGE);
                        tma_load_2d(st, &tmBhi, &b_full[s], tap * p.cpitch + chunk * 32, 0);
                        tma_load_2d(st + Cfg::BBLK, &tmBlo, &b_full[s], tap * p.cpitch + chunk * 32, 0);
                    }
                    __syncwarp();
                }
            }
        }
    } else {
        regs_inc<232>();
        const int cw = (warp >> 2) - 1;                        // MMA warpgroup: pixel rows 8 cw .. 8 cw + 7 of the tile
        const int wq = warp & 3;
        const int ct = (int)threadIdx.x - 128;
        constexpr int NR = BN / 2;
        const float inv = 1.f / (scale_from_amax(p.amax_a ? ldg_f32(p.amax_a) : 0.f) * scale_from_amax(p.amax_b ? ldg_f32(p.amax_b) : 0.f));
        const bool want_stats = p.stats != nullptr;
        float ssum = 0.f, esum = 0.f, ssq = 0.f, esq = 0.f, smin = INFINITY, smax = -INFINITY;
        float acc[2 * NR];                                     // [hi | lo]
        if (BRES) mbar_wait(&b_full[0], 0);
        const uint32_t smem_base = smem_u32(smem);
        // this warp has read activation stage `sa_` / weight stage `sb_` (< 0: none)
        auto release = [&](int sa_, int sb_) {
            __syncwarp();
            if (lane == 0) {
                if (sa_ >= 0) mbar_arrive(&a_empty[sa_]);
                if (sb_ >= 0) mbar_arrive(&b_empty[sb_]);
            }
        };
        int pend_a = -1, pend_b = -1;                          // stages whose last wgmma group may still be in flight
        unsigned ita = 0, itb = 0;
        for (int tile = (int)blockIdx.x; tile < tiles_total; tile += (int)gridDim.x) {
            uint32_t started = 0;
#pragma unroll 1
            for (int chunk = 0; chunk < NCH; ++chunk, ++ita) {
                const int sa = ita % SA;
                mbar_wait(&a_full[sa], (ita / SA) & 1);
                const uint32_t a0 = smem_base + sa * HALO_ASTAGE_BYTES + cw * 8 * (HALO_TW * 64);
#pragma unroll 1
                for (int dy = 0; dy < 3; ++dy) {
#pragma unroll
                    for (int dx = 0; dx < 3; ++dx, ++itb) {
                        int sb;
                        if (BRES) {
                            sb = chunk * 9 + dy * 3 + dx;
                        } else {
                            sb = itb % SB;
                            mbar_wait(&b_full[sb], (itb / SB) & 1);
                        }
                        const uint64_t ah = gmma_desc(a0 + dx * HALO_COPY_BYTES + dy * (HALO_TW * 64), 0, 512, GMMA_SW64);
                        const uint64_t al = ah + (uint64_t)((3 * HALO_COPY_BYTES) >> 4);
                        const uint64_t bh = gmma_desc(smem_base + Cfg::OFF_B + sb * Cfg::BSTAGE, 0, 512, GMMA_SW64);
                        const uint64_t bl = bh + (uint64_t)(Cfg::BBLK >> 4);
                        wgmma_fence();
#pragma unroll
                        for (int k = 0; k < 2; ++k) {          // 16 halves = 32 B along K inside the swizzle atom: + 2 in the descriptor
                            const uint64_t adv = (uint64_t)(2 * k);
                            wgmma<BN>(acc, ah + adv, bh + adv, started);
                            wgmma<BN>(acc + NR, ah + adv, bl + adv, started);
                            wgmma<BN>(acc + NR, al + adv, bh + adv, 1u);
                            started = 1u;
                        }
                        wgmma_commit();
                        // one tap stays in flight: every earlier group is complete, so the stages it read are free
                        wgmma_wait<1>();
                        release(pend_a, pend_b);
                        pend_a = -1;
                        pend_b = BRES ? -1 : sb;
                    }
                }
                pend_a = sa;                                   // freed once the chunk's last tap has completed
            }
            wgmma_wait<0>();
            wgmma_use<2 * NR>(acc);
            release(pend_a, pend_b);
            pend_a = pend_b = -1;
            // epilogue: rows 16 wq + lane / 4 (+ 8) of this warpgroup's 64 = pixel rows 8 cw + 2 wq (+ 1), column lane / 4
            const int img = tile / tiles_img;
            const int r = tile - img * tiles_img;
            const int ty = r / p.tiles_x, tx = r - ty * p.tiles_x;
            const int x = tx * HALO_TW + (lane >> 2);
            const int ya = ty * HALO_TH + 8 * cw + 2 * wq, yb = ya + 1;
            float* z0 = (ya < p.H && !(p.flags & 2)) ? p.z + (((long long)img * p.H + ya) * p.W + x) * p.ldz : nullptr;
            float* z1 = (yb < p.H && !(p.flags & 2)) ? p.z + (((long long)img * p.H + yb) * p.W + x) * p.ldz : nullptr;
            epi_tile<BN, true>(acc, acc + NR, inv, z0, z1, p.Cout, p.accumulate, want_stats ? sstat + (warp - 4) * BN : nullptr);
            if (want_stats) epi_fold_stats<BN>(sstat, ct, ssum, esum, ssq, esq, smin, smax);
        }
        if (want_stats && ct < BN && ct < p.Cout) {
            float* dst = p.stats + (long long)blockIdx.x * 4 * p.Cout + ct;
            dst[0] = ssum - esum; dst[p.Cout] = ssq - esq; dst[2 * p.Cout] = smin; dst[3 * p.Cout] = smax;
        }
    }
}
