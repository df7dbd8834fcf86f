// Host build of csrc/conv_halo_kernels.cuh (the halo-tile convolution) against the functional models of
// conv_tc_emul.cpp plus a model of the tiled 4-D TMA box it adds.  As there, boxes land 64-byte swizzled and the wgmma
// model reads shared memory through the device descriptor encoding and the same swizzle - which is exactly what the
// halo scheme relies on: filter tap (dy, dx) = the K-major tile starting dy * 8 rows into x-shifted copy dx.  What is
// validated: tile walk of the persistent grid, the two producer warps (activation stages / weight ring or resident
// weights), stage phases, tap addressing inside the halo copies, zero fill at the image border, clipped stores and
// statistics for tiles that overhang the image.  Test tooling only.
#include "conv_tc_emul.cpp"

namespace fsdet {

// box (32 channels, 8 x, 18 y) of an NHWC fp16 plane at signed coordinates; zero outside the tensor
static inline void tma_load_tiled_4d(void* dst, const CUtensorMap* map, uint64_t* bar, int c, int w, int h, int n) {
    const MapModel* m = model(map);
    for (int yy = 0; yy < 18; ++yy)
        for (int xx = 0; xx < 8; ++xx)
            for (int k = 0; k < 32; ++k) {
                const int y = h + yy, x = w + xx, ch = c + k;
                const bool ok = n >= 0 && n < m->B && y >= 0 && y < m->H && x >= 0 && x < m->W && ch < m->C;
                box_store(dst, yy * 8 + xx, k, 64, ok ? m->base[(((size_t)n * m->H + y) * m->W + x) * m->cpitch + ch] : (uint16_t)0);
            }
    bar_complete_tx(bar, 18 * 8 * 32 * 2);
}
#include "../../fewshot_detection_b200/csrc/conv_halo_kernels.cuh"

}  // namespace fsdet

template <int BN, int NCH>
static int run_halo(const uint16_t* x_hi, const uint16_t* x_lo, const uint16_t* w_hi, const uint16_t* w_lo, HaloArgs a, float* z,
                    int ldz, int B, int Cin, int ctas) {
    constexpr bool BRES = NCH * BN <= 64;
    using Cfg = HaloCfg<BN, NCH, BRES>;
    CUtensorMap mAh, mAl, mBh, mBl;
    auto act = [&](CUtensorMap* m, const uint16_t* base) {
        MapModel mm{}; mm.kind = 3; mm.base = base; mm.B = B; mm.H = a.H; mm.W = a.W; mm.C = Cin; mm.cpitch = a.cpitch;
        memset(m, 0, sizeof(*m)); memcpy(m, &mm, sizeof(mm));
    };
    auto wgt = [&](CUtensorMap* m, const uint16_t* base) {
        MapModel mm{}; mm.kind = 1; mm.base = base; mm.rows = a.Cout; mm.K = 9LL * a.cpitch; mm.bk = 32; mm.box_rows = BN;
        memset(m, 0, sizeof(*m)); memcpy(m, &mm, sizeof(mm));
    };
    act(&mAh, x_hi); act(&mAl, x_lo); wgt(&mBh, w_hi); wgt(&mBl, w_lo);
    a.z = z; a.ldz = ldz;
    g_deadlock.store(false);
    g_wgmma_pending_at_exit.store(false);
    emul::launch(dim3(ctas), dim3(HALO_THREADS), Cfg::SMEM_BYTES, [&]() {
        if (threadIdx.x == 0) {
            std::lock_guard<std::mutex> l(g_mu);
            g_bars.clear();
            for (auto& nb : g_named) nb = NamedBar{};
        }
        pthread_barrier_wait(&emul::g_block.bar);
        conv_halo_kernel<BN, NCH, BRES>(mAh, mAl, mBh, mBl, a);
        wgmma_block_exit();
    });
    return g_deadlock.load() ? -100 : (g_wgmma_pending_at_exit.load() ? -102 : 0);
}

template <int BN>
static int run_halo_nch(int nch, const uint16_t* x_hi, const uint16_t* x_lo, const uint16_t* w_hi, const uint16_t* w_lo, const HaloArgs& a,
                        float* z, int ldz, int B, int Cin, int ctas) {
    switch (nch) {
        case 1: return run_halo<BN, 1>(x_hi, x_lo, w_hi, w_lo, a, z, ldz, B, Cin, ctas);
        case 2: return run_halo<BN, 2>(x_hi, x_lo, w_hi, w_lo, a, z, ldz, B, Cin, ctas);
        case 4: return run_halo<BN, 4>(x_hi, x_lo, w_hi, w_lo, a, z, ldz, B, Cin, ctas);
    }
    return -1;
}

// 3x3 convolution through the halo-tile kernel on `ctas` persistent CTAs; returns 0, -100 on a barrier deadlock, -102
// when a thread ended with wgmma operations not waited for.
// stats: optional [ctas][4*Cout] partial rows
extern "C" int emul_conv_halo(const uint16_t* x_hi, const uint16_t* x_lo, const uint16_t* w_hi, const uint16_t* w_lo,
                              const float* amax_x, const float* amax_w, float* z, int ldz, int B, int H, int W, int Cin, int cpitch,
                              int Cout, int accumulate, int ctas, float* stats, int flags) {
    if (W % 8 != 0 || Cin % 32 != 0 || Cout > 128) return -1;
    HaloArgs a;
    a.amax_a = amax_x; a.amax_b = amax_w; a.stats = stats; a.H = H; a.W = W; a.Cout = Cout; a.cpitch = cpitch;
    a.tiles_x = W / 8; a.tiles_y = (H + 15) / 16; a.tiles_total = B * a.tiles_x * a.tiles_y; a.accumulate = accumulate; a.flags = flags;
    if (ctas > a.tiles_total) return -1;
    const int bn = Cout <= 32 ? 32 : (Cout <= 64 ? 64 : 128);
    if (bn == 32) return run_halo_nch<32>(Cin / 32, x_hi, x_lo, w_hi, w_lo, a, z, ldz, B, Cin, ctas);
    if (bn == 64) return run_halo_nch<64>(Cin / 32, x_hi, x_lo, w_hi, w_lo, a, z, ldz, B, Cin, ctas);
    return run_halo_nch<128>(Cin / 32, x_hi, x_lo, w_hi, w_lo, a, z, ldz, B, Cin, ctas);
}
