// Host build of csrc/conv_tc_kernels.cuh against FUNCTIONAL MODELS of the PTX wrappers it uses (tc_models_emul.h; see
// cuda_host_emul.h for the thread model).  What is modelled: mbarriers (arrival counts, transaction bytes, phase
// parity), the im2col / tiled TMA loads (boxes land 64- / 128-byte swizzled, like the hardware's), wgmma with the device
// descriptor encoding (wgmma_emul.h), named barriers.  What this validates: the kernel's CONTROL FLOW - stage phases,
// tile sequencing over a persistent grid, accumulate flags of the three-MMA hi/lo scheme and of the k-block totals,
// the epilogue's fragment -> row mapping, edge clipping, the fused statistics - and the shared-memory descriptors it
// builds.  A wrong phase shows up as a deadlock (reported after a timeout) or as a wrong result.  Test tooling only.
#include "tc_models_emul.h"

namespace fsdet {
#include "../../fewshot_detection_b200/csrc/conv_tc_kernels.cuh"

}  // namespace fsdet

using namespace fsdet;

template <int BN, int BK, int TERMS, bool PERSIST, bool FOLD>
static int run(const uint16_t* x_hi, const uint16_t* x_lo, const uint16_t* w_hi, const uint16_t* w_lo, TcArgs a, int B,
               int ctas) {
    using Cfg = TcCfg<BN, BK, TERMS, PERSIST>;
    CUtensorMap mAh, mAl, mBh, mBl;
    const long long K = (long long)a.ks * a.ks * a.cpitch;
    auto act = [&](CUtensorMap* m, const uint16_t* base) {
        MapModel mm{}; mm.kind = 0; mm.base = base; mm.B = B; mm.H = a.H; mm.W = a.W; mm.C = a.Cin; mm.cpitch = a.cpitch;
        mm.ks = a.ks; mm.pad = a.pad; mm.bk = BK; mm.box_rows = TC_BM;
        memset(m, 0, sizeof(*m)); memcpy(m, &mm, sizeof(mm));
    };
    auto wgt = [&](CUtensorMap* m, const uint16_t* base) {
        MapModel mm{}; mm.kind = 1; mm.base = base; mm.rows = a.Cout; mm.K = K; mm.bk = BK; mm.box_rows = BN;
        memset(m, 0, sizeof(*m)); memcpy(m, &mm, sizeof(mm));
    };
    static_assert(sizeof(MapModel) <= sizeof(CUtensorMap), "model must fit in the tensor map");
    // planes a term does not use must never be touched: their maps get a null base (a load would crash)
    act(&mAh, x_hi); act(&mAl, (TERMS & 1) ? x_lo : nullptr); wgt(&mBh, w_hi); wgt(&mBl, (TERMS & 2) ? w_lo : nullptr);
    a.tiles_n = ceil_div(a.Cout, BN);
    a.tiles_total = a.tiles_n * ceil_div(a.M, TC_BM);
    const int grid = PERSIST ? ctas : a.tiles_total;
    g_deadlock.store(false);
    g_fault.store(false);
    g_wgmma_pending_at_exit.store(false);
    emul::launch(dim3(grid), dim3(TC_THREADS), Cfg::SMEM_BYTES, [&]() {
        if (threadIdx.x == 0) {
            std::lock_guard<std::mutex> l(g_mu);
            g_bars.clear();
            for (auto& nb : g_named) nb = NamedBar{};
        }
        pthread_barrier_wait(&emul::g_block.bar);
        conv_tc_kernel<BN, BK, TERMS, PERSIST, FOLD>(mAh, mAl, mBh, mBl, a);
        wgmma_block_exit();
    });
    return g_deadlock.load() ? -100 : (g_fault.load() ? -101 : (g_wgmma_pending_at_exit.load() ? -102 : 0));
}

template <int BN, int BK, bool PERSIST, bool FOLD>
static int run_terms(int terms, const uint16_t* x_hi, const uint16_t* x_lo, const uint16_t* w_hi, const uint16_t* w_lo,
                     const TcArgs& a, int B, int ctas) {
    switch (terms) {
        case 0: return run<BN, BK, 0, PERSIST, FOLD>(x_hi, x_lo, w_hi, w_lo, a, B, ctas);
        case 1: return run<BN, BK, 1, PERSIST, FOLD>(x_hi, x_lo, w_hi, w_lo, a, B, ctas);
        case 2: return run<BN, BK, 2, PERSIST, FOLD>(x_hi, x_lo, w_hi, w_lo, a, B, ctas);
        default: return run<BN, BK, 3, PERSIST, FOLD>(x_hi, x_lo, w_hi, w_lo, a, B, ctas);
    }
}

// returns 0, -100 when a barrier wait timed out (deadlock: wrong phase / arrival count), -101 when a TMA load used a
// filter offset outside the map's window, or -102 when a thread ended with wgmma operations not waited for.
//   bk = 32: short-K flavour (persist = 0: one tile per CTA, `ctas` ignored; persist = 1: `ctas` CTAs walk the tiles,
//            ctas must be a multiple of ceil(Cout / bn));  bk = 64: long-K flavour (hi*hi k-blocks folded into a total)
//   stats: optional [rows][4*Cout] partial rows (rows = persist ? ctas / tiles_n : number of 128-pixel tiles)
extern "C" int emul_conv_tc(const uint16_t* x_hi, const uint16_t* x_lo, const uint16_t* w_hi, const uint16_t* w_lo,
                            const float* amax_x, const float* amax_w, float* z, int ldz, int B, int H, int W, int Cin,
                            int cpitch, int Cout, int ks, int accumulate, int bn, int bk, int terms, int persist, int ctas,
                            float* stats) {
    TcArgs a;
    a.z = z; a.amax_a = amax_x; a.amax_b = amax_w; a.stats = stats; a.ldz = ldz; a.H = H; a.W = W; a.Cin = Cin; a.Cout = Cout;
    a.ks = ks; a.pad = (ks - 1) / 2; a.cpitch = cpitch; a.M = (long long)B * H * W; a.accumulate = accumulate;
    a.tiles_n = a.tiles_total = 0;
    if (bk == 32 && persist) {
        if (bn == 64) return run_terms<64, 32, true, false>(terms, x_hi, x_lo, w_hi, w_lo, a, B, ctas);
        if (bn == 128) return run_terms<128, 32, true, false>(terms, x_hi, x_lo, w_hi, w_lo, a, B, ctas);
    } else if (bk == 32) {
        if (bn == 64) return run_terms<64, 32, false, false>(terms, x_hi, x_lo, w_hi, w_lo, a, B, ctas);
        if (bn == 128) return run_terms<128, 32, false, false>(terms, x_hi, x_lo, w_hi, w_lo, a, B, ctas);
    } else if (bk == 64 && !persist) {
        if (bn == 64) return run_terms<64, 64, false, true>(terms, x_hi, x_lo, w_hi, w_lo, a, B, ctas);
        if (bn == 128) return run_terms<128, 64, false, true>(terms, x_hi, x_lo, w_hi, w_lo, a, B, ctas);
    }
    return -1;
}

// test knob: every wgmma wait of the model sleeps this long (0 = off)
extern "C" void emul_set_ld_delay_us(int us) { fsdet::g_mma_delay_us.store(us); }
