// Host build of csrc/conv_wgrad_kernels.cuh (the wgmma weight-gradient kernel) against the functional models of
// tc_models_emul.h (see cuda_host_emul.h for the thread model).  The dz operand comes through a 2-D tiled map (64
// channels x 64 pixels), the x operand of one filter tap through an im2col map of 64-pixel boxes; both land 128-byte
// swizzled and the wgmma model reads them MN-major through the device descriptor encoding.  What this validates:
// the split-K pixel ranges (slices past the last pixel store zeros), stages that straddle images, tap pairs and the
// clamped tail tap, channel and output-channel tiles that overhang Cin / Cout, the accumulate flags of the hi/lo terms,
// the fold of every stage's hi*hi sum into the register total, the fragment -> (co, tap, ci) store mapping and the
// stage phases (deadlock = -100; a filter offset outside the im2col window = -101).  Test tooling only.
#include "tc_models_emul.h"

namespace fsdet {
#define FSDET_TC_DYN_SMEM(name) uint8_t* name = emul::g_dyn_smem
#include "../../fewshot_detection_b200/csrc/conv_wgrad_kernels.cuh"
}  // namespace fsdet

using namespace fsdet;

template <int TAPS, int TERMS>
static int run(const uint16_t* x_hi, const uint16_t* x_lo, const uint16_t* dz_hi, const uint16_t* dz_lo, const TcWgArgs& a,
               int B, int splits) {
    using Cfg = WgCfg<TERMS>;
    CUtensorMap mDh, mDl, mXh, mXl;
    auto dz = [&](CUtensorMap* m, const uint16_t* base) {   // [M][Cout] plane: box = 64 channels x 64 pixels
        MapModel mm{}; mm.kind = 1; mm.base = base; mm.rows = (int)a.M; mm.K = a.Cout; mm.bk = 64; mm.box_rows = WG_BP;
        memset(m, 0, sizeof(*m)); memcpy(m, &mm, sizeof(mm));
    };
    auto act = [&](CUtensorMap* m, const uint16_t* base) {  // [B][H][W][Cin] plane: im2col boxes of 64 pixels x 64 channels
        MapModel mm{}; mm.kind = 0; mm.base = base; mm.B = B; mm.H = a.H; mm.W = a.W; mm.C = a.Cin; mm.cpitch = a.Cin;
        mm.ks = a.ks; mm.pad = a.pad; mm.bk = 64; mm.box_rows = WG_BP;
        memset(m, 0, sizeof(*m)); memcpy(m, &mm, sizeof(mm));
    };
    static_assert(sizeof(MapModel) <= sizeof(CUtensorMap), "model must fit in the tensor map");
    // planes a term does not use must never be touched: their maps get a null base (a load would crash)
    dz(&mDh, dz_hi); dz(&mDl, (TERMS & 1) ? dz_lo : nullptr); act(&mXh, x_hi); act(&mXl, (TERMS & 2) ? x_lo : nullptr);
    constexpr int CIB = WG_BN / TAPS;
    const dim3 grid(((a.Cin + CIB - 1) / CIB) * ((a.ks * a.ks + TAPS - 1) / TAPS), (a.Cout + 127) / 128, splits);
    g_deadlock.store(false);
    g_fault.store(false);
    g_wgmma_pending_at_exit.store(false);
    emul::launch(grid, dim3(384), Cfg::SMEM_BYTES, [&]() {
        if (threadIdx.x == 0) {
            std::lock_guard<std::mutex> l(g_mu);
            g_bars.clear();
        }
        pthread_barrier_wait(&emul::g_block.bar);
        wgrad_tc_kernel<TAPS, TERMS>(mDh, mDl, mXh, mXl, a);
        wgmma_block_exit();
    });
    return g_deadlock.load() ? -100 : (g_fault.load() ? -101 : (g_wgmma_pending_at_exit.load() ? -102 : 0));
}

template <int TAPS>
static int run_terms(int terms, const uint16_t* x_hi, const uint16_t* x_lo, const uint16_t* dz_hi, const uint16_t* dz_lo,
                     const TcWgArgs& a, int B, int splits) {
    switch (terms) {
        case 0: return run<TAPS, 0>(x_hi, x_lo, dz_hi, dz_lo, a, B, splits);
        case 1: return run<TAPS, 1>(x_hi, x_lo, dz_hi, dz_lo, a, B, splits);
        case 2: return run<TAPS, 2>(x_hi, x_lo, dz_hi, dz_lo, a, B, splits);
        default: return run<TAPS, 3>(x_hi, x_lo, dz_hi, dz_lo, a, B, splits);
    }
}

// Weight gradient of an NHWC x [B][H][W][Cin] and dz [B*H*W][Cout] (fp16 hi / lo planes) into out [splits][Cout][k*k*Cin]:
// slice z holds the sum over pixels [z * pix_per_split, min((z + 1) * pix_per_split, M)), unreduced, exactly as
// fsdet_conv_tc_wgrad's workspace.  Two taps per N tile when Cin < 128 (as wg_taps in conv_tc.cu).
// Returns 0, -100 on a barrier deadlock, -101 on a TMA load outside the im2col filter window, -102 when a thread ended
// with wgmma operations not waited for, -1 on bad arguments.
extern "C" int emul_conv_wgrad(const uint16_t* x_hi, const uint16_t* x_lo, const uint16_t* dz_hi, const uint16_t* dz_lo,
                               const float* amax_x, const float* amax_dz, float* out, int B, int H, int W, int Cin, int Cout,
                               int ks, int terms, int splits, long long pix_per_split) {
    if (Cin % 64 != 0 || Cout % 64 != 0 || !(ks == 1 || ks == 3) || splits < 1 || pix_per_split % WG_BP != 0) return -1;
    TcWgArgs a;
    a.out = out; a.amax_a = amax_dz; a.amax_b = amax_x;
    a.H = H; a.W = W; a.Cin = Cin; a.Cout = Cout; a.ks = ks; a.pad = (ks - 1) / 2; a.M = (long long)B * H * W;
    a.pix_per_split = pix_per_split;
    if (Cin >= 128) return run_terms<1>(terms, x_hi, x_lo, dz_hi, dz_lo, a, B, splits);
    return run_terms<2>(terms, x_hi, x_lo, dz_hi, dz_lo, a, B, splits);
}

// test knob: every wgmma wait of the model sleeps this long (0 = off)
extern "C" void emul_set_ld_delay_us(int us) { fsdet::g_mma_delay_us.store(us); }
