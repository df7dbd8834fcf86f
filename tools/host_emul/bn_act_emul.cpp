// Host-emulated build of csrc/bn_act.cu (see cuda_host_emul.h): the BatchNorm / LeakyReLU / max-pool passes with the
// argument lists of the fsdet_* entry points (no stream; an `emul_` prefix), host pointers instead of device pointers,
// and the launch geometry of the device (chan_lanes, bwd_rows, stat_split).  Test tooling only; built by
// tests/test_bn_act_host_emul.py with g++.
#include "../../fewshot_detection_b200/csrc/bn_act.cu"

namespace emul {
Block g_block;
unsigned char* g_dyn_smem = nullptr;
}  // namespace emul
namespace fsdet {
void set_error(const char*, ...) {}
}  // namespace fsdet

using namespace fsdet;

extern "C" int emul_bn_bwd_rows(int B, int H, int W) { return bwd_rows(B, H, W); }
extern "C" int emul_bn_chan_lanes(int C) { return chan_lanes(C); }
extern "C" int emul_bn_stat_splits(int nparts) {
    int S, rps;
    stat_split(nparts, &S, &rps);
    return S;
}

// stat_partial: nparts rows of 4C floats followed by fsdet_bn_stat_scratch_rows() rows of scratch (as on the device)
extern "C" int emul_bn_finalize(const float* stat_partial, int nparts, double count, const float* gamma, const float* beta,
                                float* running_mean, float* running_var, float momentum, float eps, float* mean, float* invstd,
                                float* scale, float* shift, float slope, float* amax_y, float* xhat_absmax, int C,
                                int training) {
    if (!scale || !shift || C <= 0) return -1;
    if (training ? !(stat_partial && nparts > 0) : !(running_mean && running_var)) return -1;
    if (amax_y && !training) *amax_y = 0.f;
    const double* red = nullptr;
    int S = 0;
    if (training) {
        int rps;
        stat_split(nparts, &S, &rps);
        double* scratch = reinterpret_cast<double*>(const_cast<float*>(stat_partial) + (size_t)nparts * 4 * C);
        emul::launch(dim3(ceil_div(C, 32), S), dim3(32, 32), 0,
                     [&]() { bn_stats_reduce_kernel(stat_partial, nparts, rps, C, scratch, amax_y); });
        red = scratch;
    }
    emul::launch(dim3(ceil_div(C, 128)), dim3(128), 0, [&]() {
        bn_finalize_kernel(red, S, count, gamma, beta, running_mean, running_var, momentum, eps, mean, invstd, scale, shift,
                           slope, amax_y, xhat_absmax, C, training);
    });
    return 0;
}

extern "C" int emul_bn_act_fwd(const float* z, int ldz, const float* scale, const float* shift, float slope, float* y_full,
                               int ld_full, float* y_pool, int ld_pool, void* full_hi, void* full_lo, void* pool_hi,
                               void* pool_lo, int Cpad, const float* amax, int B, int H, int W, int C) {
    const bool planes = full_hi || pool_hi;
    if (!(z && scale && shift && (y_full || y_pool || planes)) || C % 4 || ldz % 4 || (y_full && ld_full % 4) ||
        (y_pool && ld_pool % 4) || (planes && !(amax && Cpad >= C && Cpad % 4 == 0)))
        return -1;
    FwdArgs a;
    a.z = z; a.scale = scale; a.shift = shift; a.amax = amax; a.yf = y_full; a.yp = y_pool;
    a.fh = (__half*)full_hi; a.fl = (__half*)full_lo; a.ph = (__half*)pool_hi; a.pl = (__half*)pool_lo;
    a.ldz = ldz; a.ldf = ld_full; a.ldp = ld_pool; a.Cpad = planes ? Cpad : C; a.B = B; a.H = H; a.W = W; a.C = C; a.slope = slope;
    const int CP4 = a.Cpad / 4;
    if (!y_pool && !pool_hi) {
        long long n = (long long)B * H * W * CP4;
        if (n == 0) return 0;
        emul::launch_serial(dim3(ceil_div(n, 256)), dim3(256), [&]() { bn_act_flat_kernel(a); });
    } else {
        long long nwin = (long long)B * ((H + 1) / 2) * ((W + 1) / 2);
        if (nwin == 0) return 0;
        const int TC = chan_lanes(C);
        const int TY = 256 / TC;
        const dim3 block(TC, TY), grid((unsigned)ceil_div(nwin, TY));
        if (a.yf || a.fh) emul::launch_serial(grid, block, [&]() { bn_act_pool_kernel<true>(a); });
        else emul::launch_serial(grid, block, [&]() { bn_act_pool_kernel<false>(a); });
    }
    return 0;
}

// returns 1 when the pool-only specialisation ran, 0 for the general kernel (the same dispatch as launch_bwd)
static int emul_bwd(bool apply, const BwdArgs& a) {
    const int C4 = a.C / 4;
    const int TC = chan_lanes(a.C);
    const int TY = 256 / TC;
    const dim3 block(TC, TY), grid(bwd_rows(a.B, a.H, a.W), ceil_div(C4, TC));
    const size_t smem = (size_t)TY * TC * 16 * sizeof(double);
    const bool pool_only = !a.dyf && a.dyp && a.has_bn && a.slope >= 0.f && a.slope <= 1.f;
    if (pool_only) {
        if (apply) emul::launch_serial(grid, block, [&]() { bn_act_bwd_pool_kernel<true>(a); });
        else emul::launch(grid, block, smem, [&]() { bn_act_bwd_pool_kernel<false>(a); });
    } else {
        if (apply) emul::launch_serial(grid, block, [&]() { bn_act_bwd_kernel<true>(a); });
        else emul::launch(grid, block, smem, [&]() { bn_act_bwd_kernel<false>(a); });
    }
    return pool_only ? 1 : 0;
}

// partial: bwd_rows(B, H, W) + 1 rows of 3C doubles
extern "C" int emul_bn_act_bwd_reduce(const float* z, int ldz, const float* dy_full, int ld_dyf, const float* dy_pool,
                                      int ld_dyp, const float* scale, const float* shift, const float* mean, const float* invstd,
                                      float slope, double* partial, int B, int H, int W, int C, int has_bn) {
    if (!(z && scale && shift && partial && (dy_full || dy_pool)) || (has_bn && !(mean && invstd)) || C % 4) return -1;
    BwdArgs a;
    a.z = z; a.dyf = dy_full; a.dyp = dy_pool; a.scale = scale; a.shift = shift; a.mean = mean; a.invstd = invstd;
    a.coef = nullptr; a.dz = nullptr; a.dh = nullptr; a.dl = nullptr; a.amax = nullptr; a.partial = partial;
    a.ldz = ldz; a.ld_dyf = ld_dyf; a.ld_dyp = ld_dyp; a.lddz = 0; a.cpad = 0;
    a.B = B; a.H = H; a.W = W; a.C = C; a.slope = slope; a.has_bn = has_bn;
    return emul_bwd(false, a);
}

extern "C" int emul_bn_bwd_finalize(const double* partial, int nparts, double count, const float* gamma, const float* invstd,
                                    const float* xhat_absmax, float* dgamma, float* dbeta, double* coef, float* amax_bound,
                                    int C, int has_bn) {
    if (!(partial && nparts > 0 && C > 0) || (has_bn && !(coef && gamma && invstd)) || (amax_bound && has_bn && !xhat_absmax))
        return -1;
    double* sums = const_cast<double*>(partial) + (size_t)nparts * 3 * C;
    emul::launch(dim3(ceil_div(3 * C, 32)), dim3(32, 32), 0,
                 [&]() { colsum_dd_kernel(partial, nparts, 3 * C, 2 * C, sums, amax_bound); });
    emul::launch_serial(dim3(ceil_div(C, 128)), dim3(128), [&]() {
        bn_bwd_finalize_kernel(sums, count, gamma, invstd, xhat_absmax, dgamma, dbeta, coef, amax_bound, C, has_bn);
    });
    return 0;
}

extern "C" int emul_bn_act_bwd_apply(const float* z, int ldz, const float* dy_full, int ld_dyf, const float* dy_pool,
                                     int ld_dyp, const float* scale, const float* shift, const float* mean, const float* invstd,
                                     const double* coef, float slope, float* dz, int lddz, void* dz_hi, void* dz_lo, int cpad,
                                     const float* amax, int B, int H, int W, int C, int has_bn) {
    if (!(z && scale && shift && (dz || dz_hi) && (dy_full || dy_pool)) || (has_bn && !(mean && invstd && coef)) || C % 4 ||
        (dz_hi && !(dz_lo && amax && cpad == C)))
        return -1;
    BwdArgs a;
    a.z = z; a.dyf = dy_full; a.dyp = dy_pool; a.scale = scale; a.shift = shift; a.mean = mean; a.invstd = invstd;
    a.coef = coef; a.dz = dz; a.dh = (__half*)dz_hi; a.dl = (__half*)dz_lo; a.amax = amax; a.partial = nullptr;
    a.ldz = ldz; a.ld_dyf = ld_dyf; a.ld_dyp = ld_dyp; a.lddz = lddz; a.cpad = cpad;
    a.B = B; a.H = H; a.W = W; a.C = C; a.slope = slope; a.has_bn = has_bn;
    return emul_bwd(true, a);
}
