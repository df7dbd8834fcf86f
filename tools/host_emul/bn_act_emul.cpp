// Host-emulated build of csrc/bn_act.cu (see cuda_host_emul.h): the BatchNorm / LeakyReLU / max-pool passes (plain and
// segmented) and the column statistics of z with the
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

static int finalize(const float* stat_partial, int nparts, int nseg, double count, const float* gamma, const float* beta,
                    float* running_mean, float* running_var, float momentum, float eps, float* mean, float* invstd,
                    float* scale, float* shift, float slope, float* amax_y, float* xhat_absmax, int C, int training) {
    if (!scale || !shift || C <= 0 || nseg < 1 || (!training && nseg != 1)) return -1;
    if (training ? !(stat_partial && nparts > 0) : !(running_mean && running_var)) return -1;
    if (amax_y && !training) *amax_y = 0.f;
    const double* red = nullptr;
    int S = 0;
    if (training) {
        int rps;
        stat_split(nparts, &S, &rps);
        double* scratch = reinterpret_cast<double*>(const_cast<float*>(stat_partial) + (size_t)nseg * nparts * 4 * C);
        emul::launch(dim3(ceil_div(C, 32), S, nseg), dim3(32, 32), 0,
                     [&]() {
                         if (nseg > 1) bn_stats_reduce_kernel<true>(stat_partial, nparts, rps, C, scratch, amax_y);
                         else bn_stats_reduce_kernel<false>(stat_partial, nparts, rps, C, scratch, amax_y);
                     });
        red = scratch;
    }
    emul::launch(dim3(ceil_div(C, 128), nseg), dim3(128), 0, [&]() {
        if (nseg > 1)
            bn_finalize_kernel<true>(red, S, count, gamma, beta, running_mean, running_var, momentum, eps, mean, invstd, scale,
                                     shift, slope, amax_y, xhat_absmax, C, training);
        else
            bn_finalize_kernel<false>(red, S, count, gamma, beta, running_mean, running_var, momentum, eps, mean, invstd, scale,
                                      shift, slope, amax_y, xhat_absmax, C, training);
    });
    return 0;
}

// stat_partial: nparts rows of 4C floats followed by fsdet_bn_stat_scratch_rows() rows of scratch (as on the device)
extern "C" int emul_bn_finalize(const float* stat_partial, int nparts, double count, const float* gamma, const float* beta,
                                float* running_mean, float* running_var, float momentum, float eps, float* mean, float* invstd,
                                float* scale, float* shift, float slope, float* amax_y, float* xhat_absmax, int C,
                                int training) {
    return finalize(stat_partial, nparts, 1, count, gamma, beta, running_mean, running_var, momentum, eps, mean, invstd, scale,
                    shift, slope, amax_y, xhat_absmax, C, training);
}

// nseg segments of nparts rows each, then nseg * fsdet_bn_stat_scratch_rows() rows of scratch
extern "C" int emul_bn_seg_finalize(const float* stat_partial, int nparts, int nseg, size_t seg_pix, const float* gamma,
                                    const float* beta, float* running_mean, float* running_var, float momentum, float eps,
                                    float* mean, float* invstd, float* scale, float* shift, float slope, float* amax_y,
                                    float* xhat_absmax, int C) {
    if (seg_pix == 0) return -1;
    return finalize(stat_partial, nparts, nseg, (double)seg_pix, gamma, beta, running_mean, running_var, momentum, eps, mean,
                    invstd, scale, shift, slope, amax_y, xhat_absmax, C, 1);
}

static int colstats(const float* z, int ld, long long seg_pix, int nseg, int C, float* partial) {
    if (!(z && partial && C % 4 == 0 && ld % 4 == 0 && nseg >= 1 && seg_pix >= 0)) return -1;
    if (seg_pix == 0) return 0;
    const int TCx = chan_lanes(C);
    const int TY = 256 / TCx;
    emul::launch(dim3(colstats_seg_rows(seg_pix, nseg), nseg), dim3(TCx, TY), (size_t)TY * TCx * 16 * sizeof(float),
                 [&]() { colstats_kernel(z, ld, seg_pix, C, stat_strip(seg_pix * nseg), partial); });
    return 0;
}

extern "C" int emul_colstats_rows(size_t npix) { return colstats_seg_rows((long long)npix, 1); }
extern "C" int emul_bn_seg_colstats_rows(size_t seg_pix, int nseg) { return colstats_seg_rows((long long)seg_pix, nseg); }
extern "C" int emul_colstats(const float* z, int ld, size_t npix, int C, float* partial) {
    return colstats(z, ld, (long long)npix, 1, C, partial);
}
extern "C" int emul_bn_seg_colstats(const float* z, int ld, size_t seg_pix, int nseg, int C, float* partial) {
    return colstats(z, ld, (long long)seg_pix, nseg, C, partial);
}

static int act_fwd(const float* z, int ldz, const float* scale, const float* shift, float slope, float* y_full, int ld_full,
                   float* y_pool, int ld_pool, void* full_hi, void* full_lo, void* pool_hi, void* pool_lo, int Cpad,
                   const float* amax, int B, int H, int W, int C, int nseg, int segB) {
    const bool planes = full_hi || pool_hi;
    if (!(z && scale && shift && (y_full || y_pool || planes)) || C % 4 || ldz % 4 || (y_full && ld_full % 4) ||
        (y_pool && ld_pool % 4) || (planes && !(amax && Cpad >= C && Cpad % 4 == 0)) || segB <= 0)
        return -1;
    FwdArgs a;
    a.z = z; a.scale = scale; a.shift = shift; a.amax = amax; a.yf = y_full; a.yp = y_pool;
    a.fh = (__half*)full_hi; a.fl = (__half*)full_lo; a.ph = (__half*)pool_hi; a.pl = (__half*)pool_lo;
    a.ldz = ldz; a.ldf = ld_full; a.ldp = ld_pool; a.Cpad = planes ? Cpad : C; a.B = B; a.H = H; a.W = W; a.C = C; a.slope = slope;
    a.segB = segB;
    const int CP4 = a.Cpad / 4;
    if (!y_pool && !pool_hi) {
        long long n = (long long)segB * H * W * CP4;
        if (n == 0) return 0;
        if (nseg > 1) emul::launch_serial(dim3(ceil_div(n, 256), nseg), dim3(256), [&]() { bn_act_flat_kernel<true>(a); });
        else emul::launch_serial(dim3(ceil_div(n, 256)), dim3(256), [&]() { bn_act_flat_kernel<false>(a); });
    } else {
        long long nwin = (long long)segB * ((H + 1) / 2) * ((W + 1) / 2);
        if (nwin == 0) return 0;
        const int TC = chan_lanes(C);
        const int TY = 256 / TC;
        const dim3 block(TC, TY), grid((unsigned)ceil_div(nwin, TY), nseg);
        const bool full = a.yf || a.fh;
        if (nseg > 1) {
            if (full) emul::launch_serial(grid, block, [&]() { bn_act_pool_kernel<true, true>(a); });
            else emul::launch_serial(grid, block, [&]() { bn_act_pool_kernel<false, true>(a); });
        } else {
            if (full) emul::launch_serial(grid, block, [&]() { bn_act_pool_kernel<true, false>(a); });
            else emul::launch_serial(grid, block, [&]() { bn_act_pool_kernel<false, false>(a); });
        }
    }
    return 0;
}

extern "C" int emul_bn_act_fwd(const float* z, int ldz, const float* scale, const float* shift, float slope, float* y_full,
                               int ld_full, float* y_pool, int ld_pool, void* full_hi, void* full_lo, void* pool_hi,
                               void* pool_lo, int Cpad, const float* amax, int B, int H, int W, int C) {
    return act_fwd(z, ldz, scale, shift, slope, y_full, ld_full, y_pool, ld_pool, full_hi, full_lo, pool_hi, pool_lo, Cpad, amax,
                   B, H, W, C, 1, B);
}

extern "C" int emul_bn_act_fwd_seg(const float* z, int ldz, const float* scale, const float* shift, float slope, float* y_full,
                                   int ld_full, float* y_pool, int ld_pool, void* full_hi, void* full_lo, void* pool_hi,
                                   void* pool_lo, int Cpad, const float* amax, int B, int H, int W, int C, int nseg,
                                   size_t seg_pix) {
    return act_fwd(z, ldz, scale, shift, slope, y_full, ld_full, y_pool, ld_pool, full_hi, full_lo, pool_hi, pool_lo, Cpad, amax,
                   B, H, W, C, nseg, seg_images(B, H, W, nseg, (long long)seg_pix));
}

// returns 1 when the pool-only specialisation ran, 0 for the general kernel (the same dispatch as launch_bwd)
static int emul_bwd(bool apply, const BwdArgs& a, int nseg) {
    if (a.segB <= 0) return -1;
    const int C4 = a.C / 4;
    const int TC = chan_lanes(a.C);
    const int TY = 256 / TC;
    const dim3 block(TC, TY), grid(seg_bwd_rows(a.segB, a.H, a.W, nseg), ceil_div(C4, TC), nseg);
    const size_t smem = (size_t)TY * TC * 16 * sizeof(double);
    const bool pool_only = !a.dyf && a.dyp && a.has_bn && a.slope >= 0.f && a.slope <= 1.f;
    const bool seg = nseg > 1;
    if (pool_only) {
        if (apply) emul::launch_serial(grid, block, [&]() { seg ? bn_act_bwd_pool_kernel<true, true>(a) : bn_act_bwd_pool_kernel<true, false>(a); });
        else emul::launch(grid, block, smem, [&]() { seg ? bn_act_bwd_pool_kernel<false, true>(a) : bn_act_bwd_pool_kernel<false, false>(a); });
    } else {
        if (apply) emul::launch_serial(grid, block, [&]() { seg ? bn_act_bwd_kernel<true, true>(a) : bn_act_bwd_kernel<true, false>(a); });
        else emul::launch(grid, block, smem, [&]() { seg ? bn_act_bwd_kernel<false, true>(a) : bn_act_bwd_kernel<false, false>(a); });
    }
    return pool_only ? 1 : 0;
}

extern "C" int emul_bn_seg_bwd_rows(int B, int H, int W, int nseg) { return seg_bwd_rows(B / nseg, H, W, nseg); }

static int bwd_reduce(const float* z, int ldz, const float* dy_full, int ld_dyf, const float* dy_pool, int ld_dyp,
                      const float* scale, const float* shift, const float* mean, const float* invstd, float slope,
                      double* partial, int B, int H, int W, int C, int has_bn, int nseg, int segB) {
    if (!(z && scale && shift && partial && (dy_full || dy_pool)) || (has_bn && !(mean && invstd)) || C % 4) return -1;
    BwdArgs a;
    a.z = z; a.dyf = dy_full; a.dyp = dy_pool; a.scale = scale; a.shift = shift; a.mean = mean; a.invstd = invstd;
    a.coef = nullptr; a.dz = nullptr; a.dh = nullptr; a.dl = nullptr; a.amax = nullptr; a.partial = partial;
    a.ldz = ldz; a.ld_dyf = ld_dyf; a.ld_dyp = ld_dyp; a.lddz = 0; a.cpad = 0;
    a.B = B; a.H = H; a.W = W; a.C = C; a.segB = segB; a.slope = slope; a.has_bn = has_bn;
    return emul_bwd(false, a, nseg);
}

// partial: bwd_rows(B, H, W) + 1 rows of 3C doubles
extern "C" int emul_bn_act_bwd_reduce(const float* z, int ldz, const float* dy_full, int ld_dyf, const float* dy_pool,
                                      int ld_dyp, const float* scale, const float* shift, const float* mean, const float* invstd,
                                      float slope, double* partial, int B, int H, int W, int C, int has_bn) {
    return bwd_reduce(z, ldz, dy_full, ld_dyf, dy_pool, ld_dyp, scale, shift, mean, invstd, slope, partial, B, H, W, C, has_bn, 1, B);
}

// partial: nseg * seg_bwd_rows + nseg rows of 3C doubles
extern "C" int emul_bn_act_bwd_reduce_seg(const float* z, int ldz, const float* dy_full, int ld_dyf, const float* dy_pool,
                                          int ld_dyp, const float* scale, const float* shift, const float* mean,
                                          const float* invstd, float slope, double* partial, int B, int H, int W, int C,
                                          int nseg, size_t seg_pix) {
    return bwd_reduce(z, ldz, dy_full, ld_dyf, dy_pool, ld_dyp, scale, shift, mean, invstd, slope, partial, B, H, W, C, 1, nseg,
                      seg_images(B, H, W, nseg, (long long)seg_pix));
}

static int bwd_finalize(const double* partial, int nparts, int nseg, double count, const float* gamma, const float* invstd,
                        const float* xhat_absmax, float* dgamma, float* dbeta, double* coef, float* amax_bound, int C,
                        int has_bn) {
    if (!(partial && nparts > 0 && C > 0 && nseg >= 1) || (has_bn && !(coef && gamma && invstd)) ||
        (amax_bound && has_bn && !xhat_absmax))
        return -1;
    double* sums = const_cast<double*>(partial) + (size_t)nseg * nparts * 3 * C;
    emul::launch(dim3(ceil_div(3 * C, 32), nseg), dim3(32, 32), 0,
                 [&]() {
                     if (nseg > 1) colsum_dd_kernel<true>(partial, nparts, 3 * C, 2 * C, sums, amax_bound);
                     else colsum_dd_kernel<false>(partial, nparts, 3 * C, 2 * C, sums, amax_bound);
                 });
    emul::launch_serial(dim3(ceil_div(C, 128)), dim3(128), [&]() {
        if (nseg > 1) bn_bwd_finalize_kernel<true>(sums, count, gamma, invstd, xhat_absmax, dgamma, dbeta, coef, amax_bound, C, has_bn, nseg);
        else bn_bwd_finalize_kernel<false>(sums, count, gamma, invstd, xhat_absmax, dgamma, dbeta, coef, amax_bound, C, has_bn, 1);
    });
    return 0;
}

extern "C" int emul_bn_bwd_finalize(const double* partial, int nparts, double count, const float* gamma, const float* invstd,
                                    const float* xhat_absmax, float* dgamma, float* dbeta, double* coef, float* amax_bound,
                                    int C, int has_bn) {
    return bwd_finalize(partial, nparts, 1, count, gamma, invstd, xhat_absmax, dgamma, dbeta, coef, amax_bound, C, has_bn);
}

extern "C" int emul_bn_bwd_finalize_seg(const double* partial, int nparts, int nseg, size_t seg_pix, const float* gamma,
                                        const float* invstd, const float* xhat_absmax, float* dgamma, float* dbeta,
                                        double* coef, float* amax_bound, int C) {
    return bwd_finalize(partial, nparts, nseg, (double)seg_pix, gamma, invstd, xhat_absmax, dgamma, dbeta, coef, amax_bound, C, 1);
}

static int bwd_apply(const float* z, int ldz, const float* dy_full, int ld_dyf, const float* dy_pool, int ld_dyp,
                     const float* scale, const float* shift, const float* mean, const float* invstd, const double* coef,
                     float slope, float* dz, int lddz, void* dz_hi, void* dz_lo, int cpad, const float* amax, int B, int H,
                     int W, int C, int has_bn, int nseg, int segB) {
    if (!(z && scale && shift && (dz || dz_hi) && (dy_full || dy_pool)) || (has_bn && !(mean && invstd && coef)) || C % 4 ||
        (dz_hi && !(dz_lo && amax && cpad == C)))
        return -1;
    BwdArgs a;
    a.z = z; a.dyf = dy_full; a.dyp = dy_pool; a.scale = scale; a.shift = shift; a.mean = mean; a.invstd = invstd;
    a.coef = coef; a.dz = dz; a.dh = (__half*)dz_hi; a.dl = (__half*)dz_lo; a.amax = amax; a.partial = nullptr;
    a.ldz = ldz; a.ld_dyf = ld_dyf; a.ld_dyp = ld_dyp; a.lddz = lddz; a.cpad = cpad;
    a.B = B; a.H = H; a.W = W; a.C = C; a.segB = segB; a.slope = slope; a.has_bn = has_bn;
    return emul_bwd(true, a, nseg);
}

extern "C" int emul_bn_act_bwd_apply(const float* z, int ldz, const float* dy_full, int ld_dyf, const float* dy_pool,
                                     int ld_dyp, const float* scale, const float* shift, const float* mean, const float* invstd,
                                     const double* coef, float slope, float* dz, int lddz, void* dz_hi, void* dz_lo, int cpad,
                                     const float* amax, int B, int H, int W, int C, int has_bn) {
    return bwd_apply(z, ldz, dy_full, ld_dyf, dy_pool, ld_dyp, scale, shift, mean, invstd, coef, slope, dz, lddz, dz_hi, dz_lo,
                     cpad, amax, B, H, W, C, has_bn, 1, B);
}

extern "C" int emul_bn_act_bwd_apply_seg(const float* z, int ldz, const float* dy_full, int ld_dyf, const float* dy_pool,
                                         int ld_dyp, const float* scale, const float* shift, const float* mean,
                                         const float* invstd, const double* coef, float slope, float* dz, int lddz, void* dz_hi,
                                         void* dz_lo, int cpad, const float* amax, int B, int H, int W, int C, int nseg,
                                         size_t seg_pix) {
    return bwd_apply(z, ldz, dy_full, ld_dyf, dy_pool, ld_dyp, scale, shift, mean, invstd, coef, slope, dz, lddz, dz_hi, dz_lo,
                     cpad, amax, B, H, W, C, 1, nseg, seg_images(B, H, W, nseg, (long long)seg_pix));
}
