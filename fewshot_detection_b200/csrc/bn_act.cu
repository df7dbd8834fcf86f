// Train/eval BatchNorm2d + LeakyReLU(0.1) + MaxPool2d(2,2) fused passes over
// NHWC fp32 activations (HBM-bound; float4 along channels, coalesced).
//
// Replaces nn.BatchNorm2d / nn.LeakyReLU / nn.MaxPool2d of the reference's conv
// blocks (darknet_meta.py:240-268) and their autograd backward.
//
//   forward : conv kernel writes pre-BN z once (+ per-CTA sum / sum-of-squares; or colstats reads z once more)
//             bn_finalize  -> mean, invstd, scale = gamma*invstd, shift = beta - mean*scale
//             bn_act_fwd   -> y = leaky(z*scale+shift) [and/or its 2x2/2 max-pool]
//   backward: bn_act_bwd_reduce -> sum(du), sum(du*xhat) partials (du = dy through pool+leaky)
//             bn_bwd_finalize   -> dgamma, dbeta, c1 = dbeta/N, c2 = dgamma/N
//             bn_act_bwd_apply  -> dz = scale*(du - c1 - xhat*c2)
//
// Segments: every pass also runs on a batch split into `nseg` contiguous segments of whole images, each normalised
// with its own batch statistics (the per-replica BatchNorm of nn.DataParallel).  One launch covers all segments: the
// segment is a grid dimension, per-segment vectors are [nseg][C] and partial rows never straddle a segment.  The
// element-wise kernels take a SEG template flag: their one-segment instantiation is the plain pass, instruction for
// instruction.
#include <cuda_fp16.h>

#include "common.cuh"

// tools/host_emul compiles this file with g++ (threads = OS threads) to test the kernels without a GPU
#ifdef FSDET_HOST_EMULATION
#define FSDET_DYN_SMEM_F64(name) double* name = reinterpret_cast<double*>(emul::g_dyn_smem)
#else
#define FSDET_DYN_SMEM_F64(name) extern __shared__ double name[]
#endif

namespace fsdet {

// power-of-two scale that maps a tensor with absolute maximum `a` into [512, 1024)  (same rule as conv_tc.cu)
__device__ __forceinline__ float plane_scale(float a) {
    if (!(a > 0.f) || !isfinite(a)) return 1.f;
    int ex = (int)((__float_as_uint(a) >> 23) & 0xff) - 126;
    int e = 10 - ex;
    e = e < -60 ? -60 : (e > 60 ? 60 : e);
    return __uint_as_float((uint32_t)(e + 127) << 23);
}

__device__ __forceinline__ void store_planes4(__half* hi, __half* lo, long long off, float4 v, float sc) {
    const float f[4] = {v.x * sc, v.y * sc, v.z * sc, v.w * sc};
    __half h[4], l[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        h[k] = __float2half_rn(f[k]);
        l[k] = __float2half_rn(f[k] - __half2float(h[k]));
    }
    *reinterpret_cast<uint2*>(hi + off) = *reinterpret_cast<uint2*>(h);
    *reinterpret_cast<uint2*>(lo + off) = *reinterpret_cast<uint2*>(l);
}


// ------------------------------------------------------------------ column statistics of z (BN partials)
// grid (strips per segment, nseg): one CTA per strip of `strip` pixels of segment blockIdx.y (a strip ends at its
// segment's end); partial[blockIdx.y * gridDim.x + blockIdx.x] = [sum(C) | sum of squares(C) | min(C) | max(C)]
__global__ void __launch_bounds__(256) colstats_kernel(const float* __restrict__ z, int ld, long long seg_pix, int C, int strip,
                                                       float* __restrict__ part) {
    // threads: x = channel vector lane (float4), y = pixel lane
    const int C4 = C >> 2;
    const int TC = blockDim.x, TY = blockDim.y;
    const long long send = (long long)(blockIdx.y + 1) * seg_pix;
    long long p0 = (long long)blockIdx.y * seg_pix + (long long)blockIdx.x * strip, p1 = p0 + strip < send ? p0 + strip : send;
    const long long row = (long long)blockIdx.y * gridDim.x + blockIdx.x;
    FSDET_DYN_SMEM_F64(red_d);
    float* red = reinterpret_cast<float*>(red_d);  // [TY][TC*16]
    for (int cv0 = 0; cv0 < C4; cv0 += TC) {
        int cv = cv0 + threadIdx.x;
        float s[4] = {0, 0, 0, 0}, q[4] = {0, 0, 0, 0};
        float mn[4] = {INFINITY, INFINITY, INFINITY, INFINITY}, mx[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
        if (cv < C4)
            for (long long p = p0 + threadIdx.y; p < p1; p += 4 * TY) {   // four loads in flight, accumulated in row order
                float4 v[4];
#pragma unroll
                for (int u = 0; u < 4; ++u)
                    if (p + u * TY < p1) v[u] = ldg4(z + (p + u * TY) * ld + cv * 4);
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    if (p + u * TY >= p1) break;
                    const float f[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        s[k] += f[k]; q[k] += f[k] * f[k]; mn[k] = fminf(mn[k], f[k]); mx[k] = fmaxf(mx[k], f[k]);
                    }
                }
            }
        float* mine = red + ((size_t)threadIdx.y * TC + threadIdx.x) * 16;
#pragma unroll
        for (int k = 0; k < 4; ++k) { mine[k] = s[k]; mine[4 + k] = q[k]; mine[8 + k] = mn[k]; mine[12 + k] = mx[k]; }
        __syncthreads();
        // column j = (channel lane, statistic, component) reduced over the TY pixel lanes in a fixed order, all threads busy
        for (int j = threadIdx.y * TC + threadIdx.x; j < TC * 16; j += TC * TY) {
            const int lane = j >> 4, stat = (j >> 2) & 3, comp = j & 3;
            if (cv0 + lane >= C4) continue;
            float t = red[j];
            for (int r = 1; r < TY; ++r) {
                const float o = red[(size_t)r * TC * 16 + j];
                t = stat < 2 ? t + o : (stat == 2 ? fminf(t, o) : fmaxf(t, o));
            }
            part[row * 4 * C + stat * C + (cv0 + lane) * 4 + comp] = t;
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------ finalize (fwd)
// generic double-precision column sums of float partial rows (used by the backward finalize of the bias path)
__global__ void __launch_bounds__(1024) colsum_double_kernel(const float* __restrict__ part, int nparts, int ncols,
                                                             double* __restrict__ out) {
    __shared__ double red[32][33];
    int col = blockIdx.x * 32 + threadIdx.x;
    double s = 0.0;
    if (col < ncols)
        for (int r = threadIdx.y; r < nparts; r += 32) s += (double)part[(long long)r * ncols + col];
    red[threadIdx.y][threadIdx.x] = s;
    __syncthreads();
    if (threadIdx.y == 0 && col < ncols) {
        double t = 0.0;
        for (int i = 0; i < 32; ++i) t += red[i][threadIdx.x];
        out[col] = t;
    }
}

// reduction over the double-precision partial rows of the backward pass: columns [0, nsum) are summed (fixed
// order), columns [nsum, ncols) hold maxima
// `zero`: optional device float cleared here (the atomicMax target of the kernel that follows on the same stream - one graph
// node less than a memset per layer).  blockIdx.y: segment (its nparts rows -> its row of out)
template <bool SEG>
__global__ void __launch_bounds__(1024) colsum_dd_kernel(const double* __restrict__ part, int nparts, int ncols, int nsum,
                                                         double* __restrict__ out, float* __restrict__ zero) {
    __shared__ double red[32][33];
    if (zero && blockIdx.x == 0 && (!SEG || blockIdx.y == 0) && threadIdx.x == 0 && threadIdx.y == 0) *zero = 0.f;
    if (SEG) {
        part += (long long)blockIdx.y * nparts * ncols;
        out += (long long)blockIdx.y * ncols;
    }
    int col = blockIdx.x * 32 + threadIdx.x;
    const bool is_max = col >= nsum;
    double s = 0.0;
    if (col < ncols)
        for (int r = threadIdx.y; r < nparts; r += 32) {
            const double v = part[(long long)r * ncols + col];
            s = is_max ? fmax(s, v) : s + v;
        }
    red[threadIdx.y][threadIdx.x] = s;
    __syncthreads();
    if (threadIdx.y == 0 && col < ncols) {
        double t = 0.0;
        for (int i = 0; i < 32; ++i) t = is_max ? fmax(t, red[i][threadIdx.x]) : t + red[i][threadIdx.x];
        out[col] = t;
    }
}

// Stage 1: grid (ceil(C/32), S, nseg): block (x, y, z) reduces rows [y*rps, (y+1)*rps) of segment z's conv partial
// rows [nparts][4C] = (sum | sum of squares | min | max) into red[z][y][4C] (doubles; sums accumulated in double).
template <bool SEG>
__global__ void __launch_bounds__(1024) bn_stats_reduce_kernel(const float* __restrict__ part, int nparts, int rps, int C,
                                                               double* __restrict__ red, float* __restrict__ zero) {
    __shared__ double rs[32][33], rq[32][33];
    __shared__ float rn[32][33], rx[32][33];
    if (zero && blockIdx.x == 0 && blockIdx.y == 0 && (!SEG || blockIdx.z == 0) && threadIdx.x == 0 && threadIdx.y == 0)
        *zero = 0.f;   // see colsum_dd_kernel
    if (SEG) {
        part += (long long)blockIdx.z * nparts * 4 * C;
        red += (long long)blockIdx.z * gridDim.y * 4 * C;
    }
    const int c = blockIdx.x * 32 + threadIdx.x;
    const int r0 = blockIdx.y * rps;
    const int r1 = min(r0 + rps, nparts);
    double s = 0.0, q = 0.0;
    float mn = INFINITY, mx = -INFINITY;
    if (c < C) {
        for (int r = r0 + threadIdx.y; r < r1; r += 32) {
            const float* row = part + (long long)r * 4 * C;
            s += (double)row[c];
            q += (double)row[C + c];
            mn = fminf(mn, row[2 * C + c]);
            mx = fmaxf(mx, row[3 * C + c]);
        }
    }
    rs[threadIdx.y][threadIdx.x] = s; rq[threadIdx.y][threadIdx.x] = q;
    rn[threadIdx.y][threadIdx.x] = mn; rx[threadIdx.y][threadIdx.x] = mx;
    __syncthreads();
    if (threadIdx.y == 0 && c < C) {
        s = 0.0; q = 0.0; mn = INFINITY; mx = -INFINITY;
        for (int i = 0; i < 32; ++i) {
            s += rs[i][threadIdx.x]; q += rq[i][threadIdx.x];
            mn = fminf(mn, rn[i][threadIdx.x]); mx = fmaxf(mx, rx[i][threadIdx.x]);
        }
        double* dst = red + (long long)blockIdx.y * 4 * C;
        dst[c] = s; dst[C + c] = q; dst[2 * C + c] = (double)mn; dst[3 * C + c] = (double)mx;
    }
}

// Stage 2: fold the S reduced rows, derive mean / invstd / scale / shift, update the running statistics and - from
// the per-channel range of z and the monotonicity of y = leaky(scale*z + shift) in z - the exact absolute maximum
// of the activation.  One thread per channel; blockIdx.y: segment (vectors [nseg][C], `count` pixels each).  The
// running statistics follow segment 0 only (nn.DataParallel keeps replica 0's buffers); amax_y spans all segments.
template <bool SEG>
__global__ void __launch_bounds__(128) bn_finalize_kernel(const double* __restrict__ red, int S, double count,
                                                          const float* __restrict__ gamma, const float* __restrict__ beta,
                                                          float* __restrict__ running_mean, float* __restrict__ running_var,
                                                          float momentum, float eps, float* __restrict__ mean,
                                                          float* __restrict__ invstd, float* __restrict__ scale,
                                                          float* __restrict__ shift, float slope, float* __restrict__ amax_y,
                                                          float* __restrict__ xhat_absmax, int C, int training) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (SEG) {
        const int seg = blockIdx.y;
        red += (long long)seg * S * 4 * C;
        if (seg > 0) running_mean = running_var = nullptr;
        if (mean) mean += seg * C;
        if (invstd) invstd += seg * C;
        scale += seg * C;
        shift += seg * C;
        if (xhat_absmax) xhat_absmax += seg * C;
    }
    float ymax = 0.f;
    if (c < C) {
        float m, is;
        float mn = INFINITY, mx = -INFINITY;
        if (training) {
            double s = 0.0, q = 0.0;
#pragma unroll 8
            for (int i = 0; i < S; ++i) {
                const double* row = red + (long long)i * 4 * C;
                s += row[c]; q += row[C + c];
                mn = fminf(mn, (float)row[2 * C + c]); mx = fmaxf(mx, (float)row[3 * C + c]);
            }
            double mu = s / count;
            double var = q / count - mu * mu;
            if (var < 0.0) var = 0.0;
            m = (float)mu;
            is = (float)(1.0 / sqrt(var + (double)eps));
            if (running_mean) {
                double unbiased = count > 1.0 ? var * count / (count - 1.0) : var;
                running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * m;
                running_var[c] = (1.f - momentum) * running_var[c] + momentum * (float)unbiased;
            }
        } else {
            m = running_mean[c];
            is = 1.f / sqrtf(running_var[c] + eps);
        }
        float g = gamma ? gamma[c] : 1.f;
        float b = beta ? beta[c] : 0.f;
        float sc = g * is;
        float sh = b - m * sc;
        if (mean) mean[c] = m;
        if (invstd) invstd[c] = is;
        scale[c] = sc;
        shift[c] = sh;
        if (training && mn <= mx) {
            ymax = fmaxf(fabsf(leaky(fmaf(mn, sc, sh), slope)), fabsf(leaky(fmaf(mx, sc, sh), slope)));
            // max |xhat| with xhat = (z - mean) * invstd evaluated exactly as the backward kernels do (monotone in z)
            if (xhat_absmax) xhat_absmax[c] = fmaxf(fabsf((mn - m) * is), fabsf((mx - m) * is));
        } else if (xhat_absmax) {
            xhat_absmax[c] = 0.f;
        }
    }
    if (amax_y && training) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) ymax = fmaxf(ymax, __shfl_xor_sync(0xffffffffu, ymax, o));
        if ((threadIdx.x & 31) == 0 && isfinite(ymax)) atomicMax(reinterpret_cast<int*>(amax_y), __float_as_int(ymax));
    }
}

// ------------------------------------------------------------------ forward
struct FwdArgs {
    const float* z;
    const float* scale;
    const float* shift;
    const float* amax;   // device scalar the fp16 planes are scaled by (plane_scale)
    float* yf;           // fp32 full-resolution output (optional)
    float* yp;           // fp32 pooled output (optional)
    __half *fh, *fl;     // fp16 hi/lo planes of the full-resolution output [npix][Cpad] (optional)
    __half *ph, *pl;     // fp16 hi/lo planes of the pooled output (optional)
    int ldz, ldf, ldp, Cpad;
    int B, H, W, C;
    int segB;            // images per segment (blockIdx.y = segment; scale / shift are [nseg][C])
    float slope;
};

__device__ __forceinline__ float4 act4(float4 v, float4 sc, float4 sh, float slope) {
    v.x = leaky(fmaf(v.x, sc.x, sh.x), slope);
    v.y = leaky(fmaf(v.y, sc.y, sh.y), slope);
    v.z = leaky(fmaf(v.z, sc.z, sh.z), slope);
    v.w = leaky(fmaf(v.w, sc.w, sh.w), slope);
    return v;
}

// no pooling: one thread = one pixel x 4 channels (channel index runs to Cpad: the zero padding of the planes)
// SEG: segments (blockIdx.y); the one-segment instantiation is the plain pass
template <bool SEG>
__global__ void __launch_bounds__(256) bn_act_flat_kernel(const FwdArgs a) {
    const unsigned CP4 = a.Cpad >> 2;
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;   // host guarantees npix * CP4 < 2^31
    const unsigned npix = (unsigned)(SEG ? a.segB : a.B) * a.H * a.W;   // of this segment
    if (i >= npix * CP4) return;
    const unsigned pu = i / CP4;
    const long long p = SEG ? (long long)blockIdx.y * npix + pu : (long long)pu;
    const int c = (int)(i - pu * CP4) * 4;
    const int vc = SEG ? blockIdx.y * a.C + c : c;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c < a.C) {
        v = act4(ldg4(a.z + p * a.ldz + c), ldg4(a.scale + vc), ldg4(a.shift + vc), a.slope);
        if (a.yf) *reinterpret_cast<float4*>(a.yf + p * a.ldf + c) = v;
    }
    if (a.fh) store_planes4(a.fh, a.fl, p * a.Cpad + c, v, plane_scale(__ldg(a.amax)));
}

// block (TC channel-vector lanes, TY windows): one thread = one 2x2 window x 4 channels per pass over the channel
// lanes; windows cover ceil(H/2) x ceil(W/2).  FULL = some full-resolution output is wanted; otherwise only the
// pooled activation is produced, from max(leaky(y)) == leaky(max(y)) (leaky is monotone).
template <bool FULL, bool SEG>
__global__ void __launch_bounds__(256) bn_act_pool_kernel(const FwdArgs a) {
    const int H = a.H, W = a.W;
    const int H2 = (H + 1) >> 1, W2 = (W + 1) >> 1, Hp = H >> 1, Wp = W >> 1;
    const int CP4 = a.Cpad >> 2;
    const unsigned wi = blockIdx.x * blockDim.y + threadIdx.y;   // host guarantees B*H*W < 2^31
    if (wi >= (unsigned)(SEG ? a.segB : a.B) * H2 * W2) return;
    const unsigned t = wi / W2;
    const int w2 = (int)(wi - t * W2);
    const int bl = (int)(t / H2);
    const int h2 = (int)(t - (unsigned)bl * H2);
    const int b = SEG ? blockIdx.y * a.segB + bl : bl;
    const float* scale = SEG ? a.scale + blockIdx.y * a.C : a.scale;
    const float* shift = SEG ? a.shift + blockIdx.y * a.C : a.shift;
    const bool whole = h2 < Hp && w2 < Wp;
    if (!FULL && !whole) return;                                 // no pooled output for windows cut by an odd edge
    const float psc = (a.fh || a.ph) ? plane_scale(__ldg(a.amax)) : 1.f;
    const float slope = a.slope;
    const unsigned p00 = ((unsigned)b * H + 2 * h2) * W + 2 * w2;
    const unsigned pp = ((unsigned)b * Hp + h2) * Wp + w2;
    for (int cv = threadIdx.x; cv < CP4; cv += blockDim.x) {
        const int c = cv * 4;
        const bool cok = c < a.C;
        float4 sc = make_float4(0, 0, 0, 0), sh = sc;
        if (cok) { sc = ldg4(scale + c); sh = ldg4(shift + c); }
        float4 mx;
        if (FULL) {
            mx = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                if (2 * h2 + (q >> 1) < H && 2 * w2 + (q & 1) < W) {
                    const unsigned p = p00 + (q >> 1) * W + (q & 1);
                    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (cok) {
                        v = act4(ldg4(a.z + (size_t)p * a.ldz + c), sc, sh, slope);
                        if (a.yf) *reinterpret_cast<float4*>(a.yf + (size_t)p * a.ldf + c) = v;
                    }
                    if (a.fh) store_planes4(a.fh, a.fl, (long long)p * a.Cpad + c, v, psc);
                    mx.x = fmaxf(mx.x, v.x); mx.y = fmaxf(mx.y, v.y); mx.z = fmaxf(mx.z, v.z); mx.w = fmaxf(mx.w, v.w);
                }
            }
        } else {
            mx = make_float4(0.f, 0.f, 0.f, 0.f);
            if (cok) {
                float4 v[4];
#pragma unroll
                for (int q = 0; q < 4; ++q) v[q] = ldg4(a.z + (size_t)(p00 + (q >> 1) * W + (q & 1)) * a.ldz + c);
                float4 y;
                y.x = fmaxf(fmaxf(fmaf(v[0].x, sc.x, sh.x), fmaf(v[1].x, sc.x, sh.x)), fmaxf(fmaf(v[2].x, sc.x, sh.x), fmaf(v[3].x, sc.x, sh.x)));
                y.y = fmaxf(fmaxf(fmaf(v[0].y, sc.y, sh.y), fmaf(v[1].y, sc.y, sh.y)), fmaxf(fmaf(v[2].y, sc.y, sh.y), fmaf(v[3].y, sc.y, sh.y)));
                y.z = fmaxf(fmaxf(fmaf(v[0].z, sc.z, sh.z), fmaf(v[1].z, sc.z, sh.z)), fmaxf(fmaf(v[2].z, sc.z, sh.z), fmaf(v[3].z, sc.z, sh.z)));
                y.w = fmaxf(fmaxf(fmaf(v[0].w, sc.w, sh.w), fmaf(v[1].w, sc.w, sh.w)), fmaxf(fmaf(v[2].w, sc.w, sh.w), fmaf(v[3].w, sc.w, sh.w)));
                mx = make_float4(leaky(y.x, slope), leaky(y.y, slope), leaky(y.z, slope), leaky(y.w, slope));
            }
        }
        if (whole) {
            if (a.yp && cok) *reinterpret_cast<float4*>(a.yp + (size_t)pp * a.ldp + c) = mx;
            if (a.ph) store_planes4(a.ph, a.pl, (long long)pp * a.Cpad + c, mx, psc);
        }
    }
}

// ----------------------------------------------------------------- backward
struct BwdArgs {
    const float* z;
    const float* dyf;
    const float* dyp;
    const float* scale;
    const float* shift;
    const float* mean;
    const float* invstd;
    const double* coef;
    float* dz;
    __half* dh;
    __half* dl;
    const float* amax;
    double* partial;
    int ldz, ld_dyf, ld_dyp, lddz, cpad;
    int B, H, W, C;
    int segB;            // images per segment (blockIdx.z = segment; vectors [nseg][C], coef [nseg][2C])
    float slope;
    int has_bn;
};

// compensated (Kahan) fp32 accumulation: (s, e) carries ~48 bits, read back as (double)s - (double)e
__device__ __forceinline__ void kahan_add(float& s, float& e, float x) {
    const float y = x - e;
    const float t = s + y;
    e = (t - s) - y;
    s = t;
}

// reduce-pass epilogue: red[blockDim.y][TC*16] doubles (per thread: 4 x sum(du), 4 x sum(du*xhat), 4 x max|du|,
// 4 unused) -> one partial row [3C]; column j is reduced over the blockDim.y lanes in a fixed order, all threads busy
__device__ __forceinline__ void bwd_block_reduce(const double* red, double* dst, int C, int cv0) {
    const int TC = blockDim.x, TY = blockDim.y;
    for (int j = threadIdx.y * TC + threadIdx.x; j < TC * 16; j += TC * TY) {
        const int lane = j >> 4, stat = (j >> 2) & 3, comp = j & 3;
        const int ch = (cv0 + lane) * 4 + comp;
        if (ch >= C || stat == 3) continue;
        double t = red[j];
        for (int r = 1; r < TY; ++r) {
            const double o = red[(size_t)r * TC * 16 + j];
            t = stat < 2 ? t + o : fmax(t, o);
        }
        dst[stat * C + ch] = t;
    }
}

// The BN-backward projection dz = scale*(du - mean(du) - xhat*mean(du*xhat)) cancels heavily when du is dominated
// by its per-channel mean.  The sums are therefore accumulated to double-precision accuracy (compensated fp32 per
// thread, double across threads), the coefficients are computed in double, and the apply pass subtracts mean(du)
// as a (hi, lo) float pair: a difference of close floats is exact, so nothing is lost to the cancellation.
// REDUCE writes per CTA row [sum(du) | sum(du*xhat) | max|du|] (3C doubles).
// APPLY writes dz as fp32 and/or directly as the scaled fp16 (hi, lo) planes the tensor-core GEMMs read.
template <bool APPLY, bool SEG>
__global__ void __launch_bounds__(256, 3) bn_act_bwd_kernel(const BwdArgs a) {
    const int H2 = (a.H + 1) >> 1, W2 = (a.W + 1) >> 1, Hp = a.H >> 1, Wp = a.W >> 1;
    const int C4 = a.C >> 2;
    const int TC = blockDim.x;          // channel-vector lanes
    const int cv = blockIdx.y * TC + threadIdx.x;
    const bool cok = cv < C4;
    const int c = cv * 4;
    const int vc = SEG ? blockIdx.z * a.C + c : c;   // per-segment vectors [nseg][C], coef [nseg][2C]
    const int cc = SEG ? blockIdx.z * a.C : 0;
    const long long nwin = (long long)(SEG ? a.segB : a.B) * H2 * W2;

    float scv[4] = {1, 1, 1, 1}, shv[4] = {0, 0, 0, 0}, muv[4] = {0, 0, 0, 0}, isv[4] = {1, 1, 1, 1};
    float c1h[4] = {0, 0, 0, 0}, c1l[4] = {0, 0, 0, 0}, c2f[4] = {0, 0, 0, 0};
    if (cok) {
        const float4 sc = ldg4(a.scale + vc), sh = ldg4(a.shift + vc);
        scv[0] = sc.x; scv[1] = sc.y; scv[2] = sc.z; scv[3] = sc.w;
        shv[0] = sh.x; shv[1] = sh.y; shv[2] = sh.z; shv[3] = sh.w;
        if (a.has_bn) {
            const float4 mu = ldg4(a.mean + vc), is = ldg4(a.invstd + vc);
            muv[0] = mu.x; muv[1] = mu.y; muv[2] = mu.z; muv[3] = mu.w;
            isv[0] = is.x; isv[1] = is.y; isv[2] = is.z; isv[3] = is.w;
        }
        if (APPLY && a.has_bn) {
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const double c1 = a.coef[vc + cc + k];
                c1h[k] = (float)c1;
                c1l[k] = (float)(c1 - (double)c1h[k]);
                c2f[k] = (float)a.coef[vc + cc + a.C + k];
            }
        }
    }
    const float psc = (APPLY && a.dh) ? plane_scale(__ldg(a.amax)) : 1.f;
    float s1[4] = {0, 0, 0, 0}, e1[4] = {0, 0, 0, 0}, s2[4] = {0, 0, 0, 0}, e2[4] = {0, 0, 0, 0};
    float md[4] = {0, 0, 0, 0};

    for (unsigned wi = blockIdx.x * blockDim.y + threadIdx.y; cok && wi < (unsigned)nwin; wi += gridDim.x * blockDim.y) {
        const unsigned t = wi / W2;
        const int w2 = (int)(wi - t * W2);
        const int bl = (int)(t / H2);
        const int h2 = (int)(t - (unsigned)bl * H2);
        const int b = SEG ? blockIdx.z * a.segB + bl : bl;
        float zv[4][4], yv[4][4];
        long long pix[4];
        bool ok[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            int h = h2 * 2 + (q >> 1), w = w2 * 2 + (q & 1);
            ok[q] = h < a.H && w < a.W;
            pix[q] = ((long long)b * a.H + h) * a.W + w;
            float4 v = ok[q] ? ldg4(a.z + pix[q] * a.ldz + c) : make_float4(0, 0, 0, 0);
            zv[q][0] = v.x; zv[q][1] = v.y; zv[q][2] = v.z; zv[q][3] = v.w;
        }
        float du[4][4];
#pragma unroll
        for (int q = 0; q < 4; ++q)
#pragma unroll
            for (int k = 0; k < 4; ++k) { yv[q][k] = fmaf(zv[q][k], scv[k], shv[k]); du[q][k] = 0.f; }
        if (a.dyf) {
#pragma unroll
            for (int q = 0; q < 4; ++q)
                if (ok[q]) {
                    float4 g = ldg4(a.dyf + pix[q] * a.ld_dyf + c);
                    du[q][0] = g.x; du[q][1] = g.y; du[q][2] = g.z; du[q][3] = g.w;
                }
        }
        if (a.dyp && h2 < Hp && w2 < Wp) {
            long long pp = ((long long)b * Hp + h2) * Wp + w2;
            float4 g = ldg4(a.dyp + pp * a.ld_dyp + c);
            const float gv[4] = {g.x, g.y, g.z, g.w};
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                // first maximum of the activated values in scan order (torch max_pool2d: strict >)
                int best = 0;
                float bv = leaky(yv[0][k], a.slope);
#pragma unroll
                for (int q = 1; q < 4; ++q) {
                    float v = leaky(yv[q][k], a.slope);
                    if (v > bv) { bv = v; best = q; }
                }
#pragma unroll
                for (int q = 0; q < 4; ++q)
                    if (q == best) du[q][k] += gv[k];
            }
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            if (!ok[q]) continue;
            float o[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const float d = du[q][k] * (yv[q][k] > 0.f ? 1.f : a.slope);
                const float xh = (zv[q][k] - muv[k]) * isv[k];
                if (APPLY) {
                    o[k] = a.has_bn ? scv[k] * fmaf(-xh, c2f[k], (d - c1h[k]) - c1l[k]) : d;
                } else {
                    kahan_add(s1[k], e1[k], d);
                    kahan_add(s2[k], e2[k], d * xh);
                    md[k] = fmaxf(md[k], fabsf(d));
                }
            }
            if (APPLY) {
                const float4 ov = make_float4(o[0], o[1], o[2], o[3]);
                if (a.dz) *reinterpret_cast<float4*>(a.dz + pix[q] * a.lddz + c) = ov;
                if (a.dh) store_planes4(a.dh, a.dl, pix[q] * a.cpad + c, ov, psc);
            }
        }
    }

    if (!APPLY) {
        // reduce over threadIdx.y -> one partial row per blockIdx.x
        FSDET_DYN_SMEM_F64(red);  // [blockDim.y][TC*16]
        double* mine = red + ((size_t)threadIdx.y * TC + threadIdx.x) * 16;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            mine[k] = (double)s1[k] - (double)e1[k];
            mine[4 + k] = (double)s2[k] - (double)e2[k];
            mine[8 + k] = (double)md[k];
        }
        __syncthreads();
        bwd_block_reduce(red, a.partial + ((SEG ? (long long)blockIdx.z * gridDim.x : 0ll) + blockIdx.x) * 3 * a.C, a.C, blockIdx.y * TC);
    }
}

// Specialisation for the common block conv + BN + leaky + maxpool whose full-resolution output has no other
// consumer (only dy_pool exists): du is non-zero only at the arg-max pixel of each 2x2 window, so the reduce pass
// touches one element per window and channel, and the apply pass needs the activation derivative only there.
// Same arithmetic as the general kernel (the zero terms are dropped), a fraction of the instructions.
template <bool APPLY, bool SEG>
__global__ void __launch_bounds__(256, 3) bn_act_bwd_pool_kernel(const BwdArgs a) {
    const int H2 = (a.H + 1) >> 1, W2 = (a.W + 1) >> 1, Hp = a.H >> 1, Wp = a.W >> 1;
    const int C4 = a.C >> 2;
    const int TC = blockDim.x;          // channel-vector lanes
    const int cv = blockIdx.y * TC + threadIdx.x;
    const bool cok = cv < C4;
    const int c = cv * 4;
    const int vc = SEG ? blockIdx.z * a.C + c : c;
    const int cc = SEG ? blockIdx.z * a.C : 0;
    const unsigned nwin = (unsigned)(SEG ? a.segB : a.B) * H2 * W2;

    float scv[4] = {1, 1, 1, 1}, shv[4] = {0, 0, 0, 0}, muv[4] = {0, 0, 0, 0}, isv[4] = {1, 1, 1, 1};
    float c1h[4] = {0, 0, 0, 0}, c1l[4] = {0, 0, 0, 0}, c2f[4] = {0, 0, 0, 0}, t0[4] = {0, 0, 0, 0};
    if (cok) {
        const float4 sc = ldg4(a.scale + vc), sh = ldg4(a.shift + vc), mu = ldg4(a.mean + vc), is = ldg4(a.invstd + vc);
        scv[0] = sc.x; scv[1] = sc.y; scv[2] = sc.z; scv[3] = sc.w;
        shv[0] = sh.x; shv[1] = sh.y; shv[2] = sh.z; shv[3] = sh.w;
        muv[0] = mu.x; muv[1] = mu.y; muv[2] = mu.z; muv[3] = mu.w;
        isv[0] = is.x; isv[1] = is.y; isv[2] = is.z; isv[3] = is.w;
        if (APPLY) {
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const double c1 = a.coef[vc + cc + k];
                c1h[k] = (float)c1;
                c1l[k] = (float)(c1 - (double)c1h[k]);
                c2f[k] = (float)a.coef[vc + cc + a.C + k];
                t0[k] = (0.f - c1h[k]) - c1l[k];     // du == 0
            }
        }
    }
    const float psc = (APPLY && a.dh) ? plane_scale(__ldg(a.amax)) : 1.f;
    const float slope = a.slope;
    float s1[4] = {0, 0, 0, 0}, e1[4] = {0, 0, 0, 0}, s2[4] = {0, 0, 0, 0}, e2[4] = {0, 0, 0, 0};
    float md[4] = {0, 0, 0, 0};

    for (unsigned wi = blockIdx.x * blockDim.y + threadIdx.y; cok && wi < nwin; wi += gridDim.x * blockDim.y) {
        const unsigned t = wi / W2;
        const int w2 = (int)(wi - t * W2);
        const int bl = (int)(t / H2);
        const int h2 = (int)(t - (unsigned)bl * H2);
        const int b = SEG ? blockIdx.z * a.segB + bl : bl;
        const bool whole = h2 < Hp && w2 < Wp;       // windows cut by an odd edge have no pooled output
        const unsigned p00 = ((unsigned)b * a.H + 2 * h2) * a.W + 2 * w2;
        float zv[4][4];
        bool ok[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            ok[q] = whole || ((2 * h2 + (q >> 1) < a.H) && (2 * w2 + (q & 1) < a.W));
            const unsigned pq = p00 + (q >> 1) * a.W + (q & 1);
            const float4 v = ok[q] ? ldg4(a.z + (size_t)pq * a.ldz + c) : make_float4(0, 0, 0, 0);
            zv[q][0] = v.x; zv[q][1] = v.y; zv[q][2] = v.z; zv[q][3] = v.w;
        }
        float gv[4] = {0, 0, 0, 0};
        if (whole) {
            const unsigned pp = ((unsigned)b * Hp + h2) * Wp + w2;
            const float4 g = ldg4(a.dyp + (size_t)pp * a.ld_dyp + c);
            gv[0] = g.x; gv[1] = g.y; gv[2] = g.z; gv[3] = g.w;
        }
        float o[4][4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            // first maximum of the activated values in scan order (torch max_pool2d: strict >)
            int best = 0;
            float yb = fmaf(zv[0][k], scv[k], shv[k]);
            float vb = fmaxf(yb, yb * slope);        // leaky for 0 <= slope <= 1 (checked by the host)
            float zb = zv[0][k];
#pragma unroll
            for (int q = 1; q < 4; ++q) {
                const float y = fmaf(zv[q][k], scv[k], shv[k]);
                const float v = fmaxf(y, y * slope);
                if (v > vb) { vb = v; yb = y; zb = zv[q][k]; best = q; }
            }
            const float d = gv[k] * (yb > 0.f ? 1.f : slope);
            if (APPLY) {
                const float tb = (d - c1h[k]) - c1l[k];
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const float xh = (zv[q][k] - muv[k]) * isv[k];
                    o[q][k] = scv[k] * fmaf(-xh, c2f[k], (whole && q == best) ? tb : t0[k]);
                }
            } else {
                if (whole) {
                    const float xh = (zb - muv[k]) * isv[k];
                    kahan_add(s1[k], e1[k], d);
                    kahan_add(s2[k], e2[k], d * xh);
                    md[k] = fmaxf(md[k], fabsf(d));
                }
            }
        }
        if (APPLY) {
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                if (!ok[q]) continue;
                const unsigned pq = p00 + (q >> 1) * a.W + (q & 1);
                const float4 ov = make_float4(o[q][0], o[q][1], o[q][2], o[q][3]);
                if (a.dz) *reinterpret_cast<float4*>(a.dz + (size_t)pq * a.lddz + c) = ov;
                if (a.dh) store_planes4(a.dh, a.dl, (long long)pq * a.cpad + c, ov, psc);
            }
        }
    }

    if (!APPLY) {
        FSDET_DYN_SMEM_F64(red);  // [blockDim.y][TC*16]
        double* mine = red + ((size_t)threadIdx.y * TC + threadIdx.x) * 16;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            mine[k] = (double)s1[k] - (double)e1[k];
            mine[4 + k] = (double)s2[k] - (double)e2[k];
            mine[8 + k] = (double)md[k];
        }
        __syncthreads();
        bwd_block_reduce(red, a.partial + ((SEG ? (long long)blockIdx.z * gridDim.x : 0ll) + blockIdx.x) * 3 * a.C, a.C, blockIdx.y * TC);
    }
}

// sums rows [nseg][3C] -> dgamma, dbeta (summed over the segments in order), the projection coefficients of each
// segment ([nseg][2C]), and an upper bound of max|dz| over all segments (the scale of dz's fp16 planes):
// |dz| <= |scale| * (max|du| + |c1| + max|xhat| * |c2|).  SEG == false: one segment
template <bool SEG>
__global__ void bn_bwd_finalize_kernel(const double* __restrict__ sums, double count, const float* __restrict__ gamma,
                                       const float* __restrict__ invstd, const float* __restrict__ xhat_absmax,
                                       float* __restrict__ dgamma, float* __restrict__ dbeta, double* __restrict__ coef,
                                       float* __restrict__ amax_bound, int C, int has_bn, int nseg) {
    int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    double sdu_all = 0.0, sdux_all = 0.0, bound = 0.0;
    for (int g = 0; g < (SEG ? nseg : 1); ++g) {
        const double* sg = sums + (long long)g * 3 * C;
        const double sdu = sg[c], sdux = sg[C + c];
        double bg = sg[2 * C + c];
        sdu_all = g ? sdu_all + sdu : sdu;
        sdux_all = g ? sdux_all + sdux : sdux;
        if (has_bn) {
            const double c1 = sdu / count, c2 = sdux / count;
            coef[2 * g * C + c] = c1;
            coef[2 * g * C + C + c] = c2;
            if (amax_bound)
                bg = fabs((double)gamma[c] * (double)invstd[g * C + c]) * (bg + fabs(c1) + (double)xhat_absmax[g * C + c] * fabs(c2));
        }
        bound = g ? fmax(bound, bg) : bg;
    }
    if (dbeta) dbeta[c] = (float)sdu_all;
    if (has_bn && dgamma) dgamma[c] = (float)sdux_all;
    if (amax_bound) {
        const float bf = (float)(bound * 1.0001);
        if (isfinite(bf) && bf > 0.f) atomicMax(reinterpret_cast<int*>(amax_bound), __float_as_int(bf));
    }
}

constexpr int kBnSplits = 64;

static int bwd_rows(int B, int H, int W) {
    long long nwin = (long long)B * ((H + 1) / 2) * ((W + 1) / 2);
    long long r = (nwin + 63) / 64;
    if (r > 6 * kNumSMs) r = 6 * kNumSMs;   // whole waves of the 3 resident CTAs per SM (8 x would leave a 2/3-empty third wave)
    if (r < 1) r = 1;
    return (int)r;
}

// channel-vector lanes TC of the pooled forward and the backward blocks (TC x 256/TC threads), sized by the real
// channels C
static int chan_lanes(int C) {
    const int C4 = C / 4;
    return C4 >= 32 ? 32 : (C4 >= 16 ? 16 : (C4 >= 8 ? 8 : (C4 >= 4 ? 4 : (C4 >= 2 ? 2 : 1))));
}

// stage-1 split of bn_finalize: S blocks of rps conv partial rows each (S <= kBnSplits)
static void stat_split(int nparts, int* S, int* rps) {
    int s = ceil_div(nparts, 64);
    if (s > kBnSplits) s = kBnSplits;
    *rps = ceil_div(nparts, s);
    *S = ceil_div(nparts, *rps);
}

// backward CTA rows per segment: the one-segment rows shared out, so that nseg segments fill the same waves
static int seg_bwd_rows(int segB, int H, int W, int nseg) {
    const int r = bwd_rows(segB * nseg, H, W) / nseg;
    return r < 1 ? 1 : r;
}

// pixels per partial row of colstats: large tensors use long strips (few partial rows, little reduction work
// afterwards), small ones short strips so that every SM still gets CTAs
static int stat_strip(long long npix) {
    long long s = npix / (8 * kNumSMs) / 32 * 32;
    return (int)(s < 32 ? 32 : (s > 1024 ? 1024 : s));
}

// strips per segment of nseg segments of seg_pix pixels (the strip length is that of the whole tensor)
static int colstats_seg_rows(long long seg_pix, int nseg) { return ceil_div(seg_pix, stat_strip(seg_pix * nseg)); }

// segments of whole images: nseg * seg_pix == B*H*W and seg_pix a multiple of H*W; returns images per segment or 0
static int seg_images(int B, int H, int W, int nseg, long long seg_pix) {
    const long long hw = (long long)H * W;
    if (nseg < 1 || hw <= 0 || seg_pix <= 0 || seg_pix % hw || (long long)nseg * seg_pix != (long long)B * hw) return 0;
    return (int)(seg_pix / hw);
}

}  // namespace fsdet

#ifndef FSDET_HOST_EMULATION  // tools/host_emul/bn_act_emul.cpp launches the kernels above on the same geometry

using namespace fsdet;

extern "C" int fsdet_bn_bwd_rows(int B, int H, int W) { return bwd_rows(B, H, W); }
extern "C" int fsdet_bn_seg_bwd_rows(int B, int H, int W, int nseg) {
    return nseg >= 1 && B % nseg == 0 ? seg_bwd_rows(B / nseg, H, W, nseg) : -1;
}

extern "C" int fsdet_colstats_rows(size_t npix) { return colstats_seg_rows((long long)npix, 1); }
extern "C" int fsdet_bn_seg_colstats_rows(size_t seg_pix, int nseg) {
    return nseg >= 1 ? colstats_seg_rows((long long)seg_pix, nseg) : -1;
}

static int launch_colstats(const float* z, int ld, long long seg_pix, int nseg, int C, float* partial, cudaStream_t s) {
    FSDET_CHECK_ARG(z && partial && C % 4 == 0 && ld % 4 == 0 && aligned16(z) && nseg >= 1 && seg_pix >= 0,
                    "colstats: C=%d ld=%d nseg=%d", C, ld, nseg);
    if (seg_pix == 0) return 0;
    const int TCx = chan_lanes(C);
    const int TY = 256 / TCx;
    dim3 block(TCx, TY), grid(colstats_seg_rows(seg_pix, nseg), nseg);
    size_t smem = (size_t)TY * TCx * 16 * sizeof(float);
    colstats_kernel<<<grid, block, smem, s>>>(z, ld, seg_pix, C, stat_strip(seg_pix * nseg), partial);
    return launch_status("colstats");
}

extern "C" int fsdet_colstats(const float* z, int ld, size_t npix, int C, float* partial, void* stream) {
    return launch_colstats(z, ld, (long long)npix, 1, C, partial, (cudaStream_t)stream);
}

extern "C" int fsdet_bn_seg_colstats(const float* z, int ld, size_t seg_pix, int nseg, int C, float* partial, void* stream) {
    return launch_colstats(z, ld, (long long)seg_pix, nseg, C, partial, (cudaStream_t)stream);
}

static int launch_finalize(const float* stat_partial, int nparts, int nseg, double count, const float* gamma,
                           const float* beta, float* running_mean, float* running_var, float momentum, float eps,
                           float* mean, float* invstd, float* scale, float* shift, float slope, float* amax_y,
                           float* xhat_absmax, int C, int training, cudaStream_t s) {
    FSDET_CHECK_ARG(scale && shift && C > 0 && nseg >= 1 && (training || nseg == 1), "bn_finalize: bad args");
    if (training) {
        FSDET_CHECK_ARG(stat_partial && nparts > 0, "bn_finalize: training needs the conv partials");
    } else {
        FSDET_CHECK_ARG(running_mean && running_var, "bn_finalize: eval needs running stats");
    }
    if (amax_y && !training) {       // (training: cleared by the stage-1 kernel)
        cudaError_t e = cudaMemsetAsync(amax_y, 0, sizeof(float), s);
        if (e != cudaSuccess) { set_error("bn_finalize: memset: %s", cudaGetErrorString(e)); return (int)e; }
    }
    const double* red = nullptr;
    int S = 0;
    if (training) {
        // scratch for the stage-1 result lives behind the partial rows (nseg * fsdet_bn_stat_scratch_rows() extra rows)
        int rps;
        stat_split(nparts, &S, &rps);
        double* scratch = reinterpret_cast<double*>(const_cast<float*>(stat_partial) + (size_t)nseg * nparts * 4 * C);
        dim3 block(32, 32), grid(ceil_div(C, 32), S, nseg);
        if (nseg > 1) bn_stats_reduce_kernel<true><<<grid, block, 0, s>>>(stat_partial, nparts, rps, C, scratch, amax_y);
        else bn_stats_reduce_kernel<false><<<grid, block, 0, s>>>(stat_partial, nparts, rps, C, scratch, amax_y);
        int st = launch_status("bn_finalize/reduce");
        if (st) return st;
        red = scratch;
    }
    if (nseg > 1)
        bn_finalize_kernel<true><<<dim3(ceil_div(C, 128), nseg), 128, 0, s>>>(red, S, count, gamma, beta, running_mean, running_var,
                                                                               momentum, eps, mean, invstd, scale, shift, slope,
                                                                               amax_y, xhat_absmax, C, training);
    else
        bn_finalize_kernel<false><<<ceil_div(C, 128), 128, 0, s>>>(red, S, count, gamma, beta, running_mean, running_var, momentum,
                                                                   eps, mean, invstd, scale, shift, slope, amax_y, xhat_absmax,
                                                                   C, training);
    return launch_status("bn_finalize");
}

extern "C" int fsdet_bn_finalize(const float* stat_partial, int nparts, double count, const float* gamma,
                                 const float* beta, float* running_mean, float* running_var, float momentum, float eps,
                                 float* mean, float* invstd, float* scale, float* shift, float slope, float* amax_y,
                                 float* xhat_absmax, int C, int training, void* stream) {
    return launch_finalize(stat_partial, nparts, 1, count, gamma, beta, running_mean, running_var, momentum, eps, mean,
                           invstd, scale, shift, slope, amax_y, xhat_absmax, C, training, (cudaStream_t)stream);
}

extern "C" int fsdet_bn_seg_finalize(const float* stat_partial, int nparts, int nseg, size_t seg_pix, const float* gamma,
                                     const float* beta, float* running_mean, float* running_var, float momentum, float eps,
                                     float* mean, float* invstd, float* scale, float* shift, float slope, float* amax_y,
                                     float* xhat_absmax, int C, void* stream) {
    FSDET_CHECK_ARG(seg_pix > 0, "bn_seg_finalize: empty segments");
    return launch_finalize(stat_partial, nparts, nseg, (double)seg_pix, gamma, beta, running_mean, running_var, momentum,
                           eps, mean, invstd, scale, shift, slope, amax_y, xhat_absmax, C, 1, (cudaStream_t)stream);
}

extern "C" int fsdet_bn_stat_scratch_rows(void) { return 2 * kBnSplits; }  // kBnSplits rows of 4C doubles

static int launch_act_fwd(const float* z, int ldz, const float* scale, const float* shift, float slope, float* y_full,
                          int ld_full, float* y_pool, int ld_pool, void* full_hi, void* full_lo, void* pool_hi,
                          void* pool_lo, int Cpad, const float* amax, int B, int H, int W, int C, int nseg, int segB,
                          cudaStream_t s) {
    const bool planes = full_hi || pool_hi;
    FSDET_CHECK_ARG(z && scale && shift && (y_full || y_pool || planes), "bn_act_fwd: null pointer");
    FSDET_CHECK_ARG(C % 4 == 0 && ldz % 4 == 0 && (!y_full || ld_full % 4 == 0) && (!y_pool || ld_pool % 4 == 0),
                    "bn_act_fwd: C=%d and leading dims must be multiples of 4", C);
    FSDET_CHECK_ARG(!planes || (amax && Cpad >= C && Cpad % 4 == 0 && (!full_hi || full_lo) && (!pool_hi || pool_lo)),
                    "bn_act_fwd: plane outputs need amax, lo planes and Cpad >= C");
    FwdArgs a;
    a.z = z; a.scale = scale; a.shift = shift; a.amax = amax; a.yf = y_full; a.yp = y_pool;
    a.fh = (__half*)full_hi; a.fl = (__half*)full_lo; a.ph = (__half*)pool_hi; a.pl = (__half*)pool_lo;
    a.ldz = ldz; a.ldf = ld_full; a.ldp = ld_pool; a.Cpad = planes ? Cpad : C; a.B = B; a.H = H; a.W = W; a.C = C; a.slope = slope;
    a.segB = segB;
    const int CP4 = a.Cpad / 4;
    FSDET_CHECK_ARG((long long)B * H * W * CP4 < (1ll << 31), "bn_act_fwd: tensor too large for 32-bit indexing");
    if (!y_pool && !pool_hi) {
        long long n = (long long)segB * H * W * CP4;
        if (n == 0) return 0;
        if (nseg > 1) bn_act_flat_kernel<true><<<dim3(ceil_div(n, 256), nseg), 256, 0, s>>>(a);
        else bn_act_flat_kernel<false><<<ceil_div(n, 256), 256, 0, s>>>(a);
    } else {
        long long nwin = (long long)segB * ((H + 1) / 2) * ((W + 1) / 2);
        if (nwin == 0) return 0;
        // channel-vector lanes sized by the REAL channels: the zero padding of the planes (pitch > C) is written by the
        // same threads in a second trip of their channel loop instead of by threads that never load anything
        const int TC = chan_lanes(C);
        const int TY = 256 / TC;
        dim3 block(TC, TY), grid((unsigned)ceil_div(nwin, TY), nseg);
        const bool full = a.yf || a.fh;
        if (nseg > 1) {
            if (full) bn_act_pool_kernel<true, true><<<grid, block, 0, s>>>(a);
            else bn_act_pool_kernel<false, true><<<grid, block, 0, s>>>(a);
        } else {
            if (full) bn_act_pool_kernel<true, false><<<grid, block, 0, s>>>(a);
            else bn_act_pool_kernel<false, false><<<grid, block, 0, s>>>(a);
        }
    }
    return launch_status("bn_act_fwd");
}

extern "C" int fsdet_bn_act_fwd(const float* z, int ldz, const float* scale, const float* shift, float slope, float* y_full,
                                int ld_full, float* y_pool, int ld_pool, void* full_hi, void* full_lo, void* pool_hi,
                                void* pool_lo, int Cpad, const float* amax, int B, int H, int W, int C, void* stream) {
    return launch_act_fwd(z, ldz, scale, shift, slope, y_full, ld_full, y_pool, ld_pool, full_hi, full_lo, pool_hi, pool_lo,
                          Cpad, amax, B, H, W, C, 1, B, (cudaStream_t)stream);
}

extern "C" int fsdet_bn_act_fwd_seg(const float* z, int ldz, const float* scale, const float* shift, float slope,
                                    float* y_full, int ld_full, float* y_pool, int ld_pool, void* full_hi, void* full_lo,
                                    void* pool_hi, void* pool_lo, int Cpad, const float* amax, int B, int H, int W, int C,
                                    int nseg, size_t seg_pix, void* stream) {
    const int segB = seg_images(B, H, W, nseg, (long long)seg_pix);
    FSDET_CHECK_ARG(segB > 0, "bn_act_fwd_seg: %d segments of %zu pixels do not split %d images of %dx%d", nseg, seg_pix, B, H, W);
    return launch_act_fwd(z, ldz, scale, shift, slope, y_full, ld_full, y_pool, ld_pool, full_hi, full_lo, pool_hi, pool_lo,
                          Cpad, amax, B, H, W, C, nseg, segB, (cudaStream_t)stream);
}

static int launch_bwd(bool apply, const BwdArgs& a, int nseg, cudaStream_t s) {
    FSDET_CHECK_ARG((long long)a.B * a.H * a.W < (1ll << 31), "bn_act_bwd: tensor too large for 32-bit pixel indexing");
    int C4 = a.C / 4;
    int TC = chan_lanes(a.C);
    int TY = 256 / TC;
    dim3 block(TC, TY), grid(seg_bwd_rows(a.segB, a.H, a.W, nseg), ceil_div(C4, TC), nseg);
    const size_t smem = (size_t)TY * TC * 16 * sizeof(double);  // 32 KB (reduce pass)
    const bool pool_only = !a.dyf && a.dyp && a.has_bn && a.slope >= 0.f && a.slope <= 1.f;
    if (nseg > 1) {
        if (pool_only) {
            if (apply) bn_act_bwd_pool_kernel<true, true><<<grid, block, 0, s>>>(a);
            else bn_act_bwd_pool_kernel<false, true><<<grid, block, smem, s>>>(a);
        } else {
            if (apply) bn_act_bwd_kernel<true, true><<<grid, block, 0, s>>>(a);
            else bn_act_bwd_kernel<false, true><<<grid, block, smem, s>>>(a);
        }
    } else {
        if (pool_only) {
            if (apply) bn_act_bwd_pool_kernel<true, false><<<grid, block, 0, s>>>(a);
            else bn_act_bwd_pool_kernel<false, false><<<grid, block, smem, s>>>(a);
        } else {
            if (apply) bn_act_bwd_kernel<true, false><<<grid, block, 0, s>>>(a);
            else bn_act_bwd_kernel<false, false><<<grid, block, smem, s>>>(a);
        }
    }
    return launch_status(apply ? "bn_act_bwd_apply" : "bn_act_bwd_reduce");
}

static int bwd_reduce(const float* z, int ldz, const float* dy_full, int ld_dyf, const float* dy_pool, int ld_dyp,
                      const float* scale, const float* shift, const float* mean, const float* invstd, float slope,
                      double* partial, int B, int H, int W, int C, int has_bn, int nseg, int segB, cudaStream_t s) {
    FSDET_CHECK_ARG(z && scale && shift && partial && (dy_full || dy_pool), "bn_act_bwd_reduce: null pointer");
    FSDET_CHECK_ARG(!has_bn || (mean && invstd), "bn_act_bwd_reduce: BN needs mean/invstd");
    FSDET_CHECK_ARG(C % 4 == 0 && ldz % 4 == 0 && ld_dyf % 4 == 0 && ld_dyp % 4 == 0, "bn_act_bwd_reduce: alignment");
    BwdArgs a;
    a.z = z; a.dyf = dy_full; a.dyp = dy_pool; a.scale = scale; a.shift = shift; a.mean = mean; a.invstd = invstd;
    a.coef = nullptr; a.dz = nullptr; a.dh = nullptr; a.dl = nullptr; a.amax = nullptr; a.partial = partial;
    a.ldz = ldz; a.ld_dyf = ld_dyf; a.ld_dyp = ld_dyp; a.lddz = 0; a.cpad = 0;
    a.B = B; a.H = H; a.W = W; a.C = C; a.segB = segB; a.slope = slope; a.has_bn = has_bn;
    return launch_bwd(false, a, nseg, s);
}

extern "C" int fsdet_bn_act_bwd_reduce(const float* z, int ldz, const float* dy_full, int ld_dyf, const float* dy_pool,
                                       int ld_dyp, const float* scale, const float* shift, const float* mean,
                                       const float* invstd, float slope, double* partial, int B, int H, int W, int C,
                                       int has_bn, void* stream) {
    return bwd_reduce(z, ldz, dy_full, ld_dyf, dy_pool, ld_dyp, scale, shift, mean, invstd, slope, partial, B, H, W, C, has_bn,
                      1, B, (cudaStream_t)stream);
}

extern "C" int fsdet_bn_act_bwd_reduce_seg(const float* z, int ldz, const float* dy_full, int ld_dyf, const float* dy_pool,
                                           int ld_dyp, const float* scale, const float* shift, const float* mean,
                                           const float* invstd, float slope, double* partial, int B, int H, int W, int C,
                                           int nseg, size_t seg_pix, void* stream) {
    const int segB = seg_images(B, H, W, nseg, (long long)seg_pix);
    FSDET_CHECK_ARG(segB > 0, "bn_act_bwd_reduce_seg: %d segments of %zu pixels do not split %d images of %dx%d", nseg, seg_pix, B, H, W);
    return bwd_reduce(z, ldz, dy_full, ld_dyf, dy_pool, ld_dyp, scale, shift, mean, invstd, slope, partial, B, H, W, C, 1,
                      nseg, segB, (cudaStream_t)stream);
}

static int bwd_finalize(const double* partial, int nparts, int nseg, double count, const float* gamma, const float* invstd,
                        const float* xhat_absmax, float* dgamma, float* dbeta, double* coef, float* amax_bound, int C,
                        int has_bn, cudaStream_t s) {
    FSDET_CHECK_ARG(partial && nparts > 0 && C > 0 && nseg >= 1 && (!has_bn || (coef && gamma && invstd)), "bn_bwd_finalize: bad args");
    FSDET_CHECK_ARG(!(amax_bound && has_bn) || xhat_absmax, "bn_bwd_finalize: the bound of max|dz| needs xhat_absmax");
    double* sums = const_cast<double*>(partial) + (size_t)nseg * nparts * 3 * C;  // the extra rows
    dim3 block(32, 32), grid(ceil_div(3 * C, 32), nseg);
    if (nseg > 1) colsum_dd_kernel<true><<<grid, block, 0, s>>>(partial, nparts, 3 * C, 2 * C, sums, amax_bound);
    else colsum_dd_kernel<false><<<grid, block, 0, s>>>(partial, nparts, 3 * C, 2 * C, sums, amax_bound);
    int st = launch_status("bn_bwd_finalize/colsum");
    if (st) return st;
    if (nseg > 1)
        bn_bwd_finalize_kernel<true><<<ceil_div(C, 128), 128, 0, s>>>(sums, count, gamma, invstd, xhat_absmax, dgamma, dbeta, coef,
                                                                      amax_bound, C, has_bn, nseg);
    else
        bn_bwd_finalize_kernel<false><<<ceil_div(C, 128), 128, 0, s>>>(sums, count, gamma, invstd, xhat_absmax, dgamma, dbeta, coef,
                                                                       amax_bound, C, has_bn, 1);
    return launch_status("bn_bwd_finalize");
}

extern "C" int fsdet_bn_bwd_finalize(const double* partial, int nparts, double count, const float* gamma,
                                     const float* invstd, const float* xhat_absmax, float* dgamma, float* dbeta, double* coef,
                                     float* amax_bound, int C, int has_bn, void* stream) {
    return bwd_finalize(partial, nparts, 1, count, gamma, invstd, xhat_absmax, dgamma, dbeta, coef, amax_bound, C, has_bn,
                        (cudaStream_t)stream);
}

extern "C" int fsdet_bn_bwd_finalize_seg(const double* partial, int nparts, int nseg, size_t seg_pix, const float* gamma,
                                         const float* invstd, const float* xhat_absmax, float* dgamma, float* dbeta,
                                         double* coef, float* amax_bound, int C, void* stream) {
    FSDET_CHECK_ARG(seg_pix > 0, "bn_bwd_finalize_seg: empty segments");
    return bwd_finalize(partial, nparts, nseg, (double)seg_pix, gamma, invstd, xhat_absmax, dgamma, dbeta, coef, amax_bound, C, 1,
                        (cudaStream_t)stream);
}

static int bwd_apply(const float* z, int ldz, const float* dy_full, int ld_dyf, const float* dy_pool, int ld_dyp,
                     const float* scale, const float* shift, const float* mean, const float* invstd, const double* coef,
                     float slope, float* dz, int lddz, void* dz_hi, void* dz_lo, int cpad, const float* amax, int B, int H,
                     int W, int C, int has_bn, int nseg, int segB, cudaStream_t s) {
    FSDET_CHECK_ARG(z && scale && shift && (dz || dz_hi) && (dy_full || dy_pool), "bn_act_bwd_apply: null pointer");
    FSDET_CHECK_ARG(!has_bn || (mean && invstd && coef), "bn_act_bwd_apply: BN needs mean/invstd/coef");
    FSDET_CHECK_ARG(C % 4 == 0 && ldz % 4 == 0 && ld_dyf % 4 == 0 && ld_dyp % 4 == 0 && lddz % 4 == 0,
                    "bn_act_bwd_apply: alignment");
    FSDET_CHECK_ARG(!dz_hi || (dz_lo && amax && cpad == C), "bn_act_bwd_apply: planes need lo, amax and cpad == C (%d vs %d)", cpad, C);
    BwdArgs a;
    a.z = z; a.dyf = dy_full; a.dyp = dy_pool; a.scale = scale; a.shift = shift; a.mean = mean; a.invstd = invstd;
    a.coef = coef; a.dz = dz; a.dh = (__half*)dz_hi; a.dl = (__half*)dz_lo; a.amax = amax; a.partial = nullptr;
    a.ldz = ldz; a.ld_dyf = ld_dyf; a.ld_dyp = ld_dyp; a.lddz = lddz; a.cpad = cpad;
    a.B = B; a.H = H; a.W = W; a.C = C; a.segB = segB; a.slope = slope; a.has_bn = has_bn;
    return launch_bwd(true, a, nseg, s);
}

extern "C" int fsdet_bn_act_bwd_apply(const float* z, int ldz, const float* dy_full, int ld_dyf, const float* dy_pool,
                                      int ld_dyp, const float* scale, const float* shift, const float* mean,
                                      const float* invstd, const double* coef, float slope, float* dz, int lddz,
                                      void* dz_hi, void* dz_lo, int cpad, const float* amax, int B, int H, int W, int C,
                                      int has_bn, void* stream) {
    return bwd_apply(z, ldz, dy_full, ld_dyf, dy_pool, ld_dyp, scale, shift, mean, invstd, coef, slope, dz, lddz, dz_hi, dz_lo,
                     cpad, amax, B, H, W, C, has_bn, 1, B, (cudaStream_t)stream);
}

extern "C" int fsdet_bn_act_bwd_apply_seg(const float* z, int ldz, const float* dy_full, int ld_dyf, const float* dy_pool,
                                          int ld_dyp, const float* scale, const float* shift, const float* mean,
                                          const float* invstd, const double* coef, float slope, float* dz, int lddz,
                                          void* dz_hi, void* dz_lo, int cpad, const float* amax, int B, int H, int W, int C,
                                          int nseg, size_t seg_pix, void* stream) {
    const int segB = seg_images(B, H, W, nseg, (long long)seg_pix);
    FSDET_CHECK_ARG(segB > 0, "bn_act_bwd_apply_seg: %d segments of %zu pixels do not split %d images of %dx%d", nseg, seg_pix, B, H, W);
    return bwd_apply(z, ldz, dy_full, ld_dyf, dy_pool, ld_dyp, scale, shift, mean, invstd, coef, slope, dz, lddz, dz_hi, dz_lo,
                     cpad, amax, B, H, W, C, 1, nseg, segB, (cudaStream_t)stream);
}

#endif  // FSDET_HOST_EMULATION
