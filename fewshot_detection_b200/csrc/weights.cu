// Per-step preparation of ALL convolution weights of a network for the tensor-core kernels, in two launches.
//
// The tensor-core convolutions read their weight operand as scaled fp16 (hi, lo) planes, the forward GEMM in OHWI order
// [Cout][tap][Cin], the input-gradient GEMM flip-transposed [Cin][kk-1-tap][Cout] (the weights of the transposed
// convolution; nn.Conv2d's autograd does the same inside cuDNN, darknet_meta.py:236-252).  Round 1 produced them per
// use with four small launches per layer (amax, split, flip-transpose, split: ~120 launches per step); here one
// launch computes every tensor's absolute maximum and one launch writes all planes, driven by a device table with
// one descriptor per layer and one (layer, tile) entry per 32x32 (Cout x Cin) tile of one filter tap.
//   pass 1: amax[layer] = max |w|                      (atomicMax on the int view of non-negative floats)
//   pass 2: per tile: read w once (coalesced along Cin), write the forward planes (coalesced along Cin) and - through a
//           shared-memory transpose - the input-gradient planes (coalesced along Cout).
// The channel padding of the planes (pitch > channels) is never written: the caller allocates the planes zeroed, once.
#include <cuda_fp16.h>

#include "common.cuh"

namespace fsdet {

__device__ __forceinline__ float wp_scale(float a) {   // same rule as conv_tc.cu / bn_act.cu: amax -> [512, 1024)
    if (!(a > 0.f) || !isfinite(a)) return 1.f;
    int ex = (int)((__float_as_uint(a) >> 23) & 0xff) - 126;
    int e = 10 - ex;
    e = e < -60 ? -60 : (e > 60 ? 60 : e);
    return __uint_as_float((uint32_t)(e + 127) << 23);
}

__device__ __forceinline__ void wp_tile_coords(const fsdet_weight_desc& d, int local, int& tap, int& co0, int& ci0) {
    const int per_tap = d.tiles_co * d.tiles_ci;
    tap = local / per_tap;
    const int r = local - tap * per_tap;
    co0 = (r / d.tiles_ci) * 32;
    ci0 = (r - (r / d.tiles_ci) * d.tiles_ci) * 32;
}

// block (32, 8); one 32x32 tile per block
__global__ void __launch_bounds__(256) weight_amax_kernel(const fsdet_weight_desc* __restrict__ descs,
                                                          const int2* __restrict__ tiles) {
    const int2 t = tiles[blockIdx.x];
    const fsdet_weight_desc d = descs[t.x];
    int tap, co0, ci0;
    wp_tile_coords(d, t.y, tap, co0, ci0);
    float m = 0.f;
    const int ci = ci0 + threadIdx.x;
    if (ci < d.Cin)
        for (int r = threadIdx.y; r < 32; r += 8) {
            const int co = co0 + r;
            if (co < d.Cout) m = fmaxf(m, fabsf(__ldg(d.w + ((long long)co * d.kk + tap) * d.Cin + ci)));
        }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    __shared__ float red[8];
    if (threadIdx.x == 0) red[threadIdx.y] = m;
    __syncthreads();
    if (threadIdx.x == 0 && threadIdx.y == 0) {
        for (int w = 1; w < 8; ++w) m = fmaxf(m, red[w]);
        if (isfinite(m) && m > 0.f) atomicMax(reinterpret_cast<int*>(d.amax), __float_as_int(m));
    }
}

__global__ void __launch_bounds__(256) weight_planes_kernel(const fsdet_weight_desc* __restrict__ descs,
                                                            const int2* __restrict__ tiles) {
    __shared__ float tile[32][33];
    const int2 t = tiles[blockIdx.x];
    const fsdet_weight_desc d = descs[t.x];
    int tap, co0, ci0;
    wp_tile_coords(d, t.y, tap, co0, ci0);
    const float sc = wp_scale(__ldg(d.amax));
    __half* fh = reinterpret_cast<__half*>(d.fwd_hi);
    __half* fl = reinterpret_cast<__half*>(d.fwd_lo);
    for (int r = threadIdx.y; r < 32; r += 8) {
        const int co = co0 + r, ci = ci0 + threadIdx.x;
        float v = 0.f;
        if (co < d.Cout && ci < d.Cin) {
            v = __ldg(d.w + ((long long)co * d.kk + tap) * d.Cin + ci) * sc;
            if (fh) {
                const __half h = __float2half_rn(v);
                const long long o = (long long)co * d.kk * d.fwd_pitch + (long long)tap * d.fwd_pitch + ci;
                fh[o] = h;
                fl[o] = __float2half_rn(v - __half2float(h));
            }
        }
        tile[r][threadIdx.x] = v;
    }
    if (!d.bwd_hi) return;          // block-uniform
    __syncthreads();
    __half* bh = reinterpret_cast<__half*>(d.bwd_hi);
    __half* bl = reinterpret_cast<__half*>(d.bwd_lo);
    for (int r = threadIdx.y; r < 32; r += 8) {
        const int ci = ci0 + r, co = co0 + threadIdx.x;
        if (ci < d.Cin && co < d.Cout) {
            const float v = tile[threadIdx.x][r];
            const __half h = __float2half_rn(v);
            const long long o = (long long)ci * d.kk * d.bwd_pitch + (long long)(d.kk - 1 - tap) * d.bwd_pitch + co;
            bh[o] = h;
            bl[o] = __float2half_rn(v - __half2float(h));
        }
    }
}

}  // namespace fsdet

using namespace fsdet;

extern "C" int fsdet_weight_prep(const fsdet_weight_desc* descs_dev, const int32_t* tiles_dev, int n_tiles, float* amax_all,
                                 int n_layers, void* stream) {
    FSDET_CHECK_ARG(descs_dev && tiles_dev && amax_all && n_layers > 0 && n_tiles >= 0, "weight_prep: bad args");
    if (n_tiles == 0) return 0;
    cudaStream_t s = (cudaStream_t)stream;
    cudaError_t e = cudaMemsetAsync(amax_all, 0, (size_t)n_layers * sizeof(float), s);
    if (e != cudaSuccess) { set_error("weight_prep: memset: %s", cudaGetErrorString(e)); return (int)e; }
    dim3 block(32, 8);
    weight_amax_kernel<<<n_tiles, block, 0, s>>>(descs_dev, reinterpret_cast<const int2*>(tiles_dev));
    int st = launch_status("weight_prep/amax");
    if (st) return st;
    weight_planes_kernel<<<n_tiles, block, 0, s>>>(descs_dev, reinterpret_cast<const int2*>(tiles_dev));
    return launch_status("weight_prep/planes");
}
