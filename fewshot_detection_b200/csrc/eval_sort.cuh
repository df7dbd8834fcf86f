// Block scan, stable LSD radix sort and uint64 prefix sums shared by the device evaluators (voc_eval.cu, coco_eval.cu),
// with the launch macros that run them either on the device or under host emulation (tools/host_emul).
// Internal linkage: every evaluator translation unit gets its own copy of the kernels.
#pragma once
#include "common.cuh"

namespace fsdet {
namespace {

constexpr int kVocThreads = 256;
constexpr int kVocItems = 8;                          // items per thread of a radix / scan tile
constexpr int kVocTile = kVocThreads * kVocItems;

// Exclusive prefix sum of one value per thread over a kVocThreads block (Hillis-Steele in shared memory).
__device__ __forceinline__ unsigned long long voc_block_scan(unsigned long long v, unsigned long long* s,
                                                            unsigned long long& total) {
    s[threadIdx.x] = v;
    __syncthreads();
    for (int off = 1; off < kVocThreads; off <<= 1) {
        const unsigned long long t = s[threadIdx.x] + (threadIdx.x >= (unsigned)off ? s[threadIdx.x - off] : 0ull);
        __syncthreads();
        s[threadIdx.x] = t;
        __syncthreads();
    }
    const unsigned long long incl = s[threadIdx.x];
    total = s[kVocThreads - 1];
    __syncthreads();                                  // s is reused by the caller
    return incl - v;
}

// ---- stable LSD radix sort of (rank_key, record index), 8 bits per pass ----------------------------------------
__global__ void __launch_bounds__(kVocThreads) voc_radix_hist_kernel(const uint32_t* __restrict__ keys, int n, int shift,
                                                                     int ntiles, unsigned long long* __restrict__ cnt) {
    __shared__ int h[256];
    h[threadIdx.x] = 0;
    __syncthreads();
    const int tile = blockIdx.x;
    for (int it = 0; it < kVocItems; ++it) {
        const int i = tile * kVocTile + it * kVocThreads + threadIdx.x;
        if (i < n) atomicAdd(&h[(keys[i] >> shift) & 255], 1);
    }
    __syncthreads();
    cnt[(size_t)threadIdx.x * ntiles + tile] = (unsigned long long)h[threadIdx.x];
}

// cnt_scan[d * ntiles + t] = where tile t's first item of digit d goes.  Items are taken in index order (round, warp,
// lane), and each one's place among the equal digits before it is counted exactly: the pass is stable.
__global__ void __launch_bounds__(kVocThreads) voc_radix_scatter_kernel(const uint32_t* __restrict__ keys_in,
                                                                        const int32_t* __restrict__ vals_in, int n,
                                                                        int shift, int ntiles,
                                                                        const unsigned long long* __restrict__ cnt_scan,
                                                                        uint32_t* __restrict__ keys_out,
                                                                        int32_t* __restrict__ vals_out) {
    __shared__ unsigned long long base[256];
    __shared__ int wc[kVocThreads / 32][256];
    __shared__ int tot[256];
    const int tile = blockIdx.x, lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    base[threadIdx.x] = cnt_scan[(size_t)threadIdx.x * ntiles + tile];
    for (int it = 0; it < kVocItems; ++it) {
        for (int q = 0; q < kVocThreads / 32; ++q) wc[q][threadIdx.x] = 0;
        __syncthreads();
        const int i = tile * kVocTile + it * kVocThreads + threadIdx.x;
        const bool valid = i < n;
        const uint32_t k = valid ? keys_in[i] : 0u;
        const int32_t v = valid ? (vals_in ? vals_in[i] : i) : 0;
        const int dg = (int)((k >> shift) & 255u);
        unsigned peers = __ballot_sync(0xffffffffu, valid);
        for (int b = 0; b < 8; ++b) {
            const bool bit = (dg >> b) & 1;
            const unsigned m = __ballot_sync(0xffffffffu, bit);
            peers &= bit ? m : ~m;
        }
        const unsigned below = peers & ((1u << lane) - 1u);
        if (valid && below == 0) wc[w][dg] = __popc(peers);
        __syncthreads();
        int run = 0;
        for (int q = 0; q < kVocThreads / 32; ++q) {
            const int c = wc[q][threadIdx.x];
            wc[q][threadIdx.x] = run;
            run += c;
        }
        tot[threadIdx.x] = run;
        __syncthreads();
        if (valid) {
            const unsigned long long dst = base[dg] + (unsigned long long)wc[w][dg] + (unsigned long long)__popc(below);
            keys_out[dst] = k;
            vals_out[dst] = v;
        }
        __syncthreads();
        base[threadIdx.x] += (unsigned long long)tot[threadIdx.x];
    }
}

// ---- prefix sums over uint64 (three kernels: tile sums, one block over the tile sums, tile scans) -------------------
__global__ void __launch_bounds__(kVocThreads) voc_scan_partials_kernel(const unsigned long long* __restrict__ a, long long n,
                                                                        unsigned long long* __restrict__ part) {
    __shared__ unsigned long long s[kVocThreads];
    const long long b0 = (long long)blockIdx.x * kVocTile + (long long)threadIdx.x * kVocItems;
    unsigned long long v = 0;
    for (int k = 0; k < kVocItems; ++k)
        if (b0 + k < n) v += a[b0 + k];
    unsigned long long total;
    voc_block_scan(v, s, total);
    if (threadIdx.x == 0) part[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kVocThreads) voc_scan_top_kernel(unsigned long long* __restrict__ part, int nb) {
    __shared__ unsigned long long s[kVocThreads];
    unsigned long long carry = 0;
    for (int b0 = 0; b0 < nb; b0 += kVocThreads) {
        const int b = b0 + threadIdx.x;
        const unsigned long long v = b < nb ? part[b] : 0ull;
        unsigned long long total;
        const unsigned long long pre = voc_block_scan(v, s, total);
        if (b < nb) part[b] = carry + pre;
        carry += total;
    }
}

__global__ void __launch_bounds__(kVocThreads) voc_scan_apply_kernel(unsigned long long* __restrict__ a, long long n,
                                                                     const unsigned long long* __restrict__ part,
                                                                     int inclusive) {
    __shared__ unsigned long long s[kVocThreads];
    const long long b0 = (long long)blockIdx.x * kVocTile + (long long)threadIdx.x * kVocItems;
    unsigned long long x[kVocItems], v = 0;
    for (int k = 0; k < kVocItems; ++k) {
        x[k] = b0 + k < n ? a[b0 + k] : 0ull;
        v += x[k];
    }
    unsigned long long total;
    unsigned long long run = part[blockIdx.x] + voc_block_scan(v, s, total);
    for (int k = 0; k < kVocItems; ++k) {
        const unsigned long long next = run + x[k];
        if (b0 + k < n) a[b0 + k] = inclusive ? next : run;
        run = next;
    }
}

// ---- host side, shared by the library and the host-emulation build -----------------------------------------------
#ifdef FSDET_HOST_EMULATION
#define VOC_LAUNCH(grid, block, kernel, ...) emul::launch(dim3(grid), dim3(block), 0, [&]() { kernel(__VA_ARGS__); })
#define VOC_CHECK(what) ((void)0)
#else
#define VOC_LAUNCH(grid, block, kernel, ...) kernel<<<(grid), (block), 0, st>>>(__VA_ARGS__)
#define VOC_CHECK(what)                            \
    do {                                           \
        const int rc_ = launch_status(what);       \
        if (rc_) return rc_;                       \
    } while (0)
#endif

static inline size_t voc_align(size_t b) { return (b + 255) & ~(size_t)255; }

static int voc_scan(unsigned long long* a, long long n, unsigned long long* part, int inclusive, cudaStream_t st) {
    (void)st;
    const int nb = ceil_div(n, kVocTile);
    VOC_LAUNCH(nb, kVocThreads, voc_scan_partials_kernel, a, n, part);
    VOC_CHECK("voc_scan_partials");
    VOC_LAUNCH(1, kVocThreads, voc_scan_top_kernel, part, nb);
    VOC_CHECK("voc_scan_top");
    VOC_LAUNCH(nb, kVocThreads, voc_scan_apply_kernel, a, n, part, inclusive);
    VOC_CHECK("voc_scan_apply");
    return 0;
}

}  // namespace
}  // namespace fsdet
