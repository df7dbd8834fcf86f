// Host emulation of the CUDA block model for LOGIC tests of block-cooperative kernels without a GPU (test tooling).
//
// A kernel source is compiled by g++ with `-include cuda_host_emul.h -DFSDET_HOST_EMULATION`; every CUDA thread of a
// block is an OS thread, __syncthreads() is a pthread barrier over the block, warp collectives are a barrier over the
// warp's 32 threads, `__shared__` variables are function-local statics (blocks run one after another).  Arithmetic
// intrinsics map to the plain IEEE operation (compile with -ffp-contract=off); transcendental functions are libm's,
// so values can differ from the device by an ulp - the point is the control flow: scans, sorts, barriers, indexing.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <string.h>

#include <deque>
#include <functional>
#include <thread>
#include <vector>

#undef __global__
#define __global__
#undef __device__
#define __device__
#undef __host__
#define __host__
#undef __shared__
#define __shared__ static
#undef __forceinline__
#define __forceinline__ inline
#undef __launch_bounds__
#define __launch_bounds__(...)

namespace emul {
constexpr int kMaxThreads = 1024;
struct Block {
    pthread_barrier_t bar;
    pthread_barrier_t warp_bar[kMaxThreads / 32];
    unsigned warp_flags[kMaxThreads / 32][32];
    uint64_t warp_vals[kMaxThreads / 32][32];
};
extern Block g_block;
extern unsigned char* g_dyn_smem;
}  // namespace emul

static thread_local uint3 threadIdx;
static thread_local uint3 blockIdx;
static thread_local dim3 blockDim;
static thread_local dim3 gridDim;

static inline void __syncthreads() { pthread_barrier_wait(&emul::g_block.bar); }
static inline unsigned __ballot_sync(unsigned, bool pred) {
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    emul::g_block.warp_flags[w][lane] = pred ? 1u : 0u;
    pthread_barrier_wait(&emul::g_block.warp_bar[w]);
    unsigned m = 0;
    for (int i = 0; i < 32; ++i) m |= emul::g_block.warp_flags[w][i] << i;
    pthread_barrier_wait(&emul::g_block.warp_bar[w]);
    return m;
}
static inline int __popc(unsigned v) { return __builtin_popcount(v); }
template <typename T> static inline T __ldg(const T* p) { return *p; }
static inline float __fadd_rn(float a, float b) { return a + b; }
static inline float __fsub_rn(float a, float b) { return a - b; }
static inline float __fmul_rn(float a, float b) { return a * b; }
static inline float __fdiv_rn(float a, float b) { return a / b; }
static inline double __dadd_rn(double a, double b) { return a + b; }
static inline double __dsub_rn(double a, double b) { return a - b; }
static inline double __dmul_rn(double a, double b) { return a * b; }
static inline double __ddiv_rn(double a, double b) { return a / b; }
static inline float __int_as_float(int v) { float f; memcpy(&f, &v, 4); return f; }
static inline int __float_as_int(float f) { int v; memcpy(&v, &f, 4); return v; }
static inline unsigned __float_as_uint(float f) { unsigned v; memcpy(&v, &f, 4); return v; }
static inline int atomicExch(int* p, int v) { return __atomic_exchange_n(p, v, __ATOMIC_SEQ_CST); }
static inline int atomicAdd(int* p, int v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
static inline int atomicCAS(int* p, int compare, int v) {
    __atomic_compare_exchange_n(p, &compare, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST);
    return compare;                               // the old value, whether or not it was swapped
}
static inline unsigned long long atomicOr(unsigned long long* p, unsigned long long v) {
    return __atomic_fetch_or(p, v, __ATOMIC_SEQ_CST);
}
static inline int atomicMax(int* p, int v) {   // CAS loop
    int old = __atomic_load_n(p, __ATOMIC_SEQ_CST);
    while (old < v && !__atomic_compare_exchange_n(p, &old, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {
    }
    return old;
}
static inline unsigned long long atomicMax(unsigned long long* p, unsigned long long v) {
    unsigned long long old = __atomic_load_n(p, __ATOMIC_SEQ_CST);
    while (old < v && !__atomic_compare_exchange_n(p, &old, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {
    }
    return old;
}
static inline long long __double_as_longlong(double d) { long long v; memcpy(&v, &d, 8); return v; }
static inline double __longlong_as_double(long long v) { double d; memcpy(&d, &v, 8); return d; }
static inline double atomicAdd(double* p, double v) {   // CAS loop, like pre-sm_60 devices
    uint64_t old_bits, new_bits;
    double old;
    do {
        old_bits = __atomic_load_n(reinterpret_cast<uint64_t*>(p), __ATOMIC_SEQ_CST);
        memcpy(&old, &old_bits, 8);
        const double nv = old + v;
        memcpy(&new_bits, &nv, 8);
    } while (!__atomic_compare_exchange_n(reinterpret_cast<uint64_t*>(p), &old_bits, new_bits, false, __ATOMIC_SEQ_CST,
                                          __ATOMIC_SEQ_CST));
    return old;
}
static inline float atomicAdd(float* p, float v) {
    uint32_t old_bits, new_bits;
    float old;
    do {
        old_bits = __atomic_load_n(reinterpret_cast<uint32_t*>(p), __ATOMIC_SEQ_CST);
        memcpy(&old, &old_bits, 4);
        const float nv = old + v;
        memcpy(&new_bits, &nv, 4);
    } while (!__atomic_compare_exchange_n(reinterpret_cast<uint32_t*>(p), &old_bits, new_bits, false, __ATOMIC_SEQ_CST,
                                          __ATOMIC_SEQ_CST));
    return old;
}
static inline float __double2float_rn(double v) { return (float)v; }
static inline float __uint_as_float(unsigned v) { float f; memcpy(&f, &v, 4); return f; }
static inline void __syncwarp(unsigned = 0xffffffffu) { pthread_barrier_wait(&emul::g_block.warp_bar[threadIdx.x >> 5]); }
#ifndef __grid_constant__
#define __grid_constant__
#endif
template <typename T> static inline T __shfl_xor_sync(unsigned, T v, int lane_mask) {
    static_assert(sizeof(T) <= 8, "shuffle of at most 8 bytes");
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    memcpy(&emul::g_block.warp_vals[w][lane], &v, sizeof(T));
    pthread_barrier_wait(&emul::g_block.warp_bar[w]);
    T r;
    memcpy(&r, &emul::g_block.warp_vals[w][lane ^ lane_mask], sizeof(T));
    pthread_barrier_wait(&emul::g_block.warp_bar[w]);
    return r;
}
template <typename T> static inline T __shfl_down_sync(unsigned, T v, int delta) {
    static_assert(sizeof(T) <= 8, "shuffle of at most 8 bytes");
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    memcpy(&emul::g_block.warp_vals[w][lane], &v, sizeof(T));
    pthread_barrier_wait(&emul::g_block.warp_bar[w]);
    T r = v;
    if (lane + delta < 32) memcpy(&r, &emul::g_block.warp_vals[w][lane + delta], sizeof(T));
    pthread_barrier_wait(&emul::g_block.warp_bar[w]);
    return r;
}
static inline int min(int a, int b) { return a < b ? a : b; }
static inline int max(int a, int b) { return a > b ? a : b; }

namespace emul {
// Run `body` as grid x block CUDA threads (blocks sequentially, the threads of a block concurrently).
inline void launch(dim3 grid, dim3 block, size_t dyn_smem, const std::function<void()>& body) {
    const int nthreads = (int)(block.x * block.y * block.z);
    pthread_barrier_init(&g_block.bar, nullptr, nthreads);
    for (int w = 0; w < (nthreads + 31) / 32; ++w) {
        const int n = (w + 1) * 32 <= nthreads ? 32 : nthreads - w * 32;
        pthread_barrier_init(&g_block.warp_bar[w], nullptr, n);
    }
    std::vector<unsigned char> smem(dyn_smem + 1024);     // 1 KB aligned like the device's swizzled operand tiles want
    g_dyn_smem = (unsigned char*)(((uintptr_t)smem.data() + 1023) & ~(uintptr_t)1023);
    std::vector<std::thread> ts;
    for (int t = 0; t < nthreads; ++t)
        ts.emplace_back([&, t]() {
            blockDim = block;
            gridDim = grid;
            threadIdx.x = t % block.x;
            threadIdx.y = (t / block.x) % block.y;
            threadIdx.z = t / (block.x * block.y);
            for (unsigned bz = 0; bz < grid.z; ++bz)
                for (unsigned by = 0; by < grid.y; ++by)
                    for (unsigned bx = 0; bx < grid.x; ++bx) {
                        blockIdx.x = bx; blockIdx.y = by; blockIdx.z = bz;
                        body();
                        pthread_barrier_wait(&g_block.bar);  // statics (= shared memory) are reused by the next block
                    }
        });
    for (auto& t : ts) t.join();
    pthread_barrier_destroy(&g_block.bar);
    for (int w = 0; w < (nthreads + 31) / 32; ++w) pthread_barrier_destroy(&g_block.warp_bar[w]);
}

// Kernels WITHOUT barriers or warp collectives: run the threads one after another (much faster).
inline void launch_serial(dim3 grid, dim3 block, const std::function<void()>& body) {
    blockDim = block;
    gridDim = grid;
    for (unsigned bz = 0; bz < grid.z; ++bz)
        for (unsigned by = 0; by < grid.y; ++by)
            for (unsigned bx = 0; bx < grid.x; ++bx) {
                blockIdx.x = bx; blockIdx.y = by; blockIdx.z = bz;
                for (unsigned tz = 0; tz < block.z; ++tz)
                    for (unsigned ty = 0; ty < block.y; ++ty)
                        for (unsigned tx = 0; tx < block.x; ++tx) {
                            threadIdx.x = tx; threadIdx.y = ty; threadIdx.z = tz;
                            body();
                        }
            }
}
}  // namespace emul
