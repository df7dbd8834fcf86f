// Shared helpers for libfsdet.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/fsdet.h"

namespace fsdet {

void set_error(const char* fmt, ...);

#define FSDET_CHECK_ARG(cond, ...)          \
    do {                                    \
        if (!(cond)) {                      \
            fsdet::set_error(__VA_ARGS__);  \
            return -1;                      \
        }                                   \
    } while (0)

// Launch epilogue: report a failed launch as the positive cudaError_t.
inline int launch_status(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        set_error("%s: %s", what, cudaGetErrorString(e));
        return (int)e;
    }
    return 0;
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

static inline int ceil_div(long long a, long long b) { return (int)((a + b - 1) / b); }

constexpr int kNumSMs = 132;  // H100 SXM

__device__ __forceinline__ float leaky(float u, float slope) { return u > 0.f ? u : u * slope; }

__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

}  // namespace fsdet
