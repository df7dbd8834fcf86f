// FUNCTIONAL MODELS of the PTX wrappers the TMA-fed wgmma kernels use (see cuda_host_emul.h for the thread model),
// shared by conv_tc_emul.cpp (forward / input gradient, and the halo kernel through it) and conv_wgrad_emul.cpp (weight
// gradient).  What is modelled: mbarriers (arrival counts, transaction bytes, phase parity), the im2col / tiled TMA
// loads (boxes land 64- / 128-byte swizzled, like the hardware's), wgmma with the device descriptor encoding
// (wgmma_emul.h), named barriers.  A wrong phase shows up as a deadlock (reported after a timeout); a TMA load whose
// filter offset lies outside the im2col map's window sets g_fault.  Included once per library, at file scope.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>

#include <atomic>
#include <chrono>
#include <map>
#include <mutex>

#include "../../fewshot_detection_b200/csrc/common.cuh"

namespace emul {
Block g_block;
unsigned char* g_dyn_smem = nullptr;
}  // namespace emul

namespace fsdet {
void set_error(const char*, ...) {}

// ---- helpers conv_tc.cu defines before including the kernel headers
static inline float scale_from_amax(float a) {   // conv_tc.cu: power of two mapping amax into [512, 1024)
    if (!(a > 0.f) || !std::isfinite(a)) return 1.f;
    int ex = (int)((__float_as_uint(a) >> 23) & 0xff) - 126;
    int e = 10 - ex;
    e = e < -60 ? -60 : (e > 60 ? 60 : e);
    return __uint_as_float((uint32_t)(e + 127) << 23);
}
static inline float ldg_f32(const float* p) { return *p; }

// ---- models
static std::atomic<bool> g_deadlock{false};
static std::atomic<bool> g_fault{false};
static std::mutex g_mu;
struct Bar { int count, pending; long long tx; int phase; };
static std::map<const void*, Bar> g_bars;

struct MapModel {   // lives in the first bytes of a CUtensorMap
    int kind;       // 0 = im2col activation plane, 1 = 2-D tiled plane (weights, dz), 3 = tiled 4-D activation box
    const uint16_t* base;
    float* z;
    int B, H, W, C, cpitch, ks, pad, bk, box_rows, rows, ldz;   // box_rows: pixels per im2col box, rows per tiled box
    long long K, M;
};
static inline const MapModel* model(const CUtensorMap* m) { return reinterpret_cast<const MapModel*>(m); }

static inline uint32_t smem_u32(const void* p) { return (uint32_t)((const unsigned char*)p - emul::g_dyn_smem); }

static void bar_check(Bar& b) {
    if (b.pending == 0 && b.tx == 0) { b.phase ^= 1; b.pending = b.count; }
}
static inline void mbar_init(uint64_t* bar, uint32_t count) {
    std::lock_guard<std::mutex> l(g_mu);
    g_bars[bar] = Bar{(int)count, (int)count, 0, 0};
}
static inline void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    std::lock_guard<std::mutex> l(g_mu);
    Bar& b = g_bars[bar];
    b.tx += bytes; b.pending -= 1;
    bar_check(b);
}
static inline void bar_complete_tx(uint64_t* bar, uint32_t bytes) {
    std::lock_guard<std::mutex> l(g_mu);
    Bar& b = g_bars[bar];
    b.tx -= bytes;
    bar_check(b);
}
static inline void mbar_arrive(uint64_t* bar) {
    std::lock_guard<std::mutex> l(g_mu);
    Bar& b = g_bars[bar];
    b.pending -= 1;
    bar_check(b);
}
static inline void mbar_wait(uint64_t* bar, uint32_t parity) {
    const auto t0 = std::chrono::steady_clock::now();
    for (;;) {
        {
            std::lock_guard<std::mutex> l(g_mu);
            if ((uint32_t)g_bars[bar].phase != parity) return;   // the phase with this parity has completed
        }
        if (g_deadlock.load()) return;
        if (std::chrono::steady_clock::now() - t0 > std::chrono::seconds(60)) { g_deadlock.store(true); return; }
        std::this_thread::sleep_for(std::chrono::microseconds(20));   // whole warps poll (elect_one pattern): keep the lock free
    }
}
// whole-warp wait: OS threads are not lock-step, a slow lane could miss a complete phase flip that lane 0 already acted
// on - so lane 0 polls and the warp converges behind it
static inline void mbar_wait_warp(uint64_t* bar, uint32_t parity) {
    if ((threadIdx.x & 31) == 0) mbar_wait(bar, parity);
    __syncwarp();
}
static inline void fence_barrier_init() {}
static inline void tma_prefetch_desc(const CUtensorMap*) {}

#include "wgmma_emul.h"

// element k of row r of a TMA box with rows of `row_bytes` bytes, through the shared-memory swizzle of the tensor map
static inline void box_store(void* dst, int r, int k, int row_bytes, uint16_t v) {
    const uint32_t a = swizzle_addr(smem_u32(dst) + (uint32_t)(r * row_bytes + k * 2), row_bytes == 128 ? GMMA_SW128 : GMMA_SW64);
    memcpy(emul::g_dyn_smem + a, &v, 2);
}

// box_rows consecutive output pixels starting at the pixel whose filter window has its corner at (w, h) of image n;
// one filter tap (off_w, off_h), channels c .. c+bk-1; zero outside the image / beyond the last pixel.  The hardware
// only takes offsets inside the filter window the map was encoded with (ks x ks): anything else is a fault.
static inline void tma_load_im2col_4d(void* dst, const CUtensorMap* map, uint64_t* bar, int c, int w, int h, int n,
                                      uint16_t off_w, uint16_t off_h) {
    const MapModel* m = model(map);
    if (off_w >= m->ks || off_h >= m->ks) g_fault.store(true);
    long long pix0 = ((long long)n * m->H + (h + m->pad)) * m->W + (w + m->pad);
    const long long total = (long long)m->B * m->H * m->W;
    for (int i = 0; i < m->box_rows; ++i) {
        const long long pi = pix0 + i;
        bool ok = pi < total;
        int img = 0, y = 0, x = 0;
        if (ok) {
            img = (int)(pi / ((long long)m->H * m->W));
            const int rem = (int)(pi - (long long)img * m->H * m->W);
            y = rem / m->W - m->pad + off_h;
            x = rem % m->W - m->pad + off_w;
            ok = y >= 0 && y < m->H && x >= 0 && x < m->W;
        }
        for (int k = 0; k < m->bk; ++k) {
            const int ch = c + k;
            box_store(dst, i, k, m->bk * 2, (ok && ch < m->C) ? m->base[(((size_t)img * m->H + y) * m->W + x) * m->cpitch + ch] : (uint16_t)0);
        }
    }
    bar_complete_tx(bar, (uint32_t)(m->box_rows * m->bk * 2));
}
// box of box_rows rows x bk columns of a [rows][K] plane at (column c0, row c1); zero beyond the tensor
static inline void tma_load_2d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
    const MapModel* m = model(map);
    for (int r = 0; r < m->box_rows; ++r)
        for (int k = 0; k < m->bk; ++k) {
            const long long row = c1 + r, col = c0 + k;
            box_store(dst, r, k, m->bk * 2, (row < m->rows && col < m->K) ? m->base[(size_t)row * m->K + col] : (uint16_t)0);
        }
    bar_complete_tx(bar, (uint32_t)(m->box_rows * m->bk * 2));
}
// thread-block clusters are not modelled (blocks run one after another): the cluster flavour is never instantiated here
static inline uint32_t cluster_ctarank() { return 0; }
static inline void cluster_sync_all() {}
static inline void tma_load_2d_mc(void*, const CUtensorMap*, uint64_t*, int, int, uint16_t) { g_deadlock.store(true); }
static inline void mbar_arrive_cluster(uint64_t*, uint32_t) { g_deadlock.store(true); }
static inline bool elect_one() { return (threadIdx.x & 31) == 0; }

}  // namespace fsdet
