// Functional models of the wgmma wrappers of csrc/tc_ptx.cuh for the host-emulation builds (see cuda_host_emul.h for the
// thread model).  Included inside namespace fsdet by the *_emul.cpp files, after their smem_u32() / mbarrier models.
//
// Shared memory is addressed the way the hardware does it: the descriptors have the device bit layout (start address,
// LBO, SBO, swizzle mode), the logical address of an operand element follows the canonical K-major / MN-major layouts,
// and the 64- / 128-byte swizzle is the XOR of address bits [4,6) / [4,7) with bits [7,9) / [7,10) of the (1 KB
// aligned) shared-memory offset.  The modelled TMA loads store their boxes through the same swizzle, so descriptor
// encodings, K advances inside a swizzle atom and the TMA / wgmma layout agreement are all checked on the CPU.
// Each thread computes its own accumulator fragment (rows 16 * warp + lane / 4 (+ 8), columns 8j + 2 (lane % 4) (+ 1)
// of the warpgroup's 64 x N tile).
//
// Completion is asynchronous, as on the device: wgmma() only queues the operation in the thread's open group,
// wgmma_commit() closes that group, and wgmma_wait<N>() executes the oldest committed groups - reading shared memory and
// writing the accumulators at that moment - until at most N remain.  A stage released to the producer before the group
// that reads it has been waited for, or an accumulator read before its group is complete, therefore gives a wrong result
// once the producer runs ahead (g_mma_delay_us).  Operations still queued when a block ends are a kernel bug:
// wgmma_block_exit() reports them.
#pragma once

constexpr uint32_t GMMA_SW128 = 1, GMMA_SW64 = 2;
static inline uint64_t gmma_desc(uint32_t saddr, uint32_t lbo, uint32_t sbo, uint32_t swz) {
    return (uint64_t)((saddr & 0x3FFFF) >> 4) | ((uint64_t)(lbo >> 4) << 16) | ((uint64_t)(sbo >> 4) << 32) | ((uint64_t)swz << 62);
}
static inline uint32_t swizzle_addr(uint32_t addr, uint32_t swz) {
    if (swz == GMMA_SW128) return addr ^ (((addr >> 7) & 7u) << 4);
    if (swz == GMMA_SW64) return addr ^ (((addr >> 7) & 3u) << 4);
    return addr;
}
static inline float emul_h2f(uint16_t b) { __half_raw r; r.x = b; return __half2float(__half(r)); }
static inline float gmma_operand(uint64_t desc, bool mn_major, int idx, int k) {   // idx = M or N index, k = 0..15
    const uint32_t start = (uint32_t)(desc & 0x3FFF) << 4;
    const uint32_t lbo = (uint32_t)((desc >> 16) & 0x3FFF) << 4, sbo = (uint32_t)((desc >> 32) & 0x3FFF) << 4;
    const uint32_t swz = (uint32_t)(desc >> 62);
    const uint32_t row_bytes = swz == GMMA_SW128 ? 128u : 64u;
    uint32_t a;
    if (mn_major)   // a row = one K index with 64 M/N elements; 8-row groups SBO apart; 64-element blocks LBO apart
        a = start + (uint32_t)(idx / 64) * lbo + (uint32_t)(k / 8) * sbo + (uint32_t)(k % 8) * 128u + (uint32_t)(idx % 64) * 2u;
    else            // a row = one M/N index, K contiguous inside the row; 8-row groups SBO apart
        a = start + (uint32_t)(idx / 8) * sbo + (uint32_t)(idx % 8) * row_bytes + (uint32_t)k * 2u;
    uint16_t v;
    memcpy(&v, emul::g_dyn_smem + swizzle_addr(a, swz), 2);
    return emul_h2f(v);
}

struct WgmmaOp {
    float* d;
    uint64_t da, db;
    uint32_t accumulate;
    int n;
    bool ta, tb;
};
static inline void wgmma_execute(const WgmmaOp& o) {
    const int t = (int)(threadIdx.x & 127), wq = t >> 5, lane = t & 31;
    for (int j = 0; j < o.n / 8; ++j)
        for (int e = 0; e < 4; ++e) {
            const int row = 16 * wq + (lane >> 2) + 8 * (e >> 1), col = 8 * j + 2 * (lane & 3) + (e & 1);
            float acc = o.accumulate ? o.d[4 * j + e] : 0.f;
            for (int k = 0; k < 16; ++k) acc += gmma_operand(o.da, o.ta, row, k) * gmma_operand(o.db, o.tb, col, k);
            o.d[4 * j + e] = acc;
        }
}
static thread_local std::vector<WgmmaOp> t_wgmma_open;                 // issued since the last commit
static thread_local std::deque<std::vector<WgmmaOp>> t_wgmma_groups;   // committed, not yet complete (oldest first)

template <int N, int TA = 0, int TB = 0>
static inline void wgmma(float* d, uint64_t da, uint64_t db, uint32_t accumulate) {
    t_wgmma_open.push_back(WgmmaOp{d, da, db, accumulate, N, TA != 0, TB != 0});
}
static std::atomic<int> g_mma_delay_us{0};   // slows the MMA warpgroups down so that the producers run far ahead
static inline void wgmma_fence() {}
static inline void wgmma_commit() {
    t_wgmma_groups.push_back(std::move(t_wgmma_open));
    t_wgmma_open.clear();
}
template <int N> static inline void wgmma_wait() {
    if (g_mma_delay_us.load() > 0) std::this_thread::sleep_for(std::chrono::microseconds(g_mma_delay_us.load()));
    while (t_wgmma_groups.size() > (size_t)N) {
        for (const WgmmaOp& o : t_wgmma_groups.front()) wgmma_execute(o);
        t_wgmma_groups.pop_front();
    }
}
// set when a thread ended a block with wgmma operations still queued (the emulated launches return -102)
static std::atomic<bool> g_wgmma_pending_at_exit{false};
// called by every thread when its kernel body returns
static inline void wgmma_block_exit() {
    if (!t_wgmma_open.empty() || !t_wgmma_groups.empty()) g_wgmma_pending_at_exit.store(true);
    t_wgmma_open.clear();
    t_wgmma_groups.clear();
}
template <int R> static inline void wgmma_use(float*) {}
template <int R> static inline void regs_dec() {}
template <int R> static inline void regs_inc() {}

// barrier over a subset of the block's threads (bar.sync id, n): generation counter per id
struct NamedBar { int waiting = 0; long long gen = 0; };
static NamedBar g_named[16];
static inline void named_bar_sync(int id, int nthreads) {
    long long my;
    {
        std::lock_guard<std::mutex> l(g_mu);
        NamedBar& b = g_named[id];
        my = b.gen;
        if (++b.waiting == nthreads) { b.waiting = 0; ++b.gen; return; }
    }
    const auto t0 = std::chrono::steady_clock::now();
    for (;;) {
        {
            std::lock_guard<std::mutex> l(g_mu);
            if (g_named[id].gen != my) return;
        }
        if (g_deadlock.load()) return;
        if (std::chrono::steady_clock::now() - t0 > std::chrono::seconds(20)) { g_deadlock.store(true); return; }
        std::this_thread::yield();
    }
}
