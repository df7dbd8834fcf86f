// Block scan, stable LSD radix sort, uint64 prefix sums, the gather plan and the pool merge shared by the device
// evaluators (voc_eval.cu, coco_eval.cu) and the per-image selection (detect.cu), with the launch macros that run them either on the device or under host emulation (tools/host_emul).
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
// n_live (optional, device): the number of items when only the device knows it; the grid then covers n >= *n_live
// items and the tiles past *n_live sort nothing.
__global__ void __launch_bounds__(kVocThreads) voc_radix_hist_kernel(const uint32_t* __restrict__ keys, int n, int shift,
                                                                     int ntiles, unsigned long long* __restrict__ cnt,
                                                                     const long long* __restrict__ n_live = nullptr) {
    __shared__ int h[256];
    if (n_live && *n_live < n) n = (int)*n_live;
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
                                                                        int32_t* __restrict__ vals_out,
                                                                        const long long* __restrict__ n_live = nullptr) {
    __shared__ unsigned long long base[256];
    if (n_live && *n_live < n) n = (int)*n_live;
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

// ---- gather plan: one batch of Detections (after NMS) -> group descriptors --------------------------------------
// counters (int64): [0] records in the pool, [1] groups, [2] first group of the last batch, [3] overflow flag.
// One block: the batch's rows get consecutive groups and record ranges (row order = result-file order per class); row r
// takes min(keep_count[r], row_limit) records.  A batch that does not fit, or follows an overflow, sets the flag and
// writes nothing.
__global__ void __launch_bounds__(kVocThreads) eval_gather_plan_kernel(const int32_t* __restrict__ keep_count, int N,
                                                                       int n_cls, const int32_t* __restrict__ image_index,
                                                                       int row_limit, long long pool_cap,
                                                                       int32_t* __restrict__ groups, int group_cap,
                                                                       long long* counters) {
    __shared__ unsigned long long s[kVocThreads];
    __shared__ int s_ok;
    const long long pool0 = counters[0], group0 = counters[1];
    // pass 1: total, to decide whether the batch fits
    unsigned long long sum = 0;
    for (int r = threadIdx.x; r < N; r += kVocThreads) sum += (unsigned long long)min(max(keep_count[r], 0), row_limit);
    unsigned long long total;
    voc_block_scan(sum, s, total);
    if (threadIdx.x == 0)
        s_ok = counters[3] == 0 && pool0 + (long long)total <= pool_cap && group0 + N <= (long long)group_cap;
    __syncthreads();
    if (!s_ok) {
        if (threadIdx.x == 0) counters[3] = 1;
        return;
    }
    // pass 2: ordered ranges
    unsigned long long base = 0;
    for (int r0 = 0; r0 < N; r0 += kVocThreads) {
        const int r = r0 + threadIdx.x;
        const int c = r < N ? min(max(keep_count[r], 0), row_limit) : 0;
        unsigned long long chunk;
        const unsigned long long pre = voc_block_scan((unsigned long long)c, s, chunk);
        if (r < N) {
            int32_t* g = groups + (group0 + r) * 4;
            g[0] = (int32_t)(pool0 + (long long)(base + pre));
            g[1] = c;
            g[2] = image_index[r / n_cls];
            g[3] = r % n_cls;
        }
        base += chunk;
    }
    if (threadIdx.x == 0) {
        counters[0] = pool0 + (long long)total;
        counters[1] = group0 + N;
        counters[2] = group0;
    }
}

// ---- merge:the pools of several accumulators (one per rank of a sharded evaluation) -> one pool -----------------
// Source s holds counters src_counters[s][4], records [s * src_pool_stride, + its record count) and groups
// [s * src_group_stride, + its group count).  The merged pool takes the sources in order: records are copied, each
// group's first record is rebased.  Error bits in counters[3]: overflow (a source overflowed, or the destination is
// too small: nothing is written), an image in the groups of two sources, a group outside its source's records or
// image range (written as an empty group).
constexpr long long kMergeOverflow = 1, kMergeDuplicateImage = 2, kMergeBadGroup = 4;

struct MergeWorkspace {
    long long* rec_off;                               // [n_src + 1] first merged record of each source
    long long* grp_off;                               // [n_src + 1] first merged group of each source
    int32_t* owner;                                   // [n_images] the source whose groups name the image, or -1
    size_t bytes;
};

static MergeWorkspace merge_workspace_layout(void* base, int n_src, int n_images) {
    MergeWorkspace w;
    unsigned char* p = static_cast<unsigned char*>(base);
    size_t off = 0;
    auto take = [&](size_t bytes) { unsigned char* q = p ? p + off : nullptr; off += (bytes + 255) & ~(size_t)255; return q; };
    w.rec_off = reinterpret_cast<long long*>(take((size_t)(n_src + 1) * 8));
    w.grp_off = reinterpret_cast<long long*>(take((size_t)(n_src + 1) * 8));
    w.owner = reinterpret_cast<int32_t*>(take((size_t)n_images * 4));
    w.bytes = off;
    return w;
}

// One block: owner table cleared, source offsets by a serial pass over the (few) sources, destination counters set.
__global__ void __launch_bounds__(kVocThreads) eval_merge_plan_kernel(const long long* __restrict__ src_counters, int n_src,
                                                                      long long src_pool_stride, long long src_group_stride,
                                                                      long long pool_cap, long long group_cap, int n_images,
                                                                      MergeWorkspace w, long long* __restrict__ counters) {
    for (int i = threadIdx.x; i < n_images; i += kVocThreads) w.owner[i] = -1;
    if (threadIdx.x != 0) return;
    long long r = 0, g = 0, err = 0;
    for (int s = 0; s < n_src; ++s) {
        const long long* c = src_counters + (size_t)s * 4;
        long long nr = c[0], ng = c[1];
        if (c[3] != 0 || nr < 0 || nr > src_pool_stride || ng < 0 || ng > src_group_stride) {
            err |= kMergeOverflow | (c[3] & ~kMergeOverflow);
            nr = ng = 0;
        }
        w.rec_off[s] = r;
        w.grp_off[s] = g;
        r += nr;
        g += ng;
    }
    w.rec_off[n_src] = r;
    w.grp_off[n_src] = g;
    if (r > pool_cap || g > group_cap) err |= kMergeOverflow;
    counters[0] = (err & kMergeOverflow) ? 0 : r;
    counters[1] = (err & kMergeOverflow) ? 0 : g;
    counters[2] = 0;
    counters[3] = err;
}

// grid (blocks, n_src): group i of source s -> merged group grp_off[s] + i, its first record + rec_off[s]
__global__ void __launch_bounds__(kVocThreads) eval_merge_groups_kernel(const int32_t* __restrict__ src_groups,
                                                                        long long src_group_stride, int n_images,
                                                                        MergeWorkspace w, int32_t* __restrict__ groups,
                                                                        long long* counters) {
    if (counters[3] & kMergeOverflow) return;
    const int s = blockIdx.y;
    const long long ng = w.grp_off[s + 1] - w.grp_off[s], nr = w.rec_off[s + 1] - w.rec_off[s];
    unsigned long long* flag = reinterpret_cast<unsigned long long*>(counters + 3);
    for (long long i = (long long)blockIdx.x * kVocThreads + threadIdx.x; i < ng; i += (long long)gridDim.x * kVocThreads) {
        const int32_t* g = src_groups + ((size_t)s * src_group_stride + i) * 4;
        const long long first = g[0];
        const int count = g[1], img = g[2], cls = g[3];
        int32_t* d = groups + (size_t)(w.grp_off[s] + i) * 4;
        if (first < 0 || count < 0 || first + count > nr || img < 0 || img >= n_images) {
            atomicOr(flag, (unsigned long long)kMergeBadGroup);
            d[0] = (int32_t)w.rec_off[s];
            d[1] = 0;
            d[2] = 0;
            d[3] = cls;
            continue;
        }
        d[0] = (int32_t)(w.rec_off[s] + first);
        d[1] = count;
        d[2] = img;
        d[3] = cls;
        const int prev = atomicCAS(&w.owner[img], -1, s);
        if (prev != -1 && prev != s) atomicOr(flag, (unsigned long long)kMergeDuplicateImage);
    }
}

// grid (blocks, n_src): record i of source s -> merged record rec_off[s] + i (key and box[4])
template <typename K>
__global__ void __launch_bounds__(kVocThreads) eval_merge_records_kernel(const K* __restrict__ src_key,
                                                                         const double* __restrict__ src_box,
                                                                         long long src_pool_stride, MergeWorkspace w,
                                                                         const long long* __restrict__ counters,
                                                                         K* __restrict__ key, double* __restrict__ box) {
    if (counters[3] & kMergeOverflow) return;
    const int s = blockIdx.y;
    const long long n = w.rec_off[s + 1] - w.rec_off[s], d0 = w.rec_off[s];
    const size_t s0 = (size_t)s * src_pool_stride;
    for (long long i = (long long)blockIdx.x * kVocThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kVocThreads) {
        key[d0 + i] = src_key[s0 + i];
        for (int q = 0; q < 4; ++q) box[(d0 + i) * 4 + q] = src_box[(s0 + i) * 4 + q];
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

template <typename K>
static int eval_merge_impl(int n_src, const long long* src_counters, const K* src_key, const double* src_box,
                           long long src_pool_stride, const int32_t* src_groups, long long src_group_stride, int n_images,
                           void* workspace, K* key, double* box, long long pool_cap, int32_t* groups, int group_cap,
                           long long* counters, cudaStream_t st) {
    (void)st;
    const MergeWorkspace w = merge_workspace_layout(workspace, n_src, n_images);
    VOC_LAUNCH(1, kVocThreads, eval_merge_plan_kernel, src_counters, n_src, src_pool_stride, src_group_stride, pool_cap,
               (long long)group_cap, n_images, w, counters);
    VOC_CHECK("eval_merge_plan");
    if (src_group_stride > 0) {
        const int gb = (int)(ceil_div(src_group_stride, kVocThreads) < 256 ? ceil_div(src_group_stride, kVocThreads) : 256);
        VOC_LAUNCH(dim3(gb, n_src), kVocThreads, eval_merge_groups_kernel, src_groups, src_group_stride, n_images, w,
                   groups, counters);
        VOC_CHECK("eval_merge_groups");
    }
    if (src_pool_stride > 0) {
        const int rb = (int)(ceil_div(src_pool_stride, kVocThreads) < 1024 ? ceil_div(src_pool_stride, kVocThreads) : 1024);
        VOC_LAUNCH(dim3(rb, n_src), kVocThreads, eval_merge_records_kernel<K>, src_key, src_box, src_pool_stride, w,
                   counters, key, box);
        VOC_CHECK("eval_merge_records");
    }
    return 0;
}

}  // namespace
}  // namespace fsdet
