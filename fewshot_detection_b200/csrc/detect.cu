// Detection decode + non-maximum suppression + reweighting-vector ensembling on the device (SURVEY.md §8f row 1).
//
// Replaces, for evaluation (valid_ensemble.py:86-178):
//   utils.get_region_boxes     utils.py:112-193   tensor prologue, 7 device->host copies, triple Python loop
//   utils.get_region_boxes_v2  utils.py:195-290   same + softmax across the n_cls class rows of each image
//   utils.nms                  utils.py:85-104    O(n^2) Python loop per (image, class) row
//   the running mean of the support net's vectors per class, valid_ensemble.py:86-100
//
// Number formats follow the reference under torch 0.3.1 (requirements.txt:3): tensor math in float32; everything
// that the reference does on elements indexed out of a tensor (Python floats) in float64: the confidence test
// `det_conf * cls_conf > conf_thresh`, the normalisation x/w, the NMS key float32(1 - det_conf) and the NMS IoUs
// (utils.bbox_iou, utils.py:21-52, operation order kept, no FMA contraction).
#include "common.cuh"
#include "detect_records.cuh"
#include "eval_sort.cuh"

// tools/host_emul compiles this file with g++ (threads = OS threads) to test the block-level logic without a GPU
#ifdef FSDET_HOST_EMULATION
#define FSDET_DYN_SMEM(name) unsigned char* name = emul::g_dyn_smem
#else
#define FSDET_DYN_SMEM(name) extern __shared__ __align__(16) unsigned char name[]
#endif

namespace fsdet {

constexpr int kDetThreads = 256;
constexpr int kCandFloats = 8;  // xs, ys, ws, hs, det_conf, cls_max_conf, (int) cls_max_id, (int) a*HW + cell

__device__ __forceinline__ float sigmoid_acc(float v) { return 1.f / (1.f + expf(-v)); }

// Exclusive prefix (thread order) of a per-thread flag over a 256-thread block, and the block total.
__device__ __forceinline__ int block_flag_scan(bool flag, int* s_warp, int& total) {
    const unsigned m = __ballot_sync(0xffffffffu, flag);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int pre = __popc(m & ((1u << lane) - 1u));
    if (lane == 0) s_warp[w] = __popc(m);
    __syncthreads();
    int base = 0, tot = 0;
#pragma unroll
    for (int i = 0; i < kDetThreads / 32; ++i) {
        const int c = s_warp[i];
        if (i < w) base += c;
        tot += c;
    }
    __syncthreads();  // s_warp is reused by the caller's next chunk
    total = tot;
    return base + pre;
}

struct DetArgs {
    const float* out;      // [N][A*(5+nC)][H][W]
    const float* anchors;  // [2A]
    float* cand;           // [N][cap][8]
    int32_t* count;        // [N]
    float* cls_dense;      // optional [N*A*HW][nC]
    int N, A, nC, H, W, cs, v2, only_obj, cap;
    double thresh;
};

// One CTA per row n (an image of the plain detector, an (image, class) pair of the meta detector).  Candidates are
// written in the reference's loop order (cy, cx, anchor) by an ordered block compaction.
__global__ void __launch_bounds__(kDetThreads) region_detect_kernel(DetArgs p) {
    __shared__ int s_warp[kDetThreads / 32];
    const int n = blockIdx.x;
    const int HW = p.H * p.W, K = p.A * HW, C5 = 5 + p.nC;
    const int b0 = (n / p.cs) * p.cs;  // first row of this row's image (cs == 1 for the plain detector)
    const size_t row_stride = (size_t)p.A * C5 * HW;
    int base = 0;
    for (int k0 = 0; k0 < K; k0 += kDetThreads) {
        const int k = k0 + threadIdx.x;
        bool pass = false;
        float xs = 0.f, ys = 0.f, ws = 0.f, hs = 0.f, det = 0.f, cmax = 0.f;
        int cid = 0, cell = 0, a = 0;
        if (k < K) {
            cell = k / p.A;
            a = k - cell * p.A;
            const float* o = p.out + (size_t)n * row_stride + (size_t)a * C5 * HW + cell;
            det = sigmoid_acc(__ldg(o + 4 * HW));
            cmax = -1.f;
            if (p.v2) {
                // utils.py:213-220: softmax over the cs class rows of the image, per (anchor, class channel, cell)
                for (int cc = 0; cc < p.nC; ++cc) {
                    const float* q = p.out + (size_t)b0 * row_stride + (size_t)a * C5 * HW + (size_t)(5 + cc) * HW + cell;
                    float mx = -INFINITY;
                    for (int m = 0; m < p.cs; ++m) mx = fmaxf(mx, __ldg(q + m * row_stride));
                    float sum = 0.f;
                    for (int m = 0; m < p.cs; ++m) sum += expf(__ldg(q + m * row_stride) - mx);
                    const float v = __fdiv_rn(expf(__ldg(q + (size_t)(n - b0) * row_stride) - mx), sum);
                    if (p.cls_dense) p.cls_dense[((size_t)n * K + (size_t)a * HW + cell) * p.nC + cc] = v;
                    if (v > cmax) { cmax = v; cid = cc; }
                }
            } else {
                // utils.py:141: softmax over the nC class logits of the anchor-cell
                float mx = -INFINITY;
                for (int cc = 0; cc < p.nC; ++cc) mx = fmaxf(mx, __ldg(o + (size_t)(5 + cc) * HW));
                float sum = 0.f;
                for (int cc = 0; cc < p.nC; ++cc) sum += expf(__ldg(o + (size_t)(5 + cc) * HW) - mx);
                for (int cc = 0; cc < p.nC; ++cc) {
                    const float v = __fdiv_rn(expf(__ldg(o + (size_t)(5 + cc) * HW) - mx), sum);
                    if (p.cls_dense) p.cls_dense[((size_t)n * K + (size_t)a * HW + cell) * p.nC + cc] = v;
                    if (v > cmax) { cmax = v; cid = cc; }
                }
            }
            const double conf = p.only_obj ? (double)det : __dmul_rn((double)det, (double)cmax);
            pass = conf > p.thresh;
            if (pass) {
                xs = __fadd_rn(sigmoid_acc(__ldg(o)), (float)(cell % p.W));
                ys = __fadd_rn(sigmoid_acc(__ldg(o + HW)), (float)(cell / p.W));
                ws = __fmul_rn(expf(__ldg(o + 2 * HW)), __ldg(p.anchors + 2 * a));
                hs = __fmul_rn(expf(__ldg(o + 3 * HW)), __ldg(p.anchors + 2 * a + 1));
            }
        }
        int total;
        const int slot = base + block_flag_scan(pass, s_warp, total);
        if (pass && slot < p.cap) {
            float4* dst = reinterpret_cast<float4*>(p.cand + ((size_t)n * p.cap + slot) * kCandFloats);
            dst[0] = make_float4(xs, ys, ws, hs);
            dst[1] = make_float4(det, cmax, __int_as_float(cid), __int_as_float(a * HW + cell));
        }
        base += total;
    }
    if (threadIdx.x == 0) p.count[n] = base < p.cap ? base : p.cap;
}

// float64 IoU of (cx, cy, w, h) boxes, utils.py:21-52 (x1y1x2y2=False)
__device__ __forceinline__ double nms_iou(const double4 p, const double4 q) {
    const double mx = fmin(__dsub_rn(p.x, __ddiv_rn(p.z, 2.0)), __dsub_rn(q.x, __ddiv_rn(q.z, 2.0)));
    const double Mx = fmax(__dadd_rn(p.x, __ddiv_rn(p.z, 2.0)), __dadd_rn(q.x, __ddiv_rn(q.z, 2.0)));
    const double my = fmin(__dsub_rn(p.y, __ddiv_rn(p.w, 2.0)), __dsub_rn(q.y, __ddiv_rn(q.w, 2.0)));
    const double My = fmax(__dadd_rn(p.y, __ddiv_rn(p.w, 2.0)), __dadd_rn(q.y, __ddiv_rn(q.w, 2.0)));
    const double uw = __dsub_rn(Mx, mx);
    const double uh = __dsub_rn(My, my);
    const double cw = __dsub_rn(__dadd_rn(p.z, q.z), uw);
    const double ch = __dsub_rn(__dadd_rn(p.w, q.w), uh);
    if (cw <= 0.0 || ch <= 0.0) return 0.0;
    const double area1 = __dmul_rn(p.z, p.w);
    const double area2 = __dmul_rn(q.z, q.w);
    const double carea = __dmul_rn(cw, ch);
    const double uarea = __dsub_rn(__dadd_rn(area1, area2), carea);
    return __ddiv_rn(carea, uarea);
}

// One CTA per row: bitonic sort of (float32(1 - det_conf), slot) ascending = torch.sort of utils.py:89-93 with list
// order on ties, then the greedy suppression loop of utils.py:95-103 with the inner loop spread over the block.
// Dynamic shared memory: P * (8 + 32 + 1) bytes, P = power of two >= cap.
// boxes64 != nullptr: rows of already-normalised float64 boxes [N][cap][5] = {x, y, w, h, det_conf} (the list-of-lists
// form utils.nms receives) instead of `cand`.
__global__ void __launch_bounds__(kDetThreads) nms_kernel(const float* __restrict__ cand, const double* __restrict__ boxes64,
                                                          const int32_t* __restrict__ count, int cap, int P, int H, int W,
                                                          double thresh, int32_t* __restrict__ keep,
                                                          int32_t* __restrict__ keep_count) {
    FSDET_DYN_SMEM(smem_raw);
    double4* box = reinterpret_cast<double4*>(smem_raw);                                   // [P]
    unsigned long long* keys = reinterpret_cast<unsigned long long*>(box + P);             // [P]
    unsigned char* alive = reinterpret_cast<unsigned char*>(keys + P);                     // [P]
    __shared__ int s_warp[kDetThreads / 32];
    const int row = blockIdx.x;
    const int n = min(count[row], cap);
    if (n <= 0) {
        if (threadIdx.x == 0) keep_count[row] = 0;
        return;
    }
    int Pn = 1;
    while (Pn < n) Pn <<= 1;
    const float* c = cand ? cand + (size_t)row * cap * kCandFloats : nullptr;
    const double* c64 = boxes64 ? boxes64 + (size_t)row * cap * 5 : nullptr;
    for (int t = threadIdx.x; t < Pn; t += kDetThreads) {
        unsigned long long key = ~0ull;
        if (t < n) {
            const double det = c64 ? c64[(size_t)t * 5 + 4] : (double)c[(size_t)t * kCandFloats + 4];
            const float kf = (float)__dsub_rn(1.0, det);   // det_confs[i] = 1 - boxes[i][4] into a FloatTensor
            key = ((unsigned long long)__float_as_uint(kf) << 32) | (unsigned)t;
        }
        keys[t] = key;
    }
    __syncthreads();
    for (int k = 2; k <= Pn; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int t = threadIdx.x; t < Pn; t += kDetThreads) {
                const int u = t ^ j;
                if (u > t) {
                    const unsigned long long x = keys[t], y = keys[u];
                    const bool up = (t & k) == 0;
                    if ((x > y) == up) { keys[t] = y; keys[u] = x; }
                }
            }
            __syncthreads();
        }
    }
    for (int t = threadIdx.x; t < n; t += kDetThreads) {
        const int slot = (int)(keys[t] & 0xffffffffu);
        if (c64) {
            const double* q = c64 + (size_t)slot * 5;
            box[t] = make_double4(q[0], q[1], q[2], q[3]);
            alive[t] = q[4] > 0.0 ? 1 : 0;
        } else {
            const float4 v = *reinterpret_cast<const float4*>(c + (size_t)slot * kCandFloats);
            const float det = c[(size_t)slot * kCandFloats + 4];
            box[t] = make_double4(__ddiv_rn((double)v.x, (double)W), __ddiv_rn((double)v.y, (double)H),
                                  __ddiv_rn((double)v.z, (double)W), __ddiv_rn((double)v.w, (double)H));
            alive[t] = det > 0.f ? 1 : 0;
        }
    }
    __syncthreads();
    for (int i = 0; i < n; ++i) {
        if (!alive[i]) continue;  // block-uniform: alive[i] was last written before an earlier barrier
        const double4 bi = box[i];
        for (int j = i + 1 + threadIdx.x; j < n; j += kDetThreads)
            if (alive[j] && nms_iou(bi, box[j]) > thresh) alive[j] = 0;
        __syncthreads();
    }
    int base = 0;
    for (int t0 = 0; t0 < n; t0 += kDetThreads) {
        const int t = t0 + threadIdx.x;
        const bool f = t < n && alive[t];
        int total;
        const int pos = base + block_flag_scan(f, s_warp, total);
        if (f) keep[(size_t)row * cap + pos] = (int)(keys[t] & 0xffffffffu);
        base += total;
    }
    if (threadIdx.x == 0) keep_count[row] = base;
}

// valid_ensemble.py:96-98, float32: e[c] = e[c]*cnt/(cnt+1) + dw[i]/(cnt+1) for the samples i of class c, in order.
__global__ void rw_running_mean_kernel(float* __restrict__ e, const int32_t* __restrict__ cnt_in, int32_t* __restrict__ cnt_out,
                                       const float* __restrict__ dw, const int32_t* __restrict__ ids, int n, int n_cls, int C) {
    const int c = blockIdx.y;
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    int cnt = cnt_in[c];
    float v = (k < C) ? e[(size_t)c * C + k] : 0.f;
    for (int i = 0; i < n; ++i) {
        if (ids[i] != c) continue;
        const float f0 = (float)cnt, f1 = (float)(cnt + 1);
        if (k < C) v = __fadd_rn(__fdiv_rn(__fmul_rn(v, f0), f1), __fdiv_rn(dw[(size_t)i * C + k], f1));
        ++cnt;
    }
    if (k < C) e[(size_t)c * C + k] = v;
    if (k == 0) cnt_out[c] = cnt;
}

static inline int next_pow2(int v) {
    int p = 1;
    while (p < v) p <<= 1;
    return p;
}

// ---- per-image selection of the meta detector's NMS survivors (fsdet_detect_select) ---------------------------------
// Every survivor of the batch is a record, numbered in row order (image, class) and then NMS rank.  One stable LSD
// radix sort (eval_sort.cuh) orders the records by ~bits(prob) (low word, then high word), then by image: within an
// image, prob descending with ties in record order, i.e. class ascending, then NMS rank ascending.  The record count is
// only known on the device, so the sort's grid covers every candidate slot and its kernels read the count.
struct SelectWorkspace {
    int32_t* row_off;                                 // [N + 1] first record of each row
    long long* n_rec;                                 // [1] records of the batch
    int32_t* rec;                                     // [N * cap] record -> row * cap + candidate slot
    uint32_t* keys[2];
    int32_t* vals[2];
    unsigned long long* cnt;
    unsigned long long* part;
    size_t bytes;
};

static SelectWorkspace select_workspace_layout(void* base, int N, int cap) {
    const long long n = (long long)N * cap;
    const int ntiles = ceil_div(n, kVocTile);
    const size_t n_cnt = (size_t)256 * ntiles;
    const size_t n_part = (size_t)ceil_div((long long)n_cnt, kVocTile) + 1;
    SelectWorkspace w;
    unsigned char* p = static_cast<unsigned char*>(base);
    size_t off = 0;
    auto take = [&](size_t bytes) { unsigned char* q = p ? p + off : nullptr; off += voc_align(bytes); return q; };
    w.row_off = reinterpret_cast<int32_t*>(take((size_t)(N + 1) * 4));
    w.n_rec = reinterpret_cast<long long*>(take(8));
    w.rec = reinterpret_cast<int32_t*>(take((size_t)n * 4));
    w.keys[0] = reinterpret_cast<uint32_t*>(take((size_t)n * 4));
    w.keys[1] = reinterpret_cast<uint32_t*>(take((size_t)n * 4));
    w.vals[0] = reinterpret_cast<int32_t*>(take((size_t)n * 4));
    w.vals[1] = reinterpret_cast<int32_t*>(take((size_t)n * 4));
    w.cnt = reinterpret_cast<unsigned long long*>(take(n_cnt * 8));
    w.part = reinterpret_cast<unsigned long long*>(take(n_part * 8));
    w.bytes = off;
    return w;
}

// One block: the first record of every row (exclusive prefix of keep_count) and the batch's record count.
__global__ void __launch_bounds__(kDetThreads) select_offsets_kernel(const int32_t* __restrict__ keep_count, int N,
                                                                     int cap, int32_t* __restrict__ row_off,
                                                                     long long* __restrict__ n_rec) {
    __shared__ unsigned long long s[kVocThreads];
    unsigned long long base = 0;
    for (int r0 = 0; r0 < N; r0 += kDetThreads) {
        const int r = r0 + threadIdx.x;
        const int c = r < N ? min(max(keep_count[r], 0), cap) : 0;
        unsigned long long chunk;
        const unsigned long long pre = voc_block_scan((unsigned long long)c, s, chunk);
        if (r < N) row_off[r] = (int32_t)(base + pre);
        base += chunk;
    }
    if (threadIdx.x == 0) {
        row_off[N] = (int32_t)base;
        *n_rec = (long long)base;
    }
}

// One block per row: survivor k (NMS rank) becomes record row_off[r] + k.
__global__ void __launch_bounds__(kDetThreads) select_compact_kernel(const int32_t* __restrict__ keep,
                                                                     const int32_t* __restrict__ row_off, int cap,
                                                                     int32_t* __restrict__ rec) {
    const int r = blockIdx.x;
    const int o = row_off[r], n = row_off[r + 1] - o;
    for (int k = threadIdx.x; k < n; k += kDetThreads) rec[o + k] = r * cap + keep[(size_t)r * cap + k];
}

// valid.detection_lines' prob = det_conf * cls_conf, float64 (exact: a product of two float32 values)
template <class Rows>
__device__ __forceinline__ double select_prob(const Rows& rows, size_t id) {
    return __dmul_rn((double)rows.det(id), (double)rows.cls(id));
}

// Key word `word` of the records taken in the order perm (nullptr: record order): 0 / 1 the low / high half of
// ~bits(prob) (the bits of a non-negative double order like its value, so ascending ~bits is descending prob),
// 2 the image.  Rows: a reader of detect_records.cuh.
template <class Rows>
__global__ void __launch_bounds__(kDetThreads) select_keys_kernel(const Rows rows,
                                                                  const int32_t* __restrict__ rec,
                                                                  const int32_t* __restrict__ perm,
                                                                  const long long* __restrict__ n_rec, int cap,
                                                                  int n_cls, int word, uint32_t* __restrict__ keys) {
    const long long n = *n_rec;
    for (long long j = (long long)blockIdx.x * kDetThreads + threadIdx.x; j < n; j += (long long)gridDim.x * kDetThreads) {
        const int id = rec[perm ? perm[j] : j];
        uint32_t k;
        if (word == 2) {
            k = (uint32_t)(id / cap / n_cls);
        } else {
            const unsigned long long b = ~(unsigned long long)__double_as_longlong(select_prob(rows, (size_t)id));
            k = word ? (uint32_t)(b >> 32) : (uint32_t)b;
        }
        keys[j] = k;
    }
}

// One block per image: its records are the contiguous run [row_off[b * n_cls], row_off[(b + 1) * n_cls]) of the sorted
// order; the first max_det become the image's result, in pixels with valid.detection_lines' float64 arithmetic.
// Slots past the count are written as score 0, box 0, class -1.
template <class Rows>
__global__ void __launch_bounds__(kDetThreads) select_write_kernel(const Rows rows,
                                                                   const int32_t* __restrict__ rec,
                                                                   const int32_t* __restrict__ order,
                                                                   const int32_t* __restrict__ row_off,
                                                                   const int32_t* __restrict__ sizes, int cap, int n_cls,
                                                                   int max_det, double* __restrict__ score,
                                                                   double* __restrict__ box, int32_t* __restrict__ cls,
                                                                   int32_t* __restrict__ count, int32_t* __restrict__ total) {
    const int b = blockIdx.x;
    const int s0 = row_off[b * n_cls], s1 = row_off[(b + 1) * n_cls];
    const int n = min(s1 - s0, max_det);
    const double width = (double)sizes[2 * b], height = (double)sizes[2 * b + 1];
    for (int t = threadIdx.x; t < max_det; t += kDetThreads) {
        const size_t o = (size_t)b * max_det + t;
        double4 bx = make_double4(0.0, 0.0, 0.0, 0.0);
        double sc = 0.0;
        int c = -1;
        if (t < n) {
            const int id = rec[order[s0 + t]];
            const double4 q = rows.box((size_t)id);
            const double x = q.x, y = q.y;
            const double w2 = __ddiv_rn(q.z, 2.0);
            const double h2 = __ddiv_rn(q.w, 2.0);
            bx = make_double4(__dmul_rn(__dsub_rn(x, w2), width), __dmul_rn(__dsub_rn(y, h2), height),
                              __dmul_rn(__dadd_rn(x, w2), width), __dmul_rn(__dadd_rn(y, h2), height));
            sc = select_prob(rows, (size_t)id);
            c = (id / cap) % n_cls;
        }
        score[o] = sc;
        box[o * 4 + 0] = bx.x;
        box[o * 4 + 1] = bx.y;
        box[o * 4 + 2] = bx.z;
        box[o * 4 + 3] = bx.w;
        cls[o] = c;
    }
    if (threadIdx.x == 0) {
        count[b] = n;
        total[b] = s1 - s0;
    }
}

template <class Rows>
static int detect_select_impl(const Rows& rows, const int32_t* keep, const int32_t* keep_count, int N, int cap,
                              int n_cls, const int32_t* sizes, int max_det, void* workspace, double* score, double* box,
                              int32_t* cls, int32_t* count, int32_t* total, cudaStream_t st) {
    (void)st;
    const SelectWorkspace w = select_workspace_layout(workspace, N, cap);
    const int B = N / n_cls;
    const long long n_slots = (long long)N * cap;
    const int ntiles = ceil_div(n_slots, kVocTile);
    const int kgrid = ceil_div(n_slots, kDetThreads) < 2048 ? ceil_div(n_slots, kDetThreads) : 2048;
    VOC_LAUNCH(1, kDetThreads, select_offsets_kernel, keep_count, N, cap, w.row_off, w.n_rec);
    VOC_CHECK("detect_select_offsets");
    VOC_LAUNCH(N, kDetThreads, select_compact_kernel, keep, w.row_off, cap, w.rec);
    VOC_CHECK("detect_select_compact");
    int img_bits = 0;
    while ((1 << img_bits) < B) ++img_bits;
    const int word_passes[3] = {4, 4, (img_bits + 7) / 8};
    const int32_t* perm = nullptr;                    // record order
    int cur = 0;
    for (int word = 0; word < 3; ++word) {
        if (word_passes[word] == 0) continue;
        // the word's keys in the current order go to the key buffer the next pass does not write
        VOC_LAUNCH(kgrid, kDetThreads, select_keys_kernel<Rows>, rows, w.rec, perm, w.n_rec, cap, n_cls, word,
                   w.keys[cur ^ 1]);
        VOC_CHECK("detect_select_keys");
        const uint32_t* kin = w.keys[cur ^ 1];
        for (int p = 0; p < word_passes[word]; ++p) {
            VOC_LAUNCH(ntiles, kVocThreads, voc_radix_hist_kernel, kin, (int)n_slots, 8 * p, ntiles, w.cnt, w.n_rec);
            VOC_CHECK("detect_select_radix_hist");
            const int rc = voc_scan(w.cnt, (long long)256 * ntiles, w.part, 0, st);
            if (rc) return rc;
            VOC_LAUNCH(ntiles, kVocThreads, voc_radix_scatter_kernel, kin, perm, (int)n_slots, 8 * p, ntiles, w.cnt,
                       w.keys[cur], w.vals[cur], w.n_rec);
            VOC_CHECK("detect_select_radix_scatter");
            kin = w.keys[cur];
            perm = w.vals[cur];
            cur ^= 1;
        }
    }
    VOC_LAUNCH(B, kDetThreads, select_write_kernel<Rows>, rows, w.rec, perm, w.row_off, sizes, cap, n_cls, max_det,
               score, box, cls, count, total);
    VOC_CHECK("detect_select_write");
    return 0;
}

// ---- test-time augmentation: the candidates of several passes in one table per row (fsdet_tta_merge) ----------------
// One CTA per row, one launch per pass: the pass's candidates of row r go to merged[r][merged_count[r] ...) in slot
// order, as the reference's box lists of the pass would be appended to the row's list, with the box normalised to the
// image in float64 (x = xs / W, ..., utils.py:270) and mirrored (x = 1.0 - x) for a flipped pass.  A row whose pass does
// not fit in merged_cap records takes none of it and sets *overflow.
__global__ void __launch_bounds__(kDetThreads) tta_merge_kernel(const float* __restrict__ cand,
                                                                const int32_t* __restrict__ count, int cap, int H, int W,
                                                                int flip, int pass, TtaRecord* __restrict__ merged,
                                                                int32_t* __restrict__ merged_count, int merged_cap,
                                                                int32_t* __restrict__ overflow) {
    const int r = blockIdx.x;
    const int n = min(max(count[r], 0), cap);
    const int off = merged_count[r];
    __syncthreads();                                  // every thread has read the offset before it moves
    if (off < 0 || (long long)off + n > merged_cap) {
        if (threadIdx.x == 0) *overflow = 1;
        return;
    }
    for (int t = threadIdx.x; t < n; t += kDetThreads) {
        const float* v = cand + ((size_t)r * cap + t) * kCandFloats;
        TtaRecord q;
        const double x = __ddiv_rn((double)v[0], (double)W);
        q.x = flip ? __dsub_rn(1.0, x) : x;
        q.y = __ddiv_rn((double)v[1], (double)H);
        q.w = __ddiv_rn((double)v[2], (double)W);
        q.h = __ddiv_rn((double)v[3], (double)H);
        q.det = v[4];
        q.cls = v[5];
        q.cid = __float_as_int(v[6]);
        q.src = (pass << kTtaSlotBits) | t;
        merged[(size_t)r * merged_cap + off + t] = q;
    }
    if (threadIdx.x == 0) merged_count[r] = off + n;
}

// ---- NMS over merged rows of any length (fsdet_nms_merged) ------------------------------------------------------------
// utils.nms on every row: a stable sort on float32(1 - det_conf), then greedy suppression with the float64 IoU.
// 1. Every candidate of the batch is a record (row order, then slot); one stable LSD radix sort (eval_sort.cuh) orders
//    them by the key, then by row: per row, key ascending with ties in merged order.  The workspace is the per-image
//    selection's (SelectWorkspace).
// 2. One CTA per row streams its sorted boxes through shared memory kNmsChunk at a time.  A box is kept iff its
//    det_conf > 0 and no kept box before it overlaps it by more than the threshold, so each chunk is first tested
//    against every box the earlier chunks kept (in parallel, no order needed), then suppressed greedily within itself,
//    exactly as fsdet_nms does for a whole row.
constexpr int kNmsChunk = 1024;
constexpr int kNmsMergedMaxCap = 1 << 16;

__global__ void __launch_bounds__(kDetThreads) nms_merged_compact_kernel(const int32_t* __restrict__ row_off, int cap,
                                                                         int32_t* __restrict__ rec) {
    const int r = blockIdx.x;
    const int o = row_off[r], n = row_off[r + 1] - o;
    for (int k = threadIdx.x; k < n; k += kDetThreads) rec[o + k] = r * cap + k;
}

// The bits of a float ordered like its value (so ascending key = ascending float32(1 - det_conf)).
__device__ __forceinline__ uint32_t nms_key_bits(float f) {
    const uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// word 0: the NMS key of the records taken in the order perm (nullptr: record order); 1: the row.
__global__ void __launch_bounds__(kDetThreads) nms_merged_keys_kernel(const TtaRecord* __restrict__ merged,
                                                                      const int32_t* __restrict__ rec,
                                                                      const int32_t* __restrict__ perm,
                                                                      const long long* __restrict__ n_rec, int cap,
                                                                      int word, uint32_t* __restrict__ keys) {
    const long long n = *n_rec;
    for (long long j = (long long)blockIdx.x * kDetThreads + threadIdx.x; j < n; j += (long long)gridDim.x * kDetThreads) {
        const int id = rec[perm ? perm[j] : j];
        keys[j] = word ? (uint32_t)(id / cap)
                       : nms_key_bits((float)__dsub_rn(1.0, (double)merged[id].det));   // det_confs[i] = 1 - boxes[i][4]
    }
}

__global__ void __launch_bounds__(kDetThreads) nms_merged_suppress_kernel(const TtaRecord* __restrict__ merged,
                                                                          const int32_t* __restrict__ rec,
                                                                          const int32_t* __restrict__ order,
                                                                          const int32_t* __restrict__ row_off, int cap,
                                                                          double thresh, int32_t* __restrict__ keep,
                                                                          int32_t* __restrict__ keep_count) {
    __shared__ double4 s_box[kNmsChunk];
    __shared__ double4 s_kept[kDetThreads];
    __shared__ unsigned char s_alive[kNmsChunk];
    __shared__ int s_warp[kDetThreads / 32];
    const int r = blockIdx.x;
    const int s0 = row_off[r], n = row_off[r + 1] - s0;
    const TtaRecord* row = merged + (size_t)r * cap;
    int32_t* krow = keep + (size_t)r * cap;
    int n_kept = 0;
    for (int c0 = 0; c0 < n; c0 += kNmsChunk) {
        const int m = min(kNmsChunk, n - c0);
        for (int t = threadIdx.x; t < m; t += kDetThreads) {
            const TtaRecord& q = merged[rec[order[s0 + c0 + t]]];
            s_box[t] = make_double4(q.x, q.y, q.w, q.h);
            s_alive[t] = q.det > 0.f ? 1 : 0;
        }
        // Suppressors: the boxes the earlier chunks kept, staged kDetThreads at a time, then the chunk's own boxes in
        // order.  One sweep per suppressor (one IoU call site: ptxas keeps the float64 division's slow path unspilled).
        for (int k0 = 0;; k0 += kDetThreads) {
            const bool kept = k0 < n_kept;           // block-uniform
            __syncthreads();                          // s_box / s_alive written; s_kept free
            if (kept && k0 + (int)threadIdx.x < n_kept) {
                const TtaRecord& q = row[krow[k0 + threadIdx.x]];
                s_kept[threadIdx.x] = make_double4(q.x, q.y, q.w, q.h);
            }
            if (kept) __syncthreads();
            const int ns = kept ? min(kDetThreads, n_kept - k0) : m;
            for (int v = 0; v < ns; ++v) {
                if (!kept && !s_alive[v]) continue;   // block-uniform: alive[v] was last written before a barrier
                const double4 bi = kept ? s_kept[v] : s_box[v];
                for (int j = (kept ? 0 : v + 1) + threadIdx.x; j < m; j += kDetThreads)
                    if (s_alive[j] && nms_iou(bi, s_box[j]) > thresh) s_alive[j] = 0;
                if (!kept) __syncthreads();
            }
            if (!kept) break;
        }
        for (int t0 = 0; t0 < m; t0 += kDetThreads) {
            const int t = t0 + threadIdx.x;
            const bool f = t < m && s_alive[t];
            int total;
            const int pos = n_kept + block_flag_scan(f, s_warp, total);
            if (f) krow[pos] = rec[order[s0 + c0 + t]] - r * cap;
            n_kept += total;
        }
        __syncthreads();                              // krow of this chunk visible to the block; s_box free
    }
    if (threadIdx.x == 0) keep_count[r] = n_kept;
}

static int nms_merged_impl(const TtaRecord* merged, const int32_t* count, int N, int cap, double thresh, void* workspace,
                           int32_t* keep, int32_t* keep_count, cudaStream_t st) {
    (void)st;
    const SelectWorkspace w = select_workspace_layout(workspace, N, cap);
    const long long n_slots = (long long)N * cap;
    const int ntiles = ceil_div(n_slots, kVocTile);
    const int kgrid = ceil_div(n_slots, kDetThreads) < 2048 ? ceil_div(n_slots, kDetThreads) : 2048;
    VOC_LAUNCH(1, kDetThreads, select_offsets_kernel, count, N, cap, w.row_off, w.n_rec);
    VOC_CHECK("nms_merged_offsets");
    VOC_LAUNCH(N, kDetThreads, nms_merged_compact_kernel, w.row_off, cap, w.rec);
    VOC_CHECK("nms_merged_compact");
    int row_bits = 0;
    while ((1 << row_bits) < N) ++row_bits;
    const int word_passes[2] = {4, (row_bits + 7) / 8};
    const int32_t* perm = nullptr;                    // record order
    int cur = 0;
    for (int word = 0; word < 2; ++word) {
        if (word_passes[word] == 0) continue;
        VOC_LAUNCH(kgrid, kDetThreads, nms_merged_keys_kernel, merged, w.rec, perm, w.n_rec, cap, word, w.keys[cur ^ 1]);
        VOC_CHECK("nms_merged_keys");
        const uint32_t* kin = w.keys[cur ^ 1];
        for (int p = 0; p < word_passes[word]; ++p) {
            VOC_LAUNCH(ntiles, kVocThreads, voc_radix_hist_kernel, kin, (int)n_slots, 8 * p, ntiles, w.cnt, w.n_rec);
            VOC_CHECK("nms_merged_radix_hist");
            const int rc = voc_scan(w.cnt, (long long)256 * ntiles, w.part, 0, st);
            if (rc) return rc;
            VOC_LAUNCH(ntiles, kVocThreads, voc_radix_scatter_kernel, kin, perm, (int)n_slots, 8 * p, ntiles, w.cnt,
                       w.keys[cur], w.vals[cur], w.n_rec);
            VOC_CHECK("nms_merged_radix_scatter");
            kin = w.keys[cur];
            perm = w.vals[cur];
            cur ^= 1;
        }
    }
    VOC_LAUNCH(N, kDetThreads, nms_merged_suppress_kernel, merged, w.rec, perm, w.row_off, cap, thresh, keep, keep_count);
    VOC_CHECK("nms_merged_suppress");
    return 0;
}

}  // namespace fsdet

#ifndef FSDET_HOST_EMULATION
using namespace fsdet;

extern "C" int fsdet_region_detect(const float* output, const float* anchors_f32, int N, int A, int nC, int H, int W,
                                   int n_models, int v2, int only_objectness, double conf_thresh, float* cand,
                                   int32_t* count, float* cls_dense, void* stream) {
    FSDET_CHECK_ARG(output && anchors_f32 && cand && count, "region_detect: null pointer");
    FSDET_CHECK_ARG(aligned16(cand), "region_detect: cand must be 16-byte aligned");
    FSDET_CHECK_ARG(N >= 0 && A > 0 && nC > 0 && H > 0 && W > 0, "region_detect: bad shape");
    FSDET_CHECK_ARG(n_models >= 1 && (v2 ? N % n_models == 0 : n_models == 1),
                    "region_detect: %d rows are not a multiple of n_models=%d", N, n_models);
    if (N == 0) return 0;
    DetArgs p;
    p.out = output; p.anchors = anchors_f32; p.cand = cand; p.count = count; p.cls_dense = cls_dense;
    p.N = N; p.A = A; p.nC = nC; p.H = H; p.W = W; p.cs = n_models; p.v2 = v2; p.only_obj = only_objectness;
    p.cap = A * H * W; p.thresh = conf_thresh;
    region_detect_kernel<<<N, kDetThreads, 0, (cudaStream_t)stream>>>(p);
    return launch_status("region_detect");
}

static int launch_nms(const float* cand, const double* boxes64, const int32_t* count, int N, int cap, int H, int W,
                      double nms_thresh, int32_t* keep, int32_t* keep_count, void* stream) {
    FSDET_CHECK_ARG((cand || boxes64) && count && keep && keep_count, "nms: null pointer");
    FSDET_CHECK_ARG(!cand || aligned16(cand), "nms: cand must be 16-byte aligned");
    FSDET_CHECK_ARG(cap > 0 && cap <= 4096, "nms: %d candidates per row (1..4096)", cap);
    FSDET_CHECK_ARG(H > 0 && W > 0 && N >= 0, "nms: bad shape");
    if (N == 0) return 0;
    const int P = next_pow2(cap);
    const size_t smem = (size_t)P * (sizeof(double4) + sizeof(unsigned long long) + 1);
    cudaError_t e = cudaFuncSetAttribute(nms_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { set_error("nms: smem attribute: %s", cudaGetErrorString(e)); return (int)e; }
    nms_kernel<<<N, kDetThreads, smem, (cudaStream_t)stream>>>(cand, boxes64, count, cap, P, H, W, nms_thresh, keep,
                                                               keep_count);
    return launch_status("nms");
}

extern "C" int fsdet_nms(const float* cand, const int32_t* count, int N, int cap, int H, int W, double nms_thresh,
                         int32_t* keep, int32_t* keep_count, void* stream) {
    return launch_nms(cand, nullptr, count, N, cap, H, W, nms_thresh, keep, keep_count, stream);
}

extern "C" int fsdet_nms_boxes64(const double* boxes, const int32_t* count, int N, int cap, double nms_thresh,
                                 int32_t* keep, int32_t* keep_count, void* stream) {
    return launch_nms(nullptr, boxes, count, N, cap, 1, 1, nms_thresh, keep, keep_count, stream);
}

extern "C" size_t fsdet_detect_select_workspace_bytes(int N, int cap) {
    if (N < 0 || cap <= 0) return 0;
    return select_workspace_layout(nullptr, N, cap).bytes;
}

extern "C" int fsdet_detect_select(const float* cand, const int32_t* keep, const int32_t* keep_count, int N, int cap, int H,
                                   int W, int n_cls, const int32_t* sizes, int max_det, void* workspace,
                                   size_t workspace_bytes, double* score, double* box, int32_t* cls, int32_t* count,
                                   int32_t* total, void* stream) {
    FSDET_CHECK_ARG(cand && keep && keep_count && sizes && workspace && score && box && cls && count && total,
                    "detect_select: null pointer");
    FSDET_CHECK_ARG(n_cls > 0 && N > 0 && N % n_cls == 0, "detect_select: %d rows are not images x %d classes", N, n_cls);
    FSDET_CHECK_ARG(cap > 0 && H > 0 && W > 0 && max_det > 0, "detect_select: bad shape");
    FSDET_CHECK_ARG((long long)N * cap < 0x7fffffffll, "detect_select: %d rows x %d candidates do not fit int32", N, cap);
    FSDET_CHECK_ARG(workspace_bytes >= select_workspace_layout(nullptr, N, cap).bytes,
                    "detect_select: workspace of %zu bytes, %zu needed", workspace_bytes,
                    select_workspace_layout(nullptr, N, cap).bytes);
    return detect_select_impl(CandRows{cand, H, W}, keep, keep_count, N, cap, n_cls, sizes, max_det, workspace, score,
                              box, cls, count, total, (cudaStream_t)stream);
}

extern "C" int fsdet_detect_select_merged(const void* merged, const int32_t* keep, const int32_t* keep_count, int N,
                                          int cap, int n_cls, const int32_t* sizes, int max_det, void* workspace,
                                          size_t workspace_bytes, double* score, double* box, int32_t* cls,
                                          int32_t* count, int32_t* total, void* stream) {
    FSDET_CHECK_ARG(merged && keep && keep_count && sizes && workspace && score && box && cls && count && total,
                    "detect_select_merged: null pointer");
    FSDET_CHECK_ARG(n_cls > 0 && N > 0 && N % n_cls == 0, "detect_select_merged: %d rows are not images x %d classes", N,
                    n_cls);
    FSDET_CHECK_ARG(cap > 0 && max_det > 0, "detect_select_merged: bad shape");
    FSDET_CHECK_ARG((long long)N * cap < 0x7fffffffll, "detect_select_merged: %d rows x %d candidates do not fit int32",
                    N, cap);
    FSDET_CHECK_ARG(workspace_bytes >= select_workspace_layout(nullptr, N, cap).bytes,
                    "detect_select_merged: workspace of %zu bytes, %zu needed", workspace_bytes,
                    select_workspace_layout(nullptr, N, cap).bytes);
    return detect_select_impl(MergedRows{static_cast<const TtaRecord*>(merged)}, keep, keep_count, N, cap, n_cls, sizes,
                              max_det, workspace, score, box, cls, count, total, (cudaStream_t)stream);
}

extern "C" int fsdet_tta_merge(const float* cand, const int32_t* count, int N, int cap, int H, int W, int flip,
                               int pass, void* merged, int32_t* merged_count, int merged_cap, int32_t* overflow,
                               void* stream) {
    FSDET_CHECK_ARG(cand && count && merged && merged_count && overflow, "tta_merge: null pointer");
    FSDET_CHECK_ARG(N >= 0 && cap > 0 && cap <= (1 << kTtaSlotBits) && H > 0 && W > 0 && merged_cap > 0,
                    "tta_merge: bad shape (at most %d candidates per row of a pass)", 1 << kTtaSlotBits);
    FSDET_CHECK_ARG(pass >= 0 && pass < kTtaMaxPasses, "tta_merge: pass %d outside 0..%d", pass, kTtaMaxPasses - 1);
    FSDET_CHECK_ARG(flip == 0 || flip == 1, "tta_merge: flip must be 0 or 1");
    if (N == 0) return 0;
    tta_merge_kernel<<<N, kDetThreads, 0, (cudaStream_t)stream>>>(cand, count, cap, H, W, flip, pass,
                                                                   static_cast<TtaRecord*>(merged), merged_count,
                                                                   merged_cap, overflow);
    return launch_status("tta_merge");
}

extern "C" size_t fsdet_nms_merged_workspace_bytes(int N, int cap) {
    if (N < 0 || cap <= 0) return 0;
    return select_workspace_layout(nullptr, N, cap).bytes;
}

extern "C" int fsdet_nms_merged(const void* merged, const int32_t* count, int N, int cap, double nms_thresh,
                                void* workspace, size_t workspace_bytes, int32_t* keep, int32_t* keep_count,
                                void* stream) {
    FSDET_CHECK_ARG(merged && count && workspace && keep && keep_count, "nms_merged: null pointer");
    FSDET_CHECK_ARG(N >= 0 && cap > 0 && cap <= kNmsMergedMaxCap, "nms_merged: %d candidates per row (1..%d)", cap,
                    kNmsMergedMaxCap);
    FSDET_CHECK_ARG((long long)N * cap < 0x7fffffffll, "nms_merged: %d rows x %d candidates do not fit int32", N, cap);
    FSDET_CHECK_ARG(workspace_bytes >= select_workspace_layout(nullptr, N, cap).bytes,
                    "nms_merged: workspace of %zu bytes, %zu needed", workspace_bytes,
                    select_workspace_layout(nullptr, N, cap).bytes);
    if (N == 0) return 0;
    return nms_merged_impl(static_cast<const TtaRecord*>(merged), count, N, cap, nms_thresh, workspace, keep, keep_count,
                           (cudaStream_t)stream);
}

extern "C" int fsdet_rw_running_mean(float* enews, const int32_t* cnt_in, int32_t* cnt_out, const float* dw,
                                     const int32_t* ids, int n, int n_cls, int C, void* stream) {
    FSDET_CHECK_ARG(enews && cnt_in && cnt_out && cnt_in != cnt_out, "rw_running_mean: null or aliased counters");
    FSDET_CHECK_ARG(n == 0 || (dw && ids), "rw_running_mean: null pointer");
    FSDET_CHECK_ARG(n >= 0 && n_cls > 0 && C > 0, "rw_running_mean: bad shape");
    dim3 grid(ceil_div(C, 128), n_cls);
    rw_running_mean_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(enews, cnt_in, cnt_out, dw, ids, n, n_cls, C);
    return launch_status("rw_running_mean");
}
#endif  // FSDET_HOST_EMULATION
