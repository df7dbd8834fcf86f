// COCO box AP / AR on the device (pycocotools COCOeval, iouType='bbox', useCats=1), from the detections that decode +
// NMS (detect.cu) leave there.  The host evaluator coco_eval.py defines every number; this file reproduces it bit for
// bit in float64 (explicit _rn intrinsics: no FMA contraction).
//
// Data model.  An accumulator owns a pool of detection records:
//   score double    det_conf * cls_conf
//   box   double[4] x, y, w, h: the unclipped result-line corners x1 = (bx - bw/2.0) * width, ..., w = x2 - x1
// and one group descriptor per (image, class) row: {first record, record count, image index, class}.  The gather
// writes a row's first maxDets[-1] boxes by a stable sort on score (descending) in that order, so a group's records
// are already the detections pycocotools' evaluateImg keeps, in its order; the groups tile the pool.
//
// Evaluation.
//   1. Canonical order: every group gets its place in (class, image) order from a scan over a dense table.
//   2. Match: one warp per group runs the greedy matching of evaluateImg for the 4 area ranges x 10 IoU thresholds
//      (one lane per pair, 8 lanes take a second pair) and writes per record and area a word of TP / FP bits.
//   3. Rank: a stable LSD radix sort of the canonical sequence on (class, score descending): ties keep image-set
//      order, then rank within the image, as accumulate's mergesort over the image-ordered concatenation does.
//   4. Accumulate: one block per (class, area, maxDets) scans the class's ranked records for the 10 thresholds at once.
//      A record contributes (rc, pr) = (tp / npig, tp / (tp + fp + eps)) at its TP or FP; the precision at recall
//      threshold r is the largest pr with rc >= recThrs[r], or 0: pycocotools' envelope read at searchsorted(rc, r).
#include "detect_records.cuh"
#include "eval_sort.cuh"

namespace fsdet {

constexpr int kCocoT = 10, kCocoR = 101, kCocoA = 4, kCocoM = 3;
constexpr int kCocoPairs = kCocoA * kCocoT;            // (area, IoU threshold) pairs of the matching
constexpr int kCocoFpShift = 16;                      // dt_flags word: TP bits [0, 10), FP bits [16, 26)
constexpr int kCocoMaxClasses = 1 << 16;

struct CocoParams {
    double iou[kCocoT];                               // Params.iouThrs, as computed on the host
    double rec[kCocoR];                               // Params.recThrs
    int max_det[kCocoM];                              // Params.maxDets
    double area[kCocoA][2];                           // Params.areaRng, inclusive
};

// ---- gather: one batch of Detections (after NMS) -> records + group descriptors ---------------------------------
// eval_gather_plan_kernel (eval_sort.cuh) lays out the batch's groups and counters, each row cut to max_det records;
// coco_gather_rows_kernel fills the records.
template <class Rows>
__device__ __forceinline__ double coco_score(const Rows& rows, const int32_t* __restrict__ keep, int r, int cap, int j) {
    const size_t id = (size_t)r * cap + keep[(size_t)r * cap + j];
    return __dmul_rn((double)rows.det(id), (double)rows.cls(id));
}

// One block per row: survivor t goes to rank (# survivors with a higher score, or an equal one earlier), kept if the
// rank is below max_det.  Box as coco_eval.detection_records computes it: box = [xs/W, ys/H, ws/W, hs/H] (float64 of
// the float32 candidate), x1 = (box[0] - box[2]/2.0) * width, x2 = (box[0] + box[2]/2.0) * width, w = x2 - x1.
// Rows: a reader of detect_records.cuh (the candidates of one pass, or the merged records of several).
template <class Rows>
__global__ void __launch_bounds__(kVocThreads) coco_gather_rows_kernel(const Rows rows,
                                                                       const int32_t* __restrict__ keep,
                                                                       const int32_t* __restrict__ keep_count, int cap,
                                                                       int n_cls, int max_det,
                                                                       const double* __restrict__ image_size,
                                                                       const int32_t* __restrict__ groups,
                                                                       const long long* __restrict__ counters,
                                                                       double* __restrict__ score,
                                                                       double* __restrict__ box) {
    if (counters[3]) return;
    const int r = blockIdx.x;
    const long long start = groups[(counters[2] + r) * 4];
    const int count = max(keep_count[r], 0);
    const double width = image_size[(r / n_cls) * 2], height = image_size[(r / n_cls) * 2 + 1];
    for (int t = threadIdx.x; t < count; t += kVocThreads) {
        const double s = coco_score(rows, keep, r, cap, t);
        int rank = 0;
        for (int j = 0; j < count && rank < max_det; ++j) {
            const double o = coco_score(rows, keep, r, cap, j);
            rank += (o > s || (o == s && j < t)) ? 1 : 0;
        }
        if (rank >= max_det) continue;
        const double4 b = rows.box((size_t)r * cap + keep[(size_t)r * cap + t]);
        const double bx = b.x, by = b.y, bw = b.z, bh = b.w;
        const double hw = __ddiv_rn(bw, 2.0), hh = __ddiv_rn(bh, 2.0);
        const double x1 = __dmul_rn(__dsub_rn(bx, hw), width), y1 = __dmul_rn(__dsub_rn(by, hh), height);
        const double x2 = __dmul_rn(__dadd_rn(bx, hw), width), y2 = __dmul_rn(__dadd_rn(by, hh), height);
        const long long d = start + rank;
        score[d] = s;
        box[d * 4 + 0] = x1;
        box[d * 4 + 1] = y1;
        box[d * 4 + 2] = __dsub_rn(x2, x1);
        box[d * 4 + 3] = __dsub_rn(y2, y1);
    }
}

// ---- evaluation ----------------------------------------------------------------------------------------------------
__global__ void coco_fill_kernel(unsigned long long* __restrict__ a, long long n) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        a[i] = 0ull;
}

// table[class * n_images + image] = the group's record count (each (image, class) is one group at most)
__global__ void coco_count_kernel(const int32_t* __restrict__ groups, int n_groups, int n_images,
                                  unsigned long long* __restrict__ table) {
    const int gi = blockIdx.x * blockDim.x + threadIdx.x;
    if (gi >= n_groups) return;
    const int32_t* g = groups + (size_t)gi * 4;
    table[(size_t)g[3] * n_images + g[2]] = (unsigned long long)g[1];
}

// maskApi.c bbIou of detection (dx, dy, dw, dh; area da) and ground truth k
__device__ __forceinline__ double coco_iou(double dx, double dy, double dw, double dh, double da,
                                          const double* __restrict__ gt_box, bool crowd, int k) {
    const double gx = gt_box[(size_t)k * 4], gy = gt_box[(size_t)k * 4 + 1];
    const double gw = gt_box[(size_t)k * 4 + 2], gh = gt_box[(size_t)k * 4 + 3];
    const double w = __dsub_rn(fmin(__dadd_rn(dw, dx), __dadd_rn(gw, gx)), fmax(dx, gx));
    if (w <= 0.0) return 0.0;
    const double h = __dsub_rn(fmin(__dadd_rn(dh, dy), __dadd_rn(gh, gy)), fmax(dy, gy));
    if (h <= 0.0) return 0.0;
    const double i = __dmul_rn(w, h);
    const double u = crowd ? da : __dsub_rn(__dadd_rn(da, __dmul_rn(gw, gh)), i);
    return __ddiv_rn(i, u);
}

__device__ __forceinline__ bool coco_gt_ignored(const double* __restrict__ gt_area, const uint8_t* __restrict__ gt_crowd,
                                                int k, double lo, double hi) {
    const double a = gt_area[k];
    return gt_crowd[k] != 0 || a < lo || a > hi;
}

// evaluateImg's greedy matching of detection (dx, dy, dw, dh) for one (area, threshold) pair: ground truths in the
// order of the stable sort that puts the non-ignored ones first (two passes over the json order).  Returns the
// matched ground truth or -1; *ign = its ignore flag.
__device__ __forceinline__ int coco_match_one(double dx, double dy, double dw, double dh, double da, int gb, int ge,
                                              const double* __restrict__ gt_box, const double* __restrict__ gt_area,
                                              const uint8_t* __restrict__ gt_crowd, const uint8_t* __restrict__ taken,
                                              double lo, double hi, double thr, bool* ign) {
    const double cap = 1.0 - 1e-10;
    double best = cap < thr ? cap : thr;              // min([t, 1 - 1e-10])
    int m = -1;
    bool m_ign = false;
    for (int pass = 0; pass < 2; ++pass) {
        if (pass == 1 && m >= 0 && !m_ign) break;     // a non-ignored match stops at the first ignored ground truth
        for (int k = gb; k < ge; ++k) {
            const bool gi = coco_gt_ignored(gt_area, gt_crowd, k, lo, hi);
            if (gi != (pass == 1)) continue;
            const bool crowd = gt_crowd[k] != 0;
            if (taken[k] && !crowd) continue;
            const double iou = coco_iou(dx, dy, dw, dh, da, gt_box, crowd, k);
            if (iou < best) continue;
            best = iou;
            m = k;
            m_ign = gi;
        }
    }
    *ign = m_ign;
    return m;
}

// One warp per group: the group's place in canonical order, each record's rank within its row, and the matching.
// Lane l owns the pairs p = l and p = l + 32 (< 40), p = area * 10 + threshold, with taken[p * n_gt + k] as
// evaluateImg's gtm row.  dt_flags[a * n_det + record] = TP bits | FP bits << 16, one bit per threshold.
__global__ void __launch_bounds__(kVocThreads) coco_match_kernel(const double* __restrict__ box,
                                                                 const int32_t* __restrict__ groups, int n_groups,
                                                                 const unsigned long long* __restrict__ table,
                                                                 const int32_t* __restrict__ gt_ptr,
                                                                 const double* __restrict__ gt_box,
                                                                 const double* __restrict__ gt_area,
                                                                 const uint8_t* __restrict__ gt_crowd, int n_gt,
                                                                 int n_images, int n_det, CocoParams P,
                                                                 uint8_t* __restrict__ taken, int32_t* __restrict__ canon,
                                                                 uint8_t* __restrict__ rank_of,
                                                                 uint32_t* __restrict__ dt_flags) {
    const int gi = blockIdx.x * (kVocThreads / 32) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (gi >= n_groups) return;                       // whole warps leave together
    const int32_t* g = groups + (size_t)gi * 4;
    const int first = g[0], count = g[1], img = g[2], cls = g[3];
    const size_t cell = (size_t)cls * n_images + img;
    const long long off = (long long)table[cell];
    for (int j = lane; j < count; j += 32) {
        canon[off + j] = first + j;
        rank_of[first + j] = (uint8_t)j;
    }
    const int gb = gt_ptr[cell], ge = gt_ptr[cell + 1];
    const int p0 = lane, p1 = lane + 32;
    const bool has1 = p1 < kCocoPairs;
    uint8_t* tk0 = taken + (size_t)p0 * n_gt;
    uint8_t* tk1 = taken + (size_t)(has1 ? p1 : p0) * n_gt;
    for (int k = gb; k < ge; ++k) {
        tk0[k] = 0;
        if (has1) tk1[k] = 0;
    }
    const int a0 = p0 / kCocoT, t0 = p0 % kCocoT, a1 = has1 ? p1 / kCocoT : 0, t1 = has1 ? p1 % kCocoT : 0;
    for (int d = 0; d < count; ++d) {
        const size_t rec = (size_t)first + d;
        const double dx = box[rec * 4], dy = box[rec * 4 + 1], dw = box[rec * 4 + 2], dh = box[rec * 4 + 3];
        const double da = __dmul_rn(dw, dh);
        bool tp0, fp0, tp1 = false, fp1 = false;
        {
            bool ig;
            const int m = coco_match_one(dx, dy, dw, dh, da, gb, ge, gt_box, gt_area, gt_crowd, tk0, P.area[a0][0],
                                         P.area[a0][1], P.iou[t0], &ig);
            if (m >= 0) tk0[m] = 1;
            const bool dig = m >= 0 ? ig : (da < P.area[a0][0] || da > P.area[a0][1]);
            tp0 = m >= 0 && !dig;
            fp0 = m < 0 && !dig;
        }
        if (has1) {
            bool ig;
            const int m = coco_match_one(dx, dy, dw, dh, da, gb, ge, gt_box, gt_area, gt_crowd, tk1, P.area[a1][0],
                                         P.area[a1][1], P.iou[t1], &ig);
            if (m >= 0) tk1[m] = 1;
            const bool dig = m >= 0 ? ig : (da < P.area[a1][0] || da > P.area[a1][1]);
            tp1 = m >= 0 && !dig;
            fp1 = m < 0 && !dig;
        }
        const unsigned long long tp = (unsigned long long)__ballot_sync(0xffffffffu, tp0) |
                                      ((unsigned long long)(__ballot_sync(0xffffffffu, tp1) & 0xffu) << 32);
        const unsigned long long fp = (unsigned long long)__ballot_sync(0xffffffffu, fp0) |
                                      ((unsigned long long)(__ballot_sync(0xffffffffu, fp1) & 0xffu) << 32);
        if (lane < kCocoA) {
            const uint32_t bits = (uint32_t)((tp >> (kCocoT * lane)) & 0x3ffu) |
                                  ((uint32_t)((fp >> (kCocoT * lane)) & 0x3ffu) << kCocoFpShift);
            dt_flags[(size_t)lane * n_det + rec] = bits;
        }
    }
}

// Radix keys of the ranking, per record of the current permutation `vals`: word 0 / 1 = low / high half of the
// score's order-preserving bits, complemented (descending); word 2 = the class (from the record's group via `cls_of`).
__device__ __forceinline__ unsigned long long coco_score_key(double s) {
    if (s == 0.0) s = 0.0;                            // -0 ties with +0, as in numpy's comparisons
    const unsigned long long u = (unsigned long long)__double_as_longlong(s);
    const unsigned long long ordered = (u >> 63) ? ~u : (u | (1ull << 63));
    return ~ordered;
}

__global__ void coco_keys_kernel(const double* __restrict__ score, const int32_t* __restrict__ cls_of,
                                 const int32_t* __restrict__ vals, int n, int word, uint32_t* __restrict__ keys) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int p = vals[i];
    keys[i] = word == 2 ? (uint32_t)cls_of[p] : (uint32_t)(coco_score_key(score[p]) >> (32 * word));
}

// the class of every record (from the group table): the ranking's most significant key
__global__ void coco_class_of_kernel(const int32_t* __restrict__ groups, int n_groups, int32_t* __restrict__ cls_of) {
    const int gi = blockIdx.x * (kVocThreads / 32) + (threadIdx.x >> 5);
    if (gi >= n_groups) return;
    const int32_t* g = groups + (size_t)gi * 4;
    for (int j = threadIdx.x & 31; j < g[1]; j += 32) cls_of[g[0] + j] = g[3];
}

// One block per (class k, area a, maxDets m); the class's ranked records in chunks of kVocTile, kVocItems consecutive
// records per thread.  counts per threshold: TP in the high, FP in the low 32 bits.
__global__ void __launch_bounds__(kVocThreads) coco_accumulate_kernel(const int32_t* __restrict__ order,
                                                                      const uint8_t* __restrict__ rank_of,
                                                                      const uint32_t* __restrict__ dt_flags, int n_det,
                                                                      const unsigned long long* __restrict__ table,
                                                                      int n_images, int n_cls,
                                                                      const int32_t* __restrict__ gt_ptr,
                                                                      const double* __restrict__ gt_area,
                                                                      const uint8_t* __restrict__ gt_crowd, CocoParams P,
                                                                      double* __restrict__ precision,
                                                                      double* __restrict__ recall) {
    __shared__ unsigned long long s[kVocThreads];
    __shared__ unsigned long long best[kCocoT][kCocoR];   // bits of the largest pr (>= 0) per threshold and R(rc)
    __shared__ double s_rec[kCocoR];
    __shared__ int s_cnt[kVocThreads / 32];
    const int k = blockIdx.x, a = blockIdx.y, m = blockIdx.z;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const double lo_a = P.area[a][0], hi_a = P.area[a][1];
    const int max_det = P.max_det[m];
    // npig: the class's non-ignored ground truths in the area range, over every image of the set
    int np_ = 0;
    for (int g = gt_ptr[(size_t)k * n_images] + threadIdx.x; g < gt_ptr[(size_t)(k + 1) * n_images]; g += kVocThreads)
        np_ += coco_gt_ignored(gt_area, gt_crowd, g, lo_a, hi_a) ? 0 : 1;
    for (int o = 16; o; o >>= 1) np_ += __shfl_xor_sync(0xffffffffu, np_, o);
    if (lane == 0) s_cnt[w] = np_;
    for (int i = threadIdx.x; i < kCocoT * kCocoR; i += kVocThreads) best[i / kCocoR][i % kCocoR] = 0ull;
    for (int i = threadIdx.x; i < kCocoR; i += kVocThreads) s_rec[i] = P.rec[i];
    __syncthreads();
    int npig = 0;
    for (int q = 0; q < kVocThreads / 32; ++q) npig += s_cnt[q];
    const size_t out_km = (size_t)k * kCocoA * kCocoM + (size_t)a * kCocoM + m;     // [.., K, A, M] tail of both layouts
    const size_t stride_t = (size_t)n_cls * kCocoA * kCocoM;
    if (npig == 0) {                                  // accumulate's `continue`: stays -1
        for (int i = threadIdx.x; i < kCocoT * kCocoR; i += kVocThreads) precision[(size_t)i * stride_t + out_km] = -1.0;
        for (int t = threadIdx.x; t < kCocoT; t += kVocThreads) recall[(size_t)t * stride_t + out_km] = -1.0;
        return;
    }
    const double dnpig = (double)npig;
    const double eps = 2.220446049250313e-16;         // np.spacing(1)
    const long long lo = (long long)table[(size_t)k * n_images], hi = (long long)table[(size_t)(k + 1) * n_images];
    unsigned long long carry[kCocoT];
    for (int t = 0; t < kCocoT; ++t) carry[t] = 0ull;
    for (long long c0 = lo; c0 < hi; c0 += kVocTile) {
        const long long i0 = c0 + (long long)threadIdx.x * kVocItems;
        uint32_t bits[kVocItems];
        unsigned long long mine[kCocoT];
        for (int t = 0; t < kCocoT; ++t) mine[t] = 0ull;
        for (int it = 0; it < kVocItems; ++it) {
            bits[it] = 0u;
            if (i0 + it < hi) {
                const int p = order[i0 + it];
                if (rank_of[p] < max_det) bits[it] = dt_flags[(size_t)a * n_det + p];
            }
            for (int t = 0; t < kCocoT; ++t)
                mine[t] += (((unsigned long long)(bits[it] >> t) & 1ull) << 32) | ((bits[it] >> (kCocoFpShift + t)) & 1u);
        }
        unsigned long long run[kCocoT];
        for (int t = 0; t < kCocoT; ++t) {
            unsigned long long total;
            run[t] = carry[t] + voc_block_scan(mine[t], s, total);
            carry[t] += total;
        }
        for (int it = 0; it < kVocItems; ++it) {
            if (!bits[it]) continue;                  // an ignored or cut record repeats the previous (rc, pr)
            for (int t = 0; t < kCocoT; ++t) {
                const uint32_t tpb = (bits[it] >> t) & 1u, fpb = (bits[it] >> (kCocoFpShift + t)) & 1u;
                if (!(tpb | fpb)) continue;
                run[t] += ((unsigned long long)tpb << 32) | fpb;
                const double tp = (double)(run[t] >> 32), fp = (double)(run[t] & 0xffffffffull);
                const double rc = __ddiv_rn(tp, dnpig);
                const double pr = __ddiv_rn(tp, __dadd_rn(__dadd_rn(fp, tp), eps));
                int lo_r = 0, hi_r = kCocoR;          // R = (# recall thresholds <= rc) - 1
                while (lo_r < hi_r) {
                    const int mid = (lo_r + hi_r) >> 1;
                    if (s_rec[mid] <= rc) lo_r = mid + 1;
                    else hi_r = mid;
                }
                if (lo_r > 0) atomicMax(&best[t][lo_r - 1], (unsigned long long)__double_as_longlong(pr));
            }
        }
    }
    __syncthreads();
    if (threadIdx.x < kCocoT) {
        const int t = threadIdx.x;
        double q = 0.0;
        for (int r = kCocoR - 1; r >= 0; --r) {
            q = fmax(q, __longlong_as_double((long long)best[t][r]));
            precision[((size_t)t * kCocoR + r) * stride_t + out_km] = q;
        }
        recall[(size_t)t * stride_t + out_km] = __ddiv_rn((double)(carry[t] >> 32), dnpig);
    }
}

// ---- host side, shared by the library and the host-emulation build -----------------------------------------------
struct CocoWorkspace {
    unsigned long long* table;
    int32_t* canon;
    int32_t* cls_of;
    uint8_t* rank_of;
    uint8_t* taken;
    uint32_t* keys[2];
    int32_t* vals[2];
    unsigned long long* cnt;
    unsigned long long* part;
    size_t bytes;
};

static CocoWorkspace coco_workspace_layout(void* base, int n_det, int n_gt, int n_cls, int n_images) {
    const size_t n_table = (size_t)n_cls * n_images + 1;
    const int ntiles = ceil_div(n_det, kVocTile);
    const size_t n_cnt = (size_t)256 * ntiles;
    const size_t n_scan = n_cnt > n_table ? n_cnt : n_table;
    const size_t n_part = (size_t)ceil_div((long long)n_scan, kVocTile) + 1;
    CocoWorkspace w;
    unsigned char* p = static_cast<unsigned char*>(base);
    size_t off = 0;
    auto take = [&](size_t bytes) { unsigned char* q = p ? p + off : nullptr; off += voc_align(bytes); return q; };
    w.table = reinterpret_cast<unsigned long long*>(take(n_table * 8));
    w.canon = reinterpret_cast<int32_t*>(take((size_t)n_det * 4));
    w.cls_of = reinterpret_cast<int32_t*>(take((size_t)n_det * 4));
    w.rank_of = take((size_t)n_det);
    w.taken = take((size_t)kCocoPairs * n_gt + 1);
    w.keys[0] = reinterpret_cast<uint32_t*>(take((size_t)n_det * 4));
    w.keys[1] = reinterpret_cast<uint32_t*>(take((size_t)n_det * 4));
    w.vals[0] = reinterpret_cast<int32_t*>(take((size_t)n_det * 4));
    w.vals[1] = reinterpret_cast<int32_t*>(take((size_t)n_det * 4));
    w.cnt = reinterpret_cast<unsigned long long*>(take(n_cnt * 8));
    w.part = reinterpret_cast<unsigned long long*>(take(n_part * 8));
    w.bytes = off;
    return w;
}

template <class Rows>
static int coco_gather_impl(const Rows& rows, const int32_t* keep, const int32_t* keep_count, int N, int cap, int n_cls,
                            const int32_t* image_index, const double* image_size, int max_det, double* score,
                            double* box, long long pool_cap, int32_t* groups, int group_cap, long long* counters,
                            cudaStream_t st) {
    (void)st;
    VOC_LAUNCH(1, kVocThreads, eval_gather_plan_kernel, keep_count, N, n_cls, image_index, max_det, pool_cap, groups,
               group_cap, counters);
    VOC_CHECK("coco_gather_plan");
    VOC_LAUNCH(N, kVocThreads, coco_gather_rows_kernel<Rows>, rows, keep, keep_count, cap, n_cls, max_det, image_size,
               groups, counters, score, box);
    VOC_CHECK("coco_gather_rows");
    return 0;
}

static int coco_evaluate_impl(const double* score, const double* box, int n_det, const int32_t* groups, int n_groups,
                              const int32_t* gt_ptr, const double* gt_box, const double* gt_area, const uint8_t* gt_crowd,
                              int n_gt, int n_cls, int n_images, const CocoParams& P, void* workspace,
                              uint32_t* dt_flags, int32_t* order, double* precision, double* recall, cudaStream_t st) {
    (void)st;
    CocoWorkspace w = coco_workspace_layout(workspace, n_det, n_gt, n_cls, n_images);
    const long long n_table = (long long)n_cls * n_images + 1;
    VOC_LAUNCH(ceil_div(n_table, kVocThreads), kVocThreads, coco_fill_kernel, w.table, n_table);
    VOC_CHECK("coco_fill");
    if (n_groups > 0) {
        VOC_LAUNCH(ceil_div(n_groups, kVocThreads), kVocThreads, coco_count_kernel, groups, n_groups, n_images, w.table);
        VOC_CHECK("coco_count");
    }
    int rc = voc_scan(w.table, n_table, w.part, 0, st);
    if (rc) return rc;
    if (n_det > 0) {
        VOC_LAUNCH(ceil_div(n_groups, kVocThreads / 32), kVocThreads, coco_match_kernel, box, groups, n_groups, w.table,
                   gt_ptr, gt_box, gt_area, gt_crowd, n_gt, n_images, n_det, P, w.taken, w.canon, w.rank_of, dt_flags);
        VOC_CHECK("coco_match");
        VOC_LAUNCH(ceil_div(n_groups, kVocThreads / 32), kVocThreads, coco_class_of_kernel, groups, n_groups, w.cls_of);
        VOC_CHECK("coco_class_of");
        // LSD: score low word, score high word, class; every pass stable, starting from the canonical order
        int cls_bits = 1;
        while ((1 << cls_bits) < n_cls) ++cls_bits;
        const int words[3] = {0, 1, 2}, word_passes[3] = {4, 4, (cls_bits + 7) / 8};
        const int ntiles = ceil_div(n_det, kVocTile);
        const int32_t* vin = w.canon;
        int flip = 0;
        for (int wi = 0; wi < 3; ++wi) {
            VOC_LAUNCH(ceil_div(n_det, kVocThreads), kVocThreads, coco_keys_kernel, score, w.cls_of, vin, n_det,
                       words[wi], w.keys[flip]);
            VOC_CHECK("coco_keys");
            const uint32_t* kin = w.keys[flip];
            for (int p = 0; p < word_passes[wi]; ++p) {
                const bool last = wi == 2 && p == word_passes[wi] - 1;
                uint32_t* kout = w.keys[1 - flip];
                int32_t* vout = last ? order : w.vals[flip];
                VOC_LAUNCH(ntiles, kVocThreads, voc_radix_hist_kernel, kin, n_det, 8 * p, ntiles, w.cnt);
                VOC_CHECK("voc_radix_hist");
                rc = voc_scan(w.cnt, (long long)256 * ntiles, w.part, 0, st);
                if (rc) return rc;
                VOC_LAUNCH(ntiles, kVocThreads, voc_radix_scatter_kernel, kin, vin, n_det, 8 * p, ntiles, w.cnt, kout,
                           vout);
                VOC_CHECK("voc_radix_scatter");
                kin = kout;
                vin = vout;
                flip = 1 - flip;
            }
        }
    }
    VOC_LAUNCH(dim3(n_cls, kCocoA, kCocoM), kVocThreads, coco_accumulate_kernel, order, w.rank_of, dt_flags, n_det,
               w.table, n_images, n_cls, gt_ptr, gt_area, gt_crowd, P, precision, recall);
    VOC_CHECK("coco_accumulate");
    return 0;
}

static CocoParams coco_params(const double* iou_thrs, const double* rec_thrs, const int32_t* max_dets,
                              const double* area_rng) {
    CocoParams P;
    for (int t = 0; t < kCocoT; ++t) P.iou[t] = iou_thrs[t];
    for (int r = 0; r < kCocoR; ++r) P.rec[r] = rec_thrs[r];
    for (int m = 0; m < kCocoM; ++m) P.max_det[m] = max_dets[m];
    for (int a = 0; a < kCocoA; ++a) {
        P.area[a][0] = area_rng[2 * a];
        P.area[a][1] = area_rng[2 * a + 1];
    }
    return P;
}

}  // namespace fsdet

#ifndef FSDET_HOST_EMULATION
using namespace fsdet;

extern "C" int fsdet_coco_gather(const float* cand, const int32_t* keep, const int32_t* keep_count, int N, int cap, int H,
                                 int W, int nC, int n_cls, const int32_t* image_index, const double* image_size,
                                 int max_det, double* score, double* box, long long pool_cap, int32_t* groups,
                                 int group_cap, long long* counters, void* stream) {
    FSDET_CHECK_ARG(cand && keep && keep_count && image_index && image_size && score && box && groups && counters,
                    "coco_gather: null pointer");
    FSDET_CHECK_ARG(nC == 1, "coco_gather: rows with %d (conf, id) pairs; only the meta detector's nC = 1 is supported", nC);
    FSDET_CHECK_ARG(n_cls > 0 && n_cls < kCocoMaxClasses && N >= 0 && N % n_cls == 0,
                    "coco_gather: %d rows are not images x %d classes (1..%d)", N, n_cls, kCocoMaxClasses - 1);
    FSDET_CHECK_ARG(max_det > 0 && max_det <= 255, "coco_gather: max_det %d outside 1..255", max_det);
    FSDET_CHECK_ARG(cap > 0 && H > 0 && W > 0 && pool_cap >= 0 && pool_cap <= 0x7fffffffll && group_cap >= 0,
                    "coco_gather: bad shape");
    if (N == 0) return 0;
    return coco_gather_impl(CandRows{cand, H, W}, keep, keep_count, N, cap, n_cls, image_index, image_size, max_det,
                            score, box, pool_cap, groups, group_cap, counters, (cudaStream_t)stream);
}

extern "C" int fsdet_coco_gather_merged(const void* merged, const int32_t* keep, const int32_t* keep_count, int N,
                                        int cap, int n_cls, const int32_t* image_index, const double* image_size,
                                        int max_det, double* score, double* box, long long pool_cap, int32_t* groups,
                                        int group_cap, long long* counters, void* stream) {
    FSDET_CHECK_ARG(merged && keep && keep_count && image_index && image_size && score && box && groups && counters,
                    "coco_gather_merged: null pointer");
    FSDET_CHECK_ARG(n_cls > 0 && n_cls < kCocoMaxClasses && N >= 0 && N % n_cls == 0,
                    "coco_gather_merged: %d rows are not images x %d classes (1..%d)", N, n_cls, kCocoMaxClasses - 1);
    FSDET_CHECK_ARG(max_det > 0 && max_det <= 255, "coco_gather_merged: max_det %d outside 1..255", max_det);
    FSDET_CHECK_ARG(cap > 0 && pool_cap >= 0 && pool_cap <= 0x7fffffffll && group_cap >= 0,
                    "coco_gather_merged: bad shape");
    if (N == 0) return 0;
    return coco_gather_impl(MergedRows{static_cast<const TtaRecord*>(merged)}, keep, keep_count, N, cap, n_cls,
                            image_index, image_size, max_det, score, box, pool_cap, groups, group_cap, counters,
                            (cudaStream_t)stream);
}

extern "C" int fsdet_coco_merge(int n_src, const long long* src_counters, const double* src_score, const double* src_box,
                                long long src_pool_stride, const int32_t* src_groups, long long src_group_stride,
                                int n_images, void* workspace, size_t workspace_bytes, double* score, double* box,
                                long long pool_cap, int32_t* groups, int group_cap, long long* counters, void* stream) {
    FSDET_CHECK_ARG(n_src > 0 && n_images > 0 && src_pool_stride >= 0 && src_group_stride >= 0 && pool_cap >= 0 &&
                        pool_cap <= 0x7fffffffll && group_cap >= 0, "coco_merge: bad shape");
    FSDET_CHECK_ARG(src_counters && workspace && counters && (src_group_stride == 0 || (src_groups && groups)) &&
                        (src_pool_stride == 0 || (src_score && src_box && score && box)), "coco_merge: null pointer");
    FSDET_CHECK_ARG(workspace_bytes >= merge_workspace_layout(nullptr, n_src, n_images).bytes,
                    "coco_merge: workspace of %zu bytes, %zu needed", workspace_bytes,
                    merge_workspace_layout(nullptr, n_src, n_images).bytes);
    return eval_merge_impl(n_src, src_counters, src_score, src_box, src_pool_stride, src_groups, src_group_stride,
                           n_images, workspace, score, box, pool_cap, groups, group_cap, counters, (cudaStream_t)stream);
}

extern "C" size_t fsdet_coco_workspace_bytes(int n_det, int n_gt, int n_cls, int n_images) {
    if (n_det < 0 || n_gt < 0 || n_cls <= 0 || n_images <= 0) return 0;
    return coco_workspace_layout(nullptr, n_det, n_gt, n_cls, n_images).bytes;
}

extern "C" int fsdet_coco_evaluate(const double* score, const double* box, int n_det, const int32_t* groups,
                                   int n_groups, const int32_t* gt_ptr, const double* gt_box, const double* gt_area,
                                   const uint8_t* gt_crowd, int n_gt, int n_cls, int n_images, const double* iou_thrs,
                                   const double* rec_thrs, const int32_t* max_dets, const double* area_rng,
                                   void* workspace, size_t workspace_bytes, uint32_t* dt_flags, int32_t* order,
                                   double* precision, double* recall, void* stream) {
    FSDET_CHECK_ARG(gt_ptr && iou_thrs && rec_thrs && max_dets && area_rng && workspace && precision && recall,
                    "coco_evaluate: null pointer");
    FSDET_CHECK_ARG(n_det == 0 || (score && box && groups && dt_flags && order), "coco_evaluate: null pointer");
    FSDET_CHECK_ARG(n_gt == 0 || (gt_box && gt_area && gt_crowd), "coco_evaluate: null ground-truth pointer");
    FSDET_CHECK_ARG(n_det >= 0 && n_groups >= 0 && n_gt >= 0 && n_images > 0 && n_cls > 0 && n_cls < kCocoMaxClasses,
                    "coco_evaluate: bad shape");
    FSDET_CHECK_ARG((long long)kCocoPairs * n_gt < (1ll << 40) && (long long)n_cls * n_images < 0x7fffffffll,
                    "coco_evaluate: too many ground truths or (class, image) rows");
    for (int m = 0; m < kCocoM; ++m)
        FSDET_CHECK_ARG(max_dets[m] > 0 && max_dets[m] <= 256, "coco_evaluate: maxDets[%d] = %d outside 1..256", m,
                        max_dets[m]);
    const size_t need = coco_workspace_layout(nullptr, n_det, n_gt, n_cls, n_images).bytes;
    FSDET_CHECK_ARG(workspace_bytes >= need, "coco_evaluate: workspace of %zu bytes, %zu needed", workspace_bytes, need);
    const CocoParams P = coco_params(iou_thrs, rec_thrs, max_dets, area_rng);
    return coco_evaluate_impl(score, box, n_det, groups, n_groups, gt_ptr, gt_box, gt_area, gt_crowd, n_gt, n_cls,
                              n_images, P, workspace, dt_flags, order, precision, recall, (cudaStream_t)stream);
}
#endif  // FSDET_HOST_EMULATION
