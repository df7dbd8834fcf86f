// PASCAL VOC detection AP on the device, from the detections that decode + NMS (detect.cu) leave there.
//
// Replaces, for evaluation (valid_ensemble.py:153-178 + scripts/voc_eval.py:96-243):
//   valid.detection_lines / write_detections   one '%f' text line per kept box
//   voc_eval.voc_eval                          parses the lines back
//   voc_eval.match_detections                  Python loop over every detection
//   voc_eval.voc_ap                            precision envelope / VOC07 11-point average
//
// Data model.  An accumulator owns a pool of detection records in result-file order (batch, image, survivor order):
//   rank_key uint32 = class << 20 | (2^20 - 1 - n), n = the '%f' integer of the confidence (prob = n / 1e6)
//   box      double[4] = the corners after the '%f' -> float() round trip
// and one group descriptor per (image, class) row: {first record, record count, image index, class}.  A group is a
// contiguous run of its class's result-file lines.
//
// Ranking.  Detections of a class are ranked by a STABLE sort on the confidence, descending: ties keep result-file
// order.  The host evaluator ranks with np.argsort(-conf), whose order at ties depends on numpy's sort implementation;
// the stable order is the one deliberate definition here.  Sorting by rank_key ascending, stably, gives exactly this
// order for every class at once (class-major).
//
// Arithmetic follows voc_eval.py in float64 with its operation order and no FMA contraction; see each kernel.
#include "detect_records.cuh"
#include "eval_sort.cuh"

namespace fsdet {

constexpr int kVocKeyBits = 20;                       // n <= 1e6 < 2^20 for a probability in [0, 1]
constexpr uint32_t kVocKeyMask = (1u << kVocKeyBits) - 1;
constexpr int kVocMaxClasses = 1 << (32 - kVocKeyBits);
constexpr int kVocFlagIgnored = 0, kVocFlagTP = 1, kVocFlagFP = 2;

struct VocThresholds {
    double t[11];                                     // the host's np.arange(0., 1.1, 0.1)
};

// '%f' % x followed by float(): x rounded to a multiple of 1e-6, half to even on the exact binary value, then read
// back as the correctly rounded n / 1e6.  x * 1e6 = p + e exactly (e from an fma); rint(p) is right unless p sits on
// a half (decided by the sign of e) or e itself is a half (p integral, p >= 2^52).  For |x| >= 2^33 the spacing of
// doubles exceeds 2e-6 and float() of the text returns x itself.  NaN and inf pass through.
__device__ __forceinline__ double voc_round6(double x, double* n_out) {
    if (!(fabs(x) < 8589934592.0)) {
        *n_out = x;
        return x;
    }
    const double p = __dmul_rn(x, 1e6);
    const double e = fma(x, 1e6, -p);
    double n = rint(p);
    const double d = __dsub_rn(p, n);                 // exact: |p - n| <= 0.5
    if (d == 0.5 && e > 0.0) n = __dadd_rn(n, 1.0);
    else if (d == -0.5 && e < 0.0) n = __dsub_rn(n, 1.0);
    else if (d == 0.0 && fabs(e) == 0.5 && fmod(n, 2.0) != 0.0) n = e > 0.0 ? __dadd_rn(n, 1.0) : __dsub_rn(n, 1.0);
    *n_out = n;
    return __ddiv_rn(n, 1e6);
}

__global__ void voc_round6_kernel(const double* __restrict__ x, double* __restrict__ y, double* __restrict__ n,
                                  long long count) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (long long)gridDim.x * blockDim.x) {
        double k;
        y[i] = voc_round6(x[i], &k);
        if (n) n[i] = k;
    }
}

// ---- gather: one batch of Detections (after NMS) -> records + group descriptors ---------------------------------
// eval_gather_plan_kernel (eval_sort.cuh) lays out the batch's groups and counters; the kernel below fills the records.

// One block per row: the kept boxes of row r in survivor order, as valid.detection_lines computes and prints them:
// box = [xs/W, ys/H, ws/W, hs/H, det, cls] (float64 of the float32 candidate), x1 = (box[0] - box[2]/2.0) * width, ...,
// prob = det * cls; every value through '%f' -> float().
// Rows: a reader of detect_records.cuh (the candidates of one pass, or the merged records of several).
template <class Rows>
__global__ void __launch_bounds__(kVocThreads) voc_gather_rows_kernel(const Rows rows, const int32_t* __restrict__ keep,
                                                                      int cap, int n_cls, const double* __restrict__ image_size,
                                                                      const int32_t* __restrict__ groups,
                                                                      const long long* __restrict__ counters,
                                                                      uint32_t* __restrict__ rank_key,
                                                                      double* __restrict__ box) {
    if (counters[3]) return;
    const int r = blockIdx.x;
    const int32_t* g = groups + (counters[2] + r) * 4;
    const long long start = g[0];
    const int count = g[1];
    const int cls = r % n_cls;
    const double width = image_size[(r / n_cls) * 2], height = image_size[(r / n_cls) * 2 + 1];
    for (int t = threadIdx.x; t < count; t += kVocThreads) {
        const size_t id = (size_t)r * cap + keep[(size_t)r * cap + t];
        const double4 b = rows.box(id);
        const double bx = b.x, by = b.y, bw = b.z, bh = b.w;
        const double hw = __ddiv_rn(bw, 2.0), hh = __ddiv_rn(bh, 2.0);
        double n;
        const double x1 = voc_round6(__dmul_rn(__dsub_rn(bx, hw), width), &n);
        const double y1 = voc_round6(__dmul_rn(__dsub_rn(by, hh), height), &n);
        const double x2 = voc_round6(__dmul_rn(__dadd_rn(bx, hw), width), &n);
        const double y2 = voc_round6(__dmul_rn(__dadd_rn(by, hh), height), &n);
        voc_round6(__dmul_rn((double)rows.det(id), (double)rows.cls(id)), &n);
        const uint32_t key = (uint32_t)fmin(fmax(n, 0.0), (double)kVocKeyMask);
        const long long d = start + t;
        rank_key[d] = ((uint32_t)cls << kVocKeyBits) | (kVocKeyMask - key);
        box[d * 4 + 0] = x1;
        box[d * 4 + 1] = y1;
        box[d * 4 + 2] = x2;
        box[d * 4 + 3] = y2;
    }
}

// ---- match: voc_eval.match_detections for one (image, class) group per warp ------------------------------------
__device__ __forceinline__ double np_minimum(double a, double b) { return a != a ? a : (b != b ? b : (b < a ? b : a)); }
__device__ __forceinline__ double np_maximum(double a, double b) { return a != a ? a : (b != b ? b : (b > a ? b : a)); }

// The group's detections are ranked (key descending, result-file position ascending: the class-wide stable order
// restricted to one image) by counting, then lane 0 walks them in rank order: pixel-inclusive IoU with every
// ground-truth box of the class in the image, the first maximum (np.argmax), a match needs IoU > ovthresh, a match to
// a difficult box is neither TP nor FP, a match to a claimed box or no match is an FP.
__global__ void __launch_bounds__(kVocThreads) voc_match_kernel(const uint32_t* __restrict__ rank_key,
                                                                const double* __restrict__ box,
                                                                const int32_t* __restrict__ groups, int n_groups,
                                                                const int32_t* __restrict__ gt_ptr,
                                                                const int32_t* __restrict__ gt_box,
                                                                const uint8_t* __restrict__ gt_difficult, int n_images,
                                                                double ovthresh, int32_t* __restrict__ gperm,
                                                                uint8_t* __restrict__ claimed,
                                                                uint8_t* __restrict__ flags) {
    const int gi = blockIdx.x * (kVocThreads / 32) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (gi >= n_groups) return;                       // whole warps leave together
    const int32_t* g = groups + (size_t)gi * 4;
    const int start = g[0], count = g[1], img = g[2], cls = g[3];
    for (int j = lane; j < count; j += 32) {
        const uint32_t kj = rank_key[start + j];
        int r = 0;
        for (int m = 0; m < count; ++m) {
            const uint32_t km = rank_key[start + m];
            r += (km < kj || (km == kj && m < j)) ? 1 : 0;
        }
        gperm[start + r] = j;
    }
    __syncwarp();
    if (lane != 0) return;
    const int gb = gt_ptr[(size_t)cls * n_images + img], ge = gt_ptr[(size_t)cls * n_images + img + 1];
    for (int k = gb; k < ge; ++k) claimed[k] = 0;
    for (int r = 0; r < count; ++r) {
        const int d = start + gperm[start + r];
        const double b0 = box[(size_t)d * 4], b1 = box[(size_t)d * 4 + 1], b2 = box[(size_t)d * 4 + 2], b3 = box[(size_t)d * 4 + 3];
        const double barea = __dmul_rn(__dadd_rn(__dsub_rn(b2, b0), 1.0), __dadd_rn(__dsub_rn(b3, b1), 1.0));
        double best = -INFINITY;
        int j = -1;
        for (int k = gb; k < ge; ++k) {
            const double g0 = gt_box[k * 4], g1 = gt_box[k * 4 + 1], g2 = gt_box[k * 4 + 2], g3 = gt_box[k * 4 + 3];
            const double iw = __dadd_rn(__dsub_rn(np_minimum(g2, b2), np_maximum(g0, b0)), 1.0);
            const double ih = __dadd_rn(__dsub_rn(np_minimum(g3, b3), np_maximum(g1, b1)), 1.0);
            const double inter = __dmul_rn(np_maximum(iw, 0.0), np_maximum(ih, 0.0));
            const double garea = __dmul_rn(__dadd_rn(__dsub_rn(g2, g0), 1.0), __dadd_rn(__dsub_rn(g3, g1), 1.0));
            const double iou = __ddiv_rn(inter, __dsub_rn(__dadd_rn(barea, garea), inter));
            if (j < 0 || (best == best && (iou != iou || iou > best))) {   // np.argmax: first maximum, a NaN wins
                best = iou;
                j = k;
            }
        }
        uint8_t f = kVocFlagFP;
        if (best > ovthresh) {
            if (gt_difficult[j]) f = kVocFlagIgnored;
            else if (!claimed[j]) { f = kVocFlagTP; claimed[j] = 1; }
        }
        flags[d] = f;
    }
}

// TP count in the high, FP count in the low 32 bits, in rank order: one inclusive scan gives both cumulative sums.
__global__ void voc_pack_flags_kernel(const int32_t* __restrict__ order, const uint8_t* __restrict__ flags, int n,
                                      unsigned long long* __restrict__ packed) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    const uint8_t f = flags[order[r]];
    packed[r] = f == kVocFlagTP ? (1ull << 32) : (f == kVocFlagFP ? 1ull : 0ull);
}

// ---- per-class curves and AP: one block per class ------------------------------------------------------------
__device__ __forceinline__ int voc_lower_bound(const uint32_t* k, int n, uint32_t v) {
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (k[mid] < v) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

__device__ __forceinline__ double voc_rec_at(const unsigned long long* cum, int r, unsigned long long base, double npos) {
    return __ddiv_rn((double)((cum[r] - base) >> 32), npos);
}

// rec = tp / float(npos), prec = tp / np.maximum(tp + fp, eps) over the class's ranks; VOC07: ap += max(prec[rec >= t])
// / 11. for the 11 host thresholds in order (0 where no rank qualifies); area: envelope p[i] = max(prec[i:], 0), summed
// (r[i+1] - r[i]) * p[i+1] wherever r changes, with r = [0, rec..., 1] (summation order differs from np.sum's).
__global__ void __launch_bounds__(kVocThreads) voc_ap_kernel(const uint32_t* __restrict__ skeys, int n,
                                                             const unsigned long long* __restrict__ cum,
                                                             const int32_t* __restrict__ gt_ptr,
                                                             const uint8_t* __restrict__ gt_difficult, int n_images,
                                                             VocThresholds th, double* __restrict__ rec_out,
                                                             double* __restrict__ prec_out, int32_t* __restrict__ cls_count,
                                                             int32_t* __restrict__ npos_out, double* __restrict__ ap07,
                                                             double* __restrict__ ap_area) {
    __shared__ double s_env[kVocThreads];
    __shared__ double s_red[kVocThreads / 32][12];
    __shared__ int s_cnt[kVocThreads / 32];
    __shared__ double s_carry;
    const int c = blockIdx.x, lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int lo = voc_lower_bound(skeys, n, (uint32_t)c << kVocKeyBits);
    const int hi = voc_lower_bound(skeys, n, (uint32_t)(c + 1) << kVocKeyBits);
    // npos = non-difficult ground truths of the class
    int np_ = 0;
    for (int k = gt_ptr[(size_t)c * n_images] + threadIdx.x; k < gt_ptr[(size_t)(c + 1) * n_images]; k += kVocThreads)
        np_ += gt_difficult[k] ? 0 : 1;
    for (int o = 16; o; o >>= 1) np_ += __shfl_xor_sync(0xffffffffu, np_, o);
    if (lane == 0) s_cnt[w] = np_;
    if (threadIdx.x == 0) s_carry = 0.0;
    __syncthreads();
    int npos_i = 0;
    for (int q = 0; q < kVocThreads / 32; ++q) npos_i += s_cnt[q];
    const double npos = (double)npos_i;
    const unsigned long long base = lo > 0 ? cum[lo - 1] : 0ull;
    const double eps = 2.220446049250313e-16;         // np.finfo(np.float64).eps
    double mx[11];
    for (int t = 0; t < 11; ++t) mx[t] = -1.0;        // no rank with rec >= t yet (prec >= 0)
    double area = 0.0;
    for (int end = hi; end > lo; end -= kVocThreads) {
        const int i = end - kVocThreads + (int)threadIdx.x;
        const bool valid = i >= lo;
        double rec = 0.0, prec = 0.0;
        if (valid) {
            const unsigned long long v = cum[i] - base;
            const double tp = (double)(v >> 32), fp = (double)(v & 0xffffffffull);
            const double s = __dadd_rn(tp, fp);
            rec = __ddiv_rn(tp, npos);
            prec = __ddiv_rn(tp, s > eps ? s : eps);
            rec_out[i] = rec;
            prec_out[i] = prec;
            for (int t = 0; t < 11; ++t)
                if (rec >= th.t[t] && prec > mx[t]) mx[t] = prec;
        }
        // suffix maximum of prec inside the chunk, then with everything after it
        s_env[threadIdx.x] = valid ? prec : 0.0;
        __syncthreads();
        for (int off = 1; off < kVocThreads; off <<= 1) {
            const double o = threadIdx.x + off < kVocThreads ? s_env[threadIdx.x + off] : 0.0;
            const double m = fmax(s_env[threadIdx.x], o);
            __syncthreads();
            s_env[threadIdx.x] = m;
            __syncthreads();
        }
        const double carry = s_carry;
        if (valid) {
            const double env = fmax(s_env[threadIdx.x], carry);
            const double prev = i == lo ? 0.0 : voc_rec_at(cum, i - 1, base, npos);
            if (rec != prev) area = __dadd_rn(area, __dmul_rn(__dsub_rn(rec, prev), env));
        }
        __syncthreads();
        if (threadIdx.x == 0) s_carry = fmax(carry, s_env[0]);
        __syncthreads();
    }
    if (threadIdx.x == 0) {                           // the last step, to the appended recall 1 (precision 0)
        const double last = hi > lo ? voc_rec_at(cum, hi - 1, base, npos) : 0.0;
        if (1.0 != last) area = __dadd_rn(area, __dmul_rn(__dsub_rn(1.0, last), 0.0));
    }
    for (int o = 16; o; o >>= 1) {
        area = __dadd_rn(area, __shfl_xor_sync(0xffffffffu, area, o));
        for (int t = 0; t < 11; ++t) mx[t] = fmax(mx[t], __shfl_xor_sync(0xffffffffu, mx[t], o));
    }
    if (lane == 0) {
        for (int t = 0; t < 11; ++t) s_red[w][t] = mx[t];
        s_red[w][11] = area;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        double ap = 0.0, a = 0.0;
        for (int t = 0; t < 11; ++t) {
            double m = -1.0;
            for (int q = 0; q < kVocThreads / 32; ++q) m = fmax(m, s_red[q][t]);
            ap = __dadd_rn(ap, __ddiv_rn(m < 0.0 ? 0.0 : m, 11.0));
        }
        for (int q = 0; q < kVocThreads / 32; ++q) a = __dadd_rn(a, s_red[q][11]);
        ap07[c] = ap;
        ap_area[c] = a;
        cls_count[c] = hi - lo;
        npos_out[c] = npos_i;
    }
}

struct VocWorkspace {
    int32_t* gperm;
    uint8_t* claimed;
    uint32_t* keys[2];
    int32_t* vals[2];
    uint32_t* skeys;
    unsigned long long* cnt;
    unsigned long long* part;
    unsigned long long* cum;
    size_t bytes;
};

static VocWorkspace voc_workspace_layout(void* base, int n_det, int n_gt) {
    const int ntiles = ceil_div(n_det, kVocTile);
    const size_t n_cnt = (size_t)256 * ntiles;
    const size_t n_part = (size_t)ceil_div((long long)(n_cnt > (size_t)n_det ? n_cnt : (size_t)n_det), kVocTile) + 1;
    VocWorkspace w;
    unsigned char* p = static_cast<unsigned char*>(base);
    size_t off = 0;
    auto take = [&](size_t bytes) { unsigned char* q = p ? p + off : nullptr; off += voc_align(bytes); return q; };
    w.gperm = reinterpret_cast<int32_t*>(take((size_t)n_det * 4));
    w.claimed = take((size_t)n_gt + 1);
    w.keys[0] = reinterpret_cast<uint32_t*>(take((size_t)n_det * 4));
    w.keys[1] = reinterpret_cast<uint32_t*>(take((size_t)n_det * 4));
    w.vals[0] = reinterpret_cast<int32_t*>(take((size_t)n_det * 4));
    w.vals[1] = reinterpret_cast<int32_t*>(take((size_t)n_det * 4));
    w.skeys = nullptr;
    w.cnt = reinterpret_cast<unsigned long long*>(take(n_cnt * 8));
    w.part = reinterpret_cast<unsigned long long*>(take(n_part * 8));
    w.cum = reinterpret_cast<unsigned long long*>(take((size_t)n_det * 8));
    w.bytes = off;
    return w;
}

template <class Rows>
static int voc_gather_impl(const Rows& rows, const int32_t* keep, const int32_t* keep_count, int N, int cap, int n_cls,
                           const int32_t* image_index, const double* image_size, uint32_t* rank_key, double* box,
                           long long pool_cap, int32_t* groups, int group_cap, long long* counters, cudaStream_t st) {
    (void)st;
    VOC_LAUNCH(1, kVocThreads, eval_gather_plan_kernel, keep_count, N, n_cls, image_index, cap, pool_cap, groups,
               group_cap, counters);                  // a row keeps at most cap boxes: the limit never binds
    VOC_CHECK("voc_gather_plan");
    VOC_LAUNCH(N, kVocThreads, voc_gather_rows_kernel<Rows>, rows, keep, cap, n_cls, image_size, groups, counters,
               rank_key, box);
    VOC_CHECK("voc_gather_rows");
    return 0;
}

static int voc_evaluate_impl(const uint32_t* rank_key, const double* box, int n_det, const int32_t* groups, int n_groups,
                             const int32_t* gt_ptr, const int32_t* gt_box, const uint8_t* gt_difficult, int n_gt,
                             int n_cls, int n_images, double ovthresh, const VocThresholds& th, void* workspace,
                             uint8_t* flags, int32_t* order, double* rec, double* prec, int32_t* cls_count,
                             int32_t* npos, double* ap07, double* ap_area, cudaStream_t st) {
    (void)st;
    VocWorkspace w = voc_workspace_layout(workspace, n_det, n_gt);
    const uint32_t* skeys = rank_key;
    if (n_det > 0) {
        if (n_groups > 0) {
            VOC_LAUNCH(ceil_div(n_groups, kVocThreads / 32), kVocThreads, voc_match_kernel, rank_key, box, groups,
                       n_groups, gt_ptr, gt_box, gt_difficult, n_images, ovthresh, w.gperm, w.claimed, flags);
            VOC_CHECK("voc_match");
        }
        int bits = kVocKeyBits;
        while ((1 << (bits - kVocKeyBits)) < n_cls) ++bits;
        const int passes = (bits + 7) / 8;
        const int ntiles = ceil_div(n_det, kVocTile);
        const uint32_t* kin = rank_key;
        const int32_t* vin = nullptr;
        for (int p = 0; p < passes; ++p) {
            const bool last = p == passes - 1;
            uint32_t* kout = w.keys[p & 1];
            int32_t* vout = last ? order : w.vals[p & 1];
            VOC_LAUNCH(ntiles, kVocThreads, voc_radix_hist_kernel, kin, n_det, 8 * p, ntiles, w.cnt);
            VOC_CHECK("voc_radix_hist");
            const int rc = voc_scan(w.cnt, (long long)256 * ntiles, w.part, 0, st);
            if (rc) return rc;
            VOC_LAUNCH(ntiles, kVocThreads, voc_radix_scatter_kernel, kin, vin, n_det, 8 * p, ntiles, w.cnt, kout, vout);
            VOC_CHECK("voc_radix_scatter");
            kin = kout;
            vin = vout;
        }
        skeys = kin;
        VOC_LAUNCH(ceil_div(n_det, kVocThreads), kVocThreads, voc_pack_flags_kernel, order, flags, n_det, w.cum);
        VOC_CHECK("voc_pack_flags");
        const int rc = voc_scan(w.cum, n_det, w.part, 1, st);
        if (rc) return rc;
    }
    VOC_LAUNCH(n_cls, kVocThreads, voc_ap_kernel, skeys, n_det, w.cum, gt_ptr, gt_difficult, n_images, th, rec, prec,
               cls_count, npos, ap07, ap_area);
    VOC_CHECK("voc_ap");
    return 0;
}

}  // namespace fsdet

#ifndef FSDET_HOST_EMULATION
using namespace fsdet;

extern "C" int fsdet_voc_round6(const double* x, double* y, double* n, long long count, void* stream) {
    FSDET_CHECK_ARG(count >= 0 && (count == 0 || (x && y)), "voc_round6: null pointer");
    if (count == 0) return 0;
    const int blocks = (int)(count < (1ll << 20) ? ceil_div(count, kVocThreads) : 4096);
    voc_round6_kernel<<<blocks, kVocThreads, 0, (cudaStream_t)stream>>>(x, y, n, count);
    return launch_status("voc_round6");
}

extern "C" int fsdet_voc_gather(const float* cand, const int32_t* keep, const int32_t* keep_count, int N, int cap, int H,
                                int W, int nC, int n_cls, const int32_t* image_index, const double* image_size,
                                uint32_t* rank_key, double* box, long long pool_cap, int32_t* groups, int group_cap,
                                long long* counters, void* stream) {
    FSDET_CHECK_ARG(cand && keep && keep_count && image_index && image_size && rank_key && box && groups && counters,
                    "voc_gather: null pointer");
    FSDET_CHECK_ARG(nC == 1, "voc_gather: rows with %d (conf, id) pairs; only the meta detector's nC = 1 is supported", nC);
    FSDET_CHECK_ARG(n_cls > 0 && n_cls <= kVocMaxClasses && N >= 0 && N % n_cls == 0,
                    "voc_gather: %d rows are not images x %d classes (1..%d)", N, n_cls, kVocMaxClasses);
    FSDET_CHECK_ARG(cap > 0 && H > 0 && W > 0 && pool_cap >= 0 && pool_cap <= 0x7fffffffll && group_cap >= 0,
                    "voc_gather: bad shape");
    if (N == 0) return 0;
    return voc_gather_impl(CandRows{cand, H, W}, keep, keep_count, N, cap, n_cls, image_index, image_size, rank_key, box,
                           pool_cap, groups, group_cap, counters, (cudaStream_t)stream);
}

extern "C" int fsdet_voc_gather_merged(const void* merged, const int32_t* keep, const int32_t* keep_count, int N, int cap,
                                       int n_cls, const int32_t* image_index, const double* image_size,
                                       uint32_t* rank_key, double* box, long long pool_cap, int32_t* groups,
                                       int group_cap, long long* counters, void* stream) {
    FSDET_CHECK_ARG(merged && keep && keep_count && image_index && image_size && rank_key && box && groups && counters,
                    "voc_gather_merged: null pointer");
    FSDET_CHECK_ARG(n_cls > 0 && n_cls <= kVocMaxClasses && N >= 0 && N % n_cls == 0,
                    "voc_gather_merged: %d rows are not images x %d classes (1..%d)", N, n_cls, kVocMaxClasses);
    FSDET_CHECK_ARG(cap > 0 && pool_cap >= 0 && pool_cap <= 0x7fffffffll && group_cap >= 0,
                    "voc_gather_merged: bad shape");
    if (N == 0) return 0;
    return voc_gather_impl(MergedRows{static_cast<const TtaRecord*>(merged)}, keep, keep_count, N, cap, n_cls,
                           image_index, image_size, rank_key, box, pool_cap, groups, group_cap, counters,
                           (cudaStream_t)stream);
}

extern "C" size_t fsdet_eval_merge_workspace_bytes(int n_src, int n_images) {
    if (n_src <= 0 || n_images < 0) return 0;
    return merge_workspace_layout(nullptr, n_src, n_images).bytes;
}

extern "C" int fsdet_voc_merge(int n_src, const long long* src_counters, const uint32_t* src_key, const double* src_box,
                               long long src_pool_stride, const int32_t* src_groups, long long src_group_stride,
                               int n_images, void* workspace, size_t workspace_bytes, uint32_t* rank_key, double* box,
                               long long pool_cap, int32_t* groups, int group_cap, long long* counters, void* stream) {
    FSDET_CHECK_ARG(n_src > 0 && n_images > 0 && src_pool_stride >= 0 && src_group_stride >= 0 && pool_cap >= 0 &&
                        pool_cap <= 0x7fffffffll && group_cap >= 0, "voc_merge: bad shape");
    FSDET_CHECK_ARG(src_counters && workspace && counters && (src_group_stride == 0 || (src_groups && groups)) &&
                        (src_pool_stride == 0 || (src_key && src_box && rank_key && box)), "voc_merge: null pointer");
    FSDET_CHECK_ARG(workspace_bytes >= merge_workspace_layout(nullptr, n_src, n_images).bytes,
                    "voc_merge: workspace of %zu bytes, %zu needed", workspace_bytes,
                    merge_workspace_layout(nullptr, n_src, n_images).bytes);
    return eval_merge_impl(n_src, src_counters, src_key, src_box, src_pool_stride, src_groups, src_group_stride, n_images,
                           workspace, rank_key, box, pool_cap, groups, group_cap, counters, (cudaStream_t)stream);
}

extern "C" size_t fsdet_voc_workspace_bytes(int n_det, int n_gt) {
    if (n_det < 0 || n_gt < 0) return 0;
    return voc_workspace_layout(nullptr, n_det, n_gt).bytes;
}

extern "C" int fsdet_voc_evaluate(const uint32_t* rank_key, const double* box, int n_det, const int32_t* groups,
                                  int n_groups, const int32_t* gt_ptr, const int32_t* gt_box, const uint8_t* gt_difficult,
                                  int n_gt, int n_cls, int n_images, double ovthresh, const double* thresholds,
                                  void* workspace, size_t workspace_bytes, uint8_t* flags, int32_t* order, double* rec,
                                  double* prec, int32_t* cls_count, int32_t* npos, double* ap07, double* ap_area,
                                  void* stream) {
    FSDET_CHECK_ARG(gt_ptr && thresholds && cls_count && npos && ap07 && ap_area, "voc_evaluate: null pointer");
    FSDET_CHECK_ARG(n_det == 0 || (rank_key && box && groups && flags && order && rec && prec && workspace),
                    "voc_evaluate: null pointer");
    FSDET_CHECK_ARG(n_gt == 0 || (gt_box && gt_difficult), "voc_evaluate: null ground-truth pointer");
    FSDET_CHECK_ARG(n_det >= 0 && n_groups >= 0 && n_gt >= 0 && n_images > 0 && n_cls > 0 && n_cls <= kVocMaxClasses,
                    "voc_evaluate: bad shape");
    FSDET_CHECK_ARG(workspace_bytes >= voc_workspace_layout(nullptr, n_det, n_gt).bytes,
                    "voc_evaluate: workspace of %zu bytes, %zu needed", workspace_bytes,
                    voc_workspace_layout(nullptr, n_det, n_gt).bytes);
    VocThresholds th;
    for (int t = 0; t < 11; ++t) th.t[t] = thresholds[t];
    return voc_evaluate_impl(rank_key, box, n_det, groups, n_groups, gt_ptr, gt_box, gt_difficult, n_gt, n_cls, n_images,
                             ovthresh, th, workspace, flags, order, rec, prec, cls_count, npos, ap07, ap_area,
                             (cudaStream_t)stream);
}
#endif  // FSDET_HOST_EMULATION
