// The two forms a row of detection candidates takes on the device, and one reader per form, so that the consumers of
// the NMS survivors (detect.cu's per-image selection, voc_eval.cu's and coco_eval.cu's gathers) run the same
// arithmetic on either:
//
//   cand   float32 [N][cap][8] of fsdet_region_detect: xs, ys, ws, hs in units of one H x W head grid, det_conf,
//          cls_max_conf, (int) class id, (int) a*H*W + cell;
//   merged TtaRecord [N][cap] of fsdet_tta_merge: the candidates of several passes (sides, mirrored or not) of the same
//          images, each box already normalised to the image in float64.
//
// A reader returns the normalised float64 box (x, y, w, h) = the first four entries of the reference's box list
// (utils.py:175 / :270: xs / W, ys / H, ws / W, hs / H on Python floats) and the float32 det_conf and cls_conf of a
// candidate given its flat index row * cap + slot.
#pragma once
#include "common.cuh"

namespace fsdet {

constexpr int kTtaSlotBits = 20;                      // TtaRecord::src = pass << kTtaSlotBits | slot
constexpr int kTtaMaxPasses = 1 << (31 - kTtaSlotBits);

struct TtaRecord {                                    // 48 bytes
    double x, y, w, h;                                // normalised; x already mirrored (1.0 - x) for a flipped pass
    float det, cls;                                   // det_conf, cls_max_conf
    int32_t cid;                                      // cls_max_id
    int32_t src;                                      // pass index << kTtaSlotBits | the pass's candidate slot
};
static_assert(sizeof(TtaRecord) == 48, "TtaRecord is 48 bytes (include/fsdet.h)");

struct CandRows {
    const float* cand;
    int H, W;
    __device__ __forceinline__ double4 box(size_t i) const {
        const float* v = cand + i * 8;
        return make_double4(__ddiv_rn((double)v[0], (double)W), __ddiv_rn((double)v[1], (double)H),
                            __ddiv_rn((double)v[2], (double)W), __ddiv_rn((double)v[3], (double)H));
    }
    __device__ __forceinline__ float det(size_t i) const { return cand[i * 8 + 4]; }
    __device__ __forceinline__ float cls(size_t i) const { return cand[i * 8 + 5]; }
};

struct MergedRows {
    const TtaRecord* rec;
    __device__ __forceinline__ double4 box(size_t i) const {
        const TtaRecord& q = rec[i];
        return make_double4(q.x, q.y, q.w, q.h);
    }
    __device__ __forceinline__ float det(size_t i) const { return rec[i].det; }
    __device__ __forceinline__ float cls(size_t i) const { return rec[i].cls; }
};

}  // namespace fsdet
