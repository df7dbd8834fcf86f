// Host-emulated build of csrc/coco_eval.cu (see cuda_host_emul.h): the library's orchestration of the kernels with an
// `emul_` prefix, host pointers instead of device pointers.  Test tooling only; built by the host-emulation tests.
#include "../../fewshot_detection_b200/csrc/coco_eval.cu"

namespace emul {
Block g_block;
unsigned char* g_dyn_smem = nullptr;
}  // namespace emul
namespace fsdet {
void set_error(const char*, ...) {}
}  // namespace fsdet

using namespace fsdet;

extern "C" int emul_coco_gather(const float* cand, const int32_t* keep, const int32_t* keep_count, int N, int cap, int H,
                                int W, int n_cls, const int32_t* image_index, const double* image_size, int max_det,
                                double* score, double* box, long long pool_cap, int32_t* groups, int group_cap,
                                long long* counters) {
    return coco_gather_impl(CandRows{cand, H, W}, keep, keep_count, N, cap, n_cls, image_index, image_size, max_det,
                            score, box, pool_cap, groups, group_cap, counters, nullptr);
}

extern "C" int emul_coco_gather_merged(const void* merged, const int32_t* keep, const int32_t* keep_count, int N, int cap,
                                       int n_cls, const int32_t* image_index, const double* image_size, int max_det,
                                       double* score, double* box, long long pool_cap, int32_t* groups, int group_cap,
                                       long long* counters) {
    return coco_gather_impl(MergedRows{static_cast<const TtaRecord*>(merged)}, keep, keep_count, N, cap, n_cls,
                            image_index, image_size, max_det, score, box, pool_cap, groups, group_cap, counters, nullptr);
}

extern "C" size_t emul_eval_merge_workspace_bytes(int n_src, int n_images) {
    return merge_workspace_layout(nullptr, n_src, n_images).bytes;
}

extern "C" int emul_coco_merge(int n_src, const long long* src_counters, const double* src_score, const double* src_box,
                               long long src_pool_stride, const int32_t* src_groups, long long src_group_stride,
                               int n_images, void* workspace, double* score, double* box, long long pool_cap,
                               int32_t* groups, int group_cap, long long* counters) {
    return eval_merge_impl(n_src, src_counters, src_score, src_box, src_pool_stride, src_groups, src_group_stride,
                           n_images, workspace, score, box, pool_cap, groups, group_cap, counters, nullptr);
}

extern "C" size_t emul_coco_workspace_bytes(int n_det, int n_gt, int n_cls, int n_images) {
    return coco_workspace_layout(nullptr, n_det, n_gt, n_cls, n_images).bytes;
}

extern "C" int emul_coco_evaluate(const double* score, const double* box, int n_det, const int32_t* groups, int n_groups,
                                  const int32_t* gt_ptr, const double* gt_box, const double* gt_area,
                                  const uint8_t* gt_crowd, int n_gt, int n_cls, int n_images, const double* iou_thrs,
                                  const double* rec_thrs, const int32_t* max_dets, const double* area_rng,
                                  void* workspace, uint32_t* dt_flags, int32_t* order, double* precision,
                                  double* recall) {
    const CocoParams P = coco_params(iou_thrs, rec_thrs, max_dets, area_rng);
    return coco_evaluate_impl(score, box, n_det, groups, n_groups, gt_ptr, gt_box, gt_area, gt_crowd, n_gt, n_cls,
                              n_images, P, workspace, dt_flags, order, precision, recall, nullptr);
}
