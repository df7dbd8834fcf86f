// Host-emulated build of csrc/voc_eval.cu (see cuda_host_emul.h): the library's orchestration of the kernels with an
// `emul_` prefix, host pointers instead of device pointers.  Test tooling only; built by the host-emulation tests.
#include "../../fewshot_detection_b200/csrc/voc_eval.cu"

namespace emul {
Block g_block;
unsigned char* g_dyn_smem = nullptr;
}  // namespace emul
namespace fsdet {
void set_error(const char*, ...) {}
}  // namespace fsdet

using namespace fsdet;

extern "C" int emul_voc_round6(const double* x, double* y, double* n, long long count) {
    emul::launch_serial(dim3(1), dim3(1), [&]() {
        for (long long i = 0; i < count; ++i) {
            double k;
            y[i] = voc_round6(x[i], &k);
            if (n) n[i] = k;
        }
    });
    return 0;
}

extern "C" int emul_voc_gather(const float* cand, const int32_t* keep, const int32_t* keep_count, int N, int cap, int H,
                               int W, int n_cls, const int32_t* image_index, const double* image_size, uint32_t* rank_key,
                               double* box, long long pool_cap, int32_t* groups, int group_cap, long long* counters) {
    return voc_gather_impl(CandRows{cand, H, W}, keep, keep_count, N, cap, n_cls, image_index, image_size, rank_key, box,
                           pool_cap, groups, group_cap, counters, nullptr);
}

extern "C" int emul_voc_gather_merged(const void* merged, const int32_t* keep, const int32_t* keep_count, int N, int cap,
                                      int n_cls, const int32_t* image_index, const double* image_size, uint32_t* rank_key,
                                      double* box, long long pool_cap, int32_t* groups, int group_cap,
                                      long long* counters) {
    return voc_gather_impl(MergedRows{static_cast<const TtaRecord*>(merged)}, keep, keep_count, N, cap, n_cls,
                           image_index, image_size, rank_key, box, pool_cap, groups, group_cap, counters, nullptr);
}

extern "C" size_t emul_eval_merge_workspace_bytes(int n_src, int n_images) {
    return merge_workspace_layout(nullptr, n_src, n_images).bytes;
}

extern "C" int emul_voc_merge(int n_src, const long long* src_counters, const uint32_t* src_key, const double* src_box,
                              long long src_pool_stride, const int32_t* src_groups, long long src_group_stride,
                              int n_images, void* workspace, uint32_t* rank_key, double* box, long long pool_cap,
                              int32_t* groups, int group_cap, long long* counters) {
    return eval_merge_impl(n_src, src_counters, src_key, src_box, src_pool_stride, src_groups, src_group_stride, n_images,
                           workspace, rank_key, box, pool_cap, groups, group_cap, counters, nullptr);
}

extern "C" size_t emul_voc_workspace_bytes(int n_det, int n_gt) { return voc_workspace_layout(nullptr, n_det, n_gt).bytes; }

extern "C" int emul_voc_evaluate(const uint32_t* rank_key, const double* box, int n_det, const int32_t* groups,
                                 int n_groups, const int32_t* gt_ptr, const int32_t* gt_box, const uint8_t* gt_difficult,
                                 int n_gt, int n_cls, int n_images, double ovthresh, const double* thresholds,
                                 void* workspace, uint8_t* flags, int32_t* order, double* rec, double* prec,
                                 int32_t* cls_count, int32_t* npos, double* ap07, double* ap_area) {
    VocThresholds th;
    for (int t = 0; t < 11; ++t) th.t[t] = thresholds[t];
    return voc_evaluate_impl(rank_key, box, n_det, groups, n_groups, gt_ptr, gt_box, gt_difficult, n_gt, n_cls, n_images,
                             ovthresh, th, workspace, flags, order, rec, prec, cls_count, npos, ap07, ap_area, nullptr);
}
