// Host-emulated build of csrc/detect.cu (see cuda_host_emul.h): same entry-point names with an `emul_` prefix, host
// pointers instead of device pointers.  Test tooling only; built by tests/test_detect_host_emul.py with g++.
#include "../../fewshot_detection_b200/csrc/detect.cu"

namespace emul {
Block g_block;
unsigned char* g_dyn_smem = nullptr;
}  // namespace emul
namespace fsdet {
void set_error(const char*, ...) {}
}  // namespace fsdet

using namespace fsdet;

extern "C" int emul_region_detect(const float* output, const float* anchors_f32, int N, int A, int nC, int H, int W,
                                  int n_models, int v2, int only_objectness, double conf_thresh, float* cand,
                                  int32_t* count, float* cls_dense) {
    DetArgs p;
    p.out = output; p.anchors = anchors_f32; p.cand = cand; p.count = count; p.cls_dense = cls_dense;
    p.N = N; p.A = A; p.nC = nC; p.H = H; p.W = W; p.cs = n_models; p.v2 = v2; p.only_obj = only_objectness;
    p.cap = A * H * W; p.thresh = conf_thresh;
    emul::launch(dim3(N), dim3(kDetThreads), 0, [&]() { region_detect_kernel(p); });
    return 0;
}

extern "C" int emul_nms(const float* cand, const double* boxes64, const int32_t* count, int N, int cap, int H, int W,
                        double nms_thresh, int32_t* keep, int32_t* keep_count) {
    const int P = next_pow2(cap);
    const size_t smem = (size_t)P * (sizeof(double4) + sizeof(unsigned long long) + 1);
    emul::launch(dim3(N), dim3(kDetThreads), smem,
                 [&]() { nms_kernel(cand, boxes64, count, cap, P, H, W, nms_thresh, keep, keep_count); });
    return 0;
}

extern "C" size_t emul_detect_select_workspace_bytes(int N, int cap) {
    return select_workspace_layout(nullptr, N, cap).bytes;
}

extern "C" int emul_detect_select(const float* cand, const int32_t* keep, const int32_t* keep_count, int N, int cap, int H,
                                  int W, int n_cls, const int32_t* sizes, int max_det, void* workspace, double* score,
                                  double* box, int32_t* cls, int32_t* count, int32_t* total) {
    return detect_select_impl(CandRows{cand, H, W}, keep, keep_count, N, cap, n_cls, sizes, max_det, workspace, score,
                              box, cls, count, total, nullptr);
}

extern "C" int emul_rw_running_mean(float* enews, const int32_t* cnt_in, int32_t* cnt_out, const float* dw,
                                    const int32_t* ids, int n, int n_cls, int C) {
    emul::launch(dim3(ceil_div(C, 128), n_cls), dim3(128), 0,
                 [&]() { rw_running_mean_kernel(enews, cnt_in, cnt_out, dw, ids, n, n_cls, C); });
    return 0;
}

extern "C" int emul_detect_select_merged(const void* merged, const int32_t* keep, const int32_t* keep_count, int N,
                                         int cap, int n_cls, const int32_t* sizes, int max_det, void* workspace,
                                         double* score, double* box, int32_t* cls, int32_t* count, int32_t* total) {
    return detect_select_impl(MergedRows{static_cast<const TtaRecord*>(merged)}, keep, keep_count, N, cap, n_cls, sizes,
                              max_det, workspace, score, box, cls, count, total, nullptr);
}

extern "C" int emul_tta_merge(const float* cand, const int32_t* count, int N, int cap, int H, int W, int flip, int pass,
                              void* merged, int32_t* merged_count, int merged_cap, int32_t* overflow) {
    emul::launch(dim3(N), dim3(kDetThreads), 0, [&]() {
        tta_merge_kernel(cand, count, cap, H, W, flip, pass, static_cast<TtaRecord*>(merged), merged_count, merged_cap,
                         overflow);
    });
    return 0;
}

extern "C" size_t emul_nms_merged_workspace_bytes(int N, int cap) { return select_workspace_layout(nullptr, N, cap).bytes; }

extern "C" int emul_nms_merged(const void* merged, const int32_t* count, int N, int cap, double nms_thresh,
                               void* workspace, int32_t* keep, int32_t* keep_count) {
    return nms_merged_impl(static_cast<const TtaRecord*>(merged), count, N, cap, nms_thresh, workspace, keep, keep_count,
                           nullptr);
}
