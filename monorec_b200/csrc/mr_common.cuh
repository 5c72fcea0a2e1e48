// Shared host-side plumbing for libmonorec_b200.so: thread-local error text, launch counting, CUDA checks.
#pragma once
#include <cuda_runtime.h>
#include <cstdarg>
#include <cstdio>
#include "../../include/monorec_b200.h"

namespace mr {

void set_error(const char* fmt, ...);
void count_launch(int n = 1);

// cost_volume.cu: launches the fused kernel for batch elements [b_begin, b_begin + b_count) of a B-element problem;
// depths is the plane table [D], or with per_pixel_depths != 0 one depth per plane and pixel [B,D,H,W]; out_cv / out_sfcv
// are fp32 (out_dtype MR_DT_F32) or IEEE half (MR_DT_F16); keyframe and frames have `channels` (3 or 1) planes
int launch_cost_volume(const float* keyframe, const float* const* frames, const float* proj, const float* depths,
                       void* out_cv, void* out_sfcv, int B, int F, int D, int H, int W, float alpha,
                       const float* chan_w, int b_begin, int b_count, int gather_only, cudaStream_t stream,
                       void* sf_nhwc = nullptr, int sf_nhwc_dtype = 0, int per_pixel_depths = 0,
                       int matching = MR_CV_SSIM, int centered = 1, int out_dtype = MR_DT_F32, int channels = 3);

// python slicing semantics of a roi {r0, r1, c0, c1} = [r0:r1, c0:c1] (preprocess_roi, utils/util.py:36-43, and the masking
// of PLYSaver.add_depthmap, utils/ply_utils.py:39-43): a negative bound counts from the end, a bound past the edge is clipped;
// the region may come out empty (r1 <= r0 or c1 <= c0).  roi == nullptr: the whole image
inline void clip_roi(const int* roi, int H, int W, int& r0, int& r1, int& c0, int& c1) {
    r0 = 0; r1 = H; c0 = 0; c1 = W;
    if (roi == nullptr) return;
    auto clip = [](int v, int n) { if (v < 0) v += n; return v < 0 ? 0 : (v > n ? n : v); };
    r0 = clip(roi[0], H); r1 = clip(roi[1], H); c0 = clip(roi[2], W); c1 = clip(roi[3], W);
}

inline int check_cuda(cudaError_t e, const char* what) {
    if (e == cudaSuccess) return MR_OK;
    set_error("%s: %s", what, cudaGetErrorString(e));
    return (int)e;
}

#define MR_REQUIRE(cond, ...)                  \
    do {                                       \
        if (!(cond)) {                         \
            ::mr::set_error(__VA_ARGS__);      \
            return MR_EINVAL;                  \
        }                                      \
    } while (0)

#define MR_CUDA(call)                                            \
    do {                                                         \
        int _rc = ::mr::check_cuda((call), #call);               \
        if (_rc != MR_OK) return _rc;                            \
    } while (0)

// post-launch check (does not synchronise)
#define MR_LAUNCH_CHECK(name)                                    \
    do {                                                         \
        ::mr::count_launch();                                    \
        int _rc = ::mr::check_cuda(cudaGetLastError(), name);    \
        if (_rc != MR_OK) return _rc;                            \
    } while (0)

}  // namespace mr
