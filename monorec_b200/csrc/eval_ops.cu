// Evaluation-side helpers of SURVEY.md section 8f row 2 (include/monorec_b200.h: mr_sparse_metrics, mr_images_u8_to_f32).
//
//  * the seven sparse depth metrics of model/metric_functions/sparse_metrics.py:81-251 (a1, a2, a3, rmse, rmse_log, abs_rel,
//    sq_rel; helpers utils/util.py:36-65, :101-118) in ONE pass over `result` / `target` instead of 7 x ~12 elementwise torch
//    kernels per batch (evaluater/evaluater.py:78-112 calls the seven functions one after the other);
//  * the loader's image normalisation (data_loader/kitti_odometry_dataset.py:126-132: uint8 HWC -> float CHW / 255 - .5) on the
//    device, so that uint8 images (a quarter of the bytes) cross PCIe.
#include "mr_common.cuh"
#include <cstdint>

namespace {

constexpr int kSums = 8;   // per image: valid count, a1, a2, a3 hits, sum se, sum sle, sum abs_rel, sum sq_rel

struct MetricArgs {
    const float* pred;     // [B,1,H,W] predicted inverse depth (data_dict["result"])
    const float* gt;       // [B,1,H,W] sparse ground-truth inverse depth (0 = no measurement)
    const float* mvobj;    // [B,1,H,W] moving-object mask or nullptr (use_cvmask)
    int B, H, W;
    int r0, r1, c0, c1;    // region of interest [r0, r1) x [c0, c1)
    float inv_max;         // 1 / max_distance, or 0: no clamp
    int pred_all_valid;
    double* sums;          // [B][kSums], zeroed before the launch
};

__global__ void sparse_metric_sums_kernel(const MetricArgs a) {
    const int b = blockIdx.y;
    const int rw = a.c1 - a.c0, n = (a.r1 - a.r0) * rw;
    float acc[kSums];
#pragma unroll
    for (int k = 0; k < kSums; ++k) acc[k] = 0.f;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int r = a.r0 + i / rw, c = a.c0 + i % rw;
        const size_t o = ((size_t)b * a.H + r) * a.W + c;
        float p = __ldg(a.pred + o), g = __ldg(a.gt + o);
        // get_mask (utils/util.py:101-107): True = excluded
        bool masked = (g == 0.f);
        if (a.inv_max > 0.f) masked = masked || (g < a.inv_max);
        if (!a.pred_all_valid) masked = masked || (p == 0.f);
        if (a.mvobj != nullptr) masked = masked || !(__ldg(a.mvobj + o) > 0.5f);
        if (masked) continue;
        // get_positive_depth, get_absolute_depth (utils/util.py:46-65): relu, clamp_min(1 / max_distance), 1 / x
        p = fmaxf(p, 0.f); g = fmaxf(g, 0.f);
        if (a.inv_max > 0.f) { p = fmaxf(p, a.inv_max); g = fmaxf(g, a.inv_max); }
        const float dp = __fdiv_rn(1.0f, p), dg = __fdiv_rn(1.0f, g);
        const float th = fmaxf(__fdiv_rn(dg, dp), __fdiv_rn(dp, dg));
        const float diff = dp - dg, ld = logf(dp) - logf(dg);
        acc[0] += 1.f;
        acc[1] += (th < 1.25f) ? 1.f : 0.f;
        acc[2] += (th < 1.5625f) ? 1.f : 0.f;        // 1.25 ** 2
        acc[3] += (th < 1.953125f) ? 1.f : 0.f;      // 1.25 ** 3
        acc[4] += diff * diff;
        acc[5] += ld * ld;
        acc[6] += __fdiv_rn(fabsf(diff), dg);
        acc[7] += __fdiv_rn(diff * diff, dg);
    }
    __shared__ double red[kSums][32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < kSums; ++k) {
        double v = (double)acc[k];
        for (int s = 16; s > 0; s >>= 1) v += __shfl_xor_sync(0xffffffffu, v, s);
        if (lane == 0) red[k][warp] = v;
    }
    __syncthreads();
    if (warp == 0) {
        const int nw = blockDim.x >> 5;
#pragma unroll
        for (int k = 0; k < kSums; ++k) {
            double v = lane < nw ? red[k][lane] : 0.0;
            for (int s = 16; s > 0; s >>= 1) v += __shfl_xor_sync(0xffffffffu, v, s);
            if (lane == 0) atomicAdd(a.sums + (size_t)b * kSums + k, v);
        }
    }
}

// out[7] = a1, a2, a3, rmse, rmse_log, abs_rel, sq_rel exactly as the reference combines them: the a* / *_rel metrics are
// means over every unmasked pixel of the batch (mask_mean with dim=None), rmse / rmse_log are batch means of per-image roots
__global__ void sparse_metric_finalize_kernel(const double* sums, int B, float* out) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    double tot[kSums] = {0, 0, 0, 0, 0, 0, 0, 0};
    double rm = 0.0, rl = 0.0;
    for (int b = 0; b < B; ++b) {
        const double* s = sums + (size_t)b * kSums;
        for (int k = 0; k < kSums; ++k) tot[k] += s[k];
        rm += sqrt(s[4] / s[0]);        // 0 / 0 = NaN for an image without ground truth, like the reference
        rl += sqrt(s[5] / s[0]);
    }
    out[0] = (float)(tot[1] / tot[0]);
    out[1] = (float)(tot[2] / tot[0]);
    out[2] = (float)(tot[3] / tot[0]);
    out[3] = (float)(rm / B);
    out[4] = (float)(rl / B);
    out[5] = (float)(tot[6] / tot[0]);
    out[6] = (float)(tot[7] / tot[0]);
}

__global__ void images_u8_to_f32_kernel(const unsigned char* src, float* dst, int B, int Hs, int Ws, int r0, int c0, int H, int W) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;     // output pixel of image blockIdx.y
    if (i >= H * W) return;
    const int b = blockIdx.y, r = i / W, c = i - r * W;
    const unsigned char* s = src + (((size_t)b * Hs + (r0 + r)) * Ws + (c0 + c)) * 3;
    float* d = dst + (size_t)b * 3 * H * W + i;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) d[(size_t)ch * H * W] = __fsub_rn(__fdiv_rn((float)s[ch], 255.0f), 0.5f);
}

}  // namespace

extern "C" long long mr_sparse_metrics_workspace(int B) { return B < 1 ? 0 : (long long)B * kSums * (long long)sizeof(double); }

extern "C" int mr_sparse_metrics(const float* result, const float* target, const float* mvobj_mask, int B, int H, int W,
                                 const int* roi, float max_distance, int pred_all_valid, float* out_metrics, void* workspace,
                                 long long workspace_bytes, void* stream) {
    MR_REQUIRE(result && target && out_metrics && workspace, "mr_sparse_metrics: null pointer");
    MR_REQUIRE(B >= 1 && B <= 65535 && H >= 1 && W >= 1, "mr_sparse_metrics: bad shape B=%d H=%d W=%d", B, H, W);
    if (workspace_bytes < mr_sparse_metrics_workspace(B)) {
        mr::set_error("mr_sparse_metrics: workspace too small (%lld < %lld bytes)", workspace_bytes, mr_sparse_metrics_workspace(B));
        return MR_ENOMEM;
    }
    MR_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 7) == 0, "mr_sparse_metrics: workspace must be 8-byte aligned");
    MetricArgs a{};
    a.pred = result; a.gt = target; a.mvobj = mvobj_mask; a.B = B; a.H = H; a.W = W;
    a.r0 = 0; a.r1 = H; a.c0 = 0; a.c1 = W;
    if (roi != nullptr) {      // python slicing semantics of preprocess_roi (utils/util.py:36-43): [r0:r1, c0:c1], clipped
        auto clip = [](int v, int n) { if (v < 0) v += n; return v < 0 ? 0 : (v > n ? n : v); };
        a.r0 = clip(roi[0], H); a.r1 = clip(roi[1], H); a.c0 = clip(roi[2], W); a.c1 = clip(roi[3], W);
        MR_REQUIRE(a.r1 > a.r0 && a.c1 > a.c0, "mr_sparse_metrics: empty region of interest");
    }
    a.inv_max = max_distance > 0.f ? 1.0f / max_distance : 0.f;
    a.pred_all_valid = pred_all_valid;
    a.sums = static_cast<double*>(workspace);
    cudaStream_t st = (cudaStream_t)stream;
    MR_CUDA(cudaMemsetAsync(workspace, 0, (size_t)mr_sparse_metrics_workspace(B), st));
    const int n = (a.r1 - a.r0) * (a.c1 - a.c0);
    int blocks = (n + 256 * 8 - 1) / (256 * 8);
    int dev = 0, sms = 0;
    MR_CUDA(cudaGetDevice(&dev));
    MR_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));   // at most one block per SM and image
    if (blocks > sms) blocks = sms;
    if (blocks < 1) blocks = 1;
    sparse_metric_sums_kernel<<<dim3(blocks, B), 256, 0, st>>>(a);
    MR_LAUNCH_CHECK("sparse_metric_sums_kernel");
    sparse_metric_finalize_kernel<<<1, 32, 0, st>>>(a.sums, B, out_metrics);
    MR_LAUNCH_CHECK("sparse_metric_finalize_kernel");
    return MR_OK;
}

extern "C" int mr_images_u8_to_f32(const unsigned char* src, float* dst, int B, int Hs, int Ws, int crop_top, int crop_left,
                                   int H, int W, void* stream) {
    MR_REQUIRE(src && dst, "mr_images_u8_to_f32: null pointer");
    MR_REQUIRE(B >= 1 && B <= 65535 && H >= 1 && W >= 1 && crop_top >= 0 && crop_left >= 0 && crop_top + H <= Hs && crop_left + W <= Ws,
               "mr_images_u8_to_f32: crop [%d:%d, %d:%d] outside the %dx%d source", crop_top, crop_top + H, crop_left, crop_left + W, Hs, Ws);
    images_u8_to_f32_kernel<<<dim3((H * W + 255) / 256, B), 256, 0, (cudaStream_t)stream>>>(src, dst, B, Hs, Ws, crop_top, crop_left, H, W);
    MR_LAUNCH_CHECK("images_u8_to_f32_kernel");
    return MR_OK;
}
