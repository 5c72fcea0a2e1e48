// Evaluation-side helpers of SURVEY.md section 8f row 2 (include/monorec_b200.h: mr_sparse_metrics, mr_dense_metrics,
// mr_eval_accumulate, mr_median_scaling, mr_images_u8_to_f32).
//
//  * the seven sparse depth metrics of model/metric_functions/sparse_metrics.py:81-251 (a1, a2, a3, rmse, rmse_log, abs_rel,
//    sq_rel; helpers utils/util.py:36-65, :101-118) in ONE pass over `result` / `target` instead of 7 x ~12 elementwise torch
//    kernels per batch (evaluater/evaluater.py:78-112 calls the seven functions one after the other);
//  * the twelve dense and completeness metrics (sparse_metrics.py:6-78, dense_metrics.py, completeness_metrics.py) in one pass;
//  * both passes over several evaluater batches at once (consecutive groups of images, one row of metrics per group), and the
//    evaluater's float64 totals and running average (evaluater.py:45-49, 94-103) updated on the device;
//  * the evaluater's median scaling (utils/util.py:135-142) with an exact radix select and no host synchronisation;
//  * the loader's image normalisation (data_loader/kitti_odometry_dataset.py:126-132: uint8 HWC -> float CHW / 255 - .5) on the
//    device, so that uint8 images (a quarter of the bytes) cross PCIe.
#include "mr_common.cuh"
#include <cstdint>

namespace {

constexpr int kSums = 8;   // per image: valid count, a1, a2, a3 hits, sum se, sum sle, sum abs_rel, sum sq_rel

// torch's clamp_min (and relu) keep a NaN (fmaxf would drop it)
__device__ __forceinline__ float clamp_min_nan(float x, float lo) { return isnan(x) ? x : fmaxf(x, lo); }
// torch.max(a, b) of two tensors propagates a NaN of either side
__device__ __forceinline__ float max_nan(float a, float b) { return (isnan(a) || isnan(b)) ? __int_as_float(0x7fc00000) : fmaxf(a, b); }
// torch's relu as it treats the zeros: NaN and -0.0 pass through (1 / -0.0 is -inf in the reference, a hit in a1-a3)
__device__ __forceinline__ float relu_torch(float x) { return x < 0.f ? 0.f : x; }

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
        // get_positive_depth, get_absolute_depth (utils/util.py:46-65): relu, clamp_min(1 / max_distance), 1 / x.  A NaN
        // prediction or target at an unmasked pixel stays NaN, as in the reference: rmse, rmse_log, abs_rel and sq_rel of its
        // rows are NaN (and the evaluater drops the batch), a1-a3 count it as a miss
        p = relu_torch(p); g = relu_torch(g);
        if (a.inv_max > 0.f) { p = clamp_min_nan(p, a.inv_max); g = clamp_min_nan(g, a.inv_max); }
        const float dp = __fdiv_rn(1.0f, p), dg = __fdiv_rn(1.0f, g);
        const float th = max_nan(__fdiv_rn(dg, dp), __fdiv_rn(dp, dg));
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

// out[g][7] = a1, a2, a3, rmse, rmse_log, abs_rel, sq_rel of images [g * group, min(B, (g + 1) * group)) exactly as the
// reference combines a batch: the a* / *_rel metrics are means over every unmasked pixel of the batch (mask_mean with
// dim=None), rmse / rmse_log are batch means of per-image roots.  One thread per group; group = B is the ungrouped pass
__global__ void sparse_metric_finalize_kernel(const double* sums, int B, int group, int G, float* out) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= G) return;
    const int b0 = g * group, b1 = min(B, b0 + group), nb = b1 - b0;
    double tot[kSums] = {0, 0, 0, 0, 0, 0, 0, 0};
    double rm = 0.0, rl = 0.0;
    for (int b = b0; b < b1; ++b) {
        const double* s = sums + (size_t)b * kSums;
        for (int k = 0; k < kSums; ++k) tot[k] += s[k];
        rm += sqrt(s[4] / s[0]);        // 0 / 0 = NaN for an image without ground truth, like the reference
        rl += sqrt(s[5] / s[0]);
    }
    float* o = out + (size_t)g * 7;
    o[0] = (float)(tot[1] / tot[0]);
    o[1] = (float)(tot[2] / tot[0]);
    o[2] = (float)(tot[3] / tot[0]);
    o[3] = (float)(rm / nb);
    o[4] = (float)(rl / nb);
    o[5] = (float)(tot[6] / tot[0]);
    o[6] = (float)(tot[7] / tot[0]);
}

// ---- dense metrics (model/metric_functions/sparse_metrics.py:6-78, dense_metrics.py, completeness_metrics.py) -------------
constexpr int kDenseSums = 13;  // per image: a1, a2, a3 hits, sum se, sle, abs_rel, sq_rel, E, E^2 (sc_inv), |p - g| (l1_inv),
                                // and over the whole image: result != 0, result != 0 where target == 0, target == 0

struct DenseArgs {
    const float* pred;     // [B,1,H,W] data_dict["result"]
    const float* gt;       // [B,1,H,W] data_dict["target"]
    int B, H, W;
    int r0, r1, c0, c1;    // region of interest [r0, r1) x [c0, c1)
    float min_inv;         // clamp_min bound of get_absolute_depth (1 / max_distance), or <= 0: no clamp
    double* sums;          // [B][kDenseSums], zeroed before the launch
};

__global__ void dense_metric_sums_kernel(const DenseArgs a) {
    const int b = blockIdx.y, n = a.H * a.W;
    double acc[kDenseSums];
#pragma unroll
    for (int k = 0; k < kDenseSums; ++k) acc[k] = 0.0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int r = i / a.W, c = i - r * a.W;
        const size_t o = (size_t)b * n + i;
        const float p0 = __ldg(a.pred + o), g0 = __ldg(a.gt + o);
        // completeness_metric and covered_gt_metric ignore roi and max_distance
        acc[10] += (p0 != 0.f) ? 1.0 : 0.0;
        acc[11] += (p0 != 0.f && g0 == 0.f) ? 1.0 : 0.0;
        acc[12] += (g0 == 0.f) ? 1.0 : 0.0;
        if (r < a.r0 || r >= a.r1 || c < a.c0 || c >= a.c1) continue;
        // get_positive_depth (utils/util.py:59-65); l1_inv_metric stops here
        float p = clamp_min_nan(p0, 0.f), g = clamp_min_nan(g0, 0.f);
        acc[9] += (double)fabsf(__fsub_rn(p, g));
        // get_absolute_depth (:46-56): clamp_min(1 / max_distance) only when max_distance is given, then 1 / x.  No validity
        // mask: a zero becomes inf and the IEEE outcome (inf, NaN, a miss in a1-a3) is what the reference reports
        if (a.min_inv > 0.f) { p = clamp_min_nan(p, a.min_inv); g = clamp_min_nan(g, a.min_inv); }
        const float dp = __fdiv_rn(1.0f, p), dg = __fdiv_rn(1.0f, g);
        const float th = max_nan(__fdiv_rn(dg, dp), __fdiv_rn(dp, dg));
        const float diff = __fsub_rn(dp, dg), se = __fmul_rn(diff, diff);
        const float ld = __fsub_rn(logf(dp), logf(dg)), sle = __fmul_rn(ld, ld);
        const float e = isnan(ld) ? 0.f : ld;                 // sc_inv_metric: E[isnan(E)] = 0 (an inf stays)
        acc[0] += (th < 1.25f) ? 1.0 : 0.0;
        acc[1] += (th < 1.5625f) ? 1.0 : 0.0;                 // 1.25 ** 2
        acc[2] += (th < 1.953125f) ? 1.0 : 0.0;               // 1.25 ** 3
        acc[3] += (double)se;
        acc[4] += (double)sle;
        acc[5] += (double)__fdiv_rn(fabsf(diff), dg);         // abs_rel_metric and l1_rel_metric
        acc[6] += (double)__fdiv_rn(se, dg);
        acc[7] += (double)e;
        acc[8] += (double)__fmul_rn(e, e);
    }
    __shared__ double red[kDenseSums][32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < kDenseSums; ++k) {
        double v = acc[k];
        for (int s = 16; s > 0; s >>= 1) v += __shfl_xor_sync(0xffffffffu, v, s);
        if (lane == 0) red[k][warp] = v;
    }
    __syncthreads();
    if (warp == 0) {
        const int nw = blockDim.x >> 5;
#pragma unroll
        for (int k = 0; k < kDenseSums; ++k) {
            double v = lane < nw ? red[k][lane] : 0.0;
            for (int s = 16; s > 0; s >>= 1) v += __shfl_xor_sync(0xffffffffu, v, s);
            if (lane == 0) atomicAdd(a.sums + (size_t)b * kDenseSums + k, v);
        }
    }
}

// out[g][12] = a1, a2, a3, rmse, rmse_log, abs_rel, sq_rel, sc_inv, l1_rel, l1_inv, completeness, covered_gt of images
// [g * group, min(B, (g + 1) * group)), one thread per group; group = B is the ungrouped pass
__global__ void dense_metric_finalize_kernel(const double* sums, int B, int group, int G, int H, int W, long long n_roi,
                                             float* out) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= G) return;
    const int b0 = g * group, b1 = min(B, b0 + group), nb = b1 - b0;
    double tot[kDenseSums];
    for (int k = 0; k < kDenseSums; ++k) tot[k] = 0.0;
    double rm = 0.0, rl = 0.0, si = 0.0;
    const double n = (double)n_roi, N = n * nb;
    for (int b = b0; b < b1; ++b) {
        const double* s = sums + (size_t)b * kDenseSums;
        for (int k = 0; k < kDenseSums; ++k) tot[k] += s[k];
        rm += sqrt(s[3] / n);                             // rmse / rmse_log: batch mean of per-image roots
        rl += sqrt(s[4] / n);
        const double v = sqrt(s[8] / n - s[7] * s[7] / (n * n));
        si += isnan(v) ? 0.0 : v;                         // batch_metric[isnan(batch_metric)] = 0
    }
    float* o = out + (size_t)g * 12;
    o[0] = (float)(tot[0] / N);
    o[1] = (float)(tot[1] / N);
    o[2] = (float)(tot[2] / N);
    o[3] = (float)(rm / nb);
    o[4] = (float)(rl / nb);
    o[5] = (float)(tot[5] / N);
    o[6] = (float)(tot[6] / N);
    o[7] = (float)(si / nb);
    o[8] = o[5];                                          // l1_rel_metric is abs_rel_metric's formula
    o[9] = (float)(tot[9] / N);
    o[10] = (float)(tot[10] / ((double)nb * H * W));
    o[11] = (float)(tot[11] / tot[12]);                   // mask_mean over the pixels where target == 0
}

// ---- the evaluater's bookkeeping (evaluater/evaluater.py:45-49, 94-103) ---------------------------------------------------
// state: total[M], valid[M], running_avg[M], num_samples.  Thread j owns column j and applies the groups in order, in the
// float64 operations numpy does (no contraction into an FMA): a row with a NaN adds zeros and valid 0, the first group
// ever is added to the running average, a later one of b images gives avg * (n / (n + b)) + m * (b / (n + b)).
constexpr int kAccGroups = 32;   // groups per launch; longer lists are applied by consecutive launches on the stream

struct AccArgs {
    const float* values;   // [G][M]
    double* state;         // [3M + 1]
    int G, M, g0;          // groups g0 .. g0 + G - 1 of values
    int sizes[kAccGroups];
};

__global__ void eval_accumulate_kernel(const AccArgs a) {
    const int j = threadIdx.x, M = a.M;
    double* total = a.state;
    double* valid = a.state + M;
    double* avg = a.state + 2 * M;
    double n = a.state[3 * M];
    double t = 0.0, v = 0.0, r = 0.0;
    if (j < M) { t = total[j]; v = valid[j]; r = avg[j]; }
    for (int g = 0; g < a.G; ++g) {
        const float* row = a.values + (size_t)(a.g0 + g) * M;
        bool nan_row = false;
        for (int k = 0; k < M; ++k) nan_row = nan_row || isnan(row[k]);
        const double b = (double)a.sizes[g];
        if (j < M) {
            const double m = nan_row ? 0.0 : (double)row[j];
            t = __dadd_rn(t, m);
            v = __dadd_rn(v, nan_row ? 0.0 : 1.0);
            if (n == 0.0) r = __dadd_rn(r, m);
            else r = __dadd_rn(__dmul_rn(r, __ddiv_rn(n, n + b)), __dmul_rn(m, __ddiv_rn(b, n + b)));
        }
        n += b;
    }
    __syncthreads();                                      // every thread has read num_samples
    if (j < M) { total[j] = t; valid[j] = v; avg[j] = r; }
    if (j == 0) a.state[3 * M] = n;
}

// ---- median scaling (utils/util.py:135-142) ------------------------------------------------------------------------------
// Per image, the values of target and result where target > 0 are packed into the workspace (in no particular order: a median
// does not depend on it), then an exact radix select on order-preserving keys finds the lower median of each set.

struct MedianWs {
    unsigned* count;       // [B] selected pixels per image
    float* med;            // [B][2] median of target, of result
    float* tsel;           // [B][H*W] packed target values
    float* psel;           // [B][H*W] packed result values
};

__global__ void median_pack_kernel(const float* pred, const float* gt, int HW, MedianWs w) {
    const int b = blockIdx.y, lane = threadIdx.x & 31;
    for (int base = blockIdx.x * blockDim.x + (threadIdx.x & ~31); base < HW; base += gridDim.x * blockDim.x) {
        const int i = base + lane;
        const size_t o = (size_t)b * HW + i;
        const float g = i < HW ? __ldg(gt + o) : 0.f;
        const bool sel = g > 0.f;                         // mask = target > 0 (a NaN target is not selected)
        const unsigned bal = __ballot_sync(0xffffffffu, sel);
        if (bal == 0) continue;
        unsigned pos = 0;
        if (lane == 0) pos = atomicAdd(w.count + b, (unsigned)__popc(bal));
        pos = __shfl_sync(0xffffffffu, pos, 0) + __popc(bal & ((1u << lane) - 1u));
        if (sel) {
            w.tsel[(size_t)b * HW + pos] = g;
            w.psel[(size_t)b * HW + pos] = __ldg(pred + o);
        }
    }
}

__device__ __forceinline__ unsigned float_key(float f) {       // unsigned order of the keys = numeric order of the floats
    const unsigned u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_float(unsigned k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// blockIdx = (image, 0: target / 1: result).  torch.median returns the lower median, element (n - 1) / 2 of the sorted values,
// and NaN for an empty set or a set holding a NaN
__global__ void median_select_kernel(MedianWs w, int HW) {
    const int b = blockIdx.x, which = blockIdx.y;
    const float* v = (which ? w.psel : w.tsel) + (size_t)b * HW;
    const unsigned n = w.count[b];
    __shared__ unsigned hist[256];
    __shared__ unsigned s_prefix, s_rank;
    if (n == 0) {
        if (threadIdx.x == 0) w.med[2 * b + which] = __int_as_float(0x7fc00000);
        return;
    }
    unsigned prefix = 0, rank = (n - 1) / 2;
    for (int shift = 24; shift >= 0; shift -= 8) {
        for (int j = threadIdx.x; j < 256; j += blockDim.x) hist[j] = 0;
        __syncthreads();
        const unsigned hi = shift == 24 ? 0u : (0xffffffffu << (shift + 8));   // the digits already fixed
        int nan_seen = 0;
        for (unsigned i = threadIdx.x; i < n; i += blockDim.x) {
            const float x = v[i];
            if (isnan(x)) { nan_seen = 1; continue; }
            const unsigned k = float_key(x);
            if ((k & hi) == prefix) atomicAdd(&hist[(k >> shift) & 255u], 1u);
        }
        if (__syncthreads_or(nan_seen)) {
            if (threadIdx.x == 0) w.med[2 * b + which] = __int_as_float(0x7fc00000);
            return;
        }
        if (threadIdx.x == 0) {
            unsigned below = 0, d = 0;
            for (; d < 255u && below + hist[d] <= rank; ++d) below += hist[d];
            s_prefix = prefix | (d << shift);
            s_rank = rank - below;
        }
        __syncthreads();
        prefix = s_prefix;
        rank = s_rank;
        __syncthreads();
    }
    if (threadIdx.x == 0) w.med[2 * b + which] = key_float(prefix);
}

// result * ratios.view(-1, 1, 1, 1) with ratio = median(target) / median(result), both in fp32 as in the reference
__global__ void median_scale_kernel(const float* pred, float* out, int HW, const float* med) {
    const int b = blockIdx.y;
    const float ratio = __fdiv_rn(med[2 * b], med[2 * b + 1]);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += gridDim.x * blockDim.x) {
        const size_t o = (size_t)b * HW + i;
        out[o] = __fmul_rn(__ldg(pred + o), ratio);
    }
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

// blocks per image of a grid-stride pass over n pixels: ~8 pixels per thread, at most one block per SM and image
int blocks_per_image(int n, int threads, int* blocks) {
    int dev = 0, sms = 0;
    MR_CUDA(cudaGetDevice(&dev));
    MR_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    int nb = (n + threads * 8 - 1) / (threads * 8);
    if (nb > sms) nb = sms;
    *blocks = nb < 1 ? 1 : nb;
    return MR_OK;
}

// bytes of the median-scaling workspace before the packed values: count [B], med [B][2]
long long median_header_bytes(int B) { return (12LL * B + 255) / 256 * 256; }

}  // namespace

extern "C" long long mr_sparse_metrics_workspace(int B) { return B < 1 ? 0 : (long long)B * kSums * (long long)sizeof(double); }

extern "C" long long mr_dense_metrics_workspace(int B) { return B < 1 ? 0 : (long long)B * kDenseSums * (long long)sizeof(double); }

extern "C" int mr_dense_metrics(const float* result, const float* target, int B, int group, int H, int W, const int* roi,
                                float min_inv_depth, float* out_metrics, void* workspace, long long workspace_bytes, void* stream) {
    MR_REQUIRE(result && target && out_metrics && workspace, "mr_dense_metrics: null pointer (result, target, out_metrics, workspace)");
    MR_REQUIRE(B >= 1 && B <= 65535 && H >= 1 && W >= 1 && (long long)H * W <= 0x7fffffffLL,
               "mr_dense_metrics: bad shape B=%d H=%d W=%d", B, H, W);
    MR_REQUIRE(group >= 1, "mr_dense_metrics: group=%d must be >= 1", group);
    if (workspace_bytes < mr_dense_metrics_workspace(B)) {
        mr::set_error("mr_dense_metrics: workspace too small (%lld < %lld bytes)", workspace_bytes, mr_dense_metrics_workspace(B));
        return MR_ENOMEM;
    }
    MR_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 7) == 0, "mr_dense_metrics: workspace must be 8-byte aligned");
    DenseArgs a{};
    a.pred = result; a.gt = target; a.B = B; a.H = H; a.W = W;
    mr::clip_roi(roi, H, W, a.r0, a.r1, a.c0, a.c1);
    MR_REQUIRE(a.r1 > a.r0 && a.c1 > a.c0, "mr_dense_metrics: empty region of interest (roi)");
    a.min_inv = min_inv_depth;
    a.sums = static_cast<double*>(workspace);
    cudaStream_t st = (cudaStream_t)stream;
    MR_CUDA(cudaMemsetAsync(workspace, 0, (size_t)mr_dense_metrics_workspace(B), st));
    int blocks = 1;
    int rc = blocks_per_image(H * W, 256, &blocks);
    if (rc != MR_OK) return rc;
    dense_metric_sums_kernel<<<dim3(blocks, B), 256, 0, st>>>(a);
    MR_LAUNCH_CHECK("dense_metric_sums_kernel");
    const int G = (B + group - 1) / group;
    dense_metric_finalize_kernel<<<(G + 31) / 32, 32, 0, st>>>(a.sums, B, group, G, H, W,
                                                               (long long)(a.r1 - a.r0) * (a.c1 - a.c0), out_metrics);
    MR_LAUNCH_CHECK("dense_metric_finalize_kernel");
    return MR_OK;
}

extern "C" long long mr_median_scaling_workspace(int B, int H, int W) {
    if (B < 1 || H < 1 || W < 1) return 0;
    return median_header_bytes(B) + 2LL * B * H * W * (long long)sizeof(float);
}

extern "C" int mr_median_scaling(const float* result, const float* target, float* out, int B, int H, int W, void* workspace,
                                 long long workspace_bytes, void* stream) {
    MR_REQUIRE(result && target && out && workspace, "mr_median_scaling: null pointer (result, target, out, workspace)");
    MR_REQUIRE(B >= 1 && B <= 65535 && H >= 1 && W >= 1 && (long long)H * W <= 0x7fffffffLL,
               "mr_median_scaling: bad shape B=%d H=%d W=%d", B, H, W);
    MR_REQUIRE(out != result, "mr_median_scaling: out must not alias result (the input is left unmodified)");
    if (workspace_bytes < mr_median_scaling_workspace(B, H, W)) {
        mr::set_error("mr_median_scaling: workspace too small (%lld < %lld bytes)", workspace_bytes, mr_median_scaling_workspace(B, H, W));
        return MR_ENOMEM;
    }
    MR_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 3) == 0, "mr_median_scaling: workspace must be 4-byte aligned");
    const int HW = H * W;
    char* base = static_cast<char*>(workspace);
    MedianWs w;
    w.count = reinterpret_cast<unsigned*>(base);
    w.med = reinterpret_cast<float*>(base + 4LL * B);
    w.tsel = reinterpret_cast<float*>(base + median_header_bytes(B));
    w.psel = w.tsel + (size_t)B * HW;
    cudaStream_t st = (cudaStream_t)stream;
    MR_CUDA(cudaMemsetAsync(w.count, 0, sizeof(unsigned) * (size_t)B, st));
    int blocks = 1;
    int rc = blocks_per_image(HW, 256, &blocks);
    if (rc != MR_OK) return rc;
    median_pack_kernel<<<dim3(blocks, B), 256, 0, st>>>(result, target, HW, w);
    MR_LAUNCH_CHECK("median_pack_kernel");
    median_select_kernel<<<dim3(B, 2), 512, 0, st>>>(w, HW);
    MR_LAUNCH_CHECK("median_select_kernel");
    median_scale_kernel<<<dim3(blocks, B), 256, 0, st>>>(result, out, HW, w.med);
    MR_LAUNCH_CHECK("median_scale_kernel");
    return MR_OK;
}

extern "C" int mr_sparse_metrics(const float* result, const float* target, const float* mvobj_mask, int B, int group, int H, int W,
                                 const int* roi, float max_distance, int pred_all_valid, float* out_metrics, void* workspace,
                                 long long workspace_bytes, void* stream) {
    MR_REQUIRE(result && target && out_metrics && workspace, "mr_sparse_metrics: null pointer");
    MR_REQUIRE(B >= 1 && B <= 65535 && H >= 1 && W >= 1, "mr_sparse_metrics: bad shape B=%d H=%d W=%d", B, H, W);
    MR_REQUIRE(group >= 1, "mr_sparse_metrics: group=%d must be >= 1", group);
    if (workspace_bytes < mr_sparse_metrics_workspace(B)) {
        mr::set_error("mr_sparse_metrics: workspace too small (%lld < %lld bytes)", workspace_bytes, mr_sparse_metrics_workspace(B));
        return MR_ENOMEM;
    }
    MR_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 7) == 0, "mr_sparse_metrics: workspace must be 8-byte aligned");
    MetricArgs a{};
    a.pred = result; a.gt = target; a.mvobj = mvobj_mask; a.B = B; a.H = H; a.W = W;
    mr::clip_roi(roi, H, W, a.r0, a.r1, a.c0, a.c1);
    MR_REQUIRE(a.r1 > a.r0 && a.c1 > a.c0, "mr_sparse_metrics: empty region of interest");
    a.inv_max = max_distance > 0.f ? 1.0f / max_distance : 0.f;
    a.pred_all_valid = pred_all_valid;
    a.sums = static_cast<double*>(workspace);
    cudaStream_t st = (cudaStream_t)stream;
    MR_CUDA(cudaMemsetAsync(workspace, 0, (size_t)mr_sparse_metrics_workspace(B), st));
    int blocks = 1;
    int rc = blocks_per_image((a.r1 - a.r0) * (a.c1 - a.c0), 256, &blocks);
    if (rc != MR_OK) return rc;
    sparse_metric_sums_kernel<<<dim3(blocks, B), 256, 0, st>>>(a);
    MR_LAUNCH_CHECK("sparse_metric_sums_kernel");
    const int G = (B + group - 1) / group;
    sparse_metric_finalize_kernel<<<(G + 31) / 32, 32, 0, st>>>(a.sums, B, group, G, out_metrics);
    MR_LAUNCH_CHECK("sparse_metric_finalize_kernel");
    return MR_OK;
}

extern "C" int mr_eval_accumulate(const float* values, int G, int M, const int* group_sizes, double* state, void* stream) {
    MR_REQUIRE(values && group_sizes && state, "mr_eval_accumulate: null pointer (values, group_sizes, state)");
    MR_REQUIRE(G >= 1 && M >= 1 && M <= 1024, "mr_eval_accumulate: bad shape G=%d M=%d (1 <= M <= 1024)", G, M);
    for (int g = 0; g < G; ++g)
        MR_REQUIRE(group_sizes[g] >= 1, "mr_eval_accumulate: group_sizes[%d] = %d must be >= 1", g, group_sizes[g]);
    MR_REQUIRE((reinterpret_cast<uintptr_t>(state) & 7) == 0, "mr_eval_accumulate: state must be 8-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    for (int g0 = 0; g0 < G; g0 += kAccGroups) {
        AccArgs a{};
        a.values = values; a.state = state; a.M = M; a.g0 = g0;
        a.G = G - g0 < kAccGroups ? G - g0 : kAccGroups;
        for (int g = 0; g < a.G; ++g) a.sizes[g] = group_sizes[g0 + g];
        eval_accumulate_kernel<<<1, (M + 31) / 32 * 32, 0, st>>>(a);
        MR_LAUNCH_CHECK("eval_accumulate_kernel");
    }
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
