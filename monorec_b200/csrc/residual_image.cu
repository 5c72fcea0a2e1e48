// Photometric residual image for sm_90a: the reference's ground-truth-free check of a depth map.
//
// Replaces ResidualImageModule.forward (reference: model/layers.py:161-217) and the ResidualImage wrapper (:147-158):
// per source frame, the back-projection of every keyframe pixel at the given inverse depth, point_projection (:63-71, with
// the +1e-7 and the (W-1) / (H-1) normalisation and no clamp), F.grid_sample of frame + 1 (bilinear, zero padding,
// align_corners=False), the mask any_c(warped == 0), the reflection-padded 3x3-box SSIM of warped - 0.5 against
// keyframe + 0.5 (:91-139, not comp mode), the channel mean, +inf where masked, the minimum over the frames and 0 where
// every frame is masked.  The reference materialises per frame the points, the grid, the warped image, five pooled maps and a
// [B,F,C,H,W] stack; here one launch reads each input once and writes the [B,1,H,W] map:
//   one CTA = 32 x 8 pixels of one keyframe.  The keyframe tile and its 1-px ring (+0.5) go to shared memory once and each
//   pixel keeps its keyframe window sums in registers.  Per source frame the warped samples of the tile and its ring go to
//   shared memory (homography from the mr_projection_tables rows with z = 1 / inv_depth), each pixel evaluates the SSIM of
//   every channel from there, takes the channel mean and folds it into a running minimum and mask in registers.
// The ring follows the reference's ReflectionPad2d(1): at the image border a ring position holds the sample of the mirrored
// pixel (-1 -> 1, n -> n - 2); between tiles it holds the neighbouring tile's sample.
// Grayscale frames (NC = 1) are read as one plane and the single SSIM value enters the channel mean three times, in the
// three-channel expression, so the result is that of the replicated frames bit for bit.
#include "mr_common.cuh"
#include <cstdint>

namespace {

constexpr int kTW = 32, kTH = 8;                  // output pixels per CTA
constexpr int kPitch = kTW + 2 + 1;               // row pitch of the (kTH + 2) x (kTW + 2) sample tiles
constexpr int kRows = kTH + 2;
constexpr int kPlane = kRows * kPitch;
constexpr int kRing = kRows * (kTW + 2);          // tile + ring positions
constexpr float kC1 = 0.01f * 0.01f;              // layers.py:116
constexpr float kC2 = 0.03f * 0.03f;              // layers.py:117

struct RiArgs {
    const float* key;                    // [B,NC,H,W]
    const float* frames[MR_MAX_FRAMES];  // each [B,NC,H,W]
    const float* proj;                   // [B,F,12] rows of mr_projection_tables
    const float* invd;                   // [B,1,H,W] predicted_inverse_depths[0]
    const float* range;                  // {inv_depth_max, inv_depth_min} on the device, or null: {0, 1} (ResidualImage)
    float* out;                          // [B,1,H,W]
    int B, F, H, W;
};

// ReflectionPad2d(1) index: -1 -> 1, n -> n - 2; clamped so that positions past a ragged tile edge stay addressable
__device__ __forceinline__ int reflect(int i, int n) {
    i = i < 0 ? -i : (i >= n ? 2 * n - 2 - i : i);
    return min(max(i, 0), n - 1);
}

// torch.clamp(x, 0, 1), which keeps a NaN (fminf / fmaxf would drop it)
__device__ __forceinline__ float clamp01(float x) { return x < 0.f ? 0.f : (x > 1.f ? 1.f : x); }

// The warped sample of keyframe pixel (u, v) in one frame: layers.py:193-205.  depth = (1 - p) inv_depth_max + p inv_depth_min
// (:172) rounded op by op as torch does, back-projected at z = 1 / depth, projected with the table row m (K_f T K^-1 scaled by
// W/(W-1), H/(H-1), +1e-7 on the translation's z), bilinear sample of frame + 1 with zero taps outside the image.
// x[c] = sample - 0.5 (:205); masked = some channel of the sample is exactly 0 (:204).  A position that is not finite gives a
// NaN sample, as the reference's grid_sample on the CPU does (zero taps times NaN weights); NaN != 0, so it is not masked.
template <int NC>
__device__ __forceinline__ bool warp_sample(const float* __restrict__ img, const float* m, float fu, float fv, float p,
                                            float dmax, float dmin, int H, int W, float* x) {
    const float depth = __fadd_rn(__fmul_rn(__fsub_rn(1.0f, p), dmax), __fmul_rn(p, dmin));
    const float z = 1.0f / depth;
    const float ax = fmaf(m[0], fu, fmaf(m[1], fv, m[2]));
    const float ay = fmaf(m[4], fu, fmaf(m[5], fv, m[6]));
    const float az = fmaf(m[8], fu, fmaf(m[9], fv, m[10]));
    const float cx = fmaf(ax, z, m[3]), cy = fmaf(ay, z, m[7]), cz = fmaf(az, z, m[11]);
    const float inv = 1.0f / cz;
    const float sx = fmaf(cx, inv, -0.5f), sy = fmaf(cy, inv, -0.5f);
    if (!(isfinite(sx) && isfinite(sy))) {
#pragma unroll
        for (int c = 0; c < NC; ++c) x[c] = __int_as_float(0x7fffffff);
        return false;
    }
    bool masked = false;
    if (!(sx > -1.0f && sx < (float)W && sy > -1.0f && sy < (float)H)) {   // no tap inside the image: every channel is 0
#pragma unroll
        for (int c = 0; c < NC; ++c) x[c] = -0.5f;
        return true;
    }
    const float x0f = floorf(sx), y0f = floorf(sy);
    const int x0 = (int)x0f, y0 = (int)y0f;
    const float fx = sx - x0f, fy = sy - y0f;
    const float wnw = (1.0f - fx) * (1.0f - fy), wne = fx * (1.0f - fy), wsw = (1.0f - fx) * fy, wse = fx * fy;
    const bool inx0 = x0 >= 0, inx1 = x0 + 1 < W, iny0 = y0 >= 0, iny1 = y0 + 1 < H;
    const size_t plane = (size_t)H * W;
    const float* q = img + (ptrdiff_t)y0 * W + x0;
#pragma unroll
    for (int c = 0; c < NC; ++c, q += plane) {
        const float nw = (inx0 && iny0) ? __ldg(q) + 1.0f : 0.f;
        const float ne = (inx1 && iny0) ? __ldg(q + 1) + 1.0f : 0.f;
        const float sw = (inx0 && iny1) ? __ldg(q + W) + 1.0f : 0.f;
        const float se = (inx1 && iny1) ? __ldg(q + W + 1) + 1.0f : 0.f;
        const float v = fmaf(se, wse, fmaf(sw, wsw, fmaf(ne, wne, nw * wnw)));
        masked = masked || (v == 0.f);
        x[c] = v - 0.5f;
    }
    return masked;
}

template <int NC>
__global__ void __launch_bounds__(kTW * kTH)
residual_image_kernel(const RiArgs a) {
    __shared__ float ys[NC * kPlane];                 // keyframe + 0.5, tile + ring
    __shared__ float xs[NC * kPlane];                 // warped - 0.5 of the current frame, tile + ring
    __shared__ float pj[MR_MAX_FRAMES * 12];
    __shared__ bool mks[kRows * kPitch];              // the sample of the tile position is masked
    __shared__ const float* fptr[MR_MAX_FRAMES];      // (a dynamic index into the parameter struct would copy it to the stack)
    const int tx = threadIdx.x, ty = threadIdx.y, tid = ty * kTW + tx;
    const int b = blockIdx.z, u0 = blockIdx.x * kTW, v0 = blockIdx.y * kTH;
    const int H = a.H, W = a.W, F = a.F;
    const size_t plane = (size_t)H * W;
    if (tid < F * 12) pj[tid] = __ldg(a.proj + (size_t)b * F * 12 + tid);
#pragma unroll
    for (int f = 0; f < MR_MAX_FRAMES; ++f)
        if (tid == f) fptr[f] = a.frames[f];
    const float dmax = a.range ? __ldg(a.range) : 0.0f;
    const float dmin = a.range ? __ldg(a.range + 1) : 1.0f;
    const float* key = a.key + (size_t)b * NC * plane;
    const float* invd = a.invd + (size_t)b * plane;
    for (int k = tid; k < kRing; k += kTW * kTH) {
        const int r = k / (kTW + 2), c = k - r * (kTW + 2);
        const size_t o = (size_t)reflect(v0 - 1 + r, H) * W + reflect(u0 - 1 + c, W);
#pragma unroll
        for (int ch = 0; ch < NC; ++ch) ys[ch * kPlane + r * kPitch + c] = __ldg(key + ch * plane + o) + 0.5f;
    }
    __syncthreads();
    // the keyframe's window sums at the thread's pixel (AvgPool2d(3, 1) of y and y^2: sum / 9), kept for every frame
    float my[NC], syy[NC];
#pragma unroll
    for (int ch = 0; ch < NC; ++ch) {
        float s = 0.f, s2 = 0.f;
#pragma unroll
        for (int dy = 0; dy < 3; ++dy)
#pragma unroll
            for (int dx = 0; dx < 3; ++dx) {
                const float y = ys[ch * kPlane + (ty + dy) * kPitch + tx + dx];
                s += y; s2 = fmaf(y, y, s2);
            }
        my[ch] = s / 9.0f; syy[ch] = s2 / 9.0f;
    }
    const int u = u0 + tx, v = v0 + ty;
    const float inf = __int_as_float(0x7f800000);
    float best = inf;
    bool all_masked = true;
    for (int f = 0; f < F; ++f) {
        const float* img = fptr[f] + (size_t)b * NC * plane;
        const float* m = pj + f * 12;
        if (f > 0) __syncthreads();                   // the previous frame's tile has been consumed
        for (int k = tid; k < kRing; k += kTW * kTH) {
            const int r = k / (kTW + 2), c = k - r * (kTW + 2);
            const int pv = reflect(v0 - 1 + r, H), pu = reflect(u0 - 1 + c, W);
            float x[NC];
            const bool mk = warp_sample<NC>(img, m, (float)pu, (float)pv, __ldg(invd + (size_t)pv * W + pu), dmax, dmin, H, W, x);
#pragma unroll
            for (int ch = 0; ch < NC; ++ch) xs[ch * kPlane + r * kPitch + c] = x[ch];
            mks[r * kPitch + c] = mk;
        }
        __syncthreads();
        const bool masked = mks[(ty + 1) * kPitch + tx + 1];
        float e[NC];
#pragma unroll
        for (int ch = 0; ch < NC; ++ch) {
            float s = 0.f, s2 = 0.f, sxy = 0.f;
#pragma unroll
            for (int dy = 0; dy < 3; ++dy)
#pragma unroll
                for (int dx = 0; dx < 3; ++dx) {
                    const int o = ch * kPlane + (ty + dy) * kPitch + tx + dx;
                    const float x = xs[o], y = ys[o];
                    s += x; s2 = fmaf(x, x, s2); sxy = fmaf(x, y, sxy);
                }
            // layers.py:123-137 in the reference's order, rounded op by op (no contraction: one expression for both
            // channel counts)
            const float mx = s / 9.0f;
            const float mxx = __fmul_rn(mx, mx), myy = __fmul_rn(my[ch], my[ch]), mxy = __fmul_rn(mx, my[ch]);
            const float sigx = __fsub_rn(s2 / 9.0f, mxx), sigy = __fsub_rn(syy[ch], myy), sigxy = __fsub_rn(sxy / 9.0f, mxy);
            const float n = __fmul_rn(__fadd_rn(__fmul_rn(2.0f, mxy), kC1), __fadd_rn(__fmul_rn(2.0f, sigxy), kC2));
            const float d = __fmul_rn(__fadd_rn(__fadd_rn(mxx, myy), kC1), __fadd_rn(__fadd_rn(sigx, sigy), kC2));
            e[ch] = clamp01(__fsub_rn(1.0f, n / d) / 2.0f);
        }
        // channel mean (a one-channel value enters all three terms); masked entries are +inf (:212)
        float mean;
        if constexpr (NC == 3) mean = __fadd_rn(__fadd_rn(e[0], e[1]), e[2]) / 3.0f;
        else mean = __fadd_rn(__fadd_rn(e[0], e[0]), e[0]) / 3.0f;
        const float r = masked ? inf : mean;
        // torch.min over the frames (:214), which keeps a NaN
        if (!(best != best) && !(r >= best)) best = r;
        all_masked = all_masked && masked;
    }
    if (u < W && v < H) a.out[(size_t)b * plane + (size_t)v * W + u] = all_masked ? 0.0f : best;   // :215
}

}  // namespace

extern "C" int mr_residual_image(const float* keyframe, const float* const* frames, const float* proj, const float* inv_depth,
                                 const float* inv_depth_range, int B, int F, int C, int H, int W, float* out, void* stream) {
    const char* who = "mr_residual_image";
    MR_REQUIRE(keyframe && frames && proj && inv_depth && out, "%s: null pointer", who);
    MR_REQUIRE(B >= 1 && B <= 65535, "%s: batch %d out of range", who, B);
    MR_REQUIRE(F >= 1 && F <= MR_MAX_FRAMES, "%s: 1 <= F <= %d required (got %d)", who, MR_MAX_FRAMES, F);
    MR_REQUIRE(C == 1 || C == 3, "%s: channels must be 1 or 3 (got %d)", who, C);
    MR_REQUIRE(H >= 2 && W >= 2 && H <= 16384 && W <= 16384, "%s: image size %dx%d out of range (2..16384)", who, H, W);
    RiArgs a{};
    auto aligned = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 3) == 0; };
    for (int f = 0; f < F; ++f) {
        MR_REQUIRE(frames[f] != nullptr, "%s: null frame pointer %d", who, f);
        MR_REQUIRE(aligned(frames[f]), "%s: frame %d must be 4-byte aligned", who, f);
        a.frames[f] = frames[f];
    }
    MR_REQUIRE(aligned(keyframe) && aligned(proj) && aligned(inv_depth) && aligned(out) && aligned(inv_depth_range),
               "%s: keyframe, proj, inv_depth, inv_depth_range and out must be 4-byte aligned", who);
    a.key = keyframe; a.proj = proj; a.invd = inv_depth; a.range = inv_depth_range; a.out = out;
    a.B = B; a.F = F; a.H = H; a.W = W;
    dim3 grid((W + kTW - 1) / kTW, (H + kTH - 1) / kTH, B), block(kTW, kTH);
    if (C == 3)
        residual_image_kernel<3><<<grid, block, 0, (cudaStream_t)stream>>>(a);
    else
        residual_image_kernel<1><<<grid, block, 0, (cudaStream_t)stream>>>(a);
    MR_LAUNCH_CHECK("residual_image_kernel");
    return MR_OK;
}
