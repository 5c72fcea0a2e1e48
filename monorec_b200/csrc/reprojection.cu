// Photometric reprojection loss, forward and backward, for sm_90a (SURVEY.md 8f row 4: the training-side sibling of the
// cost-volume kernel -- one predicted depth per pixel instead of D planes, Gaussian-window SSIM, a gradient).
//
// Replaces reprojection_loss (reference: model/loss_functions/common_losses.py:16-114) for the argument sets the reference's
// losses use (model/loss_functions/monorec_loss.py:185-188, :264-265, :355, :361: error_function=compute_errors,
// combine_frames="min", mono_auto=False, reduce=False) together with compute_errors (:10-13), Backprojection /
// point_projection (model/layers.py:43-71), F.grid_sample x2 (:52, :54), create_mask (utils/util.py:130-132) and the
// Gaussian-window zero-padded comp-mode SSIM (layers.py:79-139) -- and torch autograd of all of that w.r.t. the predicted
// inverse depth (trainer/monorec_trainer.py:143-145).
//
// The reference materialises per source frame the back-projected points, the sampling grid, the warped image, five Gaussian
// filtered maps and a dozen element-wise temporaries, all kept alive for the backward pass.  Here:
//   forward   one CTA = 32 x 8 pixels of one keyframe; per source frame the warped samples of the tile and its 1-px ring go
//             to shared memory (homography from the mr_projection_tables rows with z = 1 / inv_depth, bilinear taps with
//             zero padding), the error 0.85 mean_c ssim + 0.15 mean_c |x - y| is evaluated from there, masked / auto-masked,
//             and the minimum over the frames and its index are written: [B,H,W] errors (+inf: no usable frame) and winners.
//   backward  nothing but the winners is saved.  Per frame the warped samples of the tile and a 2-px ring are recomputed,
//             every pixel p of the 1-px ring whose winner is this frame turns its upstream gradient into three coefficients
//             per channel (d ssim(p) / d x(q) = g(p - q) (alpha + beta y(q) + gamma x(q)) for the 9 pixels q of its window), and
//             each pixel q gathers the 9 windows it belongs to, adds the L1 term and chains through the bilinear sample
//             (d x / d sx, d x / d sy from the in-bounds taps) and the projection (d s / d inv_depth): one [B,1,H,W] gradient.
// Both kernels read each image a small constant number of times and write one map: they are far from any roofline that
// matters next to the D-plane cost volume (0.1 ms per batch of 8 at 256 x 512) and are written for clarity.
#include "mr_common.cuh"
#include <cstdint>

namespace {

constexpr int kTW = 32, kTH = 8;                  // output pixels per CTA
constexpr float kC1 = 0.01f * 0.01f;              // layers.py:116
constexpr float kC2 = 0.03f * 0.03f;              // layers.py:117
constexpr float kGc = 0.0947f, kGe = 0.1183f, kGm = 0.1478f;   // layers.py:82-85: corner, edge, centre of the window

struct RpArgs {
    const float* key;                    // [B,3,H,W]
    const float* frames[MR_MAX_FRAMES];  // each [B,3,H,W]
    const float* proj;                   // [B,F,12] rows of mr_projection_tables
    const float* invd;                   // [B,1,H,W] predicted inverse depth
    const float* gerr;                   // backward: [B,H,W] upstream gradient of the errors
    float* errors;                       // forward: [B,H,W]
    int* winner;                         // [B,H,W] index of the frame that gives the minimum, -1: none
    float* ginvd;                        // backward: [B,1,H,W]
    int B, F, H, W, automask, border;
};

struct Sample {
    float x[3];                          // warped value (reprojections after the -1.0 of common_losses.py:58)
    float gx[3], gy[3];                  // d x / d (sample column), d x / d (sample row)
    float dsx, dsy;                      // d (sample column) / d inv_depth, d (sample row) / d inv_depth
    bool masked;                         // common_losses.py:57 / :60-61
};

__device__ __forceinline__ float gweight(int dy, int dx) {   // dy, dx in {0,1,2}
    return (dy == 1 && dx == 1) ? kGm : ((dy == 1 || dx == 1) ? kGe : kGc);
}

// Back-projection with depth 1 / inv_depth, projection into frame f (the table holds K_f T K^-1 rows scaled by W/(W-1),
// H/(H-1) and the +1e-7 of layers.py:66), bilinear sample of frame + 1.5 with zero padding, minus 1.
template <bool GRAD>
__device__ __forceinline__ void warp_sample(const float* __restrict__ img, const float* m, float fu, float fv, float invd, int H,
                                            int W, int border, Sample& s) {
    const float z = 1.0f / invd;
    const float ax = fmaf(m[0], fu, fmaf(m[1], fv, m[2]));
    const float ay = fmaf(m[4], fu, fmaf(m[5], fv, m[6]));
    const float az = fmaf(m[8], fu, fmaf(m[9], fv, m[10]));
    const float cx = fmaf(ax, z, m[3]), cy = fmaf(ay, z, m[7]), cz = fmaf(az, z, m[11]);
    const float inv = 1.0f / cz;
    const float sxp = cx * inv, syp = cy * inv;             // sample position + 0.5
    const float sx = sxp - 0.5f, sy = syp - 0.5f;
    s.x[0] = s.x[1] = s.x[2] = -1.0f;
    s.masked = true;
    if (GRAD) { s.gx[0] = s.gx[1] = s.gx[2] = s.gy[0] = s.gy[1] = s.gy[2] = 0.f; s.dsx = s.dsy = 0.f; }
    // no tap inside the image (also NaN / inf positions): value 0, no gradient
    if (!(sx > -1.0f && sx < (float)W && sy > -1.0f && sy < (float)H)) return;
    const float x0f = floorf(sx), y0f = floorf(sy);
    const int x0 = (int)x0f, y0 = (int)y0f;
    const float fx = sx - x0f, fy = sy - y0f;
    const float wnw = (1.0f - fx) * (1.0f - fy), wne = fx * (1.0f - fy), wsw = (1.0f - fx) * fy, wse = fx * fy;
    const bool inx0 = x0 >= 0, inx1 = x0 + 1 < W, iny0 = y0 >= 0, iny1 = y0 + 1 < H;
    const size_t plane = (size_t)H * W;
    const float* p = img + (ptrdiff_t)y0 * W + x0;
    float raw0 = 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c, p += plane) {
        const float nw = (inx0 && iny0) ? __ldg(p) + 1.5f : 0.f;
        const float ne = (inx1 && iny0) ? __ldg(p + 1) + 1.5f : 0.f;
        const float sw = (inx0 && iny1) ? __ldg(p + W) + 1.5f : 0.f;
        const float se = (inx1 && iny1) ? __ldg(p + W + 1) + 1.5f : 0.f;
        const float v = nw * wnw + ne * wne + sw * wsw + se * wse;
        if (c == 0) raw0 = v;
        s.x[c] = v - 1.0f;
        if (GRAD) {
            s.gx[c] = (ne - nw) * (1.0f - fy) + (se - sw) * fy;
            s.gy[c] = (sw - nw) * (1.0f - fx) + (se - ne) * fx;
        }
    }
    if (border > 0) {
        // bilinear sample of the interior indicator (1 inside a ring of `border` pixels), masked unless > 0.5
        const bool bx0 = x0 >= border && x0 < W - border, bx1 = x0 + 1 >= border && x0 + 1 < W - border;
        const bool by0 = y0 >= border && y0 < H - border, by1 = y0 + 1 >= border && y0 + 1 < H - border;
        const float mval = ((bx0 && by0) ? wnw : 0.f) + ((bx1 && by0) ? wne : 0.f) + ((bx0 && by1) ? wsw : 0.f) + ((bx1 && by1) ? wse : 0.f);
        s.masked = !(mval > 0.5f);
    } else {
        s.masked = (raw0 == 0.f);
    }
    if (GRAD) {
        // c = a z + t, z = 1 / inv_depth: d (cx / cz) / d inv_depth = -z^2 (ax - sxp az) / cz
        const float dz = -z * z;
        s.dsx = dz * (ax - sxp * az) * inv;
        s.dsy = dz * (ay - syp * az) * inv;
    }
}

// Gaussian-window statistics of one channel at one pixel: xs / ys point at the window's top-left sample, stride = row pitch
struct Stats { float mx, my, sxx, syy, sxy; };
__device__ __forceinline__ Stats window_stats(const float* xs, const float* ys, int stride) {
    Stats t{0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int dy = 0; dy < 3; ++dy)
#pragma unroll
        for (int dx = 0; dx < 3; ++dx) {
            const float g = gweight(dy, dx), x = xs[dy * stride + dx], y = ys[dy * stride + dx];
            t.mx = fmaf(g, x, t.mx); t.my = fmaf(g, y, t.my);
            t.sxx = fmaf(g * x, x, t.sxx); t.syy = fmaf(g * y, y, t.syy); t.sxy = fmaf(g * x, y, t.sxy);
        }
    return t;
}

// compute_errors (common_losses.py:10-13) at the pixel whose window starts at xs / ys; xc / yc = the pixel itself
__device__ __forceinline__ float pixel_error(const float* xs, const float* ys, int stride, int chan_stride) {
    float ssim = 0.f, l1 = 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float* xc = xs + c * chan_stride;
        const float* yc = ys + c * chan_stride;
        const Stats t = window_stats(xc, yc, stride);
        const float mxx = t.mx * t.mx, myy = t.my * t.my, mxy = t.mx * t.my;
        const float n = (2.0f * mxy + kC1) * (2.0f * (t.sxy - mxy) + kC2);
        const float d = (mxx + myy + kC1) * ((t.sxx - mxx) + (t.syy - myy) + kC2);
        ssim += fminf(fmaxf(1.0f - n / d, 0.f), 1.f) * 0.5f;
        l1 += fabsf(xc[stride + 1] - yc[stride + 1]);
    }
    return 0.85f * (ssim / 3.0f) + 0.15f * (l1 / 3.0f);
}

constexpr int kFS = kTW + 2 + 1;                  // forward: row pitch of the (kTH + 2) x (kTW + 2) sample tile
constexpr int kFRows = kTH + 2;
constexpr int kFChan = kFRows * kFS;

__global__ void __launch_bounds__(kTW * kTH)
reprojection_fwd_kernel(const RpArgs a) {
    __shared__ float ys[3 * kFChan];
    __shared__ float xs[3 * kFChan];
    __shared__ float pj[12];
    const int tx = threadIdx.x, ty = threadIdx.y, tid = ty * kTW + tx;
    const int b = blockIdx.z, u0 = blockIdx.x * kTW, v0 = blockIdx.y * kTH;
    const int H = a.H, W = a.W;
    const size_t plane = (size_t)H * W;
    // tile positions: the thread's own pixel first, then the ring (84 positions) on the first threads
    auto position = [&](int it, int& r, int& c) -> bool {
        if (it == 0) { r = ty + 1; c = tx + 1; return true; }
        int k = tid;
        if (k >= 2 * (kTW + 2) + 2 * kTH) return false;
        if (k < kTW + 2) { r = 0; c = k; }
        else if (k < 2 * (kTW + 2)) { r = kTH + 1; c = k - (kTW + 2); }
        else { k -= 2 * (kTW + 2); r = 1 + (k >> 1); c = (k & 1) ? kTW + 1 : 0; }
        return true;
    };
    const float* key = a.key + (size_t)b * 3 * plane;
    for (int it = 0; it < 2; ++it) {
        int r, c;
        if (!position(it, r, c)) continue;
        const int v = v0 - 1 + r, u = u0 - 1 + c;
        const bool in = (u >= 0 && u < W && v >= 0 && v < H);
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) ys[ch * kFChan + r * kFS + c] = in ? __ldg(key + ch * plane + (size_t)v * W + u) + 0.5f : 0.f;
    }
    const int u = u0 + tx, v = v0 + ty;
    const bool own = (u < W && v < H);
    float best = __int_as_float(0x7f800000);
    int besti = -1;
    for (int f = 0; f < a.F; ++f) {
        __syncthreads();                                    // the previous frame's tile has been consumed
        if (tid < 12) pj[tid] = __ldg(a.proj + ((size_t)b * a.F + f) * 12 + tid);
        __syncthreads();
        const float* img = a.frames[f] + (size_t)b * 3 * plane;
        bool masked = true;
        for (int it = 0; it < 2; ++it) {
            int r, c;
            if (!position(it, r, c)) continue;
            const int pv = v0 - 1 + r, pu = u0 - 1 + c;
            Sample s;
            s.x[0] = s.x[1] = s.x[2] = 0.f;                 // outside the image: the zero padding of the SSIM (layers.py:112)
            s.masked = true;
            if (pu >= 0 && pu < W && pv >= 0 && pv < H)
                warp_sample<false>(img, pj, (float)pu, (float)pv, __ldg(a.invd + (size_t)b * plane + (size_t)pv * W + pu), H, W, a.border, s);
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) xs[ch * kFChan + r * kFS + c] = s.x[ch];
            if (it == 0) masked = s.masked;
        }
        __syncthreads();
        float e = pixel_error(xs + ty * kFS + tx, ys + ty * kFS + tx, kFS, kFChan);
        if (masked) e = __int_as_float(0x7f800000);         // common_losses.py:78
        if (a.automask) {                                   // :80-83: the unwarped frame explains the pixel better
            __syncthreads();
            for (int it = 0; it < 2; ++it) {
                int r, c;
                if (!position(it, r, c)) continue;
                const int pv = v0 - 1 + r, pu = u0 - 1 + c;
                const bool in = (pu >= 0 && pu < W && pv >= 0 && pv < H);
#pragma unroll
                for (int ch = 0; ch < 3; ++ch) xs[ch * kFChan + r * kFS + c] = in ? __ldg(img + ch * plane + (size_t)pv * W + pu) + 0.5f : 0.f;
            }
            __syncthreads();
            const float e0 = pixel_error(xs + ty * kFS + tx, ys + ty * kFS + tx, kFS, kFChan);
            if (e0 < e) e = __int_as_float(0x7f800000);
        }
        if (e < best) { best = e; besti = f; }              // :94 torch.min over the frames (first minimum)
    }
    if (own) {
        a.errors[(size_t)b * plane + (size_t)v * W + u] = best;
        a.winner[(size_t)b * plane + (size_t)v * W + u] = besti;
    }
}

constexpr int kBS = kTW + 4 + 1;                  // backward: row pitch of the (kTH + 4) x (kTW + 4) sample tile
constexpr int kBRows = kTH + 4;
constexpr int kBChan = kBRows * kBS;
constexpr int kCS = kTW + 2 + 1;                  // coefficient tile (kTH + 2) x (kTW + 2)
constexpr int kCRows = kTH + 2;
constexpr int kCChan = kCRows * kCS;

__global__ void __launch_bounds__(kTW * kTH)
reprojection_bwd_kernel(const RpArgs a) {
    __shared__ float ys[3 * kBChan];
    __shared__ float xs[3 * kBChan];
    __shared__ float ca[3 * kCChan], cb[3 * kCChan], cg[3 * kCChan];   // alpha, beta, gamma times the upstream gradient
    __shared__ float pj[12];
    const int tx = threadIdx.x, ty = threadIdx.y, tid = ty * kTW + tx;
    const int b = blockIdx.z, u0 = blockIdx.x * kTW, v0 = blockIdx.y * kTH;
    const int H = a.H, W = a.W;
    const size_t plane = (size_t)H * W;
    const float* key = a.key + (size_t)b * 3 * plane;
    for (int k = tid; k < kBRows * (kTW + 4); k += kTW * kTH) {
        const int r = k / (kTW + 4), c = k - r * (kTW + 4);
        const int pv = v0 - 2 + r, pu = u0 - 2 + c;
        const bool in = (pu >= 0 && pu < W && pv >= 0 && pv < H);
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) ys[ch * kBChan + r * kBS + c] = in ? __ldg(key + ch * plane + (size_t)pv * W + pu) + 0.5f : 0.f;
    }
    const int u = u0 + tx, v = v0 + ty;
    const bool own = (u < W && v < H);
    const size_t pix = (size_t)b * plane + (size_t)(own ? v : 0) * W + (own ? u : 0);
    const float invd_own = own ? __ldg(a.invd + pix) : 1.0f;
    const int win_own = own ? __ldg(a.winner + pix) : -1;
    const float g_own = own ? __ldg(a.gerr + pix) : 0.f;
    float grad = 0.f;
    for (int f = 0; f < a.F; ++f) {
        __syncthreads();
        if (tid < 12) pj[tid] = __ldg(a.proj + ((size_t)b * a.F + f) * 12 + tid);
        __syncthreads();
        const float* img = a.frames[f] + (size_t)b * 3 * plane;
        // the thread's own pixel with the derivatives of the sample, then the other positions of the 2-px ring tile
        Sample so;
        so.x[0] = so.x[1] = so.x[2] = 0.f;
        so.gx[0] = so.gx[1] = so.gx[2] = so.gy[0] = so.gy[1] = so.gy[2] = 0.f; so.dsx = so.dsy = 0.f;
        if (own) warp_sample<true>(img, pj, (float)u, (float)v, invd_own, H, W, a.border, so);
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) xs[ch * kBChan + (ty + 2) * kBS + tx + 2] = so.x[ch];
        for (int k = tid; k < kBRows * (kTW + 4); k += kTW * kTH) {
            const int r = k / (kTW + 4), c = k - r * (kTW + 4);
            if (r >= 2 && r < 2 + kTH && c >= 2 && c < 2 + kTW) continue;
            const int pv = v0 - 2 + r, pu = u0 - 2 + c;
            Sample s;
            s.x[0] = s.x[1] = s.x[2] = 0.f;
            if (pu >= 0 && pu < W && pv >= 0 && pv < H)
                warp_sample<false>(img, pj, (float)pu, (float)pv, __ldg(a.invd + (size_t)b * plane + (size_t)pv * W + pu), H, W, a.border, s);
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) xs[ch * kBChan + r * kBS + c] = s.x[ch];
        }
        __syncthreads();
        // coefficients of every pixel p of the 1-px ring tile whose minimum is this frame
        for (int k = tid; k < kCRows * (kTW + 2); k += kTW * kTH) {
            const int r = k / (kTW + 2), c = k - r * (kTW + 2);
            const int pv = v0 - 1 + r, pu = u0 - 1 + c;
            float g = 0.f;
            if (pu >= 0 && pu < W && pv >= 0 && pv < H) {
                const size_t pp = (size_t)b * plane + (size_t)pv * W + pu;
                if (__ldg(a.winner + pp) == f) g = __ldg(a.gerr + pp);
            }
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) {
                float al = 0.f, be = 0.f, ga = 0.f;
                if (g != 0.f) {
                    const Stats t = window_stats(xs + ch * kBChan + r * kBS + c, ys + ch * kBChan + r * kBS + c, kBS);
                    const float mxx = t.mx * t.mx, myy = t.my * t.my, mxy = t.mx * t.my;
                    const float A1 = 2.0f * mxy + kC1, A2 = 2.0f * (t.sxy - mxy) + kC2;
                    const float B1 = mxx + myy + kC1, B2 = (t.sxx - mxx) + (t.syy - myy) + kC2;
                    const float invden = 1.0f / (B1 * B2);
                    const float R = A1 * A2 * invden;
                    const float val = 1.0f - R;
                    if (val >= 0.f && val <= 1.f) {        // torch.clamp passes the gradient on the closed interval
                        // d ssim(p) / d x(q) = -0.5 g(p - q) (alpha + beta y(q) + gamma x(q)), times 0.85 / 3 and the upstream gradient
                        const float sc = -0.5f * (0.85f / 3.0f) * g;
                        al = sc * (2.0f * t.my * (A2 - A1) * invden - 2.0f * R * invden * t.mx * (B2 - B1));
                        be = sc * (2.0f * A1 * invden);
                        ga = sc * (-2.0f * R * invden * B1);
                    }
                }
                ca[ch * kCChan + r * kCS + c] = al;
                cb[ch * kCChan + r * kCS + c] = be;
                cg[ch * kCChan + r * kCS + c] = ga;
            }
        }
        __syncthreads();
        if (own) {
            float acc = 0.f;
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) {
                float sa = 0.f, sb = 0.f, sg = 0.f;
#pragma unroll
                for (int dy = 0; dy < 3; ++dy)
#pragma unroll
                    for (int dx = 0; dx < 3; ++dx) {
                        const float gw = gweight(dy, dx);
                        const int o = ch * kCChan + (ty + dy) * kCS + tx + dx;
                        sa = fmaf(gw, ca[o], sa); sb = fmaf(gw, cb[o], sb); sg = fmaf(gw, cg[o], sg);
                    }
                const float x = so.x[ch], y = ys[ch * kBChan + (ty + 2) * kBS + tx + 2];
                float gxv = sa + sb * y + sg * x;
                if (win_own == f) {                        // 0.15 mean_c |x - y|
                    const float dlt = x - y;
                    gxv += g_own * (0.15f / 3.0f) * ((dlt > 0.f) ? 1.0f : ((dlt < 0.f) ? -1.0f : 0.f));
                }
                acc += gxv * (so.gx[ch] * so.dsx + so.gy[ch] * so.dsy);
            }
            grad += acc;
        }
    }
    if (own) a.ginvd[pix] = grad;
}

int fill_args(RpArgs& a, const float* keyframe, const float* const* frames, const float* proj, const float* inv_depth, int B,
              int F, int H, int W, const char* who) {
    MR_REQUIRE(keyframe && frames && proj && inv_depth, "%s: null pointer", who);
    MR_REQUIRE(B >= 1 && B <= 65535, "%s: batch %d out of range", who, B);
    MR_REQUIRE(F >= 1 && F <= MR_MAX_FRAMES, "%s: 1 <= F <= %d required (got %d)", who, MR_MAX_FRAMES, F);
    MR_REQUIRE(H >= 3 && W >= 3 && H <= 16384 && W <= 16384, "%s: image size %dx%d out of range", who, H, W);
    a.key = keyframe;
    for (int f = 0; f < F; ++f) {
        MR_REQUIRE(frames[f] != nullptr, "%s: null frame pointer %d", who, f);
        a.frames[f] = frames[f];
    }
    a.proj = proj; a.invd = inv_depth; a.B = B; a.F = F; a.H = H; a.W = W;
    return MR_OK;
}

}  // namespace

extern "C" int mr_reprojection_loss_fwd(const float* keyframe, const float* const* frames, const float* proj,
                                        const float* inv_depth, int B, int F, int H, int W, int automasking, int border,
                                        float* out_errors, int* out_winner, void* stream) {
    RpArgs a{};
    int rc = fill_args(a, keyframe, frames, proj, inv_depth, B, F, H, W, "mr_reprojection_loss_fwd");
    if (rc != MR_OK) return rc;
    MR_REQUIRE(out_errors && out_winner, "mr_reprojection_loss_fwd: null output pointer");
    MR_REQUIRE(border >= 0 && 2 * border < H && 2 * border < W, "mr_reprojection_loss_fwd: border %d does not fit %dx%d", border, H, W);
    a.errors = out_errors; a.winner = out_winner; a.automask = automasking ? 1 : 0; a.border = border;
    dim3 grid((W + kTW - 1) / kTW, (H + kTH - 1) / kTH, B), block(kTW, kTH);
    reprojection_fwd_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(a);
    MR_LAUNCH_CHECK("reprojection_fwd_kernel");
    return MR_OK;
}

extern "C" int mr_reprojection_loss_bwd(const float* keyframe, const float* const* frames, const float* proj,
                                        const float* inv_depth, const float* grad_errors, const int* winner, int B, int F, int H,
                                        int W, float* out_grad_inv_depth, void* stream) {
    RpArgs a{};
    int rc = fill_args(a, keyframe, frames, proj, inv_depth, B, F, H, W, "mr_reprojection_loss_bwd");
    if (rc != MR_OK) return rc;
    MR_REQUIRE(grad_errors && winner && out_grad_inv_depth, "mr_reprojection_loss_bwd: null pointer");
    a.gerr = grad_errors; a.winner = const_cast<int*>(winner); a.ginvd = out_grad_inv_depth; a.border = 0;
    dim3 grid((W + kTW - 1) / kTW, (H + kTH - 1) / kTH, B), block(kTW, kTH);
    reprojection_bwd_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(a);
    MR_LAUNCH_CHECK("reprojection_bwd_kernel");
    return MR_OK;
}
