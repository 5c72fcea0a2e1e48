// Fused plane-sweep cost volume for sm_90a (H100), second generation: TMA-staged source windows.
//
// Replaces CostVolumeModule.forward (reference: model/monorec/monorec_model.py:150-280) together with
// Backprojection / point_projection (model/layers.py:43-71), F.grid_sample x2, SSIM (layers.py:119-137), the
// conv3d patch cost (:246-248) and the view weighting / fusion (:257-269).  Closed form: SURVEY.md Appendix C.
//
// Work decomposition:
//   CTA   = one keyframe tile of 60 x TH output pixels (64 x (TH+4) with the 2-px stencil halo), all D planes, all F
//           source frames.  grid = (ceil(W/60), ceil(H/TH), B).
//   plan  = per tile and source frame the D planes are cut into groups of consecutive planes whose source footprints
//           (projective image of the tile rectangle: extremes at its 4 corners) share one window of kPitch x kWinRows
//           pixels.  A window is the [C][rows][kPitch] fp32 copy of that frame region (C = 3, or 1 for grayscale
//           frames), brought into shared memory by TMA boxes {kPitch, 8, 1} straight from the NCHW frame
//           (cp.async.bulk.tensor, mbarrier complete_tx, kBuf
//           buffers in flight); out-of-image box parts are zero-filled by the TMA unit, which is exactly
//           F.grid_sample(padding_mode="zeros") once integer tap coordinates are clamped to the 2-px zero ring.
//   unit  = (frame, plane).  Warps claim units from a shared counter (units of one window are consecutive), wait for
//           the window's mbarrier, and march down the tile rows:
//             stage 1 (lane = columns l, l+32): homography, floor by magic-number rounding, 4 C bilinear taps per
//                      sample as conflict-free LDS from the window (immediate offsets), warped row -> smem row buffer;
//             stage 2 (lane = columns 2l, 2l+1): 3x3 box sums of X, X^2, XY (horizontal in registers, vertical rolling),
//                      SSIM in 81x-scaled form, channel weights, second 3x3 box -> 1 - 2 sad streamed to HBM.
//           Stage 1 of row t+1 and stage 2 of row t are issued together (double-buffered row buffer, one __syncwarp
//           per row).  The last warp to finish a window's units re-arms the buffer with the window after next.
//           Units whose footprint does not fit a window (strong zoom), groups of fewer than kMinGroup planes and
//           launches whose frames TMA cannot address (W % 4 != 0, unaligned base) gather from global memory instead.
//   CTA phase 2 (thread = pixel): view weight from max_d / sum_d exp(..), zeroing of invalid pixels, fusion over
//           frames from the L2-hot single-frame volumes.
// Template parameters: the depth source (plane table / per-pixel cv_depths), the error mode of stage 2 (SSIM, SSIM + L1 or
// the 3x3 box of L1: the reference's use_ssim, monorec_model.py:227-243), the centring of the fused volume
// (not_center_cv, :267-269) and the storage type of both volumes (fp32, or IEEE half: stores round, arithmetic stays fp32).
// Keyframe-only terms (9 mu_y, 81 (sigma_y + C2)) are hoisted into a smem table per tile; pixels whose reprojection leaves
// the source for any plane (valid_f = 0) are found by a projection pre-pass over the two extreme planes (the samples of
// one pixel lie on a line, monotone in depth, so the extremes decide) and whole row ranges / frames of a tile are skipped.
#include "mr_common.cuh"
#include <cuda.h>
#include <cuda_fp16.h>
#include <atomic>
#include <cstdint>
#include <type_traits>

namespace {

constexpr int kTileCols = 64;   // buffer columns per tile row (output columns + 2-px halo each side)
constexpr int kOutCols = 60;    // output columns per tile
constexpr int kRowStride = 68;  // floats per smem image row: column b lives at index b+1 (so [2l-1, 2l+2] is 8B aligned)
constexpr int kWarps = 16;
constexpr int kThreads = kWarps * 32;
constexpr int kMinBlocks = 1;                     // resident CTAs per SM the register allocator must leave room for
constexpr int kBuf = 2;                           // source windows in flight per CTA
constexpr int kPitch = 128;                       // pixels per window row (512 bytes)
constexpr int kWinRows = 40;                      // rows per window (multiple of 8)
constexpr int kChanStride = kWinRows * kPitch;    // floats between the channel planes of a window (NC of them)
constexpr int kBoxRows = 8;                      // rows per TMA box
constexpr int kMinGroup = 3;                      // plane groups smaller than this gather from global memory
constexpr int kTileRows = 16;                     // tile height when shared memory allows it (halved until it fits)
static_assert(kWinRows % kBoxRows == 0, "window rows must be a multiple of the TMA box height");
static_assert(MR_MAX_FRAMES <= kWarps, "the plan gives every source frame its own warp");

constexpr float kC1 = 0.01f * 0.01f;  // layers.py:116
constexpr float kC2 = 0.03f * 0.03f;  // layers.py:117
constexpr float kMagic = 12582912.0f;      // 1.5 * 2^23: adding it rounds to the nearest integer in the low mantissa bits
constexpr int kMagicBits = 0x4B400000;
constexpr int kChunk = 32;                 // planes the per-pixel phase keeps in registers at once

struct CvArgs {
    const float* key;                    // [B,C,H,W], C = the kernel's channel count NC (3, or 1 for grayscale frames)
    const float* frames[MR_MAX_FRAMES];  // each [B,C,H,W]
    const float* proj;                   // [B,F,12]
    const float* depths;                 // [D]
    void* cv;                            // [B,D,H,W] in the kernel's storage type OUT (fp32 or IEEE half)
    void* sfcv;                          // [F,B,D,H,W], OUT
    void* sf_nhwc;                       // optional [F,B,H,W,D] copy of sfcv for the conv engine (D <= 32, D % 8 == 0) or nullptr
    int sf_nhwc_half;                    // 1: that copy is IEEE half, 0: fp32
    int B, F, D, H, W, TH, b0;
    int use_tma;                         // 0: every unit gathers from global memory
    float alpha, inv_dm1;
    float cw0, cw1, cw2;                 // channel weights / 9
};

struct CvMaps {
    CUtensorMap m[MR_MAX_FRAMES];        // frame f as a (W, H, C B) fp32 tensor, box {kPitch, kBoxRows, 1}, zero fill
};

struct GroupInfo {                       // one window (a run of consecutive planes of one frame)
    short wx0, wy0;                      // image coordinates of the window origin (may be negative: zero ring)
    short nrows;                         // rows actually loaded (multiple of kBoxRows)
    short f;
    short count;                         // planes in the group
    short seq;                           // running number of the window inside the tile (buffer = seq % kBuf)
    short pad0, pad1;
};

struct SmemLayout {
    int win, ytile, cst, xbuf, pjs, zs, vmask, rowrng, bbox, gid, uflag, ginfo, seq2g, nwin, bars, ctr;  // byte offsets
    int zpix, zrow;      // per-pixel depths only: [TH][kTileCols] and [D][TH+4] float2 (min, max) depth tables
    int total;
};

constexpr int kLSlotFloats = 3 * 64;              // kErrSsimL1: a warp's carried L1 terms, three float2 per lane (ssim_row)

// Every channel-dependent size is NC (1 or 3) planes of its one-plane size: the windows, the keyframe tile, the hoisted
// SSIM table and the warped-row buffers.  The geometry (window rows, tile rows) is the same for both channel counts.
// A warp's two warped-row buffers:
__host__ __device__ constexpr int xb_warp_floats(int nc) { return 2 * nc * kRowStride; }

// pix: the per-pixel depth source (cv_depths) appends its two depth tables; the plane layout is unchanged.
// err: the error mode (MR_CV_*).  MR_CV_SSIM_L1 warps keep kLSlotFloats behind their row buffers; MR_CV_BOX_L1 reads no
// hoisted SSIM table, so its cst region is empty.  NC: the frames' channel count (a template parameter: the kernel's
// offsets are then the constant expressions of the three-channel layout, which keeps its code unchanged)
template <int NC>
__host__ __device__ inline SmemLayout make_layout(int D, int TH, int F, int use_tma, bool pix = false, int err = MR_CV_SSIM) {
    SmemLayout L;
    int off = 0;
    auto take = [&](int bytes, int align) { off = (off + align - 1) / align * align; int o = off; off += bytes; return o; };
    L.win = take(use_tma ? kBuf * (NC * kChanStride) * 4 : 0, 128);
    L.ytile = take(NC * (TH + 4) * kRowStride * 4, 16);
    L.cst = take(err == MR_CV_BOX_L1 ? 0 : NC * (TH + 2) * kTileCols * 8, 16);
    L.xbuf = take(kWarps * (xb_warp_floats(NC) + (err == MR_CV_SSIM_L1 ? kLSlotFloats : 0)) * 4, 16);
    L.pjs = take(F * 12 * 4, 16);
    L.zs = take(((D + 3) / 4) * 16, 16);
    L.vmask = take(F * TH * kTileCols, 16);
    L.rowrng = take(F * 2 * 4, 16);
    L.bbox = take(F * D * 8, 8);
    L.gid = take(F * D * 2, 4);
    L.uflag = take(F * D, 4);
    L.ginfo = take(F * D * (int)sizeof(GroupInfo), 16);
    L.seq2g = take(F * D * 2, 4);
    L.nwin = take(MR_MAX_FRAMES * 4, 4);
    L.bars = take(kBuf * 8, 8);
    L.ctr = take((2 + 2 * kBuf) * 4, 4);
    if (pix) {
        L.zpix = take(TH * kTileCols * 8, 16);
        L.zrow = take(D * (TH + 4) * 8, 16);
    } else {
        L.zpix = L.zrow = 0;
    }
    L.total = off;
    return L;
}

// ---- fp32 pairs (a pair is either two columns or two samples of one lane).  sm_90a has no packed fp32x2 arithmetic: the
// march is written per scalar.  Stage 2 uses an explicit fmaf wherever a product feeds an add; stage 1 rounds every sample
// position and weight separately (see bilinear_weights). ---------------------------------------------------------------
__device__ __forceinline__ float2 bc2(float a) { return make_float2(a, a); }

// single MUFU.RCP (flush-to-zero variant: no denormal pre/post-scaling code; operands here are never denormal)
__device__ __forceinline__ float fast_rcp(float x) {
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}

// L2 residency hints: the single-frame volume is written by the march and read back once by the per-pixel phase of the same
// CTA, so its lines are asked to stay (evict_last); the fused volume is written once and never read here (evict_first).
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
    uint64_t p;
    asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
    uint64_t p;
    asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ void st_hint_f2(float* ptr, float2 v, uint64_t pol) {
    asm volatile("st.global.L2::cache_hint.v2.f32 [%0], {%1, %2}, %3;" ::"l"(ptr), "f"(v.x), "f"(v.y), "l"(pol) : "memory");
}
__device__ __forceinline__ void st_hint_f1(float* ptr, float v, uint64_t pol) {
    asm volatile("st.global.L2::cache_hint.f32 [%0], %1, %2;" ::"l"(ptr), "f"(v), "l"(pol) : "memory");
}

// Stores of the volumes in their storage type OUT (float or IEEE half).  Half rounds each fp32 value once, to nearest even
// (__floats2half2_rn rounds both halves exactly like two __float2half_rn).
__device__ __forceinline__ void st_vol2(float* ptr, float2 v, uint64_t pol) { st_hint_f2(ptr, v, pol); }
__device__ __forceinline__ void st_vol1(float* ptr, float v, uint64_t pol) { st_hint_f1(ptr, v, pol); }
__device__ __forceinline__ void st_vol2(__half* ptr, float2 v, uint64_t pol) {
    const __half2 h = __floats2half2_rn(v.x, v.y);
    asm volatile("st.global.L2::cache_hint.b32 [%0], %1, %2;" ::"l"(ptr), "r"(*reinterpret_cast<const uint32_t*>(&h)), "l"(pol)
                 : "memory");
}
__device__ __forceinline__ void st_vol1(__half* ptr, float v, uint64_t pol) {
    asm volatile("st.global.L2::cache_hint.b16 [%0], %1, %2;" ::"l"(ptr), "h"(__half_as_ushort(__float2half_rn(v))), "l"(pol)
                 : "memory");
}
// the per-pixel phase's read-back of one single-frame value (L2 only: written by this CTA's march), widened to fp32
__device__ __forceinline__ float ld_vol(const float* ptr) { return __ldcg(ptr); }
__device__ __forceinline__ float ld_vol(const __half* ptr) { return __half2float(__ldcg(ptr)); }

// ---- mbarrier / TMA wrappers ----------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// Bounded wait: a window that never arrives (a bug, not a load condition) traps instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t done = 0;
    for (uint32_t spin = 0; !done; ++spin) {
        asm volatile(
            "{\n\t"
            ".reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t"
            "}\n"
            : "=r"(done)
            : "r"(bar), "r"(parity)
            : "memory");
        if (spin > (1u << 24)) __trap();
    }
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}

// ---- explicit shared-memory accesses (32-bit shared addresses, immediate offsets) ---------------------------------------
// volatile: never hoisted over the mbarrier wait / __syncwarp that orders them; ptxas still schedules them freely
template <int OFF>
__device__ __forceinline__ float lds32(uint32_t a) {
    float v;
    asm volatile("ld.shared.f32 %0, [%1+%2];" : "=f"(v) : "r"(a), "n"(OFF));
    return v;
}
template <int OFF>
__device__ __forceinline__ float2 lds64(uint32_t a) {
    float2 v;
    asm volatile("ld.shared.v2.f32 {%0, %1}, [%2+%3];" : "=f"(v.x), "=f"(v.y) : "r"(a), "n"(OFF));
    return v;
}
template <int OFF>
__device__ __forceinline__ float4 lds128(uint32_t a) {
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4+%5];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a), "n"(OFF));
    return v;
}
template <int OFF>
__device__ __forceinline__ void sts32(uint32_t a, float v) {
    asm volatile("st.shared.f32 [%0+%1], %2;" ::"r"(a), "n"(OFF), "f"(v) : "memory");
}
template <int OFF>
__device__ __forceinline__ void sts64(uint32_t a, float2 v) {
    asm volatile("st.shared.v2.f32 [%0+%1], {%2, %3};" ::"r"(a), "n"(OFF), "f"(v.x), "f"(v.y) : "memory");
}

// per channel plane (NC of them in each):
constexpr int kXbBytes = kRowStride * 4;          // one warped-row buffer: [channel][kRowStride]
constexpr int kYRowBytes = kRowStride * 4;        // keyframe tile: [row][channel][kRowStride]
constexpr int kCRowBytes = (kTileCols / 2) * 16;  // hoisted table: [e-row][channel][32 column pairs] float4

// ---- stage 1 of the march: homography of one tile row (pair = columns lane, lane + 32) and its 8 NC bilinear taps -----
struct Stage1Ctx {
    float2 pzx, pzy, pzz;                // per-lane column part of the projection (already times the plane depth)
    float rax, rbx, ray, rby, raz, rbz;  // per-row part: c = pz(u) + ra * v + rb
    uint32_t kaddr;                      // window modes: shared address of the window minus the unit's constant (see march)
    const float* img;                    // global mode: source frame of this batch element, [NC][H][W]
    int W, H, planei;
    float sx_lo, sx_hi, sy_lo, sy_hi;    // == grid clamp(-2, 2) + 0.5, monorec_model.py:208
    // per-pixel depths only: the depth changes from sample to sample, so setup_stage1's products are formed per sample
    float2 mu0, mu4, mu8;                // rn(m0 u), rn(m4 u), rn(m8 u) of the lane's two columns
    float m1, m2, m3, m5, m6, m7, m9, m10, m11;
    const float* zp;                     // the unit's depth plane cv_depths[b, d], [H][W]
    int zc0, zc1;                        // the lane's two columns clamped into the image
};

__device__ __forceinline__ void setup_stage1(Stage1Ctx& c, const float* m, float z, float2 fu2) {
    // projection c = M [u v 1]^T z + p split into a per-lane column part and a per-row part
    c.pzx = make_float2(__fmul_rn(m[0] * fu2.x, z), __fmul_rn(m[0] * fu2.y, z));
    c.pzy = make_float2(__fmul_rn(m[4] * fu2.x, z), __fmul_rn(m[4] * fu2.y, z));
    c.pzz = make_float2(__fmul_rn(m[8] * fu2.x, z), __fmul_rn(m[8] * fu2.y, z));
    c.rax = m[1] * z; c.rbx = fmaf(m[2], z, m[3]);
    c.ray = m[5] * z; c.rby = fmaf(m[6], z, m[7]);
    c.raz = m[9] * z; c.rbz = fmaf(m[10], z, m[11]);
}

// The per-pixel counterpart: only the depth-free factors are kept; warp_row_issue<MODE, true> rounds every product of
// setup_stage1 per sample in the same order, so a depth map that repeats one depth per plane gives the plane path's bits.
__device__ __forceinline__ void setup_stage1_pix(Stage1Ctx& c, const float* m, float2 fu2, const float* zp) {
    c.mu0 = make_float2(__fmul_rn(m[0], fu2.x), __fmul_rn(m[0], fu2.y));
    c.mu4 = make_float2(__fmul_rn(m[4], fu2.x), __fmul_rn(m[4], fu2.y));
    c.mu8 = make_float2(__fmul_rn(m[8], fu2.x), __fmul_rn(m[8], fu2.y));
    c.m1 = m[1]; c.m2 = m[2]; c.m3 = m[3];
    c.m5 = m[5]; c.m6 = m[6]; c.m7 = m[7];
    c.m9 = m[9]; c.m10 = m[10]; c.m11 = m[11];
    c.zp = zp;
}

// depth of the lane's two columns in image row v (clamped into the image: halo rows only feed invalid outputs)
__device__ __forceinline__ float2 load_row_depths(const Stage1Ctx& c, const int v) {
    const int o = min(max(v, 0), c.H - 1) * c.W;
    return make_float2(__ldg(c.zp + (o + c.zc0)), __ldg(c.zp + (o + c.zc1)));
}

// Bilinear weights of one sample at u = cx / cz (sample position + 0.5) with tap origin x0f, y0f.  Stage 1 rounds every
// position and weight separately (the _rn intrinsics keep ptxas from contracting them): the SSIM of low-variance windows
// amplifies a last-bit move of the sample position far more than any other rounding of the march.
__device__ __forceinline__ void bilinear_weights(float ux, float uy, float x0f, float y0f, float& w00, float& w01, float& w10,
                                                 float& w11) {
    const float wx1 = __fadd_rn(__fadd_rn(ux, -0.5f), -x0f), wy1 = __fadd_rn(__fadd_rn(uy, -0.5f), -y0f);
    const float wx0 = __fadd_rn(1.0f, -wx1), wy0 = __fadd_rn(1.0f, -wy1);
    w00 = __fmul_rn(wx0, wy0); w01 = __fmul_rn(wx1, wy0); w10 = __fmul_rn(wx0, wy1); w11 = __fmul_rn(wx1, wy1);
}

template <int NC>
struct Taps {                            // the 8 NC taps and 4 weight pairs of one row step (two samples per lane)
    float a[NC][4], b[NC][4];            // [channel][nw, ne, sw, se] of the sample at column lane / lane + 32
    float2 w00, w01, w10, w11;
};

// MODE 0: taps from the window, every sample of the unit strictly inside the image (decided by the plan): no clamps
// MODE 1: taps from the window, coordinates clamped to the 2-px zero ring (== zero padding of F.grid_sample)
// MODE 2: taps from global memory with per-tap zero padding
// PIX: z = the depths of the lane's two samples in this row (per-pixel depth source); unused for the plane table
// NC: channels of the frames.  The weights do not depend on the channel, so a one-channel frame's taps are those of each
// plane of its three-channel replica.
template <int MODE, bool PIX, int NC>
__device__ __forceinline__ void warp_row_issue(const Stage1Ctx& c, const float fv, Taps<NC>& t, const float2 z = float2{}) {
    float inv[2], ux[2], uy[2];
    if constexpr (!PIX) {
        const float rcx = fmaf(c.rax, fv, c.rbx), rcy = fmaf(c.ray, fv, c.rby), rcz = fmaf(c.raz, fv, c.rbz);
        inv[0] = fast_rcp(__fadd_rn(c.pzz.x, rcz)); inv[1] = fast_rcp(__fadd_rn(c.pzz.y, rcz));
        // sample position + 0.5
        ux[0] = __fmul_rn(__fadd_rn(c.pzx.x, rcx), inv[0]); ux[1] = __fmul_rn(__fadd_rn(c.pzx.y, rcx), inv[1]);
        uy[0] = __fmul_rn(__fadd_rn(c.pzy.x, rcy), inv[0]); uy[1] = __fmul_rn(__fadd_rn(c.pzy.y, rcy), inv[1]);
    } else {
        // setup_stage1 and the row part above, per sample: rn(rn(m0 u) z) + fma(rn(m1 z), v, fma(m2, z, m3)), ...
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            const float zk = k ? z.y : z.x;
            const float rcx = fmaf(__fmul_rn(c.m1, zk), fv, fmaf(c.m2, zk, c.m3));
            const float rcy = fmaf(__fmul_rn(c.m5, zk), fv, fmaf(c.m6, zk, c.m7));
            const float rcz = fmaf(__fmul_rn(c.m9, zk), fv, fmaf(c.m10, zk, c.m11));
            inv[k] = fast_rcp(__fadd_rn(__fmul_rn(k ? c.mu8.y : c.mu8.x, zk), rcz));
            ux[k] = __fmul_rn(__fadd_rn(__fmul_rn(k ? c.mu0.y : c.mu0.x, zk), rcx), inv[k]);
            uy[k] = __fmul_rn(__fadd_rn(__fmul_rn(k ? c.mu4.y : c.mu4.x, zk), rcy), inv[k]);
        }
    }
    // floor by magic-number rounding: rn(s - 0.5) differs from floor(s) only for integral s, where the interpolated value
    // is the same (weight 1 on the tap both conventions share)
    float tx[2], ty[2];
#pragma unroll
    for (int k = 0; k < 2; ++k) {
        if (MODE == 1) {   // == .clamp(-2, 2) of the normalised grid (monorec_model.py:208); also maps NaN to the low bound
            ux[k] = fminf(fmaxf(ux[k], c.sx_lo), c.sx_hi); uy[k] = fminf(fmaxf(uy[k], c.sy_lo), c.sy_hi);
        }
        tx[k] = __fadd_rn(ux[k], kMagic - 1.0f); ty[k] = __fadd_rn(uy[k], kMagic - 1.0f);
    }
    if (MODE <= 1) {
        bilinear_weights(ux[0], uy[0], tx[0] - kMagic, ty[0] - kMagic, t.w00.x, t.w01.x, t.w10.x, t.w11.x);
        bilinear_weights(ux[1], uy[1], tx[1] - kMagic, ty[1] - kMagic, t.w00.y, t.w01.y, t.w10.y, t.w11.y);
        uint32_t aa, ab;
        if (MODE == 0) {
            // address = window + 4 ((y0 - wy0) kPitch + x0 - wx0) with y0 = bits(ty) - kMagicBits: every constant is in kaddr
            aa = ((((uint32_t)__float_as_int(ty[0]) << 7) + (uint32_t)__float_as_int(tx[0])) << 2) + c.kaddr;
            ab = ((((uint32_t)__float_as_int(ty[1]) << 7) + (uint32_t)__float_as_int(tx[1])) << 2) + c.kaddr;
        } else {
            // integer tap origin clamped to [-2, W] x [-2, H]: taps of the ring [-2,-1] / [W, W+1] are zero-filled by TMA
            const int xa = min(max(__float_as_int(tx[0]) - kMagicBits, -2), c.W);
            const int xb = min(max(__float_as_int(tx[1]) - kMagicBits, -2), c.W);
            const int ya = min(max(__float_as_int(ty[0]) - kMagicBits, -2), c.H);
            const int yb = min(max(__float_as_int(ty[1]) - kMagicBits, -2), c.H);
            aa = ((((uint32_t)ya << 7) + (uint32_t)xa) << 2) + c.kaddr;
            ab = ((((uint32_t)yb << 7) + (uint32_t)xb) << 2) + c.kaddr;
        }
        static_assert(kPitch == 128, "the tap address uses a shift by 7");
#pragma unroll
        for (int ch = 0; ch < NC; ++ch) {
            // (ch is a compile-time constant after unrolling: the offsets are immediates)
            if (ch == 0) {
                t.a[0][0] = lds32<0>(aa); t.a[0][1] = lds32<4>(aa); t.a[0][2] = lds32<kPitch * 4>(aa); t.a[0][3] = lds32<kPitch * 4 + 4>(aa);
                t.b[0][0] = lds32<0>(ab); t.b[0][1] = lds32<4>(ab); t.b[0][2] = lds32<kPitch * 4>(ab); t.b[0][3] = lds32<kPitch * 4 + 4>(ab);
            } else if (ch == 1) {
                constexpr int o = kChanStride * 4;
                t.a[1][0] = lds32<o>(aa); t.a[1][1] = lds32<o + 4>(aa); t.a[1][2] = lds32<o + kPitch * 4>(aa); t.a[1][3] = lds32<o + kPitch * 4 + 4>(aa);
                t.b[1][0] = lds32<o>(ab); t.b[1][1] = lds32<o + 4>(ab); t.b[1][2] = lds32<o + kPitch * 4>(ab); t.b[1][3] = lds32<o + kPitch * 4 + 4>(ab);
            } else {
                constexpr int o = 2 * kChanStride * 4;
                t.a[2][0] = lds32<o>(aa); t.a[2][1] = lds32<o + 4>(aa); t.a[2][2] = lds32<o + kPitch * 4>(aa); t.a[2][3] = lds32<o + kPitch * 4 + 4>(aa);
                t.b[2][0] = lds32<o>(ab); t.b[2][1] = lds32<o + 4>(ab); t.b[2][2] = lds32<o + kPitch * 4>(ab); t.b[2][3] = lds32<o + kPitch * 4 + 4>(ab);
            }
        }
    } else {
        const int W = c.W, H = c.H;
        const int x0a = __float_as_int(tx[0]) - kMagicBits, x0b = __float_as_int(tx[1]) - kMagicBits;
        const int y0a = __float_as_int(ty[0]) - kMagicBits, y0b = __float_as_int(ty[1]) - kMagicBits;
        const bool inb = ((unsigned)x0a <= (unsigned)(W - 2)) && ((unsigned)x0b <= (unsigned)(W - 2)) &&
                         ((unsigned)y0a <= (unsigned)(H - 2)) && ((unsigned)y0b <= (unsigned)(H - 2));
        int oa, ob, dxa, dxb, dya, dyb;
        if (__all_sync(0xffffffffu, inb)) {
            bilinear_weights(ux[0], uy[0], tx[0] - kMagic, ty[0] - kMagic, t.w00.x, t.w01.x, t.w10.x, t.w11.x);
            bilinear_weights(ux[1], uy[1], tx[1] - kMagic, ty[1] - kMagic, t.w00.y, t.w01.y, t.w10.y, t.w11.y);
            oa = y0a * W + x0a; ob = y0b * W + x0b;
            dxa = dxb = 1; dya = dyb = W;
        } else {
            // border path: per-tap zero padding exactly like F.grid_sample(padding_mode="zeros"): clamp the tap address, zero
            // the weight of every tap that falls outside the image
            float wx0s[2], wx1s[2], wy0s[2], wy1s[2];
            int os[2], dxs[2], dys[2];
#pragma unroll
            for (int k = 0; k < 2; ++k) {
                const float sxk = fminf(fmaxf(ux[k], c.sx_lo), c.sx_hi) - 0.5f;
                const float syk = fminf(fmaxf(uy[k], c.sy_lo), c.sy_hi) - 0.5f;
                const float x0f = floorf(sxk), y0f = floorf(syk);
                float wx1 = sxk - x0f, wy1 = syk - y0f;
                float wx0 = (x0f + 1.0f) - sxk, wy0 = (y0f + 1.0f) - syk;
                const int x0 = (int)x0f, y0 = (int)y0f;
                if ((unsigned)x0 >= (unsigned)W) wx0 = 0.f;
                if ((unsigned)(x0 + 1) >= (unsigned)W) wx1 = 0.f;
                if ((unsigned)y0 >= (unsigned)H) wy0 = 0.f;
                if ((unsigned)(y0 + 1) >= (unsigned)H) wy1 = 0.f;
                const int xa = min(max(x0, 0), W - 1), xb = min(max(x0 + 1, 0), W - 1);
                const int ya = min(max(y0, 0), H - 1), yb = min(max(y0 + 1, 0), H - 1);
                wx0s[k] = wx0; wx1s[k] = wx1; wy0s[k] = wy0; wy1s[k] = wy1;
                os[k] = ya * W + xa; dxs[k] = xb - xa; dys[k] = (yb - ya) * W;
            }
            t.w00 = make_float2(wx0s[0] * wy0s[0], wx0s[1] * wy0s[1]); t.w01 = make_float2(wx1s[0] * wy0s[0], wx1s[1] * wy0s[1]);
            t.w10 = make_float2(wx0s[0] * wy1s[0], wx0s[1] * wy1s[1]); t.w11 = make_float2(wx1s[0] * wy1s[0], wx1s[1] * wy1s[1]);
            oa = os[0]; ob = os[1]; dxa = dxs[0]; dxb = dxs[1]; dya = dys[0]; dyb = dys[1];
        }
#pragma unroll
        for (int ch = 0; ch < NC; ++ch) {
            const float* pa0 = c.img + (oa + ch * c.planei);
            const float* pb0 = c.img + (ob + ch * c.planei);
            t.a[ch][0] = __ldg(pa0); t.a[ch][1] = __ldg(pa0 + dxa); t.a[ch][2] = __ldg(pa0 + dya); t.a[ch][3] = __ldg(pa0 + dya + dxa);
            t.b[ch][0] = __ldg(pb0); t.b[ch][1] = __ldg(pb0 + dxb); t.b[ch][2] = __ldg(pb0 + dyb); t.b[ch][3] = __ldg(pb0 + dyb + dxb);
        }
    }
}

// interpolation (same order as grid_sample: nw, ne, sw, se; + 0.5: monorec_model.py:231) and the warped row -> row buffer
// xw = shared address of this lane's first column in the row buffer to fill
template <int NC>
__device__ __forceinline__ void warp_row_finish(const Taps<NC>& t, const uint32_t xw) {
    float va[NC], vb[NC];
#pragma unroll
    for (int ch = 0; ch < NC; ++ch) {
        float a = fmaf(t.a[ch][0], t.w00.x, 0.5f), b = fmaf(t.b[ch][0], t.w00.y, 0.5f);
        a = fmaf(t.a[ch][1], t.w01.x, a); b = fmaf(t.b[ch][1], t.w01.y, b);
        a = fmaf(t.a[ch][2], t.w10.x, a); b = fmaf(t.b[ch][2], t.w10.y, b);
        a = fmaf(t.a[ch][3], t.w11.x, a); b = fmaf(t.b[ch][3], t.w11.y, b);
        va[ch] = a; vb[ch] = b;
    }
    sts32<0>(xw, va[0]);                  sts32<128>(xw, vb[0]);
    if constexpr (NC == 3) {
        sts32<kRowStride * 4>(xw, va[1]);     sts32<kRowStride * 4 + 128>(xw, vb[1]);
        sts32<2 * kRowStride * 4>(xw, va[2]); sts32<2 * kRowStride * 4 + 128>(xw, vb[2]);
    }
}

// ---- stage 2 of the march: SSIM + patch cost of one row; lane owns buffer columns 2l, 2l+1 (a pair) ---------------------
// Error modes: the per-pixel, per-channel difference that the 3x3 patch cost sums (monorec_model.py:227-243, chosen by
// use_ssim; the values are the C ABI's MR_CV_*).  All three have the footprint of a 3x3 box around the pixel, so the tile,
// its 2-px ring and the validity rule are the same for every mode.
constexpr int kErrSsim = MR_CV_SSIM;      // SSIM error of w + .5, k + .5 (layers.py:119-137)
constexpr int kErrSsimL1 = MR_CV_SSIM_L1; // 0.85 SSIM + 0.15 |w - k|
constexpr int kErrBoxL1 = MR_CV_BOX_L1;   // avg_pool2d(|w - k|, 3, 1, padding=1): the 3x3 box sum of |w - k| / 9

struct Stage2Ctx {
    float2 cw0, cw1, cw2;    // channel weights / 9 (kErrBoxL1: times 1/9, the box average)
    int pairflag;            // 1: both columns of this lane are output pixels and W is even (one 8-byte store)
    bool st0, st1;           // otherwise: column 2l / 2l+1 is an output pixel (one 4-byte store each)
    uint64_t pol_keep;
};

// rolling state: horizontal 3-sums of X, X^2, XY per channel for the last rows, indexed by (row step mod 3) so that no
// register moves are needed.  kErrBoxL1 keeps horizontal 3-sums of |X - Y| instead.  [row slot][channel]
template <int ERR, int NC>
struct Stage2State {
    float2 hs1[3][NC], hsx[3][NC], hsy[3][NC], hE[3];
    __device__ __forceinline__ void clear() {
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            hE[i] = bc2(0.f);
#pragma unroll
            for (int c = 0; c < NC; ++c) hs1[i][c] = hsx[i][c] = hsy[i][c] = bc2(0.f);
        }
    }
};
template <int NC>
struct Stage2State<kErrBoxL1, NC> {
    float2 hd[3][NC], hE[3];
    __device__ __forceinline__ void clear() {
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            hE[i] = bc2(0.f);
#pragma unroll
            for (int c = 0; c < NC; ++c) hd[i][c] = bc2(0.f);
        }
    }
};

// The channel whose error enters the channel-weighted sum with weight k (k = 0, 1, 2).  A one-channel frame stands for
// three equal planes: its error enters with all three weights, in the three-channel sum's own expression
// fmaf(w2, e, fmaf(w1, e, w0 * e)), so its cost is the replicated frame's bit for bit.
template <int NC>
__host__ __device__ constexpr int wchan(int k) { return NC == 1 ? 0 : k; }

// Patch cost of one row step, common to every error mode: E is the channel-weighted error of the lane's two columns in the
// row whose error was just finished; its horizontal 3-sum joins the two rows before it in hE (rolling like Stage2State).
template <int P, typename OUT>
__device__ __forceinline__ void patch_cost_row(float2 (&hE)[3], const Stage2Ctx& c, const float2 E, OUT* out,
                                               const bool store) {
    constexpr int P1 = (P + 1) % 3, P2 = (P + 2) % 3;
    const float eL = __shfl_up_sync(0xffffffffu, E.y, 1);
    const float eR = __shfl_down_sync(0xffffffffu, E.x, 1);
    const float mid = E.x + E.y;
    const float2 hEc = make_float2(eL + mid, mid + eR);
    // single-frame volume 1 - 2 sad (monorec_model.py:251) straight to HBM; the validity mask is applied by the
    // per-pixel phase (which zeroes invalid pixels) once all planes are known
    const float2 sv = make_float2(fmaf(-2.0f, (hE[P1].x + hE[P2].x) + hEc.x, 1.0f),
                                  fmaf(-2.0f, (hE[P1].y + hE[P2].y) + hEc.y, 1.0f));
    // predicated stores (no divergent branch in the row loop): the lane's pair as one 8-byte (half: 4-byte) store, or its
    // single column
    if (store && c.pairflag) st_vol2(out, sv, c.pol_keep);
    if (store && c.st0) st_vol1(out, sv.x, c.pol_keep);
    if (store && c.st1) st_vol1(out + 1, sv.y, c.pol_keep);
    hE[P] = hEc;
}

// One row step: horizontal sums of the new warped row, SSIM error of the row above it (windows complete from the third
// row of a unit on; earlier rows produce finite throw-away values from the zeroed state: 9 sxx >= s^2 for partial
// windows too), patch cost of the row above that.  `store` is warp-uniform (false for the first four rows of a unit).
//   xr: shared address of the warped row (this lane's columns 2l-1..2l+2); yr: keyframe tile row (+0.5), same columns;
//   cr: hoisted (Y, Y, Sg, Sg) table row of the SSIM row; out: single-frame volume, output row of this step.
// ERR: kErrSsim or kErrSsimL1 (kErrBoxL1 is box_l1_row below).  The row buffer and the keyframe tile both hold values
// + 0.5, so the |X - Y| of kErrSsimL1 and kErrBoxL1 is |(w + .5) - (k + .5)|: it differs from the reference's |w - k| by the
// rounding of the two additions (of order 1e-7).
template <int P, int ERR, int NC, typename OUT>
__device__ __forceinline__ void ssim_row(Stage2State<ERR, NC>& st, const Stage2Ctx& c, const uint32_t xr, const uint32_t yr,
                                         const uint32_t cr, OUT* out, const bool store, const uint32_t xb) {
    constexpr int P1 = (P + 1) % 3, P2 = (P + 2) % 3;
    float2 xl[NC], xrr[NC], yl[NC], yrr[NC];
    float4 k4[NC];
    xl[0] = lds64<0>(xr);                  xrr[0] = lds64<8>(xr);
    if constexpr (NC == 3) {
        xl[1] = lds64<kRowStride * 4>(xr);     xrr[1] = lds64<kRowStride * 4 + 8>(xr);
        xl[2] = lds64<2 * kRowStride * 4>(xr); xrr[2] = lds64<2 * kRowStride * 4 + 8>(xr);
    }
    yl[0] = lds64<0>(yr);                  yrr[0] = lds64<8>(yr);
    if constexpr (NC == 3) {
        yl[1] = lds64<kRowStride * 4>(yr);     yrr[1] = lds64<kRowStride * 4 + 8>(yr);
        yl[2] = lds64<2 * kRowStride * 4>(yr); yrr[2] = lds64<2 * kRowStride * 4 + 8>(yr);
        k4[0] = lds128<0>(cr); k4[1] = lds128<512>(cr); k4[2] = lds128<1024>(cr);
    } else {
        k4[0] = lds128<0>(cr);
    }
    // horizontal 3-sums of X, X^2, XY: the middle pair (columns 2l, 2l+1) is shared by both columns of the lane, and every
    // product is folded into an FFMA of its sum
    float2 h1[NC], hx[NC], hy[NC];
    float2 L;   // kErrSsimL1: sum_c w_c |X - Y|_c of columns 2l, 2l+1, formed channel by channel while their values are loaded
#pragma unroll
    for (int ch = 0; ch < NC; ++ch) {
        const float2 l = xl[ch], r = xrr[ch], ly = yl[ch], ry = yrr[ch];
        const float m1 = l.y + r.x, mx = fmaf(l.y, l.y, r.x * r.x), my = fmaf(l.y, ly.y, r.x * ry.x);
        h1[ch] = make_float2(l.x + m1, m1 + r.y);
        hx[ch] = make_float2(fmaf(l.x, l.x, mx), fmaf(r.y, r.y, mx));
        hy[ch] = make_float2(fmaf(l.x, ly.x, my), fmaf(r.y, ry.y, my));
        if constexpr (ERR == kErrSsimL1) {
            const float2 d = make_float2(fabsf(l.y - ly.y), fabsf(r.x - ry.x));
            // (one channel: its difference enters with all three weights, see wchan)
#pragma unroll
            for (int k = ch; k < (NC == 1 ? 3 : ch + 1); ++k) {
                const float2 w = k == 0 ? c.cw0 : k == 1 ? c.cw1 : c.cw2;
                L = k == 0 ? make_float2(w.x * d.x, w.y * d.y) : make_float2(fmaf(w.x, d.x, L.x), fmaf(w.y, d.y, L.y));
            }
        }
    }
    if constexpr (ERR == kErrSsimL1) {
        // kErrSsimL1: the row's 0.15 L waits one step in the lane's shared memory slot P behind the warp's row buffers,
        // until this row's SSIM is finished.  (Carried in registers, or in one slot that is read before it is rewritten,
        // it pushed the per-pixel gather march into local memory.)
        sts64<2 * NC * kXbBytes + 256 * P>(xb, make_float2(0.15f * L.x, 0.15f * L.y));
    }
    float e[NC][2];
#pragma unroll
    for (int ch = 0; ch < NC; ++ch) {
        // SSIM with every factor scaled by 81 (layers.py:123-137 through 3x3 box sums s = sum x, sxx, sxy; Y = 9 mu_y,
        // Sg = 81 (sigma_y + C2) hoisted):  n/d = (2 s Y + 81 C1)(2 (9 sxy - s Y) + 81 C2) / ((s^2 + Y^2 + 81 C1)(9 sxx - s^2 + Sg))
        const float Y[2] = {k4[ch].x, k4[ch].y}, Sg[2] = {k4[ch].z, k4[ch].w};
        const float h1c[2] = {h1[ch].x, h1[ch].y}, hxc[2] = {hx[ch].x, hx[ch].y}, hyc[2] = {hy[ch].x, hy[ch].y};
        const float a1[2] = {st.hs1[P1][ch].x, st.hs1[P1][ch].y}, b1[2] = {st.hs1[P2][ch].x, st.hs1[P2][ch].y};
        const float ax[2] = {st.hsx[P1][ch].x, st.hsx[P1][ch].y}, bx[2] = {st.hsx[P2][ch].x, st.hsx[P2][ch].y};
        const float ay[2] = {st.hsy[P1][ch].x, st.hsy[P1][ch].y}, by[2] = {st.hsy[P2][ch].x, st.hsy[P2][ch].y};
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            const float s = (a1[k] + b1[k]) + h1c[k], sxx = (ax[k] + bx[k]) + hxc[k], sxy = (ay[k] + by[k]) + hyc[k];
            const float p = s * Y[k];
            const float n1h = -p - 40.5f * kC1;                                // -(N1 / 2)
            const float n2 = fmaf(2.0f, fmaf(9.0f, sxy, -p), 81.0f * kC2);
            const float d1 = fmaf(s, s, fmaf(Y[k], Y[k], 81.0f * kC1));        // s^2 + Y^2 + 81 C1
            const float d2 = fmaf(-s, s, fmaf(9.0f, sxx, Sg[k]));              // 9 sxx - s^2 + Sg
            // clamp((1 - n/d) / 2, 0, 1)   (layers.py:137)
            e[ch][k] = __saturatef(fmaf(n1h * n2, fast_rcp(d1 * d2), 0.5f));
        }
    }
    float2 E;
    constexpr int c1 = wchan<NC>(1), c2 = wchan<NC>(2);
    if constexpr (ERR == kErrSsimL1) {
        // 0.85 SSIM + 0.15 |X - Y| per channel (monorec_model.py:237-241), channel-weighted as sums of their own; the L1
        // sum of the SSIM row is the one the previous step stored
        const float2 Lp = lds64<2 * NC * kXbBytes + 256 * P2>(xb);
        E = make_float2(fmaf(0.85f, fmaf(c.cw2.x, e[c2][0], fmaf(c.cw1.x, e[c1][0], c.cw0.x * e[0][0])), Lp.x),
                        fmaf(0.85f, fmaf(c.cw2.y, e[c2][1], fmaf(c.cw1.y, e[c1][1], c.cw0.y * e[0][1])), Lp.y));
    } else {
        E = make_float2(fmaf(c.cw2.x, e[c2][0], fmaf(c.cw1.x, e[c1][0], c.cw0.x * e[0][0])),
                        fmaf(c.cw2.y, e[c2][1], fmaf(c.cw1.y, e[c1][1], c.cw0.y * e[0][1])));
    }
    patch_cost_row<P>(st.hE, c, E, out, store);
#pragma unroll
    for (int ch = 0; ch < NC; ++ch) { st.hs1[P][ch] = h1[ch]; st.hsx[P][ch] = hx[ch]; st.hsy[P][ch] = hy[ch]; }
}

// kErrBoxL1: horizontal 3-sums of |X - Y| of the new row, their vertical 3-sum over the rolling rows (the 3x3 box of the
// row above, at the step where the SSIM modes finish that row's SSIM), patch cost of the row above that
template <int P, int NC, typename OUT>
__device__ __forceinline__ void box_l1_row(Stage2State<kErrBoxL1, NC>& st, const Stage2Ctx& c, const uint32_t xr,
                                           const uint32_t yr, OUT* out, const bool store) {
    constexpr int P1 = (P + 1) % 3, P2 = (P + 2) % 3;
    float2 xl[NC], xrr[NC], yl[NC], yrr[NC];
    xl[0] = lds64<0>(xr);                  xrr[0] = lds64<8>(xr);
    if constexpr (NC == 3) {
        xl[1] = lds64<kRowStride * 4>(xr);     xrr[1] = lds64<kRowStride * 4 + 8>(xr);
        xl[2] = lds64<2 * kRowStride * 4>(xr); xrr[2] = lds64<2 * kRowStride * 4 + 8>(xr);
    }
    yl[0] = lds64<0>(yr);                  yrr[0] = lds64<8>(yr);
    if constexpr (NC == 3) {
        yl[1] = lds64<kRowStride * 4>(yr);     yrr[1] = lds64<kRowStride * 4 + 8>(yr);
        yl[2] = lds64<2 * kRowStride * 4>(yr); yrr[2] = lds64<2 * kRowStride * 4 + 8>(yr);
    }
    float2 hd[NC], v[NC];
#pragma unroll
    for (int ch = 0; ch < NC; ++ch) {
        const float2 l = xl[ch], r = xrr[ch], ly = yl[ch], ry = yrr[ch];
        const float m = fabsf(l.y - ly.y) + fabsf(r.x - ry.x);
        hd[ch] = make_float2(fabsf(l.x - ly.x) + m, m + fabsf(r.y - ry.y));
        v[ch] = make_float2((st.hd[P1][ch].x + st.hd[P2][ch].x) + hd[ch].x, (st.hd[P1][ch].y + st.hd[P2][ch].y) + hd[ch].y);
    }
    // (the box's 1/9 is folded into the channel weights)
    constexpr int c1 = wchan<NC>(1), c2 = wchan<NC>(2);
    const float2 E = make_float2(fmaf(c.cw2.x, v[c2].x, fmaf(c.cw1.x, v[c1].x, c.cw0.x * v[0].x)),
                                 fmaf(c.cw2.y, v[c2].y, fmaf(c.cw1.y, v[c1].y, c.cw0.y * v[0].y)));
    patch_cost_row<P>(st.hE, c, E, out, store);
#pragma unroll
    for (int ch = 0; ch < NC; ++ch) st.hd[P][ch] = hd[ch];
}

// xb: the lane's address in the warp's first row buffer (xr without the buffer toggle)
template <int P, int ERR, int NC, typename OUT>
__device__ __forceinline__ void stage2_row(Stage2State<ERR, NC>& st, const Stage2Ctx& c, const uint32_t xr, const uint32_t yr,
                                           const uint32_t cr, OUT* out, const bool store, const uint32_t xb) {
    if constexpr (ERR == kErrBoxL1) box_l1_row<P>(st, c, xr, yr, out, store);
    else ssim_row<P, ERR>(st, c, xr, yr, cr, out, store, xb);
}

// The march of one unit over tile rows rlo-2 .. rhi+2 (nsteps = rhi - rlo + 5 >= 5 rows).  Stage 1 of the next row is
// issued with stage 2 of the current one; the three-step loop body is entered at the slot that makes the last step end
// a triple (the rolling state is symmetric under rotation of its slots).
//   xb: shared address of this warp's two row buffers; yr / cr: keyframe row rlo-2 / table row rlo-2 (lane columns);
//   out: single-frame volume at output row rlo - 4 (advanced every step, stored from the fifth step on); wstride = W
//   PIX: per-pixel depths, read from image row v0 (= fv0) on; each row's depths are loaded one row step before they are used
//   ERR: the error mode of stage 2; NC: the channels of the frames; OUT: the storage type of the single-frame volume
template <int MODE, bool PIX, int ERR, int NC, typename OUT>
__device__ __forceinline__ void march_unit(const Stage1Ctx& c1, const Stage2Ctx& c2, const uint32_t xb, const int lane,
                                           const float fv0, const int nsteps, uint32_t yr, uint32_t cr, OUT* out,
                                           const int wstride, const int v0 = 0) {
    constexpr uint32_t kXb = NC * kXbBytes;   // one warped-row buffer
    Stage2State<ERR, NC> st;
    st.clear();
    if constexpr (ERR == kErrSsimL1) {   // the L1 slots start at 0 like st
        sts64<2 * kXb>(xb + 8 * lane, bc2(0.f));
        sts64<2 * kXb + 256>(xb + 8 * lane, bc2(0.f));
        sts64<2 * kXb + 512>(xb + 8 * lane, bc2(0.f));
    }
    float fv = fv0;
    uint32_t off = 0;                      // byte offset of the row buffer stage 2 reads next
    const uint32_t xw = xb + 4 * (lane + 1), xr = xb + 8 * lane;
    int zv = v0 + 1;                       // PIX: image row of the depths in flight (zn)
    float2 zn{};
    if constexpr (PIX) zn = load_row_depths(c1, v0);
    {
        Taps<NC> t;
        if constexpr (PIX) {
            const float2 zc = zn;
            zn = load_row_depths(c1, zv);
            warp_row_issue<MODE, true>(c1, fv, t, zc);
        } else {
            warp_row_issue<MODE, false>(c1, fv, t);
        }
        warp_row_finish(t, xw);
    }
    __syncwarp();
    const int n = nsteps - 1;              // steps that also run stage 1 of the following row
    int t = -((3 - n % 3) % 3);
    int done = 0;                          // rows stage 2 has consumed
    auto both = [&](auto tag) {
        fv += 1.0f;
        Taps<NC> tp;
        if constexpr (PIX) {
            const float2 zc = zn;
            zn = load_row_depths(c1, ++zv);
            warp_row_issue<MODE, true>(c1, fv, tp, zc);
        } else {
            warp_row_issue<MODE, false>(c1, fv, tp);
        }
        // stage 1 of row t+1 completes before stage 2 of row t: measured faster than keeping the taps in flight across
        // stage 2 (1.07 against 1.12 ms)
        warp_row_finish(tp, xw + (kXb - off));
        stage2_row<decltype(tag)::value, ERR>(st, c2, xr + off, yr, cr, out, done >= 4, xr);
        __syncwarp();
        off = kXb - off;
        yr += NC * kYRowBytes;
        cr += NC * kCRowBytes;
        // (kErrSsimL1: the stride as an unsigned step, whose high word is the constant 0: the signed step's high word held a
        // register across the loop, and the per-pixel gather march spilled it)
        if constexpr (ERR == kErrSsimL1) out += (size_t)(uint32_t)wstride;
        else out += wstride;
        ++done;
    };
    using I0 = std::integral_constant<int, 0>;
    using I1 = std::integral_constant<int, 1>;
    using I2 = std::integral_constant<int, 2>;
    for (; t < n; t += 3) {
        if (t >= 0) both(I0{});
        if (t + 1 >= 0) both(I1{});
        both(I2{});
    }
    stage2_row<0, ERR>(st, c2, xr + off, yr, cr, out, true, xr);
    __syncwarp();
}

// ---- per-pixel phase: view weights (monorec_model.py:257-260), zeroing of invalid pixels (:251) and fusion
//      cv = sum_f w_f (1 - 2 sad_f) / sum_f w_f, 0 where sum_f w_f == 0 (:262-269).  T lanes share a pixel, each with a chunk of
//      kChunk planes in registers (T = 1 for D <= 32, 2 for D <= 64, 4 for D <= 128): every (L2-hot) single-frame value is
//      read back exactly once; max / sum over the planes are combined across the T lanes by shuffles.
//      CENTER = false (not_center_cv, :267-269) stores the fused sad sum_f w_f sad_f / sum_f w_f = (1 - cv) / 2 instead,
//      still 0 where sum_f w_f == 0.
//      OUT = __half: the single-frame values are read back as half and widened; weights, fusion and centring stay fp32 and
//      only the store of the fused volume rounds to half.
struct PixelPhase {
    void* cv;                            // OUT [B,D,H,W]
    void* sfcv;                          // OUT [F,B,D,H,W]
    void* sf_nhwc;
    int sf_nhwc_half;
    const unsigned char* vmask;
    int B, F, D, H, W, TH, b, u0, v0;
    float inv_dm1, kq;
    uint64_t pol_stream;
};

template <int T, bool CENTER, typename OUT>
__device__ __forceinline__ void pixel_phase(const PixelPhase& c) {
    constexpr int kSlots = 32 / T;                       // pixels per warp iteration
    // the thread index is read again here (volatile: not merged with the kernel's own read) instead of being kept live in a
    // register across the march, where ptxas spilled it and reloaded it on every pixel iteration
    int tid;
    asm volatile("mov.u32 %0, %%tid.x;" : "=r"(tid));
    const int lane = tid & 31, warp = tid >> 5;
    const int sub = lane % kSlots, chunk = lane / kSlots;
    const int D = c.D, F = c.F, TH = c.TH;
    const int d_lo = chunk * kChunk;                     // this lane's planes [d_lo, d_lo + kChunk) of D
    const size_t plane = (size_t)c.H * c.W;
    const size_t pstride = plane * sizeof(OUT);          // bytes between the planes of a pixel
    const size_t fstride = (size_t)c.B * D * pstride;    // bytes between the frames
    const int vstride = TH * kTileCols;
    const int per_iter = kWarps * kSlots;
    for (int p0 = 0; p0 < TH * kTileCols; p0 += per_iter) {
        const int p = p0 + warp * kSlots + sub;
        const int r = p >> 6, bc = p & 63;
        const int u = c.u0 + bc, v = c.v0 + r;
        const bool own = (p < TH * kTileCols) && (bc >= 2) && (bc < 2 + kOutCols) && (u < c.W) && (v < c.H);
        if (T == 1 && !own) continue;                    // (with T > 1 every lane stays for the shuffles)
        const size_t pix = own ? (size_t)v * c.W + u : 0;
        // addresses advance by pointer increments (one 64-bit add per access; an index expression costs a wide multiply each)
        char* cv_out = reinterpret_cast<char*>(static_cast<OUT*>(c.cv) + ((size_t)c.b * D + d_lo) * plane + pix);
        char* sf = reinterpret_cast<char*>(static_cast<OUT*>(c.sfcv) + ((size_t)c.b * D + d_lo) * plane + pix);  // frame f: + f * fstride
        float acc[kChunk], vv[kChunk], nv[kChunk];
#pragma unroll
        for (int j = 0; j < kChunk; ++j) acc[j] = 0.f;
        float wsum = 0.f;
        // this lane's planes of frame f -> nv (-2 for planes >= D and invalid pixels).  With T == 1 the loads of frame f + 1
        // are issued before frame f is reduced, so one frame's memory round trip overlaps the arithmetic of the previous one
        auto fetch = [&](const int f, const char* q) {
            if (own && (c.vmask[f * vstride + p] != 0)) {
                if (D == T * kChunk) {                   // 32 / 64 / 128 planes: no per-plane predicates
#pragma unroll
                    for (int j = 0; j < kChunk; ++j, q += pstride) nv[j] = ld_vol(reinterpret_cast<const OUT*>(q));
                } else {
#pragma unroll
                    for (int j = 0; j < kChunk; ++j, q += pstride) nv[j] = (d_lo + j < D) ? ld_vol(reinterpret_cast<const OUT*>(q)) : -2.0f;
                }
            } else {
#pragma unroll
                for (int j = 0; j < kChunk; ++j) nv[j] = -2.0f;
            }
        };
        // (T == 1 only: with T > 1 a lane's chunk is a quarter or half of the pixel's planes, and a second chunk of registers
        // would spill)
        if (T == 1) fetch(0, sf);
        for (int f = 0; f < F; ++f, sf += fstride) {
            const bool valid = own && (c.vmask[f * vstride + p] != 0);
            if (T > 1) fetch(f, sf);
#pragma unroll
            for (int j = 0; j < kChunk; ++j) vv[j] = nv[j];
            if (T == 1 && f + 1 < F) fetch(f + 1, sf + fstride);
            char* nh = nullptr;                          // this pixel's D channels of frame f in the NHWC copy (T == 1 only)
            if (T == 1 && c.sf_nhwc != nullptr)
                nh = static_cast<char*>(c.sf_nhwc) + (((size_t)f * c.B + c.b) * plane + pix) * D * (c.sf_nhwc_half ? 2 : 4);
            char* q = sf;
            if (own && !valid) {                         // invalid pixel of frame f: the whole plane stack is 0
#pragma unroll 4
                for (int j = 0; j < kChunk; ++j, q += pstride) {
                    if constexpr (std::is_same<OUT, float>::value) {
                        if (d_lo + j < D) *reinterpret_cast<float*>(q) = 0.f;
                    } else {
                        if (d_lo + j < D) *reinterpret_cast<unsigned short*>(q) = 0;   // +0 in half
                    }
                }
                if (nh != nullptr)
                    for (int o = 0; o < D * (c.sf_nhwc_half ? 2 : 4); o += 16) *reinterpret_cast<uint4*>(nh + o) = make_uint4(0, 0, 0, 0);
            }
            if (T == 1 && !valid) continue;
            float m4[4] = {-2.0f, -2.0f, -2.0f, -2.0f};
#pragma unroll
            for (int j = 0; j < kChunk; ++j) m4[j & 3] = fmaxf(m4[j & 3], vv[j]);
            float m = fmaxf(fmaxf(m4[0], m4[1]), fmaxf(m4[2], m4[3]));
#pragma unroll
            for (int s = kSlots; s < 32; s <<= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, s));
            const float km = c.kq * m;
            float s4[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int j = 0; j < kChunk; ++j) {
                const float t = fmaf(-c.kq, vv[j], km);
                float e;
                asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-t * t));
                if (D == T * kChunk || d_lo + j < D) s4[j & 3] += e;
            }
            float sum = (s4[0] + s4[1]) + (s4[2] + s4[3]);
#pragma unroll
            for (int s = kSlots; s < 32; s <<= 1) sum += __shfl_xor_sync(0xffffffffu, sum, s);
            // weight = 1 - 1/(D-1) * (sum - 1): separate roundings as in the reference so that flat-cost pixels
            // (sum == D) give exactly 0 (monorec_model.py:258, :265-269)
            const float w = valid ? __fsub_rn(1.0f, __fmul_rn(c.inv_dm1, __fsub_rn(sum, 1.0f))) : 0.f;
            wsum += w;
#pragma unroll
            for (int j = 0; j < kChunk; ++j) acc[j] = fmaf(w, vv[j], acc[j]);
            if (nh != nullptr) {                         // the MaskModule's input layout, written while the values are in registers
                if (c.sf_nhwc_half) {
#pragma unroll
                    for (int j = 0; j < kChunk; j += 8) {
                        if (j >= D) break;
                        uint4 pk;
                        __half2* h = reinterpret_cast<__half2*>(&pk);
#pragma unroll
                        for (int k = 0; k < 4; ++k) h[k] = __floats2half2_rn(vv[j + 2 * k], vv[j + 2 * k + 1]);
                        *reinterpret_cast<uint4*>(nh + 2 * j) = pk;
                    }
                } else {
#pragma unroll
                    for (int j = 0; j < kChunk; j += 4) {
                        if (j >= D) break;
                        *reinterpret_cast<float4*>(nh + 4 * j) = make_float4(vv[j], vv[j + 1], vv[j + 2], vv[j + 3]);
                    }
                }
            }
        }
        if (!own) continue;
        const float inv = (wsum == 0.f) ? 0.f : 1.0f / wsum;
        char* q = cv_out;
        if constexpr (CENTER) {
#pragma unroll
            for (int j = 0; j < kChunk; ++j, q += pstride)
                if (D == T * kChunk || d_lo + j < D) st_vol1(reinterpret_cast<OUT*>(q), acc[j] * inv, c.pol_stream);
        } else {
            const float h = (wsum == 0.f) ? 0.f : 0.5f;
#pragma unroll
            for (int j = 0; j < kChunk; ++j, q += pstride)
                if (D == T * kChunk || d_lo + j < D) st_vol1(reinterpret_cast<OUT*>(q), fmaf(-h, acc[j] * inv, h), c.pol_stream);
        }
    }
}

// PIX selects the depth source: false = one depth per plane (a.depths = zs[D], the default linspace planes), true = one depth
// per plane and pixel (a.depths = cv_depths [B,D,H,W]).  ERR is the error mode of stage 2 (use_ssim), CENTER false stores the
// uncentred fused volume (not_center_cv).  OUT is the storage type of both volumes: float, or __half (the march and the
// per-pixel phase compute in fp32 either way; only the stores round, and the per-pixel phase widens what it reads back).
// NC is the channel count of the keyframe and the frames: 3, or 1 for a grayscale stream, whose outputs are those of its
// three-channel replica bit for bit (see wchan).
template <bool PIX, int ERR, bool CENTER, typename OUT, int NC>
__global__ void __launch_bounds__(kThreads, kMinBlocks)
cost_volume_kernel(const CvArgs a, const __grid_constant__ CvMaps maps) {
    static_assert(NC == 1 || NC == 3, "frames have 1 or 3 channels");
    extern __shared__ __align__(128) unsigned char smem[];
    const SmemLayout L = make_layout<NC>(a.D, a.TH, a.F, a.use_tma, PIX, ERR);
    float* win = reinterpret_cast<float*>(smem + L.win);
    float* ytile = reinterpret_cast<float*>(smem + L.ytile);
    float* cst = reinterpret_cast<float*>(smem + L.cst);
    float* pjs = reinterpret_cast<float*>(smem + L.pjs);
    float* zs = reinterpret_cast<float*>(smem + L.zs);
    unsigned char* vmask = smem + L.vmask;
    int* rowrng = reinterpret_cast<int*>(smem + L.rowrng);
    short4* bbox = reinterpret_cast<short4*>(smem + L.bbox);
    unsigned short* gid = reinterpret_cast<unsigned short*>(smem + L.gid);
    unsigned char* uflag = smem + L.uflag;
    GroupInfo* ginfo = reinterpret_cast<GroupInfo*>(smem + L.ginfo);
    unsigned short* seq2g = reinterpret_cast<unsigned short*>(smem + L.seq2g);
    int* nwin = reinterpret_cast<int*>(smem + L.nwin);
    // [0] next unit, [1] number of windows, [2 + buf] finished units of the window in buffer buf, [2 + kBuf + buf] number of
    // the last window whose TMA has been issued into buffer buf (-1: none)
    int* ctr = reinterpret_cast<int*>(smem + L.ctr);
    const uint32_t bars = smem_u32(smem + L.bars);

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int H = a.H, W = a.W, D = a.D, TH = a.TH, F = a.F;
    const int b = blockIdx.z + a.b0;
    const int u0 = blockIdx.x * kOutCols - 2;  // image column of buffer column 0
    const int v0 = blockIdx.y * TH;            // image row of tile row 0
    const size_t plane = (size_t)H * W;
    const int planei = H * W;
    float* xbuf = reinterpret_cast<float*>(smem + L.xbuf) + warp * (xb_warp_floats(NC) + (ERR == kErrSsimL1 ? kLSlotFloats : 0));

    // ---- keyframe tile (+0.5, monorec_model.py:232) and hoisted SSIM terms -------------------------------------
    const float* key = a.key + (size_t)b * NC * plane;
    for (int line = warp; line < NC * (TH + 4); line += kWarps) {     // line = (tile row + 2) * NC + channel
        const int rr = line / NC, ch = line - NC * rr;
        const int v = v0 - 2 + rr;
        const float* src = key + ch * plane + (size_t)v * W;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const int idx = lane + 32 * k;
            if (idx >= 66) break;
            const int u = u0 + idx - 1;
            float val = 0.f;
            if (u >= 0 && u < W && v >= 0 && v < H) val = __ldg(src + u) + 0.5f;
            ytile[line * kRowStride + idx] = val;
        }
    }
    if constexpr (!PIX) {
        for (int i = tid; i < D; i += kThreads) zs[i] = __ldg(a.depths + i);
    } else {
        // Depth extremes.  fminf / fmaxf drop NaN, so a hypothesis that is not finite is recorded explicitly: it turns the
        // entry into (NaN, NaN), which fails every comparison of the validity pre-pass and of the plan.
        const float* zb = a.depths + (size_t)b * D * plane;
        const float kFinite = 3.40282347e38f;
        // per output pixel, over its own D hypotheses (validity pre-pass); only pixels that can be valid are evaluated.  A
        // hypothesis <= 0 is no point in front of the keyframe camera: like a non-finite one, it makes the pixel invalid.
        float2* zpix = reinterpret_cast<float2*>(smem + L.zpix);
        for (int p = tid; p < TH * kTileCols; p += kThreads) {
            const int r = p >> 6, bc = p & 63;
            const int u = u0 + bc, v = v0 + r;
            float lo = __int_as_float(0x7fc00000), hi = lo;
            if (bc >= 2 && bc < 2 + kOutCols && u >= 2 && u < W - 2 && v >= 2 && v < H - 2) {
                const float* q = zb + (size_t)v * W + u;
                lo = 3.0e38f; hi = -3.0e38f;
                bool bad = false;
                for (int d = 0; d < D; ++d, q += plane) {
                    const float z = __ldg(q);
                    bad = bad || !(z > 0.f && z <= kFinite);
                    lo = fminf(lo, z); hi = fmaxf(hi, z);
                }
                if (bad) lo = hi = __int_as_float(0x7fc00000);
            }
            zpix[p] = make_float2(lo, hi);
        }
        // per plane and tile row -2 .. TH+1, over the 64 buffer columns, rows and columns clamped into the image as stage 1
        // reads them (the plan reduces the rows each frame's march touches)
        float2* zrow = reinterpret_cast<float2*>(smem + L.zrow);
        for (int line = warp; line < D * (TH + 4); line += kWarps) {
            const int d = line / (TH + 4), rr = line - d * (TH + 4);
            const float* q = zb + (size_t)d * plane + (size_t)min(max(v0 - 2 + rr, 0), H - 1) * W;
            const float z0 = __ldg(q + min(max(u0 + lane, 0), W - 1)), z1 = __ldg(q + min(max(u0 + lane + 32, 0), W - 1));
            const bool bad = __any_sync(0xffffffffu, !(fabsf(z0) <= kFinite) || !(fabsf(z1) <= kFinite));
            float lo = fminf(z0, z1), hi = fmaxf(z0, z1);
#pragma unroll
            for (int s = 16; s >= 1; s >>= 1) {
                lo = fminf(lo, __shfl_xor_sync(0xffffffffu, lo, s));
                hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, s));
            }
            if (lane == 0) zrow[line] = bad ? make_float2(__int_as_float(0x7fc00000), __int_as_float(0x7fc00000)) : make_float2(lo, hi);
        }
    }
    if (lane < 2 * NC) {   // columns -1 and 64 of both row buffers stay zero
        const int rb = lane / NC, ch = lane % NC;
        xbuf[(rb * NC + ch) * kRowStride] = 0.f;
        xbuf[(rb * NC + ch) * kRowStride + kTileCols + 1] = 0.f;
    }
    if (tid < 2 * F) rowrng[tid] = (tid & 1) ? -1 : TH;
    if (tid < 12 * F) pjs[tid] = __ldg(a.proj + (size_t)b * F * 12 + tid);
    if (tid < 2 + 2 * kBuf) ctr[tid] = (tid < 2 + kBuf) ? 0 : -1;
    if (tid == 0 && a.use_tma) {
        for (int i = 0; i < kBuf; ++i) mbar_init(bars + 8 * i, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    // table entry for the column pair (2j, 2j+1) of e-row er, channel ch: (Y[2j], Y[2j+1], Sg[2j], Sg[2j+1]) with
    // Y = 9 mu_y = sum y, Sg = 81 (sigma_y + C2) = 9 sum y^2 - Y^2 + 81 C2 (kErrBoxL1 reads no table)
    for (int line = warp; line < (ERR == kErrBoxL1 ? 0 : NC * (TH + 2)); line += kWarps) {     // line = e-row * NC + channel
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            const int bc = lane + 32 * k;
            const float* y = ytile + line * kRowStride + bc;  // rows er..er+2 of this channel, idx bc..bc+2
            float s1 = 0.f, s2 = 0.f;
#pragma unroll
            for (int dy = 0; dy < 3; ++dy)
#pragma unroll
                for (int dx = 0; dx < 3; ++dx) {
                    float q = y[dy * NC * kRowStride + dx];
                    s1 += q;
                    s2 = fmaf(q, q, s2);
                }
            float* dst = cst + (line * (kTileCols / 2) + (bc >> 1)) * 4 + (bc & 1);
            dst[0] = s1;
            dst[2] = fmaf(9.0f, s2, -s1 * s1) + 81.0f * kC2;
        }
    }

    const float fW = (float)W, fH = (float)H;
    const float sx_lo = -fW * 0.5f, sx_hi = 1.5f * fW;  // == grid clamp(-2, 2) in sample + 0.5 units, monorec_model.py:208
    const float sy_lo = -fH * 0.5f, sy_hi = 1.5f * fH;

    // ---- validity pre-pass for every frame: valid_f(v,u) = interior(v,u) & all_d [ sample strictly inside
    //      (1,W-2)x(1,H-2) ]  (monorec_model.py:212-219: bilinear sample of the interior mask != 0 for every plane).
    //      The D samples of a pixel lie on one line and move monotonically with the depth while the denominator keeps
    //      its sign, so the farthest and the nearest plane decide.  A denominator < 0 is a point behind the source camera:
    //      the reference still samples its mirrored projection (layers.py:66 divides by z + 1e-7 whatever its sign), so
    //      such samples count like any other.  Where the denominator changes sign between the two ends, the ray crosses the
    //      source camera's plane and its samples do not lie on one segment: every depth of the pixel is checked. -----------
    for (int q = tid; q < F * TH * kTileCols; q += kThreads) {
        const int fr = q >> 6, bc = q & 63;            // fr = f * TH + r
        const int f = fr / TH, r = fr - f * TH;
        const int u = u0 + bc, v = v0 + r;
        bool ok = (bc >= 2) && (bc < 2 + kOutCols) && (u >= 2) && (u < W - 2) && (v >= 2) && (v < H - 2);
        if (ok) {
            const float* m = pjs + 12 * f;
            const float fu = (float)u, fv = (float)v;
            const float ax = fmaf(m[0], fu, fmaf(m[1], fv, m[2]));
            const float ay = fmaf(m[4], fu, fmaf(m[5], fv, m[6]));
            const float az = fmaf(m[8], fu, fmaf(m[9], fv, m[10]));
            const float m03 = m[3], m13 = m[7], m23 = m[11];
            auto inside = [&](const float z, float& den) {
                den = fmaf(az, z, m23);
                const float inv = fast_rcp(den);
                const float sx = fmaf(fmaf(ax, z, m03), inv, -0.5f);
                const float sy = fmaf(fmaf(ay, z, m13), inv, -0.5f);
                return (sx > 1.0f) && (sx < fW - 2.0f) && (sy > 1.0f) && (sy < fH - 2.0f);
            };
            float den[2] = {1.0f, 1.0f};
#pragma unroll
            for (int k = 0; k < 2; ++k) {
                float z;
                if constexpr (PIX) {   // the pixel's own nearest and farthest hypothesis (NaN: one is not finite)
                    const float2 e = reinterpret_cast<const float2*>(smem + L.zpix)[r * kTileCols + bc];
                    z = k ? e.y : e.x;
                } else {
                    z = zs[k ? D - 1 : 0];
                }
                ok = ok && inside(z, den[k]);
            }
            if (ok && ((den[0] > 0.f) != (den[1] > 0.f))) {
                for (int d = 0; d < D && ok; ++d) {
                    float dd;
                    if constexpr (PIX) ok = inside(__ldg(a.depths + ((size_t)b * D + d) * plane + (size_t)v * W + u), dd);
                    else ok = inside(zs[d], dd);
                }
            }
        }
        vmask[q] = ok ? 1 : 0;
        // (a warp covers half a tile row of one frame: one pair of shared-memory atomics per warp, not per pixel)
        if (__any_sync(0xffffffffu, ok) && lane == 0) { atomicMin(&rowrng[2 * f], r); atomicMax(&rowrng[2 * f + 1], r); }
    }
    __syncthreads();

    // ---- plan: source footprint of every unit (4 corners of the rows / columns its march touches), then windows ------
    const int nunits = F * D;
    for (int u = tid; u < nunits; u += kThreads) {
        const int f = u / D, d = u - f * D;
        const int rlo = rowrng[2 * f], rhi = rowrng[2 * f + 1];
        short4 bb = make_short4(0, 0, 0, 0);
        unsigned char fl = 0;          // bit 0: footprint usable for a window, bit 1: strictly inside the image
        if (rhi >= rlo && a.use_tma) {
            const float* m = pjs + 12 * f;
            float zlo, zhi = 0.f;
            bool good = true;
            if constexpr (PIX) {
                // depth interval of plane d over the rows rlo-2 .. rhi+2 this frame's march touches.  The unit's samples lie
                // in the hull of the 8 points (tile corner, zlo / zhi) and the denominator is affine in that point, so while
                // it is > 0 at the 8 corners their projections bound every sample.  Not finite, or far beyond any scene
                // depth (where the products of stage 1 could overflow): the unit gathers with clamped taps.
                const float2* zrow = reinterpret_cast<const float2*>(smem + L.zrow) + d * (TH + 4);
                zlo = zrow[rlo].x; zhi = zrow[rlo].y;
                bool finite = (zlo == zlo) && (zhi == zhi);
                for (int rr = rlo + 1; rr <= rhi + 4; ++rr) {
                    const float2 e = zrow[rr];
                    finite = finite && (e.x == e.x) && (e.y == e.y);
                    zlo = fminf(zlo, e.x); zhi = fmaxf(zhi, e.y);
                }
                good = finite && fmaxf(-zlo, zhi) < 1.0e20f;
            } else {
                zlo = zs[d];
            }
            float xmin = 3.0e38f, xmax = -3.0e38f, ymin = 3.0e38f, ymax = -3.0e38f;
#pragma unroll
            for (int k = 0; k < (PIX ? 8 : 4); ++k) {
                const float fu = (float)(u0 + ((k & 1) ? kTileCols - 1 : 0));
                const float fv = (float)(v0 + ((k & 2) ? rhi + 2 : rlo - 2));
                const float z = (PIX && (k & 4)) ? zhi : zlo;
                const float cx = fmaf(fmaf(m[0], fu, fmaf(m[1], fv, m[2])), z, m[3]);
                const float cy = fmaf(fmaf(m[4], fu, fmaf(m[5], fv, m[6])), z, m[7]);
                const float cz = fmaf(fmaf(m[8], fu, fmaf(m[9], fv, m[10])), z, m[11]);
                good = good && (cz > 1e-6f);
                const float inv = 1.0f / cz;
                const float sx = fminf(fmaxf(cx * inv, sx_lo), sx_hi) - 0.5f, sy = fminf(fmaxf(cy * inv, sy_lo), sy_hi) - 0.5f;
                xmin = fminf(xmin, sx); xmax = fmaxf(xmax, sx);
                ymin = fminf(ymin, sy); ymax = fmaxf(ymax, sy);
            }
            if (good) {
                // one pixel of slack on every side for the rounding differences between this estimate and stage 1
                // (the window origin is rounded down to a multiple of 4 pixels: TMA wants the innermost box coordinate
                // 16-byte aligned; negative coordinates are fine)
                const int xl = (max((int)floorf(xmin) - 1, -2) >> 2) << 2, xh = min((int)floorf(xmax) + 2, W + 1);
                const int yl = max((int)floorf(ymin) - 1, -2), yh = min((int)floorf(ymax) + 2, H + 1);
                if (xh >= xl && yh >= yl && xh - xl < kPitch && yh - yl < kWinRows) {
                    fl = 1;
                    if (xmin >= 0.05f && xmax <= fW - 1.05f && ymin >= 0.05f && ymax <= fH - 1.05f) fl = 3;
                    bb = make_short4((short)xl, (short)xh, (short)yl, (short)yh);
                }
            }
        }
        bbox[u] = bb;
        uflag[u] = fl;
        gid[u] = 0xFFFF;
    }
    __syncthreads();
    if (lane == 0 && warp < F) {   // one frame per warp: the F serial scans run side by side instead of as divergent lanes
        // greedy runs of consecutive planes whose union still fits one window
        const int f = warp;
        int ng = 0;
        const int rlo = rowrng[2 * f], rhi = rowrng[2 * f + 1];
        if (rhi >= rlo && a.use_tma) {
            int d = 0;
            while (d < D) {
                if (!(uflag[f * D + d] & 1)) { ++d; continue; }
                short4 g = bbox[f * D + d];
                int e = d + 1;
                while (e < D && (uflag[f * D + e] & 1)) {
                    const short4 o = bbox[f * D + e];
                    const int xl = min(g.x, o.x), xh = max(g.y, o.y), yl = min(g.z, o.z), yh = max(g.w, o.w);
                    if (xh - xl >= kPitch || yh - yl >= kWinRows) break;
                    g = make_short4((short)xl, (short)xh, (short)yl, (short)yh);
                    ++e;
                }
                if (e - d >= kMinGroup) {
                    GroupInfo gi;
                    gi.wx0 = g.x; gi.wy0 = g.z;
                    gi.nrows = (short)(((g.w - g.z + 1) + kBoxRows - 1) / kBoxRows * kBoxRows);
                    gi.f = (short)f; gi.count = (short)(e - d); gi.seq = (short)ng; gi.pad0 = gi.pad1 = 0;
                    ginfo[f * D + ng] = gi;
                    for (int k = d; k < e; ++k) gid[f * D + k] = (unsigned short)(f * D + ng);
                    ++ng;
                }
                d = e;
            }
        }
        nwin[f] = ng;
    }
    __syncthreads();
    if (lane == 0 && warp < F) {
        const int f = warp;
        int base = 0;
        for (int k = 0; k < f; ++k) base += nwin[k];
        for (int g = 0; g < nwin[f]; ++g) {
            ginfo[f * D + g].seq = (short)(base + g);
            seq2g[base + g] = (unsigned short)(f * D + g);
        }
        if (f == F - 1) ctr[1] = base + nwin[f];
    }
    __syncthreads();

    // window `seq` -> buffer seq % kBuf: NC channel planes of nrows rows, TMA boxes of kBoxRows rows
    auto issue_window = [&](int seq) {
        const GroupInfo gi = ginfo[seq2g[seq]];
        const int buf = seq % kBuf;
        const uint32_t bar = bars + 8 * buf;
        const uint32_t dst = smem_u32(win + (size_t)buf * (NC * kChanStride));
        atomicExch(&ctr[2 + kBuf + buf], seq);   // (an atomic, like its readers: a flag, not a data race)
        mbar_expect_tx(bar, (uint32_t)(NC * gi.nrows * kPitch * 4));
        for (int ch = 0; ch < NC; ++ch)
            for (int r8 = 0; r8 < gi.nrows; r8 += kBoxRows)
                tma_load_3d(dst + (uint32_t)((ch * kWinRows + r8) * kPitch * 4), &maps.m[gi.f], bar, gi.wx0, gi.wy0 + r8, b * NC + ch);
    };
    if (tid == 0 && a.use_tma) {
        const int nw = ctr[1];
        for (int s = 0; s < kBuf && s < nw; ++s) issue_window(s);
    }

    const float2 fu2 = make_float2((float)(u0 + lane), (float)(u0 + lane + 32));
    // stage 2 writes the single-frame volume for output columns u0 + 2l, u0 + 2l + 1 (lanes 1..30)
    const int ucol = u0 + 2 * lane;
    const bool st0 = (lane >= 1) && (lane <= 30) && (ucol < W);
    const bool st1 = (lane >= 1) && (lane <= 30) && (ucol + 1 < W);
    const uint64_t pol_keep = l2_policy_evict_last(), pol_stream = l2_policy_evict_first();

    // ---- march over the F*D (frame, plane) units; no CTA-wide barrier in here ------------------------------------
    Stage2Ctx c2;
    if constexpr (ERR != kErrBoxL1) {
        c2.cw0 = bc2(a.cw0); c2.cw1 = bc2(a.cw1); c2.cw2 = bc2(a.cw2);
    } else {
        c2.cw0 = bc2(a.cw0 / 9.0f); c2.cw1 = bc2(a.cw1 / 9.0f); c2.cw2 = bc2(a.cw2 / 9.0f);
    }
    c2.pairflag = (st0 && st1 && ((W & 1) == 0)) ? 1 : 0;
    c2.st0 = st0 && !c2.pairflag; c2.st1 = st1 && !c2.pairflag; c2.pol_keep = pol_keep;
    Stage1Ctx c1;
    c1.W = W; c1.H = H; c1.planei = planei;
    c1.sx_lo = sx_lo; c1.sx_hi = sx_hi; c1.sy_lo = sy_lo; c1.sy_hi = sy_hi;
    if constexpr (PIX) { c1.zc0 = min(max(u0 + lane, 0), W - 1); c1.zc1 = min(max(u0 + lane + 32, 0), W - 1); }
    // per-lane shared addresses for stage 2 (columns 2l-1 .. 2l+2 live at float index 2l .. 2l+3 of a row)
    const uint32_t xb_s = smem_u32(xbuf);
    const uint32_t ys_s = smem_u32(ytile) + 8 * lane;
    const uint32_t cs_s = smem_u32(cst) + 16 * lane;
    const uint32_t win_s = smem_u32(win);
    for (;;) {
        int unit = 0;
        if (lane == 0) unit = atomicAdd(&ctr[0], 1);
        unit = __shfl_sync(0xffffffffu, unit, 0);
        if (unit >= nunits) break;
        const int f = unit / D, d = unit - f * D;
        const int rlo = rowrng[2 * f], rhi = rowrng[2 * f + 1];
        if (rhi < rlo) continue;  // no valid pixel of this tile for frame f: the per-pixel phase zero-fills
        if constexpr (PIX) setup_stage1_pix(c1, pjs + 12 * f, fu2, a.depths + ((size_t)b * D + d) * plane);
        else setup_stage1(c1, pjs + 12 * f, zs[d], fu2);
        const int nsteps = rhi - rlo + 5;
        const float fv0 = (float)(v0 + rlo - 2);
        const uint32_t yr = ys_s + rlo * (NC * kYRowBytes);   // tile row rlo-2 is keyframe-tile row rlo
        // the SSIM row of step t is tile row rlo-3+t, whose table row is rlo-2+t (t = 0, 1 read throw-away rows, possibly
        // in front of the table: still inside this CTA's shared memory, see make_layout)
        const uint32_t cr = cs_s + (rlo - 2) * (NC * kCRowBytes);
        OUT* out = static_cast<OUT*>(a.sfcv) + (((size_t)f * a.B + b) * D + d) * plane + ((ptrdiff_t)(v0 + rlo - 4) * W + ucol);
        const unsigned g = gid[unit];
        if (g != 0xFFFFu) {
            const GroupInfo gi = ginfo[g];
            const int buf = gi.seq % kBuf;
            // A parity wait is only meaningful on the phase in progress or the one before: first make sure this window's
            // load has been issued (the buffer's previous window is then complete and consumed), then wait for its bytes.
            for (uint32_t spin = 0;; ++spin) {
                int armed = 0;
                if (lane == 0) armed = atomicAdd(&ctr[2 + kBuf + buf], 0);
                if (__shfl_sync(0xffffffffu, armed, 0) >= gi.seq) break;
                if (spin > (1u << 22)) __trap();
            }
            mbar_wait(bars + 8 * buf, (uint32_t)((gi.seq / kBuf) & 1));
            const uint32_t wb = win_s + (uint32_t)buf * (NC * kChanStride * 4);
            if (uflag[unit] & 2) {
                // tap address = wb + 4 ((bits(ty) - kMagicBits - wy0) kPitch + bits(tx) - kMagicBits - wx0), mod 2^32
                c1.kaddr = wb - 4u * ((uint32_t)(kMagicBits + gi.wy0) * kPitch + (uint32_t)(kMagicBits + gi.wx0));
                march_unit<0, PIX, ERR, NC>(c1, c2, xb_s, lane, fv0, nsteps, yr, cr, out, W, v0 + rlo - 2);
            } else {
                c1.kaddr = wb - 4u * ((uint32_t)(int)gi.wy0 * kPitch + (uint32_t)(int)gi.wx0);
                march_unit<1, PIX, ERR, NC>(c1, c2, xb_s, lane, fv0, nsteps, yr, cr, out, W, v0 + rlo - 2);
            }
            // hand the buffer on: the last unit of the window re-arms it with the window after next
            if (lane == 0) {
                __threadfence_block();
                const int fin = atomicAdd(&ctr[2 + buf], 1) + 1;
                if (fin == gi.count) {
                    ctr[2 + buf] = 0;
                    __threadfence_block();
                    if (gi.seq + kBuf < ctr[1]) {
                        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                        issue_window(gi.seq + kBuf);
                    }
                }
            }
            __syncwarp();
        } else {
            c1.img = a.frames[f] + (size_t)b * NC * plane;
            march_unit<2, PIX, ERR, NC>(c1, c2, xb_s, lane, fv0, nsteps, yr, cr, out, W, v0 + rlo - 2);
        }
    }
    __syncthreads();  // the marching warps' global stores are visible to the whole CTA from here on

    // ---- per-pixel phase: view weights (monorec_model.py:257-260), zeroing of invalid pixels (:251) and fusion
    //      cv = sum_f w_f (1 - 2 sad_f) / sum_f w_f, 0 where sum_f w_f == 0 (:262-269).  Each thread reads back the
    //      L2-hot single-frame values of its pixel once per frame. ------------------------------------------------------
    PixelPhase pp;
    pp.cv = a.cv; pp.sfcv = a.sfcv; pp.sf_nhwc = a.sf_nhwc; pp.sf_nhwc_half = a.sf_nhwc_half;
    pp.vmask = vmask; pp.B = a.B; pp.F = F; pp.D = D; pp.H = H; pp.W = W; pp.TH = TH; pp.b = b; pp.u0 = u0; pp.v0 = v0;
    pp.inv_dm1 = a.inv_dm1;
    // exp(-alpha (sad - min sad)^2) with sad = (1 - sv) / 2 is ex2(-(k (max sv - sv))^2), k = sqrt(alpha log2(e)) / 2
    pp.kq = 0.5f * sqrtf(a.alpha * 1.4426950408889634f);
    pp.pol_stream = pol_stream;
    if (D <= kChunk) pixel_phase<1, CENTER, OUT>(pp);
    else if (D <= 2 * kChunk) pixel_phase<2, CENTER, OUT>(pp);
    else pixel_phase<4, CENTER, OUT>(pp);
}

// ----------------------------------------------------------------------------------------------------------------
// projection tables (fp64 on device, one thread per (b,f)); see include/monorec_b200.h
// ----------------------------------------------------------------------------------------------------------------
struct PtrPack {
    const float* p[MR_MAX_FRAMES];
};

__device__ bool invert4(const float* src, double* out) {
    double m[4][8];
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) {
            m[i][j] = (double)src[i * 4 + j];
            m[i][4 + j] = (i == j) ? 1.0 : 0.0;
        }
    for (int c = 0; c < 4; ++c) {
        int piv = c;
        double best = fabs(m[c][c]);
        for (int r = c + 1; r < 4; ++r)
            if (fabs(m[r][c]) > best) { best = fabs(m[r][c]); piv = r; }
        if (best == 0.0) return false;
        if (piv != c)
            for (int j = 0; j < 8; ++j) { double t = m[c][j]; m[c][j] = m[piv][j]; m[piv][j] = t; }
        double inv = 1.0 / m[c][c];
        for (int j = 0; j < 8; ++j) m[c][j] *= inv;
        for (int r = 0; r < 4; ++r)
            if (r != c) {
                double fct = m[r][c];
                for (int j = 0; j < 8; ++j) m[r][j] -= fct * m[c][j];
            }
    }
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) out[i * 4 + j] = m[i][4 + j];
    return true;
}

__global__ void projection_tables_kernel(const float* kf_pose, const float* kf_K, PtrPack poses, PtrPack intr,
                                         int B, int F, int H, int W, float* proj, float* depths, int D,
                                         float lo, float hi) {
    int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (depths != nullptr && idx < D) {
        // torch.linspace (fp32, symmetric fill) followed by 1/x  -- monorec_model.py:184
        float step = __fdiv_rn(hi - lo, (float)(D - 1));
        float x = (idx < D / 2) ? fmaf(step, (float)idx, lo) : fmaf(-step, (float)(D - 1 - idx), hi);
        depths[idx] = __frcp_rn(x);
    }
    if (idx >= B * F) return;
    int b = idx / F, f = idx % F;
    double kinv[16], pinv[16], T[16], P[12];
    bool ok = invert4(kf_K + b * 16, kinv);
    ok = invert4(poses.p[f] + b * 16, pinv) && ok;
    const float* kp = kf_pose + b * 16;
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) {
            double s = 0;
            for (int k = 0; k < 4; ++k) s += pinv[i * 4 + k] * (double)kp[k * 4 + j];
            T[i * 4 + j] = s;
        }
    const float* Kf = intr.p[f] + b * 16;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 4; ++j) {
            double s = 0;
            for (int k = 0; k < 4; ++k) s += (double)Kf[i * 4 + k] * T[k * 4 + j];
            P[i * 4 + j] = s;
        }
    double sc[3] = {(double)W / (double)(W - 1), (double)H / (double)(H - 1), 1.0};
    float* o = proj + (size_t)idx * 12;
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) {
            double s = 0;
            for (int k = 0; k < 3; ++k) s += P[i * 4 + k] * kinv[k * 4 + j];
            o[i * 4 + j] = ok ? (float)(s * sc[i]) : __int_as_float(0x7fc00000);
        }
        double t = P[i * 4 + 3] + (i == 2 ? 1e-7 : 0.0);
        o[i * 4 + 3] = ok ? (float)(t * sc[i]) : __int_as_float(0x7fc00000);
    }
}

// the launch's layout for nc channels
SmemLayout layout_for(int nc, int D, int TH, int F, int use_tma, bool pix, int err) {
    return nc == 1 ? make_layout<1>(D, TH, F, use_tma, pix, err) : make_layout<3>(D, TH, F, use_tma, pix, err);
}

int pick_tile_rows(int D, int F, int use_tma, bool pix, int err, int nc) {
    const int limit = 227 * 1024;
    for (int th = kTileRows; th >= 2; th >>= 1)
        if (layout_for(nc, D, th, F, use_tma, pix, err).total <= limit) return th;
    return 0;
}

template <bool PIX, int ERR, bool CENTER, typename OUT, int NC>
int launch_kernel(dim3 grid, int smem, cudaStream_t stream, const CvArgs& a, const CvMaps& maps) {
    // The opt-in is per function and per device context, so it is remembered per device (bit d: device d; devices from 64 on
    // set it before every launch).  Two threads that both find the bit clear both set the attribute: harmless.
    static std::atomic<unsigned long long> opted_in{0};
    int dev = 0;
    MR_CUDA(cudaGetDevice(&dev));
    const unsigned long long bit = dev < 64 ? 1ull << dev : 0ull;
    if ((opted_in.load(std::memory_order_acquire) & bit) == 0) {
        MR_CUDA(cudaFuncSetAttribute(cost_volume_kernel<PIX, ERR, CENTER, OUT, NC>,
                                     cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        opted_in.fetch_or(bit, std::memory_order_release);
    }
    cost_volume_kernel<PIX, ERR, CENTER, OUT, NC><<<grid, kThreads, smem, stream>>>(a, maps);
    MR_LAUNCH_CHECK("cost_volume_kernel");
    return MR_OK;
}

// the instantiation for (error mode, centring); matching was checked by the caller
template <bool PIX, typename OUT, int NC>
int launch_variant(int matching, int centered, dim3 grid, int smem, cudaStream_t stream, const CvArgs& a, const CvMaps& maps) {
    if (matching == kErrSsimL1)
        return centered ? launch_kernel<PIX, kErrSsimL1, true, OUT, NC>(grid, smem, stream, a, maps)
                        : launch_kernel<PIX, kErrSsimL1, false, OUT, NC>(grid, smem, stream, a, maps);
    if (matching == kErrBoxL1)
        return centered ? launch_kernel<PIX, kErrBoxL1, true, OUT, NC>(grid, smem, stream, a, maps)
                        : launch_kernel<PIX, kErrBoxL1, false, OUT, NC>(grid, smem, stream, a, maps);
    return centered ? launch_kernel<PIX, kErrSsim, true, OUT, NC>(grid, smem, stream, a, maps)
                    : launch_kernel<PIX, kErrSsim, false, OUT, NC>(grid, smem, stream, a, maps);
}

// the instantiation for (depth source, storage type, channels)
template <int NC>
int launch_channels(bool pix, int out_dtype, int matching, int centered, dim3 grid, int smem, cudaStream_t stream,
                    const CvArgs& a, const CvMaps& maps) {
    if (out_dtype == MR_DT_F16)
        return pix ? launch_variant<true, __half, NC>(matching, centered, grid, smem, stream, a, maps)
                   : launch_variant<false, __half, NC>(matching, centered, grid, smem, stream, a, maps);
    return pix ? launch_variant<true, float, NC>(matching, centered, grid, smem, stream, a, maps)
               : launch_variant<false, float, NC>(matching, centered, grid, smem, stream, a, maps);
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;   // benign race: every thread resolves the same pointer
    if (fn == nullptr) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}

}  // namespace

extern "C" int mr_projection_tables(const float* keyframe_pose, const float* keyframe_K, const float* const* poses,
                                    const float* const* intrinsics, int B, int F, int H, int W, float* proj,
                                    float* depths, int D, float inv_depth_lo, float inv_depth_hi, void* stream) {
    MR_REQUIRE(keyframe_pose && keyframe_K && poses && intrinsics && proj, "mr_projection_tables: null pointer");
    MR_REQUIRE(B >= 1 && F >= 1 && F <= MR_MAX_FRAMES, "mr_projection_tables: need B>=1, 1<=F<=%d (got B=%d F=%d)",
               MR_MAX_FRAMES, B, F);
    MR_REQUIRE(H >= 5 && W >= 5, "mr_projection_tables: image too small (%dx%d)", H, W);
    MR_REQUIRE(depths == nullptr || D >= 2, "mr_projection_tables: D must be >= 2 (got %d)", D);
    PtrPack pp{}, ip{};
    for (int f = 0; f < F; ++f) {
        MR_REQUIRE(poses[f] && intrinsics[f], "mr_projection_tables: null pose/intrinsics pointer for frame %d", f);
        pp.p[f] = poses[f];
        ip.p[f] = intrinsics[f];
    }
    int n = B * F > D ? B * F : D;
    projection_tables_kernel<<<(n + 63) / 64, 64, 0, (cudaStream_t)stream>>>(
        keyframe_pose, keyframe_K, pp, ip, B, F, H, W, proj, depths, depths ? D : 0, inv_depth_lo, inv_depth_hi);
    MR_LAUNCH_CHECK("projection_tables_kernel");
    return MR_OK;
}

int mr::launch_cost_volume(const float* keyframe, const float* const* frames, const float* proj,
                           const float* depths, void* out_cv, void* out_sfcv, int B, int F, int D, int H, int W,
                           float alpha, const float* chan_w, int b_begin, int b_count, int gather_only,
                           cudaStream_t stream, void* sf_nhwc, int sf_nhwc_dtype, int per_pixel_depths, int matching,
                           int centered, int out_dtype, int channels) {
    MR_REQUIRE(keyframe && frames && proj && depths && out_cv && out_sfcv, "mr_cost_volume_fwd: null pointer");
    MR_REQUIRE(out_dtype == MR_DT_F32 || out_dtype == MR_DT_F16, "mr_cost_volume_fwd: unknown out_dtype %d", out_dtype);
    MR_REQUIRE(channels == 1 || channels == 3, "mr_cost_volume_fwd: channels must be 1 or 3 (got %d)", channels);
    MR_REQUIRE(b_begin >= 0 && b_count >= 1 && b_begin + b_count <= B, "mr_cost_volume_fwd: bad batch range");
    MR_REQUIRE(B >= 1 && B <= 21845, "mr_cost_volume_fwd: batch %d out of range", B);
    MR_REQUIRE(F >= 1 && F <= MR_MAX_FRAMES, "mr_cost_volume_fwd: 1 <= F <= %d required (got %d)", MR_MAX_FRAMES, F);
    MR_REQUIRE(D >= 2 && D <= 128, "mr_cost_volume_fwd: 2 <= D <= 128 required (got %d)", D);
    MR_REQUIRE(H >= 5 && W >= 5 && H <= 16384 && W <= 16384, "mr_cost_volume_fwd: image size %dx%d out of range", H, W);
    MR_REQUIRE(matching == MR_CV_SSIM || matching == MR_CV_SSIM_L1 || matching == MR_CV_BOX_L1,
               "mr_cost_volume_fwd: unknown matching %d", matching);
    CvArgs a{};
    a.key = keyframe;
    for (int f = 0; f < F; ++f) {
        MR_REQUIRE(frames[f] != nullptr, "mr_cost_volume_fwd: null frame pointer %d", f);
        a.frames[f] = frames[f];
    }
    a.proj = proj; a.depths = depths; a.cv = out_cv; a.sfcv = out_sfcv;
    MR_REQUIRE(sf_nhwc == nullptr || (D <= kChunk && (D % 8) == 0 && (reinterpret_cast<uintptr_t>(sf_nhwc) & 15) == 0 &&
                                      (sf_nhwc_dtype == MR_DT_F32 || sf_nhwc_dtype == MR_DT_F16)),
               "mr_cost_volume_fwd_nhwc: the NHWC copy needs D <= %d, D %% 8 == 0, a 16-byte aligned buffer and an fp32 / half type", kChunk);
    a.sf_nhwc = sf_nhwc; a.sf_nhwc_half = (sf_nhwc_dtype == MR_DT_F16) ? 1 : 0;
    a.B = B; a.F = F; a.D = D; a.H = H; a.W = W; a.b0 = b_begin;
    // TMA addresses the frames as (W, H, C B) tensors: the row pitch must be a multiple of 16 bytes and the base 16-byte
    // aligned; otherwise (ragged widths) every unit takes the global gather of the same kernel.
    CvMaps local{};       // by-value kernel parameter (__grid_constant__): one tensor map per source frame
    a.use_tma = 0;
    EncodeTiledFn encode = gather_only ? nullptr : get_encode_fn();
    if (encode != nullptr && (W % 4) == 0) {
        bool ok = true;
        for (int f = 0; f < F && ok; ++f) {
            if (reinterpret_cast<uintptr_t>(frames[f]) & 15) { ok = false; break; }
            const cuuint64_t gdim[3] = {(cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)channels * B};
            const cuuint64_t gstr[2] = {(cuuint64_t)W * 4, (cuuint64_t)H * W * 4};
            const cuuint32_t box[3] = {(cuuint32_t)kPitch, (cuuint32_t)kBoxRows, 1};
            const cuuint32_t estr[3] = {1, 1, 1};
            const CUresult r = encode(&local.m[f], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(frames[f]), gdim, gstr,
                                      box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                                      CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            ok = (r == CUDA_SUCCESS);
        }
        if (ok) {
            for (int f = F; f < MR_MAX_FRAMES; ++f) local.m[f] = local.m[0];
            a.use_tma = 1;
        }
    }
    const bool pix = per_pixel_depths != 0;
    a.TH = pick_tile_rows(D, F, a.use_tma, pix, matching, channels);
    MR_REQUIRE(a.TH > 0, "mr_cost_volume_fwd: no tile height fits shared memory for D=%d F=%d", D, F);
    a.alpha = alpha;
    a.inv_dm1 = (float)(1.0 / (double)(D - 1));
    const float def_w[3] = {5.f / 32.f, 16.f / 32.f, 11.f / 32.f};  // monorec_model.py:133
    const float* cw = chan_w ? chan_w : def_w;
    a.cw0 = cw[0] / 9.f; a.cw1 = cw[1] / 9.f; a.cw2 = cw[2] / 9.f;  // monorec_model.py:141 (weights / patch_size^2)
    const SmemLayout L = layout_for(channels, D, a.TH, F, a.use_tma, pix, matching);
    dim3 grid((W + kOutCols - 1) / kOutCols, (H + a.TH - 1) / a.TH, b_count);
    return channels == 1 ? launch_channels<1>(pix, out_dtype, matching, centered, grid, L.total, stream, a, local)
                         : launch_channels<3>(pix, out_dtype, matching, centered, grid, L.total, stream, a, local);
}

extern "C" int mr_cost_volume_fwd(const float* keyframe, const float* const* frames, const float* proj,
                                  const float* depths, float* out_cv, float* out_sfcv, int B, int F, int D, int H,
                                  int W, float alpha, const float* chan_w, void* stream) {
    return mr::launch_cost_volume(keyframe, frames, proj, depths, out_cv, out_sfcv, B, F, D, H, W, alpha, chan_w, 0,
                                  B, 0, (cudaStream_t)stream, nullptr, 0);
}

extern "C" int mr_cost_volume_fwd_gather(const float* keyframe, const float* const* frames, const float* proj,
                                         const float* depths, float* out_cv, float* out_sfcv, int B, int F, int D, int H,
                                         int W, float alpha, const float* chan_w, void* stream) {
    return mr::launch_cost_volume(keyframe, frames, proj, depths, out_cv, out_sfcv, B, F, D, H, W, alpha, chan_w, 0,
                                  B, 1, (cudaStream_t)stream, nullptr, 0);
}

extern "C" int mr_cost_volume_fwd_nhwc(const float* keyframe, const float* const* frames, const float* proj, const float* depths,
                                       float* out_cv, float* out_sfcv, void* out_sfcv_nhwc, int nhwc_dtype, int B, int F, int D,
                                       int H, int W, float alpha, const float* chan_w, void* stream) {
    MR_REQUIRE(out_sfcv_nhwc != nullptr, "mr_cost_volume_fwd_nhwc: null NHWC buffer");
    return mr::launch_cost_volume(keyframe, frames, proj, depths, out_cv, out_sfcv, B, F, D, H, W, alpha, chan_w, 0, B, 0,
                                  (cudaStream_t)stream, out_sfcv_nhwc, nhwc_dtype);
}

extern "C" int mr_cost_volume_fwd_depthmap(const float* keyframe, const float* const* frames, const float* proj,
                                           const float* pixel_depths, float* out_cv, float* out_sfcv, void* out_sfcv_nhwc,
                                           int nhwc_dtype, int B, int F, int D, int H, int W, float alpha,
                                           const float* chan_w, void* stream) {
    MR_REQUIRE(pixel_depths != nullptr, "mr_cost_volume_fwd_depthmap: null pixel_depths");
    MR_REQUIRE((reinterpret_cast<uintptr_t>(pixel_depths) & 3) == 0,
               "mr_cost_volume_fwd_depthmap: pixel_depths must be 4-byte aligned");
    MR_REQUIRE(D >= 2 && D <= 128, "mr_cost_volume_fwd_depthmap: 2 <= D <= 128 required (got D=%d)", D);
    MR_REQUIRE(F >= 1 && F <= MR_MAX_FRAMES, "mr_cost_volume_fwd_depthmap: 1 <= F <= %d required (got F=%d)", MR_MAX_FRAMES, F);
    MR_REQUIRE(nhwc_dtype == MR_DT_F32 || nhwc_dtype == MR_DT_F16,
               "mr_cost_volume_fwd_depthmap: nhwc_dtype must be MR_DT_F32 or MR_DT_F16 (got %d)", nhwc_dtype);
    return mr::launch_cost_volume(keyframe, frames, proj, pixel_depths, out_cv, out_sfcv, B, F, D, H, W, alpha, chan_w, 0, B,
                                  0, (cudaStream_t)stream, out_sfcv_nhwc, nhwc_dtype, 1);
}

namespace {
// the checks the general entries share; fn names the entry in the messages
int check_general_args(const char* fn, const float* depths, const float* pixel_depths, int nhwc_dtype, int F, int D,
                       int matching, int centered) {
    if (matching == 0) {   // use_ssim falsy: the plain |w - k| difference (monorec_model.py:227-228)
        ::mr::set_error("%s: matching 0 (plain L1 difference) is not implemented", fn);
        return MR_ENOSUPPORT;
    }
    MR_REQUIRE(matching == MR_CV_SSIM || matching == MR_CV_SSIM_L1 || matching == MR_CV_BOX_L1,
               "%s: unknown matching %d (MR_CV_SSIM, MR_CV_SSIM_L1 or MR_CV_BOX_L1)", fn, matching);
    MR_REQUIRE(centered == 0 || centered == 1, "%s: centered must be 0 or 1 (got %d)", fn, centered);
    MR_REQUIRE((depths == nullptr) != (pixel_depths == nullptr),
               "%s: exactly one of depths / pixel_depths must be given (got %s)", fn, depths ? "both" : "neither");
    MR_REQUIRE((reinterpret_cast<uintptr_t>(pixel_depths) & 3) == 0, "%s: pixel_depths must be 4-byte aligned", fn);
    MR_REQUIRE(D >= 2 && D <= 128, "%s: 2 <= D <= 128 required (got D=%d)", fn, D);
    MR_REQUIRE(F >= 1 && F <= MR_MAX_FRAMES, "%s: 1 <= F <= %d required (got F=%d)", fn, MR_MAX_FRAMES, F);
    MR_REQUIRE(nhwc_dtype == MR_DT_F32 || nhwc_dtype == MR_DT_F16,
               "%s: nhwc_dtype must be MR_DT_F32 or MR_DT_F16 (got %d)", fn, nhwc_dtype);
    return MR_OK;
}
}  // namespace

extern "C" int mr_cost_volume_fwd_matching(const float* keyframe, const float* const* frames, const float* proj,
                                           const float* depths, const float* pixel_depths, float* out_cv, float* out_sfcv,
                                           void* out_sfcv_nhwc, int nhwc_dtype, int B, int F, int D, int H, int W, float alpha,
                                           const float* chan_w, int matching, int centered, void* stream) {
    const int rc = check_general_args("mr_cost_volume_fwd_matching", depths, pixel_depths, nhwc_dtype, F, D, matching, centered);
    if (rc != MR_OK) return rc;
    const int pix = pixel_depths != nullptr;
    return mr::launch_cost_volume(keyframe, frames, proj, pix ? pixel_depths : depths, out_cv, out_sfcv, B, F, D, H, W, alpha,
                                  chan_w, 0, B, 0, (cudaStream_t)stream, out_sfcv_nhwc, nhwc_dtype, pix, matching, centered);
}

namespace {
// mr_cost_volume_fwd_typed on frames of `channels` channels; fn names the entry in the messages
int cost_volume_typed(const char* fn, const float* keyframe, const float* const* frames, const float* proj,
                      const float* depths, const float* pixel_depths, void* out_cv, void* out_sfcv, void* out_sfcv_nhwc,
                      int nhwc_dtype, int B, int F, int D, int H, int W, float alpha, const float* chan_w, int matching,
                      int centered, int out_dtype, int channels, void* stream) {
    MR_REQUIRE(channels == 1 || channels == 3, "%s: channels must be 1 or 3 (got %d)", fn, channels);
    MR_REQUIRE(out_dtype == MR_DT_F32 || out_dtype == MR_DT_F16, "%s: out_dtype must be MR_DT_F32 or MR_DT_F16 (got %d)", fn,
               out_dtype);
    const int rc = check_general_args(fn, depths, pixel_depths, nhwc_dtype, F, D, matching, centered);
    if (rc != MR_OK) return rc;
    // the march stores two columns at once: 8 bytes (fp32) / 4 bytes (half)
    const uintptr_t align = out_dtype == MR_DT_F16 ? 3 : 7;
    MR_REQUIRE(out_cv != nullptr && (reinterpret_cast<uintptr_t>(out_cv) & align) == 0,
               "%s: out_cv must be a non-null, %d-byte aligned buffer", fn, (int)align + 1);
    MR_REQUIRE(out_sfcv != nullptr && (reinterpret_cast<uintptr_t>(out_sfcv) & align) == 0,
               "%s: out_sfcv must be a non-null, %d-byte aligned buffer", fn, (int)align + 1);
    const int pix = pixel_depths != nullptr;
    return mr::launch_cost_volume(keyframe, frames, proj, pix ? pixel_depths : depths, out_cv, out_sfcv, B, F, D, H, W, alpha,
                                  chan_w, 0, B, 0, (cudaStream_t)stream, out_sfcv_nhwc, nhwc_dtype, pix, matching, centered,
                                  out_dtype, channels);
}
}  // namespace

extern "C" int mr_cost_volume_fwd_typed(const float* keyframe, const float* const* frames, const float* proj,
                                        const float* depths, const float* pixel_depths, void* out_cv, void* out_sfcv,
                                        void* out_sfcv_nhwc, int nhwc_dtype, int B, int F, int D, int H, int W, float alpha,
                                        const float* chan_w, int matching, int centered, int out_dtype, void* stream) {
    return cost_volume_typed("mr_cost_volume_fwd_typed", keyframe, frames, proj, depths, pixel_depths, out_cv, out_sfcv,
                             out_sfcv_nhwc, nhwc_dtype, B, F, D, H, W, alpha, chan_w, matching, centered, out_dtype, 3, stream);
}

extern "C" int mr_cost_volume_fwd_channels(const float* keyframe, const float* const* frames, const float* proj,
                                           const float* depths, const float* pixel_depths, void* out_cv, void* out_sfcv,
                                           void* out_sfcv_nhwc, int nhwc_dtype, int B, int F, int D, int H, int W,
                                           float alpha, const float* chan_w, int matching, int centered, int out_dtype,
                                           int channels, void* stream) {
    return cost_volume_typed("mr_cost_volume_fwd_channels", keyframe, frames, proj, depths, pixel_depths, out_cv, out_sfcv,
                             out_sfcv_nhwc, nhwc_dtype, B, F, D, H, W, alpha, chan_w, matching, centered, out_dtype, channels,
                             stream);
}
