// Convolution engine, CUDA-core fp32 path (sm_90a).  See include/monorec_b200.h (mr_conv_desc) for what one call fuses:
// TF-"SAME" padding, channel concatenation of up to three sources, nearest x2 upsampling on read, bias, activation and
// strided (sub-pixel) output placement.  NHWC activations, weights [kh][kw][Cin][Cout].
//
// Reference being replaced: PadSameConv2d + nn.Conv2d + LeakyReLU (model/layers.py:220-335), Upconv (:338-356),
// Refine / ConvTranspose2d (:380-400), the heads (monorec_model.py:340-343, :521-524, :554-557).
//
// Kernel shape: implicit GEMM.  A CTA owns an 8x16 tile of output pixels (M = 128) and TN output channels; the K loop
// runs over (tap, source, 16-channel chunk), staging A (pixels x channels, gathered with zero fill) and B (channels x
// Cout) through shared memory; each thread accumulates 4 pixels x TN/8 channels in registers.
#include "mr_common.cuh"
#include <cstdint>
#include <cuda_fp16.h>

namespace {

constexpr int kTileH = 8, kTileW = 16, kTileP = kTileH * kTileW;  // 128 output pixels per CTA
constexpr int kKC = 16;                                           // channels per K chunk
constexpr int kConvThreads = 256;

__device__ __forceinline__ float apply_act(float v, int act, float a, float b) {
    switch (act) {
        case MR_ACT_LEAKY: return v >= 0.f ? v : a * v;
        case MR_ACT_SIGMOID: return 1.0f / (1.0f + expf(-v));
        case MR_ACT_ABSTANH: return fmaf(b, fabsf(tanhf(v)), a);
        default: return v;
    }
}

template <int TN>
__global__ void __launch_bounds__(kConvThreads) conv2d_nhwc_kernel(const mr_conv_desc d, const int cin_total) {
    constexpr int CH = TN / 8;  // channels per thread (8 channel groups)
    __shared__ __align__(16) float As[kKC][kTileP];
    __shared__ __align__(16) float Bs[kKC][TN];

    const int tid = threadIdx.x;
    const int tiles_x = (d.Wo + kTileW - 1) / kTileW;
    const int tile_y = blockIdx.x / tiles_x, tile_x = blockIdx.x - tile_y * tiles_x;
    const int n0 = blockIdx.y * TN;
    const int b = blockIdx.z;
    const int oy0 = tile_y * kTileH, ox0 = tile_x * kTileW;
    const int Hv = d.upsample2 ? 2 * d.Hs : d.Hs, Wv = d.upsample2 ? 2 * d.Ws : d.Ws;  // virtual input size

    // staging role: this thread gathers channel quad `aq` (and aq + 2) of pixel `ap`
    const int ap = tid & (kTileP - 1), aq = tid >> 7;
    const int apy = oy0 + (ap >> 4), apx = ox0 + (ap & 15);
    // compute role: 4 consecutive pixels x CH consecutive channels
    const int cg = tid & 7, pg = tid >> 3;

    float acc[4][CH];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < CH; ++j) acc[i][j] = 0.f;

    for (int ky = 0; ky < d.kh; ++ky) {
        for (int kx = 0; kx < d.kw; ++kx) {
            int iy = apy * d.sy - d.pad_t + ky, ix = apx * d.sx - d.pad_l + kx;
            const bool inside = (iy >= 0) && (iy < Hv) && (ix >= 0) && (ix < Wv) && (apy < d.Ho) && (apx < d.Wo);
            if (d.upsample2) { iy >>= 1; ix >>= 1; }
            const size_t pix = ((size_t)b * d.Hs + iy) * d.Ws + ix;
            int cbase = 0;  // channel offset of the current source inside the concatenation
            for (int s = 0; s < d.n_src; ++s) {
                const int C = d.src_c[s];
                const float* sp = d.src[s] + pix * C;
                const bool vec_ok = (C & 3) == 0;
                for (int c0 = 0; c0 < C; c0 += kKC) {
                    // ---- stage A: 128 pixels x 16 channels (zero fill outside the image / beyond C) ----
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int cq = c0 + 4 * (aq + 2 * h);
                        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                        if (inside) {
                            if (vec_ok && cq + 4 <= C) {
                                v = __ldg(reinterpret_cast<const float4*>(sp + cq));
                            } else {
                                if (cq + 0 < C) v.x = __ldg(sp + cq + 0);
                                if (cq + 1 < C) v.y = __ldg(sp + cq + 1);
                                if (cq + 2 < C) v.z = __ldg(sp + cq + 2);
                                if (cq + 3 < C) v.w = __ldg(sp + cq + 3);
                            }
                        }
                        const int kq = 4 * (aq + 2 * h);
                        As[kq + 0][ap] = v.x; As[kq + 1][ap] = v.y; As[kq + 2][ap] = v.z; As[kq + 3][ap] = v.w;
                    }
                    // ---- stage B: 16 channels x TN output channels ----
                    const float* wrow = d.weight + ((size_t)(ky * d.kw + kx) * cin_total + cbase + c0) * d.Cout + n0;
                    for (int i = tid; i < kKC * TN; i += kConvThreads) {
                        const int k = i / TN, n = i - k * TN;
                        float w = 0.f;
                        if (c0 + k < C && n0 + n < d.Cout) w = __ldg(wrow + (size_t)k * d.Cout + n);
                        Bs[k][n] = w;
                    }
                    __syncthreads();
#pragma unroll
                    for (int k = 0; k < kKC; ++k) {
                        const float4 a4 = *reinterpret_cast<const float4*>(&As[k][4 * pg]);
                        float bv[CH];
#pragma unroll
                        for (int j = 0; j < CH; j += 4) {
                            const float4 b4 = *reinterpret_cast<const float4*>(&Bs[k][CH * cg + j]);
                            bv[j] = b4.x; bv[j + 1] = b4.y; bv[j + 2] = b4.z; bv[j + 3] = b4.w;
                        }
#pragma unroll
                        for (int j = 0; j < CH; ++j) {
                            acc[0][j] = fmaf(a4.x, bv[j], acc[0][j]);
                            acc[1][j] = fmaf(a4.y, bv[j], acc[1][j]);
                            acc[2][j] = fmaf(a4.z, bv[j], acc[2][j]);
                            acc[3][j] = fmaf(a4.w, bv[j], acc[3][j]);
                        }
                    }
                    __syncthreads();
                }
                cbase += C;
            }
        }
    }

    // ---- epilogue: bias, activation, NHWC store into the channel slice of the destination ----
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int p = 4 * pg + i;
        const int oy = oy0 + (p >> 4), ox = ox0 + (p & 15);
        if (oy >= d.Ho || ox >= d.Wo) continue;
        const int dy = oy * d.oy_step + d.oy_off, dx = ox * d.ox_step + d.ox_off;
        float* op = d.dst + (((size_t)b * d.dst_H + dy) * d.dst_W + dx) * d.dst_c + d.dst_coff + n0 + CH * cg;
#pragma unroll
        for (int j = 0; j < CH; ++j) {
            const int n = n0 + CH * cg + j;
            if (n < d.Cout) {
                float v = acc[i][j] + (d.bias ? __ldg(d.bias + n) : 0.f);
                op[j] = apply_act(v, d.act, d.act_a, d.act_b);
            }
        }
    }
}

// Single-output-channel layers (1x1 mask classifier, 3x3 depth heads: monorec_model.py:340-343, :521-524): a per-pixel dot
// product, HBM-bound -- not a dense contraction, so no tensor cores and no 32-wide channel tile.  One thread per output
// pixel, float4 channel loads (adjacent pixels are adjacent in NHWC, so a warp streams one contiguous block per filter row).
__device__ __forceinline__ float4 ld4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ float4 ld4(const __half* p) {
    const uint2 u = __ldg(reinterpret_cast<const uint2*>(p));
    const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&u.x)), b = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
    return make_float4(a.x, a.y, b.x, b.y);
}

template <typename T>
__global__ void __launch_bounds__(256) conv_cout1_kernel(const mr_conv_desc d) {
    extern __shared__ float wsm[];   // [kh*kw][C]
    const int C = d.src_c[0];
    const int nw = d.kh * d.kw * C;
    for (int i = threadIdx.x; i < nw; i += blockDim.x) wsm[i] = __ldg(d.weight + i);
    __syncthreads();
    const size_t total = (size_t)d.B * d.Ho * d.Wo;
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const int ox = (int)(idx % d.Wo);
    const int oy = (int)((idx / d.Wo) % d.Ho);
    const int b = (int)(idx / ((size_t)d.Wo * d.Ho));
    float acc0 = 0.f, acc1 = 0.f, acc2 = 0.f, acc3 = 0.f;
    for (int ky = 0; ky < d.kh; ++ky) {
        const int iy = oy * d.sy - d.pad_t + ky;
        if (iy < 0 || iy >= d.Hs) continue;
        for (int kx = 0; kx < d.kw; ++kx) {
            const int ix = ox * d.sx - d.pad_l + kx;
            if (ix < 0 || ix >= d.Ws) continue;
            const T* p = reinterpret_cast<const T*>(d.src[0]) + (((size_t)b * d.Hs + iy) * d.Ws + ix) * C;
            const float4* w = reinterpret_cast<const float4*>(wsm + (ky * d.kw + kx) * C);
            for (int c = 0; c < C / 4; ++c) {
                const float4 v = ld4(p + 4 * c), q = w[c];
                acc0 = fmaf(v.x, q.x, acc0); acc1 = fmaf(v.y, q.y, acc1);
                acc2 = fmaf(v.z, q.z, acc2); acc3 = fmaf(v.w, q.w, acc3);
            }
        }
    }
    float v = (acc0 + acc1) + (acc2 + acc3) + (d.bias ? __ldg(d.bias) : 0.f);
    const int dy = oy * d.oy_step + d.oy_off, dx = ox * d.ox_step + d.ox_off;
    d.dst[(((size_t)b * d.dst_H + dy) * d.dst_W + dx) * d.dst_c + d.dst_coff] = apply_act(v, d.act, d.act_a, d.act_b);
}

__device__ __forceinline__ void st1(float* p, float v) { *p = v; }
__device__ __forceinline__ void st1(__half* p, float v) { *p = __float2half_rn(v); }

// source element widened to fp32 (the half cost volumes of mr_cost_volume_fwd_typed)
__device__ __forceinline__ float ld1(const float* p) { return __ldg(p); }
__device__ __forceinline__ float ld1(const __half* p) { return __half2float(__ldg(p)); }

template <typename T, typename S>
__global__ void nchw_to_nhwc_kernel(const S* __restrict__ src, T* __restrict__ dst, int C, int HW, int dst_c,
                                    int dst_coff, const float* __restrict__ oms) {
    // one CTA: 32 pixels x 32 channels tile transposed through shared memory (coalesced on both sides)
    __shared__ float t[32][33];
    const int b = blockIdx.z, p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    const int tx = threadIdx.x, ty = threadIdx.y;  // 32 x 8
    for (int j = ty; j < 32; j += 8) {
        const int c = c0 + j, p = p0 + tx;
        t[j][tx] = (c < C && p < HW) ? ld1(src + ((size_t)b * C + c) * HW + p) : 0.f;
    }
    __syncthreads();
    for (int j = ty; j < 32; j += 8) {
        const int p = p0 + j, c = c0 + tx;
        if (p < HW && c < C) {
            float v = t[tx][j];
            if (oms) v *= 1.0f - __ldg(oms + (size_t)b * HW + p);
            st1(dst + ((size_t)b * HW + p) * dst_c + dst_coff + c, v);
        }
    }
}

// Half-precision fast path of the layout change (C % 32 == 0, HW % 128 == 0, 16-byte aligned channel slice): a CTA moves
// 32 channels x 128 pixels; 128-byte coalesced reads per channel row, conflict-free shared-memory transpose (pitch 129),
// one 16-byte store (8 channels) per thread so that a warp writes 8 pixels x 64 contiguous bytes.
template <typename S>
__global__ void __launch_bounds__(256)
nchw_to_nhwc_f16_tile_kernel(const S* __restrict__ src, __half* __restrict__ dst, int C, int HW, int dst_c, int dst_coff,
                             const float* __restrict__ oms) {
    __shared__ float t[32][129];
    const int b = blockIdx.z, p0 = blockIdx.x * 128, c0 = blockIdx.y * 32;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int j = warp; j < 32; j += 8) {
        const S* s = src + ((size_t)b * C + c0 + j) * HW + p0 + lane;
#pragma unroll
        for (int k = 0; k < 4; ++k) t[j][lane + 32 * k] = ld1(s + 32 * k);
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int i = threadIdx.x + 256 * r, p = i >> 2, g = i & 3;
        uint4 q;
        __half2* h = reinterpret_cast<__half2*>(&q);
        if (oms) {   // same operation order as the generic kernel: v * (1 - m), then round
            const float sc = 1.0f - __ldg(oms + (size_t)b * HW + p0 + p);
#pragma unroll
            for (int j = 0; j < 4; ++j) h[j] = __floats2half2_rn(t[8 * g + 2 * j][p] * sc, t[8 * g + 2 * j + 1][p] * sc);
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) h[j] = __floats2half2_rn(t[8 * g + 2 * j][p], t[8 * g + 2 * j + 1][p]);
        }
        *reinterpret_cast<uint4*>(dst + ((size_t)b * HW + p0 + p) * dst_c + dst_coff + c0 + 8 * g) = q;
    }
}

template <typename T>
__global__ void mask_volume_kernel(const T* __restrict__ vol, const float* __restrict__ mask,
                                   T* __restrict__ out, int D, int HW, size_t total) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const size_t b = i / ((size_t)D * HW);
    const int p = (int)(i % HW);
    st1(out + i, (1.0f - __ldg(mask + b * HW + p)) * ld1(vol + i));
}

// the layout change for a source of type S: the half tile kernel when the destination is half and the slice is aligned for
// its 16-byte stores, else the generic kernel
template <typename S>
int nchw_to_nhwc_launch(const S* src, void* dst, int dst_dtype, int B, int C, int HW, int dst_c, int dst_coff, const float* oms,
                        cudaStream_t st) {
    if (dst_dtype == MR_DT_F16 && C % 32 == 0 && HW % 128 == 0 && dst_c % 8 == 0 && dst_coff % 8 == 0 &&
        (reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
        dim3 tgrid(HW / 128, C / 32, B);
        nchw_to_nhwc_f16_tile_kernel<S><<<tgrid, 256, 0, st>>>(src, static_cast<__half*>(dst), C, HW, dst_c, dst_coff, oms);
        MR_LAUNCH_CHECK("nchw_to_nhwc_f16_tile_kernel");
        return MR_OK;
    }
    dim3 grid((HW + 31) / 32, (C + 31) / 32, B), block(32, 8);
    if (dst_dtype == MR_DT_F16)
        nchw_to_nhwc_kernel<__half, S><<<grid, block, 0, st>>>(src, static_cast<__half*>(dst), C, HW, dst_c, dst_coff, oms);
    else
        nchw_to_nhwc_kernel<float, S><<<grid, block, 0, st>>>(src, static_cast<float*>(dst), C, HW, dst_c, dst_coff, oms);
    MR_LAUNCH_CHECK("nchw_to_nhwc_kernel");
    return MR_OK;
}

}  // namespace

extern "C" int mr_mask_volume(const void* volume, const float* mask, void* out, int dtype, int B, int D, int HW, void* stream) {
    MR_REQUIRE(dtype == MR_DT_F32 || dtype == MR_DT_F16, "mr_mask_volume: dtype must be MR_DT_F32 or MR_DT_F16 (got %d)", dtype);
    MR_REQUIRE(volume && mask && out && B >= 1 && D >= 1 && HW >= 1, "mr_mask_volume: bad argument");
    const size_t total = (size_t)B * D * HW;
    const unsigned grid = (unsigned)((total + 255) / 256);
    if (dtype == MR_DT_F16)
        mask_volume_kernel<__half><<<grid, 256, 0, (cudaStream_t)stream>>>(static_cast<const __half*>(volume), mask,
                                                                           static_cast<__half*>(out), D, HW, total);
    else
        mask_volume_kernel<float><<<grid, 256, 0, (cudaStream_t)stream>>>(static_cast<const float*>(volume), mask,
                                                                          static_cast<float*>(out), D, HW, total);
    MR_LAUNCH_CHECK("mask_volume_kernel");
    return MR_OK;
}

extern "C" int mr_sizeof_conv_desc(void) { return (int)sizeof(mr_conv_desc); }

extern "C" int mr_conv2d_nhwc(const mr_conv_desc* desc, void* stream) {
    MR_REQUIRE(desc != nullptr, "mr_conv2d_nhwc: null descriptor");
    const mr_conv_desc& d = *desc;
    MR_REQUIRE(d.n_src >= 1 && d.n_src <= MR_CONV_MAX_SRC, "mr_conv2d_nhwc: n_src=%d out of range", d.n_src);
    int cin = 0;
    for (int s = 0; s < d.n_src; ++s) {
        MR_REQUIRE(d.src[s] != nullptr && d.src_c[s] >= 1, "mr_conv2d_nhwc: bad source %d", s);
        cin += d.src_c[s];
    }
    MR_REQUIRE(d.weight && d.dst, "mr_conv2d_nhwc: null weight/dst");
    MR_REQUIRE(d.B >= 1 && d.B <= 65535 && d.Hs >= 1 && d.Ws >= 1 && d.Ho >= 1 && d.Wo >= 1 && d.Cout >= 1,
               "mr_conv2d_nhwc: bad shape");
    MR_REQUIRE(d.kh >= 1 && d.kw >= 1 && d.sy >= 1 && d.sx >= 1 && d.oy_step >= 1 && d.ox_step >= 1,
               "mr_conv2d_nhwc: bad kernel/stride");
    MR_REQUIRE(d.dst_coff >= 0 && d.dst_coff + d.Cout <= d.dst_c, "mr_conv2d_nhwc: channel slice out of range");
    MR_REQUIRE(d.oy_off >= 0 && d.ox_off >= 0, "mr_conv2d_nhwc: oy_off=%d / ox_off=%d must be >= 0", d.oy_off, d.ox_off);
    MR_REQUIRE((d.Ho - 1) * d.oy_step + d.oy_off < d.dst_H && (d.Wo - 1) * d.ox_step + d.ox_off < d.dst_W,
               "mr_conv2d_nhwc: output placement out of range");
    MR_REQUIRE(d.act >= MR_ACT_NONE && d.act <= MR_ACT_ABSTANH, "mr_conv2d_nhwc: unknown activation %d", d.act);
    if (d.Cout == 1 && d.n_src == 1 && !d.upsample2 && (d.src_c[0] % 4) == 0 && d.kh * d.kw * d.src_c[0] * 4 <= 40 * 1024) {
        const size_t total = (size_t)d.B * d.Ho * d.Wo;
        MR_REQUIRE(d.dst_dtype == MR_DT_F32, "mr_conv2d_nhwc: the single-channel heads write fp32");
        if (d.src_dtype == MR_DT_F16)
            conv_cout1_kernel<__half><<<(unsigned)((total + 255) / 256), 256, (size_t)d.kh * d.kw * d.src_c[0] * 4, (cudaStream_t)stream>>>(d);
        else
            conv_cout1_kernel<float><<<(unsigned)((total + 255) / 256), 256, (size_t)d.kh * d.kw * d.src_c[0] * 4, (cudaStream_t)stream>>>(d);
        MR_LAUNCH_CHECK("conv_cout1_kernel");
        return MR_OK;
    }
    MR_REQUIRE(d.src_dtype == MR_DT_F32 && d.dst_dtype == MR_DT_F32, "mr_conv2d_nhwc: the CUDA-core kernel is fp32 only");
    const int tiles = ((d.Ho + kTileH - 1) / kTileH) * ((d.Wo + kTileW - 1) / kTileW);
    // the per-thread float4 weight reads need Cout-tile-aligned rows: TN=64 only when Cout is a multiple of 4
    if (d.Cout >= 64 && d.Cout % 4 == 0) {
        dim3 grid(tiles, (d.Cout + 63) / 64, d.B);
        conv2d_nhwc_kernel<64><<<grid, kConvThreads, 0, (cudaStream_t)stream>>>(d, cin);
    } else {
        dim3 grid(tiles, (d.Cout + 31) / 32, d.B);
        conv2d_nhwc_kernel<32><<<grid, kConvThreads, 0, (cudaStream_t)stream>>>(d, cin);
    }
    MR_LAUNCH_CHECK("conv2d_nhwc_kernel");
    return MR_OK;
}

extern "C" int mr_nchw_to_nhwc(const void* src, int src_dtype, void* dst, int dst_dtype, int B, int C, int H, int W, int dst_c,
                               int dst_coff, const float* one_minus_scale, void* stream) {
    MR_REQUIRE(src_dtype == MR_DT_F32 || src_dtype == MR_DT_F16, "mr_nchw_to_nhwc: src_dtype must be MR_DT_F32 or MR_DT_F16 (got %d)",
               src_dtype);
    MR_REQUIRE(dst_dtype == MR_DT_F32 || dst_dtype == MR_DT_F16, "mr_nchw_to_nhwc: dst_dtype must be MR_DT_F32 or MR_DT_F16 (got %d)",
               dst_dtype);
    MR_REQUIRE(src && dst && B >= 1 && C >= 1 && H >= 1 && W >= 1, "mr_nchw_to_nhwc: bad argument");
    MR_REQUIRE(dst_coff >= 0 && dst_coff + C <= dst_c, "mr_nchw_to_nhwc: channel slice out of range");
    if (src_dtype == MR_DT_F16)
        return nchw_to_nhwc_launch(static_cast<const __half*>(src), dst, dst_dtype, B, C, H * W, dst_c, dst_coff, one_minus_scale,
                                   (cudaStream_t)stream);
    return nchw_to_nhwc_launch(static_cast<const float*>(src), dst, dst_dtype, B, C, H * W, dst_c, dst_coff, one_minus_scale,
                               (cudaStream_t)stream);
}

namespace {
// element-wise max of two channel vectors: VEC = uint4 (8 half) or float4 (4 fp32)
template <typename VEC, bool HALF>
__device__ __forceinline__ VEC vmax(const VEC a, const VEC b) {
    VEC o;
    if (HALF) {
        const __half2* ah = reinterpret_cast<const __half2*>(&a);
        const __half2* bh = reinterpret_cast<const __half2*>(&b);
        __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
        for (int k = 0; k < 4; ++k) oh[k] = __hmax2(ah[k], bh[k]);
    } else {
        const float* af = reinterpret_cast<const float*>(&a);
        const float* bf = reinterpret_cast<const float*>(&b);
        float* of = reinterpret_cast<float*>(&o);
#pragma unroll
        for (int k = 0; k < 4; ++k) of[k] = fmaxf(af[k], bf[k]);
    }
    return o;
}
// nn.MaxPool2d(2) (monorec_model.py:304-316) and the element-wise max over the leading frame axis (:362-365) on NHWC tensors
template <typename VEC, bool HALF>
__global__ void maxpool2_nhwc_kernel(const VEC* __restrict__ src, VEC* __restrict__ dst, int H, int W, int CV, size_t total) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int Wo = W / 2, Ho = H / 2;
    const int c = (int)(i % CV);
    size_t r = i / CV;
    const int x = (int)(r % Wo); r /= Wo;
    const int y = (int)(r % Ho);
    const size_t b = r / Ho;
    const VEC* p = src + ((b * H + 2 * y) * W + 2 * x) * CV + c;
    const VEC q0 = __ldg(p), q1 = __ldg(p + CV), q2 = __ldg(p + (size_t)W * CV), q3 = __ldg(p + (size_t)W * CV + CV);
    dst[i] = vmax<VEC, HALF>(vmax<VEC, HALF>(q0, q1), vmax<VEC, HALF>(q2, q3));
}
template <typename VEC, bool HALF>
__global__ void max_over_frames_kernel(const VEC* __restrict__ src, VEC* __restrict__ dst, int F, size_t n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    VEC m = __ldg(src + i);
    for (int f = 1; f < F; ++f) m = vmax<VEC, HALF>(m, __ldg(src + (size_t)f * n + i));
    dst[i] = m;
}
// MaskModule encoder, between two levels (monorec_model.py:357-365 with :304-316): the level's output x [F*B,H,W,C] feeds both
// the element-wise max over the frames (-> decoder skip connection) and the 2x2 max-pool (-> next level).  One pass over x
// writes both (the two kernels above read the 268 MB level-0 tensor twice).
template <typename VEC, bool HALF>
__global__ void pool_and_frame_max_kernel(const VEC* __restrict__ src, VEC* __restrict__ pooled, VEC* __restrict__ fmax, int F, int B,
                                          int H, int W, int CV, size_t total) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;   // over (b, y/2, x/2, channel vector)
    if (i >= total) return;
    const int Wo = W / 2, Ho = H / 2;
    const int c = (int)(i % CV);
    size_t r = i / CV;
    const int x = (int)(r % Wo); r /= Wo;
    const int y = (int)(r % Ho);
    const size_t b = r / Ho;
    const size_t frame = (size_t)B * H * W * CV, frame_o = (size_t)B * Ho * Wo * CV;
    const size_t o00 = ((b * H + 2 * y) * W + 2 * x) * CV + c, oo = ((b * Ho + y) * Wo + x) * CV + c;
    VEC m[4];
    for (int f = 0; f < F; ++f) {
        const VEC* p = src + (size_t)f * frame + o00;
        const VEC q0 = __ldg(p), q1 = __ldg(p + CV), q2 = __ldg(p + (size_t)W * CV), q3 = __ldg(p + (size_t)W * CV + CV);
        pooled[(size_t)f * frame_o + oo] = vmax<VEC, HALF>(vmax<VEC, HALF>(q0, q1), vmax<VEC, HALF>(q2, q3));
        if (f == 0) { m[0] = q0; m[1] = q1; m[2] = q2; m[3] = q3; }
        else { m[0] = vmax<VEC, HALF>(m[0], q0); m[1] = vmax<VEC, HALF>(m[1], q1); m[2] = vmax<VEC, HALF>(m[2], q2); m[3] = vmax<VEC, HALF>(m[3], q3); }
    }
    VEC* d = fmax + o00;
    d[0] = m[0]; d[CV] = m[1]; d[(size_t)W * CV] = m[2]; d[(size_t)W * CV + CV] = m[3];
}
// ResNet stem max-pool (torchvision resnet18.maxpool = MaxPool2d(3, stride 2, padding 1), monorec_model.py:122) on an NHWC
// (channels-last) tensor: ATen's max_pool_forward_nhwc needs 75 us for the 64-channel half stem output of a batch of 8
// (33.5 MB in, 8.4 MB out: 14 us of HBM time).  Window taps outside the image are skipped (= -inf padding).
template <typename VEC, bool HALF>
__global__ void maxpool3s2_nhwc_kernel(const VEC* __restrict__ src, VEC* __restrict__ dst, int H, int W, int Ho, int Wo, int CV,
                                       size_t total) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int c = (int)(i % CV);
    size_t r = i / CV;
    const int x = (int)(r % Wo); r /= Wo;
    const int y = (int)(r % Ho);
    const size_t b = r / Ho;
    const int y0 = max(2 * y - 1, 0), y1 = min(2 * y + 1, H - 1), x0 = max(2 * x - 1, 0), x1 = min(2 * x + 1, W - 1);
    VEC m = __ldg(src + ((b * H + y0) * W + x0) * CV + c);
    for (int yy = y0; yy <= y1; ++yy)
        for (int xx = x0; xx <= x1; ++xx) m = vmax<VEC, HALF>(m, __ldg(src + ((b * H + yy) * W + xx) * CV + c));
    dst[i] = m;
}
__global__ void cast_f32_to_f16_kernel(const float4* __restrict__ src, uint2* __restrict__ dst, size_t n4) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n4) return;
    const float4 v = __ldg(src + i);
    uint2 o;
    *reinterpret_cast<__half2*>(&o.x) = __floats2half2_rn(v.x, v.y);
    *reinterpret_cast<__half2*>(&o.y) = __floats2half2_rn(v.z, v.w);
    dst[i] = o;
}
}  // namespace

extern "C" int mr_pool_and_frame_max(const void* src, void* pooled, void* frame_max, int dtype, int F, int B, int H, int W, int C,
                                     void* stream) {
    const int v = dtype == MR_DT_F16 ? 8 : 4;
    MR_REQUIRE(src && pooled && frame_max && (dtype == MR_DT_F16 || dtype == MR_DT_F32) && F >= 1 && B >= 1 && C >= v && (C % v) == 0 &&
                   H >= 2 && W >= 2 && (H % 2) == 0 && (W % 2) == 0,
               "mr_pool_and_frame_max: need even H, W and C %% %d == 0 (got F=%d B=%d H=%d W=%d C=%d)", v, F, B, H, W, C);
    const size_t total = (size_t)B * (H / 2) * (W / 2) * (C / v);
    const unsigned grid = (unsigned)((total + 255) / 256);
    if (dtype == MR_DT_F16)
        pool_and_frame_max_kernel<uint4, true><<<grid, 256, 0, (cudaStream_t)stream>>>(
            static_cast<const uint4*>(src), static_cast<uint4*>(pooled), static_cast<uint4*>(frame_max), F, B, H, W, C / v, total);
    else
        pool_and_frame_max_kernel<float4, false><<<grid, 256, 0, (cudaStream_t)stream>>>(
            static_cast<const float4*>(src), static_cast<float4*>(pooled), static_cast<float4*>(frame_max), F, B, H, W, C / v, total);
    MR_LAUNCH_CHECK("pool_and_frame_max_kernel");
    return MR_OK;
}

extern "C" int mr_maxpool3s2_nhwc(const void* src, void* dst, int dtype, int B, int H, int W, int C, void* stream) {
    const int v = dtype == MR_DT_F16 ? 8 : 4;
    MR_REQUIRE(src && dst && (dtype == MR_DT_F16 || dtype == MR_DT_F32) && B >= 1 && H >= 1 && W >= 1 && C >= v && (C % v) == 0,
               "mr_maxpool3s2_nhwc: need C %% %d == 0 (got B=%d H=%d W=%d C=%d)", v, B, H, W, C);
    const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
    const size_t total = (size_t)B * Ho * Wo * (C / v);
    const unsigned grid = (unsigned)((total + 255) / 256);
    if (dtype == MR_DT_F16)
        maxpool3s2_nhwc_kernel<uint4, true><<<grid, 256, 0, (cudaStream_t)stream>>>(static_cast<const uint4*>(src), static_cast<uint4*>(dst),
                                                                                    H, W, Ho, Wo, C / v, total);
    else
        maxpool3s2_nhwc_kernel<float4, false><<<grid, 256, 0, (cudaStream_t)stream>>>(static_cast<const float4*>(src),
                                                                                      static_cast<float4*>(dst), H, W, Ho, Wo, C / v, total);
    MR_LAUNCH_CHECK("maxpool3s2_nhwc_kernel");
    return MR_OK;
}

extern "C" int mr_cast_f32_to_f16(const float* src, void* dst, long long n, void* stream) {
    MR_REQUIRE(src && dst && n >= 4 && (n % 4) == 0, "mr_cast_f32_to_f16: n must be a positive multiple of 4");
    const size_t n4 = (size_t)n / 4;
    cast_f32_to_f16_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const float4*>(src), static_cast<uint2*>(dst), n4);
    MR_LAUNCH_CHECK("cast_f32_to_f16_kernel");
    return MR_OK;
}

extern "C" int mr_maxpool2_nhwc(const void* src, void* dst, int dtype, int B, int H, int W, int C, void* stream) {
    MR_REQUIRE(dtype == MR_DT_F32 || dtype == MR_DT_F16, "mr_maxpool2_nhwc: dtype must be MR_DT_F32 or MR_DT_F16 (got %d)", dtype);
    const int v = dtype == MR_DT_F16 ? 8 : 4;
    MR_REQUIRE(B >= 1 && C >= v && (C % v) == 0 && H >= 2 && W >= 2 && (H % 2) == 0 && (W % 2) == 0,
               "mr_maxpool2_nhwc: need even H, W and C %% %d == 0 (got B=%d H=%d W=%d C=%d)", v, B, H, W, C);
    MR_REQUIRE(src && dst, "mr_maxpool2_nhwc: null pointer (src, dst)");
    const size_t total = (size_t)B * (H / 2) * (W / 2) * (C / v);
    const unsigned grid = (unsigned)((total + 255) / 256);
    if (dtype == MR_DT_F16)
        maxpool2_nhwc_kernel<uint4, true><<<grid, 256, 0, (cudaStream_t)stream>>>(static_cast<const uint4*>(src), static_cast<uint4*>(dst),
                                                                                  H, W, C / v, total);
    else
        maxpool2_nhwc_kernel<float4, false><<<grid, 256, 0, (cudaStream_t)stream>>>(static_cast<const float4*>(src),
                                                                                    static_cast<float4*>(dst), H, W, C / v, total);
    MR_LAUNCH_CHECK("maxpool2_nhwc_kernel");
    return MR_OK;
}

extern "C" int mr_max_over_frames(const void* src, void* dst, int dtype, int F, long long n_per_frame, void* stream) {
    MR_REQUIRE(dtype == MR_DT_F32 || dtype == MR_DT_F16, "mr_max_over_frames: dtype must be MR_DT_F32 or MR_DT_F16 (got %d)", dtype);
    const int v = dtype == MR_DT_F16 ? 8 : 4;
    MR_REQUIRE(F >= 1 && n_per_frame >= v && (n_per_frame % v) == 0,
               "mr_max_over_frames: need F >= 1 and n_per_frame a positive multiple of %d (got F=%d n_per_frame=%lld)", v, F,
               n_per_frame);
    MR_REQUIRE(src && dst, "mr_max_over_frames: null pointer (src, dst)");
    const size_t n = (size_t)n_per_frame / v;
    const unsigned grid = (unsigned)((n + 255) / 256);
    if (dtype == MR_DT_F16)
        max_over_frames_kernel<uint4, true><<<grid, 256, 0, (cudaStream_t)stream>>>(static_cast<const uint4*>(src),
                                                                                    static_cast<uint4*>(dst), F, n);
    else
        max_over_frames_kernel<float4, false><<<grid, 256, 0, (cudaStream_t)stream>>>(static_cast<const float4*>(src),
                                                                                      static_cast<float4*>(dst), F, n);
    MR_LAUNCH_CHECK("max_over_frames_kernel");
    return MR_OK;
}
