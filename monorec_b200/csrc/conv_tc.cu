// Convolution engine, tensor-core path: implicit GEMM on Hopper warpgroup MMA (wgmma) for sm_90a.
//
//   D[128 pixels x Cout] (fp32, registers)  +=  A[128 pixels x 32 ch] (smem, TMA)  x  B[Cout x 32 ch]^T (smem, TMA)     tf32
//
// One CTA owns 128 output pixels and all Cout (MMA N = Cout padded to 16, <= 256).  The K loop runs over (filter tap,
// concatenated source, 32-channel chunk):
//   * the A operand of a tap is the NHWC input tile shifted by the tap offset, fetched by ONE 4-D TMA box
//     {32 ch, 16 px, 8 px, 1 img} (traversal stride = conv stride).  Out-of-bounds elements are zero-filled by the TMA unit,
//     which IS the reference's PadSameConv2d (model/layers.py:220-252); channel concatenation (torch.cat,
//     monorec_model.py:372-380, :541-545) is just one tensor map per source;
//   * the B operand is the matching [Cout x 32] slice of the packed weights (2-D TMA);
//   * both land in 128-byte-swizzled K-major shared-memory tiles that wgmma.mma_async reads through smem descriptors.
// Warp roles (288 threads): warps 0..7 = two consumer warpgroups, warpgroup g owns accumulator rows 64 g .. 64 g + 63 (one
// m64nNk8 / m64nNk16 chain each, accumulator in registers, then bias -> activation -> NHWC store, optional sub-pixel
// placement); warp 8 = TMA producer.  The producer loop runs on a CONVERGED warp with elect-predicated instructions (see
// tma_load_4d_elect): its operands stay in uniform registers.
// Pipeline: smem full/empty mbarrier ring between TMA and the consumers; one wgmma group stays in flight, and a stage is
// released (one arrival per warpgroup) once the group that read it has retired.  The kernels are persistent over output
// tiles, so the producer fills the next tile's stages while the consumers run an epilogue.
// MMA N is a template parameter (Cout padded to 16); it is issued as m64n256 / n128 / n64 / n32 / n16 pieces.
// Two kernels, chosen by the host code at the bottom of this file:
//   conv_tc_halo_kernel  stride-1 layers: ONE input box per (tile, K chunk) with its halo, every filter tap a shifted
//                        shared-memory descriptor into it; weights resident in shared memory, or -- when they do not fit
//                        next to two input stages -- streamed slice by slice through a second ring; 64- or 128-byte rows;
//   conv_tc_kernel       everything else (strided layers, the sub-pixel phases of Refine / Upconv -- up to four phases share
//                        one launch): one input box and one weight slice per (tap, K chunk).
// K steps that hold only the zero padding behind a source's channels are skipped.
//
// Reference being replaced: nn.Conv2d / nn.ConvTranspose2d + bias + LeakyReLU of model/layers.py:289-400 as used by
// MaskModule / DepthModule (model/monorec/monorec_model.py:287-385, :476-557).
#include "mr_common.cuh"
#include <cuda.h>
#include <cstdint>
#include <cstdlib>
#include <cuda_fp16.h>

namespace {

constexpr int kTcThreads = 288;
constexpr int kProducerWarp = 8;
constexpr int kKC = 32;                 // fp32 channels per K chunk = one 128-byte swizzle row
constexpr int kTileH = 8, kTileW = 16;  // 128 output pixels per CTA

struct TcArgs {
    int n_src;
    int chunks[MR_CONV_MAX_SRC];   // K chunks per source
    int tail_ksteps[MR_CONV_MAX_SRC];   // MMA K steps (32 bytes of channels each) that hold data in the LAST chunk of each source: the
                                        // zero padding behind a source's channels is neither multiplied nor read from shared memory
    int kh, kw, sy, sx, pad_t, pad_l;
    int Ho, Wo, Cout, n_pad, tiles_x, tiles_per_img, total_tiles, stages;
    const float* bias;
    float* dst;
    int dst_H, dst_W, dst_c, dst_coff, oy_step, ox_step, oy_off, ox_off;
    int act;
    float act_a, act_b;
    int round_out;                 // 1: round stored activations to TF32 (nearest) so the next layer's truncation is exact
    int kc;                        // channels per K chunk: 32 (fp32 sources, tf32 MMA) or 64 (half sources, f16 MMA)
    int out_f16;                   // half destination
    int row_bytes;                 // bytes of one K chunk row in shared memory = swizzle span: 128, or 64 (half sources, 32-channel chunks)
    // tap-refetch kernel: up to 4 "phases" (the sub-pixel convolutions of one Refine / Upconv layer) share one launch; tile
    // index = spatial tile * n_phase + phase, so the phases of a spatial tile run side by side and its input boxes are L2 hits
    int n_phase;
    int ph_kh[4], ph_kw[4], ph_pad_t[4], ph_pad_l[4], ph_oy_off[4], ph_ox_off[4];
    int b_stream;                  // halo kernel: 0 = the layer's weights stay resident in shared memory; n > 0 = they do not fit: the
                                   // [n_pad x chunk] slice of every (chunk, tap) streams through a ring of n stages instead
    int halo_pitch;                // halo kernel: pixels per input row of the shared-memory box (8 outputs + kw - 1 taps to the right)
    uint32_t halo_a_bytes;         // halo kernel: bytes of one input stage (box rounded up to 1 KB)
};

// ---- PTX wrappers -------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "DONE:\n\t"
        "}\n" ::"r"(bar), "r"(parity)
        : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}
// ---- single-lane instructions issued from a CONVERGED warp --------------------------------------------------------------
// All 32 lanes of the producer warp execute its loops (uniform arithmetic only) and the instruction itself is predicated on
// elect.sync: inside an `if (lane == 0)` region ptxas cannot keep the operands in uniform registers.
__device__ __forceinline__ void mbar_expect_tx_elect(uint32_t bar, uint32_t bytes) {
    asm volatile(
        "{\n\t"
        ".reg .pred pe;\n\t"
        "elect.sync _|pe, 0xffffffff;\n\t"
        "@pe mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n\t"
        "}\n" ::"r"(bar), "r"(bytes)
        : "memory");
}
__device__ __forceinline__ void tma_load_4d_elect(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2, int c3) {
    asm volatile(
        "{\n\t"
        ".reg .pred pe;\n\t"
        "elect.sync _|pe, 0xffffffff;\n\t"
        "@pe cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];\n\t"
        "}\n" ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}
__device__ __forceinline__ void tma_load_2d_elect(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
    asm volatile(
        "{\n\t"
        ".reg .pred pe;\n\t"
        "elect.sync _|pe, 0xffffffff;\n\t"
        "@pe cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];\n\t"
        "}\n" ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1)
        : "memory");
}

// K-major swizzled shared-memory matrix descriptor of wgmma:
//   [0,14) start address >> 4 | [16,30) leading byte offset >> 4 (1: unused for swizzled K-major) |
//   [32,46) stride byte offset >> 4 (distance between 8-row groups) | [49,52) base offset (0) | [62,64) layout: 1 = SWIZZLE_128B,
//   2 = SWIZZLE_64B.  The swizzle is a function of the absolute shared-memory address (as TMA writes it), so a start address
//   shifted by whole rows -- a filter tap inside the halo box -- needs no other field changed.  Everything but the start address
//   is layer-constant (desc_hi()); advancing the low word by n moves the start by 16 n bytes.
__device__ __forceinline__ uint32_t desc_lo(uint32_t saddr) { return ((saddr & 0x3FFFFu) >> 4) | (1u << 16); }
__device__ __forceinline__ uint32_t desc_hi(uint32_t sbo_bytes, uint32_t row_bytes) {
    return (sbo_bytes >> 4) | ((row_bytes == 128 ? 1u : 2u) << 30);
}
__device__ __forceinline__ uint64_t desc(uint32_t lo, uint32_t hi) { return ((uint64_t)hi << 32) | lo; }

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// m64nNk8 (tf32) / m64nNk16 (f16) with fp32 accumulators d[N / 2]; acc = 0 overwrites d (first K step of a tile)
template <int N, bool F16>
__device__ __forceinline__ void wgmma(float* d, uint64_t da, uint64_t db, uint32_t acc);

template <> __device__ __forceinline__ void wgmma<16, false>(float* d, uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7}, "
        "%8, %9, p, 1, 1;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(da), "l"(db), "r"(acc));
}
template <> __device__ __forceinline__ void wgmma<16, true>(float* d, uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7}, "
        "%8, %9, p, 1, 1, 0, 0;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(da), "l"(db), "r"(acc));
}
template <> __device__ __forceinline__ void wgmma<32, false>(float* d, uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
        "%16, %17, p, 1, 1;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(da), "l"(db), "r"(acc));
}
template <> __device__ __forceinline__ void wgmma<32, true>(float* d, uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
        "%16, %17, p, 1, 1, 0, 0;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(da), "l"(db), "r"(acc));
}
template <> __device__ __forceinline__ void wgmma<64, false>(float* d, uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "%32, %33, p, 1, 1;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(acc));
}
template <> __device__ __forceinline__ void wgmma<64, true>(float* d, uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "%32, %33, p, 1, 1, 0, 0;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(acc));
}
template <> __device__ __forceinline__ void wgmma<128, false>(float* d, uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(acc));
}
template <> __device__ __forceinline__ void wgmma<128, true>(float* d, uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1, 0, 0;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(acc));
}
template <> __device__ __forceinline__ void wgmma<256, false>(float* d, uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
        "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
        "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
        "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
        "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
        "%128, %129, p, 1, 1;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
          "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
          "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
          "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
          "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
          "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
          "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
          "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
          "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(da), "l"(db), "r"(acc));
}
template <> __device__ __forceinline__ void wgmma<256, true>(float* d, uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
        "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
        "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
        "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
        "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
        "%128, %129, p, 1, 1, 0, 0;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
          "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
          "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
          "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
          "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
          "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
          "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
          "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
          "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(da), "l"(db), "r"(acc));
}

// The whole accumulator row block [64 x N] as descending power-of-two pieces (N = 48 -> n32 + n16): piece p reads the weight
// rows [n0, n0 + p) (descriptor start advanced by n0 rows of b_row16 * 16 bytes) into d[n0 / 2 ..).
template <int N, bool F16>
__device__ __forceinline__ void mma_tile(float* d, uint64_t da, uint64_t db, uint32_t b_row16, uint32_t acc) {
    constexpr int P = N >= 256 ? 256 : N >= 128 ? 128 : N >= 64 ? 64 : N >= 32 ? 32 : 16;
    wgmma<P, F16>(d, da, db, acc);
    if constexpr (N > P) mma_tile<N - P, F16>(d + P / 2, da, db + (uint64_t)(P * b_row16), b_row16, acc);
}

__device__ __forceinline__ float act_fn(float v, int act, float a, float b) {
    switch (act) {
        case MR_ACT_LEAKY: return v >= 0.f ? v : a * v;
        case MR_ACT_SIGMOID: return 1.0f / (1.0f + expf(-v));
        case MR_ACT_ABSTANH: return fmaf(b, fabsf(tanhf(v)), a);
        default: return v;
    }
}

// Epilogue of one warpgroup's 64 accumulator rows.  wgmma fragment: warp w of the warpgroup holds rows 16 w + lane / 4 (+ 8),
// d[4 j + 2 i + c] is row 16 w + lane / 4 + 8 i, column 8 j + 2 (lane % 4) + c.  Row p of the tile is pixel (p / TW, p % TW).
// Bias from shared memory, activation, optional TF32 rounding; two adjacent channels per store (4 lanes = 8 channels).
template <int N, int TW, int TH>
__device__ __forceinline__ void epilogue_wg(const float* d, const TcArgs& a, const float* bias_s, int p0, int lane, int b, int tile_y,
                                            int tile_x, int oy_off, int ox_off) {
    const bool pair_ok = ((a.dst_c | a.dst_coff) & 1) == 0 && (reinterpret_cast<uintptr_t>(a.dst) & (a.out_f16 ? 3 : 7)) == 0;
    const float slope = a.act == MR_ACT_LEAKY ? a.act_a : 1.0f;
    const bool generic_act = a.act != MR_ACT_NONE && a.act != MR_ACT_LEAKY;
    const int c0 = 2 * (lane & 3);
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int p = p0 + (lane >> 2) + 8 * i;
        const int oy = tile_y * TH + p / TW, ox = tile_x * TW + p % TW;
        if (oy >= a.Ho || ox >= a.Wo) continue;
        const size_t oidx = (((size_t)b * a.dst_H + (oy * a.oy_step + oy_off)) * a.dst_W + (ox * a.ox_step + ox_off)) * a.dst_c +
                            a.dst_coff;
#pragma unroll
        for (int j = 0; j < N / 8; ++j) {
            const int ch = 8 * j + c0;
            if (ch >= a.Cout) break;
            float v[2];
#pragma unroll
            for (int c = 0; c < 2; ++c) {
                float x = d[4 * j + 2 * i + c] + bias_s[ch + c];
                x = generic_act ? act_fn(x, a.act, a.act_a, a.act_b) : fmaxf(x, slope * x);
                if (a.round_out) x = __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u);
                v[c] = x;
            }
            const bool two = ch + 1 < a.Cout;
            if (a.out_f16) {
                __half* o = reinterpret_cast<__half*>(a.dst) + oidx + ch;
                if (pair_ok && two) *reinterpret_cast<__half2*>(o) = __floats2half2_rn(v[0], v[1]);
                else { o[0] = __float2half_rn(v[0]); if (two) o[1] = __float2half_rn(v[1]); }
            } else {
                float* o = a.dst + oidx + ch;
                if (pair_ok && two) *reinterpret_cast<float2*>(o) = make_float2(v[0], v[1]);
                else { o[0] = v[0]; if (two) o[1] = v[1]; }
            }
        }
    }
}

// Stage release behind the in-flight wgmma group: after the group that read stages X is committed, the previous group is
// waited for and the barriers of ITS stages get this warpgroup's arrival.
struct Releaser {
    uint32_t prev0 = 0, prev1 = 0;
    __device__ __forceinline__ void after_commit(uint32_t bar0, uint32_t bar1, bool leader) {
        wgmma_wait<1>();
        if (leader) { if (prev0) mbar_arrive(prev0); if (prev1) mbar_arrive(prev1); }
        prev0 = bar0; prev1 = bar1;
    }
    __device__ __forceinline__ void drain(bool leader) {
        wgmma_wait<0>();
        if (leader) { if (prev0) mbar_arrive(prev0); if (prev1) mbar_arrive(prev1); }
        prev0 = prev1 = 0;
    }
};

// Persistent: each CTA loops over output tiles (tile = blockIdx.x, += gridDim.x).  The TMA ring keeps flowing across tile
// boundaries, so the loads of tile i+1 overlap the epilogue of tile i.  Tile = 8 rows x 16 columns, accumulator row
// p = y * 16 + x.
template <int N, bool F16>
__global__ void __launch_bounds__(kTcThreads)
conv_tc_kernel(const __grid_constant__ CUtensorMap tmA0, const __grid_constant__ CUtensorMap tmA1,
               const __grid_constant__ CUtensorMap tmA2, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmB1,
               const __grid_constant__ CUtensorMap tmB2, const __grid_constant__ CUtensorMap tmB3, const TcArgs a) {
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t bars[2 * 8];   // full[8], empty[8]
    __shared__ float bias_s[256];

    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;   // (the broadcast tells ptxas the role branches are warp-uniform)
    const uint32_t tile_base = (smem_u32(smem_raw) + 1023u) & ~1023u;   // SWIZZLE_128B tiles need 1024-byte alignment
    const uint32_t a_bytes = 128u * (uint32_t)a.row_bytes, b_bytes = (uint32_t)a.n_pad * (uint32_t)a.row_bytes;
    const uint32_t stage_bytes = a_bytes + b_bytes;
    const int stages = a.stages;
    const uint32_t full0 = smem_u32(&bars[0]), empty0 = smem_u32(&bars[8]);
    const int chunks_per_tap = a.chunks[0] + a.chunks[1] + a.chunks[2];
    const int n_phase = a.n_phase;

    if (threadIdx.x == 0) {
        for (int s = 0; s < stages; ++s) { mbar_init(full0 + 8 * s, 1); mbar_init(empty0 + 8 * s, 2); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    for (int i = threadIdx.x; i < 256; i += kTcThreads) bias_s[i] = (a.bias != nullptr && i < a.Cout) ? __ldg(a.bias + i) : 0.f;
    if (warp == kProducerWarp && lane == 0) {
        prefetch_tmap(&tmA0);
        if (a.n_src > 1) prefetch_tmap(&tmA1);
        if (a.n_src > 2) prefetch_tmap(&tmA2);
        prefetch_tmap(&tmB);
        if (n_phase > 1) { prefetch_tmap(&tmB1); prefetch_tmap(&tmB2); prefetch_tmap(&tmB3); }
    }
    __syncthreads();

    if (warp == kProducerWarp) {
        // ===================== TMA producer (whole warp, converged; the copies are issued by an elected lane) =====================
        int st = 0;
        uint32_t ph = 0;
        for (int tile = blockIdx.x; tile < a.total_tiles; tile += gridDim.x) {
            const int sp = tile / n_phase, phs = tile - sp * n_phase;
            const int b = sp / a.tiles_per_img, t = sp - b * a.tiles_per_img;
            const int tile_y = t / a.tiles_x, tile_x = t - tile_y * a.tiles_x;
            const int oy0 = tile_y * kTileH, ox0 = tile_x * kTileW;
            const int kh = a.ph_kh[phs], kw = a.ph_kw[phs], pad_t = a.ph_pad_t[phs], pad_l = a.ph_pad_l[phs];
            const CUtensorMap* tb = (phs == 0) ? &tmB : ((phs == 1) ? &tmB1 : ((phs == 2) ? &tmB2 : &tmB3));
            int brow = 0;
            for (int ky = 0; ky < kh; ++ky)
                for (int kx = 0; kx < kw; ++kx, brow += a.n_pad) {
                    const int ix0 = ox0 * a.sx - pad_l + kx, iy0 = oy0 * a.sy - pad_t + ky;
                    int kbase = 0;
                    for (int s = 0; s < a.n_src; ++s) {
                        const CUtensorMap* tm = (s == 0) ? &tmA0 : ((s == 1) ? &tmA1 : &tmA2);
                        for (int j = 0; j < a.chunks[s]; ++j, kbase += a.kc) {
                            mbar_wait(empty0 + 8 * st, ph ^ 1u);
                            const uint32_t sa = tile_base + st * stage_bytes, sb = sa + a_bytes;
                            mbar_expect_tx_elect(full0 + 8 * st, stage_bytes);
                            tma_load_4d_elect(sa, tm, full0 + 8 * st, j * a.kc, ix0, iy0, b);
                            tma_load_2d_elect(sb, tb, full0 + 8 * st, kbase, brow);
                            if (++st == stages) { st = 0; ph ^= 1u; }
                        }
                    }
                }
        }
    } else if (warp < kProducerWarp) {
        // ===================== consumer warpgroup wg: accumulator rows [64 wg, 64 wg + 64) =====================
        const int wg = warp >> 2;
        const bool leader = (threadIdx.x & 127) == 0;
        const uint32_t dhi = desc_hi(8u * (uint32_t)a.row_bytes, (uint32_t)a.row_bytes);
        const uint32_t a_off = 64u * (uint32_t)a.row_bytes * (uint32_t)wg;
        const uint32_t b_row16 = (uint32_t)a.row_bytes >> 4;
        const int ksteps = a.row_bytes / 32;   // MMA K = 32 bytes (8 tf32 / 16 half): 4 (2) steps inside the 128 (64)-byte swizzle row
        float d[N / 2];
        Releaser rel;
        int st = 0;
        uint32_t ph = 0;
        for (int tile = blockIdx.x; tile < a.total_tiles; tile += gridDim.x) {
            const int sp = tile / n_phase, phs = tile - sp * n_phase;
            const int b = sp / a.tiles_per_img, t = sp - b * a.tiles_per_img;
            const int tile_y = t / a.tiles_x, tile_x = t - tile_y * a.tiles_x;
            const int total = a.ph_kh[phs] * a.ph_kw[phs] * chunks_per_tap;
            uint32_t accf = 0;
            int src = 0, jc = 0;                                             // source / chunk inside the source of step c
            for (int c = 0; c < total; ++c) {
                mbar_wait(full0 + 8 * st, ph);
                const uint32_t sa = tile_base + st * stage_bytes;
                const uint32_t alo = desc_lo(sa + a_off), blo = desc_lo(sa + a_bytes);
                const int ks = (jc == a.chunks[src] - 1) ? a.tail_ksteps[src] : ksteps;
                if (++jc == a.chunks[src]) { jc = 0; if (++src == a.n_src) src = 0; }
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    if (k < ks) mma_tile<N, F16>(d, desc(alo + 2 * k, dhi), desc(blo + 2 * k, dhi), b_row16, accf);
                    accf = 1u;
                }
                wgmma_commit();
                rel.after_commit(empty0 + 8 * st, 0, leader);                 // frees the previous stage once its group retired
                if (++st == stages) { st = 0; ph ^= 1u; }
            }
            rel.drain(leader);
            epilogue_wg<N, kTileW, kTileH>(d, a, bias_s, 64 * wg + 16 * (warp & 3), lane, b, tile_y, tile_x, a.ph_oy_off[phs],
                                           a.ph_ox_off[phs]);
        }
    }
}

// -------------------------------------------------------------------------------------------------------------------------
// Stride-1 layers with small weights (the full-resolution 24..64-channel layers that dominate the stacks): "halo" variant.
//   * the whole packed weight tensor of the layer is loaded into shared memory ONCE per CTA (resident B);
//   * per (tile, source, K chunk) ONE TMA box {chunk, P px, 16 + kh - 1 px}, P = 8 + kw - 1, brings the input tile with its halo
//     (exactly the pixels the taps touch: a (k x 1) layer loads 8-px rows, a 3 x 3 layer 10-px rows);
//     every filter tap is then just a different shared-memory descriptor into that box: start address shifted by
//     (ky * P + kx) rows of 128 / 64 B, stride between 8-row groups = one halo row (P rows); the swizzle is a function of the
//     absolute shared-memory address, so neither shift needs to be a multiple of the 8-row swizzle atom.
//     L2->SM traffic drops from kh*kw boxes per tile to one.
// Output tile = 16 rows x 8 columns (an 8-row MMA group = 8 adjacent pixels of one output row); warpgroup wg computes output
// rows 8 wg .. 8 wg + 7, accumulator row p = y * 8 + x.
// -------------------------------------------------------------------------------------------------------------------------
template <int N, bool F16>
__global__ void __launch_bounds__(kTcThreads)
conv_tc_halo_kernel(const __grid_constant__ CUtensorMap tmA0, const __grid_constant__ CUtensorMap tmA1,
                    const __grid_constant__ CUtensorMap tmA2, const __grid_constant__ CUtensorMap tmB, const TcArgs a) {
    extern __shared__ uint8_t smem_raw[];
    // afull[4], aempty[4], bfull, streamed weights: bsfull[8], bsempty[8]
    __shared__ __align__(8) uint64_t bars[2 * 4 + 1 + 16];
    __shared__ float bias_s[256];

    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;   // (the broadcast tells ptxas the role branches are warp-uniform)
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t row_bytes = (uint32_t)a.row_bytes;
    const uint32_t b_bytes = (uint32_t)a.n_pad * row_bytes;
    const int chunks_per_tap = a.chunks[0] + a.chunks[1] + a.chunks[2];
    const int taps = a.kh * a.kw;
    const int nbs = a.b_stream;                                                    // weight ring stages (0: resident)
    // bytes in front of the input stages: all weights, or the ring (multiple of 1024: n_pad % 16 == 0)
    const uint32_t bres_bytes = (uint32_t)(nbs > 0 ? nbs : taps * chunks_per_tap) * b_bytes;
    const uint32_t a_bytes = a.halo_a_bytes;                                       // multiple of 1024
    const uint32_t pitch = (uint32_t)a.halo_pitch;
    const uint32_t a_tx = (uint32_t)(16 + a.kh - 1) * pitch * row_bytes;           // bytes one box delivers
    const uint32_t a_base = base + ((bres_bytes + 1023u) & ~1023u);
    const int stages = a.stages;
    const uint32_t afull0 = smem_u32(&bars[0]), aempty0 = smem_u32(&bars[4]), bfull = smem_u32(&bars[8]);
    const uint32_t bsfull0 = smem_u32(&bars[9]), bsempty0 = smem_u32(&bars[17]);

    if (threadIdx.x == 0) {
        for (int s = 0; s < stages; ++s) { mbar_init(afull0 + 8 * s, 1); mbar_init(aempty0 + 8 * s, 2); }
        mbar_init(bfull, 1);
        for (int s = 0; s < nbs; ++s) { mbar_init(bsfull0 + 8 * s, 1); mbar_init(bsempty0 + 8 * s, 2); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    for (int i = threadIdx.x; i < 256; i += kTcThreads) bias_s[i] = (a.bias != nullptr && i < a.Cout) ? __ldg(a.bias + i) : 0.f;
    if (warp == kProducerWarp && lane == 0) {
        prefetch_tmap(&tmA0);
        if (a.n_src > 1) prefetch_tmap(&tmA1);
        if (a.n_src > 2) prefetch_tmap(&tmA2);
        prefetch_tmap(&tmB);
    }
    __syncthreads();

    if (warp == kProducerWarp) {
        // ===================== TMA producer (whole warp, converged; the copies are issued by an elected lane) =====================
        // resident weights: every (tap, chunk) slice [n_pad x chunk] once
        if (nbs == 0) {
            mbar_expect_tx_elect(bfull, bres_bytes);
            for (int tp = 0; tp < taps; ++tp)
                for (int cg = 0; cg < chunks_per_tap; ++cg)
                    tma_load_2d_elect(base + (uint32_t)(tp * chunks_per_tap + cg) * b_bytes, &tmB, bfull, cg * a.kc, tp * a.n_pad);
        }
        int st = 0, bs = 0;
        uint32_t ph = 0, bph = 0;
        for (int tile = blockIdx.x; tile < a.total_tiles; tile += gridDim.x) {
            const int b = tile / a.tiles_per_img, t = tile - b * a.tiles_per_img;
            const int tile_y = t / a.tiles_x, tile_x = t - tile_y * a.tiles_x;
            const int ix0 = tile_x * 8 - a.pad_l, iy0 = tile_y * 16 - a.pad_t;
            int kbase = 0;
            for (int s = 0; s < a.n_src; ++s) {
                const CUtensorMap* tm = (s == 0) ? &tmA0 : ((s == 1) ? &tmA1 : &tmA2);
                for (int j = 0; j < a.chunks[s]; ++j, kbase += a.kc) {
                    mbar_wait(aempty0 + 8 * st, ph ^ 1u);
                    mbar_expect_tx_elect(afull0 + 8 * st, a_tx);
                    tma_load_4d_elect(a_base + st * a_bytes, tm, afull0 + 8 * st, j * a.kc, ix0, iy0, b);
                    if (++st == stages) { st = 0; ph ^= 1u; }
                    if (nbs > 0) {   // streamed weights: the slices of this chunk, tap by tap, behind its input box
                        int brow = 0;
                        for (int tp = 0; tp < taps; ++tp, brow += a.n_pad) {
                            mbar_wait(bsempty0 + 8 * bs, bph ^ 1u);
                            mbar_expect_tx_elect(bsfull0 + 8 * bs, b_bytes);
                            tma_load_2d_elect(base + (uint32_t)bs * b_bytes, &tmB, bsfull0 + 8 * bs, kbase, brow);
                            if (++bs == nbs) { bs = 0; bph ^= 1u; }
                        }
                    }
                }
            }
        }
    } else if (warp < kProducerWarp) {
        // ===================== consumer warpgroup wg: output rows [8 wg, 8 wg + 8) of the 16-row tile =====================
        const int wg = warp >> 2;
        const bool leader = (threadIdx.x & 127) == 0;
        const uint32_t dhi_a = desc_hi(pitch * row_bytes, row_bytes);      // stride between 8-row groups = one halo row
        const uint32_t dhi_b = desc_hi(8u * row_bytes, row_bytes);
        const uint32_t tap_dx = row_bytes >> 4, tap_dy = (pitch * row_bytes) >> 4;   // descriptor steps of one tap to the right / down
        const uint32_t b_step = b_bytes >> 4, b_row16 = row_bytes >> 4;
        const uint32_t a_off = 8u * pitch * row_bytes * (uint32_t)wg;
        const int ksteps = a.row_bytes / 32;
        if (nbs == 0) mbar_wait(bfull, 0);
        float d[N / 2];
        Releaser rel;
        int st = 0, bs = 0;
        uint32_t ph = 0, bph = 0;
        for (int tile = blockIdx.x; tile < a.total_tiles; tile += gridDim.x) {
            const int b = tile / a.tiles_per_img, t = tile - b * a.tiles_per_img;
            const int tile_y = t / a.tiles_x, tile_x = t - tile_y * a.tiles_x;
            uint32_t accf = 0;
            int src = 0, jc = 0;                                             // source / chunk inside the source of chunk cg
            for (int cg = 0; cg < chunks_per_tap; ++cg) {
                const int ks = (jc == a.chunks[src] - 1) ? a.tail_ksteps[src] : ksteps;
                if (++jc == a.chunks[src]) { jc = 0; ++src; }
                mbar_wait(afull0 + 8 * st, ph);
                uint32_t alo_row = desc_lo(a_base + st * a_bytes + a_off);
                uint32_t blo = desc_lo(base) + (uint32_t)cg * b_step;                 // resident: slice (tap 0, chunk cg)
                for (int ky = 0; ky < a.kh; ++ky, alo_row += tap_dy) {
                    uint32_t alo = alo_row;
                    for (int kx = 0; kx < a.kw; ++kx, alo += tap_dx) {
                        if (nbs > 0) {
                            mbar_wait(bsfull0 + 8 * bs, bph);
                            blo = desc_lo(base + (uint32_t)bs * b_bytes);
                        }
                        wgmma_fence();
#pragma unroll
                        for (int k = 0; k < 4; ++k) {   // 32 bytes of K per MMA (8 tf32 / 16 half): 4 per 128-byte row, 2 per 64-byte row
                            if (k < ks) mma_tile<N, F16>(d, desc(alo + 2 * k, dhi_a), desc(blo + 2 * k, dhi_b), b_row16, accf);
                            accf = 1u;
                        }
                        if (nbs > 0) {   // one group per tap: frees the weight stage (and after the last tap the input stage)
                            wgmma_commit();
                            const bool last = ky == a.kh - 1 && kx == a.kw - 1;
                            rel.after_commit(bsempty0 + 8 * bs, last ? aempty0 + 8 * st : 0u, leader);
                            if (++bs == nbs) { bs = 0; bph ^= 1u; }
                        } else {
                            blo += (uint32_t)chunks_per_tap * b_step;   // next tap, same chunk
                        }
                    }
                }
                if (nbs == 0) {
                    wgmma_commit();
                    rel.after_commit(aempty0 + 8 * st, 0u, leader);
                }
                if (++st == stages) { st = 0; ph ^= 1u; }
            }
            rel.drain(leader);
            epilogue_wg<N, 8, 16>(d, a, bias_s, 64 * wg + 16 * (warp & 3), lane, b, tile_y, tile_x, a.oy_off, a.ox_off);
        }
    }
}

// ---- host side: tensor maps ---------------------------------------------------------------------------------------------
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

// the two kernels for MMA N = n_pad (16..256, multiple of 16) and the source type
struct TcKernels {
    const void* tap;
    const void* halo;
};
template <int N>
TcKernels tc_kernels_n(bool f16) {
    if (f16) return {(const void*)conv_tc_kernel<N, true>, (const void*)conv_tc_halo_kernel<N, true>};
    return {(const void*)conv_tc_kernel<N, false>, (const void*)conv_tc_halo_kernel<N, false>};
}
TcKernels tc_kernels(int n_pad, bool f16) {
    switch (n_pad / 16) {
        case 1: return tc_kernels_n<16>(f16);
        case 2: return tc_kernels_n<32>(f16);
        case 3: return tc_kernels_n<48>(f16);
        case 4: return tc_kernels_n<64>(f16);
        case 5: return tc_kernels_n<80>(f16);
        case 6: return tc_kernels_n<96>(f16);
        case 7: return tc_kernels_n<112>(f16);
        case 8: return tc_kernels_n<128>(f16);
        case 9: return tc_kernels_n<144>(f16);
        case 10: return tc_kernels_n<160>(f16);
        case 11: return tc_kernels_n<176>(f16);
        case 12: return tc_kernels_n<192>(f16);
        case 13: return tc_kernels_n<208>(f16);
        case 14: return tc_kernels_n<224>(f16);
        case 15: return tc_kernels_n<240>(f16);
        default: return tc_kernels_n<256>(f16);
    }
}

// CTAs of `kernel` one SM can hold as far as registers and static shared memory go
int resident_ctas(const void* kernel) {
    int n = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kernel, kTcThreads, 0) != cudaSuccess) return 1;
    return n > 0 ? n : 1;
}

// bytes of one input stage of the halo kernel: a box of (16 + kh - 1) rows x pitch pixels of one K chunk, rounded up to 1 KB
size_t halo_box_bytes(int kh, int pitch, int row_bytes) { return ((size_t)(16 + kh - 1) * pitch * row_bytes + 1023) & ~size_t(1023); }

// Every argument check of mr_conv2d_nhwc_tc / _phases / _plan.  Makes no CUDA call, so a bad descriptor is rejected the same
// way with or without a GPU.  *kc_out: channels per K chunk (32 or 64), derived from k_pad.
int tc_validate(const mr_conv_desc* desc, int n_phases, int n_pad, int k_pad, int* kc_out) {
    MR_REQUIRE(desc != nullptr, "mr_conv2d_nhwc_tc: null descriptor");
    MR_REQUIRE(n_phases >= 1 && n_phases <= 4, "mr_conv2d_nhwc_tc_phases: 1..4 phases (got %d)", n_phases);
    const mr_conv_desc& d = desc[0];
    MR_REQUIRE(d.n_src >= 1 && d.n_src <= MR_CONV_MAX_SRC, "mr_conv2d_nhwc_tc: n_src=%d out of range", d.n_src);
    for (int p = 1; p < n_phases; ++p) {   // phases share everything but the filter (size, padding, weights) and the output offset
        const mr_conv_desc& e = desc[p];
        bool same = e.n_src == d.n_src && e.B == d.B && e.Hs == d.Hs && e.Ws == d.Ws && e.upsample2 == d.upsample2 && e.sy == d.sy &&
                    e.sx == d.sx && e.Ho == d.Ho && e.Wo == d.Wo && e.Cout == d.Cout && e.bias == d.bias && e.dst == d.dst &&
                    e.dst_H == d.dst_H && e.dst_W == d.dst_W && e.dst_c == d.dst_c && e.dst_coff == d.dst_coff &&
                    e.oy_step == d.oy_step && e.ox_step == d.ox_step && e.act == d.act && e.act_a == d.act_a && e.act_b == d.act_b &&
                    e.src_dtype == d.src_dtype && e.dst_dtype == d.dst_dtype;
        for (int s = 0; same && s < d.n_src; ++s) same = e.src[s] == d.src[s] && e.src_c[s] == d.src_c[s];
        MR_REQUIRE(same, "mr_conv2d_nhwc_tc_phases: phase %d differs from phase 0 in more than filter size, padding, weights and output offset", p);
    }
    MR_REQUIRE(d.upsample2 == 0, "mr_conv2d_nhwc_tc: upsample2: upsample-on-read is expressed as sub-pixel convolutions on this path");
    MR_REQUIRE(d.dst != nullptr, "mr_conv2d_nhwc_tc: null dst");
    MR_REQUIRE(d.src_dtype == MR_DT_F32 || d.src_dtype == MR_DT_F16, "mr_conv2d_nhwc_tc: bad src_dtype %d", d.src_dtype);
    MR_REQUIRE(d.dst_dtype == MR_DT_F32 || d.dst_dtype == MR_DT_F16, "mr_conv2d_nhwc_tc: bad dst_dtype %d", d.dst_dtype);
    MR_REQUIRE(d.Cout >= 1 && d.Cout <= 256 && n_pad >= d.Cout && n_pad <= 256 && (n_pad % 16) == 0,
               "mr_conv2d_nhwc_tc: Cout=%d n_pad=%d unsupported (Cout <= 256, n_pad multiple of 16)", d.Cout, n_pad);
    MR_REQUIRE(d.B >= 1 && d.B <= 65535 && d.Hs >= 1 && d.Ws >= 1 && d.Ho >= 1 && d.Wo >= 1, "mr_conv2d_nhwc_tc: bad shape");
    MR_REQUIRE(d.sy >= 1 && d.sx >= 1 && d.sy <= 4 && d.sx <= 4, "mr_conv2d_nhwc_tc: stride sy=%d sx=%d out of 1..4", d.sy, d.sx);
    MR_REQUIRE(d.oy_step >= 1 && d.ox_step >= 1, "mr_conv2d_nhwc_tc: oy_step=%d / ox_step=%d must be >= 1", d.oy_step, d.ox_step);
    MR_REQUIRE(d.act >= MR_ACT_NONE && d.act <= MR_ACT_ABSTANH, "mr_conv2d_nhwc_tc: unknown act %d", d.act);
    MR_REQUIRE(d.dst_coff >= 0 && d.dst_coff + d.Cout <= d.dst_c, "mr_conv2d_nhwc_tc: channel slice dst_coff=%d + Cout=%d out of dst_c=%d",
               d.dst_coff, d.Cout, d.dst_c);
    for (int p = 0; p < n_phases; ++p) {
        const mr_conv_desc& e = desc[p];
        MR_REQUIRE(e.weight != nullptr && (reinterpret_cast<uintptr_t>(e.weight) & 15) == 0,
                   "mr_conv2d_nhwc_tc: phase %d: weight is null or not 16-byte aligned", p);
        MR_REQUIRE(e.kh >= 1 && e.kw >= 1, "mr_conv2d_nhwc_tc: phase %d: bad filter size kh=%d kw=%d", p, e.kh, e.kw);
        MR_REQUIRE(e.oy_off >= 0 && e.ox_off >= 0, "mr_conv2d_nhwc_tc: phase %d: oy_off=%d / ox_off=%d must be >= 0", p, e.oy_off, e.ox_off);
        MR_REQUIRE((e.Ho - 1) * e.oy_step + e.oy_off < e.dst_H && (e.Wo - 1) * e.ox_step + e.ox_off < e.dst_W,
                   "mr_conv2d_nhwc_tc: phase %d: output placement out of range (dst_H=%d dst_W=%d)", p, e.dst_H, e.dst_W);
    }
    const bool f16 = d.src_dtype == MR_DT_F16;
    const int cmult = f16 ? 8 : 4;            // pixel stride must be a multiple of 16 bytes for TMA
    for (int s = 0; s < d.n_src; ++s) {
        MR_REQUIRE(d.src[s] != nullptr && d.src_c[s] >= cmult && (d.src_c[s] % cmult) == 0,
                   "mr_conv2d_nhwc_tc: source %d needs src_c a multiple of %d (got %d)", s, cmult, d.src_c[s]);
        MR_REQUIRE((reinterpret_cast<uintptr_t>(d.src[s]) & 15) == 0, "mr_conv2d_nhwc_tc: source %d is not 16-byte aligned", s);
    }
    // K chunk = one swizzle row of channels: 32 fp32 or 64 half (128 bytes).  Half sources whose channel counts waste less
    // with 32-channel chunks (32, 96, ... channels) are packed that way by the caller (k_pad tells): 64-byte rows, SWIZZLE_64B,
    // so that neither TMA nor the MMA spends time on the zero half of a 128-byte row.
    int kc = f16 ? 64 : kKC;
    if (f16) {
        int k64 = 0, k32 = 0;
        for (int s = 0; s < d.n_src; ++s) { k64 += (d.src_c[s] + 63) / 64 * 64; k32 += (d.src_c[s] + 31) / 32 * 32; }
        if (k_pad != k64 && k_pad == k32) kc = 32;
    }
    int ksum = 0;
    for (int s = 0; s < d.n_src; ++s) ksum += (d.src_c[s] + kc - 1) / kc * kc;
    MR_REQUIRE(ksum == k_pad, "mr_conv2d_nhwc_tc: packed weight k_pad (%d) does not match the sources (%d)", k_pad, ksum);
    *kc_out = kc;
    return MR_OK;
}

// The kernel choice for a validated descriptor: tap-refetch or halo kernel, resident or streamed weights, CTAs per SM,
// stages, grid.  The launch below runs exactly this plan; mr_conv2d_nhwc_tc_plan reports it.
int tc_plan(const mr_conv_desc* desc, int n_phases, int n_pad, int kc, mr_tc_plan* out) {
    const mr_conv_desc& d = desc[0];
    const bool f16 = d.src_dtype == MR_DT_F16;
    const int row_bytes = kc * (f16 ? 2 : 4);
    const TcKernels kern = tc_kernels(n_pad, f16);
    // "halo" variant (one input box per tile, resident weights): stride 1, taps reach at most 8 px to the right, weights fit
    int chunks_all = 0;
    for (int s = 0; s < d.n_src; ++s) chunks_all += (d.src_c[s] + kc - 1) / kc;
    const size_t bres = (size_t)d.kh * d.kw * chunks_all * n_pad * row_bytes;
    // MONOREC_B200_TC_HALO: unset = automatic, 0 = never, n = 1..4: at most n CTAs per SM (1: also layers that only fit once).
    // Box rows are 8 + kw - 1 px, so a box holds exactly the pixels the taps touch and the 48-channel full-resolution layers
    // fit twice per SM next to their weights.
    static const int halo_env = getenv("MONOREC_B200_TC_HALO") ? atoi(getenv("MONOREC_B200_TC_HALO")) : -1;
    // (64-byte rows are fine inside the halo box too: half sources of <= 32 channels packed with 32-channel chunks)
    const int halo_pitch = 8 + d.kw - 1;
    const size_t halo_a_bytes = halo_box_bytes(d.kh, halo_pitch, row_bytes);
    const size_t bres_al = (bres + 1023) & ~size_t(1023);
    // CTAs per SM the accumulator registers allow (the wider N, the more registers per consumer thread)
    const int halo_reg_ctas = resident_ctas(kern.halo);
    auto halo_fit = [&](int ctas) {   // A stages that fit next to the resident weights with `ctas` CTAs per SM
        if (ctas > halo_reg_ctas) return 0;
        // 228 KB per SM, 1 KB reserved per CTA; static per CTA: 1 KB bias + barriers; 1 KB alignment slack
        const size_t budget = (size_t)(ctas == 1 ? 210 : 228) * 1024 / ctas - (1 + 1 + 1) * 1024 - 512;
        int st = bres_al + 1024 < budget ? (int)((budget - 1024 - bres_al) / halo_a_bytes) : 0;
        return st > 4 ? 4 : st;
    };
    // CTAs per SM: up to three, each with at least two input stages (up to 4).
    // MONOREC_B200_TC_HALO=n (1..4) caps / forces the count (1: also layers that only fit once).
    const bool halo_shape = n_phases == 1 && halo_env != 0 && d.sy == 1 && d.sx == 1 && d.kw <= 9 && d.kh <= 7;
    int halo_ctas = 0;
    if (halo_shape) {
        const int cap = (halo_env >= 1 && halo_env <= 4) ? halo_env : 3;
        for (int c = cap; c >= (halo_env == 1 ? 1 : 2) && halo_ctas == 0; --c)
            if (halo_fit(c) >= 2) halo_ctas = c;
    }
    // Weights that do not fit next to two input stages stream instead: the [n_pad x chunk] slice of each (chunk, tap) goes through
    // a ring of 3..8 stages behind the chunk's input box.  Per tile that is all the weights once (L2 hits) plus ONE input box per
    // chunk, against kh*kw input boxes + the same weights in the tap-refetch kernel, whose L2->SM traffic bounds the
    // multi-source decoder layers.  MONOREC_B200_TC_STREAM=0 disables it.
    static const bool stream_on = getenv("MONOREC_B200_TC_STREAM") ? (atoi(getenv("MONOREC_B200_TC_STREAM")) != 0) : true;
    int b_stream = 0, stream_stages = 0;
    const size_t b_slice = (size_t)n_pad * row_bytes;
    if (halo_ctas == 0 && stream_on && halo_shape && d.kh * d.kw > 1 && halo_reg_ctas >= 2) {
        const size_t budget = (size_t)228 * 1024 / 2 - (1 + 1 + 1) * 1024 - 512 - 1024;
        if (budget > 2 * halo_a_bytes + 3 * b_slice) {
            int nb = (int)((budget - 2 * halo_a_bytes) / b_slice);
            if (nb > 8) nb = 8;
            int st = (int)((budget - (size_t)nb * b_slice) / halo_a_bytes);
            b_stream = nb;
            stream_stages = st > 4 ? 4 : st;
            halo_ctas = 2;
        }
    }
    const bool halo = halo_ctas > 0;
    const int tiles_x = halo ? (d.Wo + 7) / 8 : (d.Wo + kTileW - 1) / kTileW;
    const int tiles = tiles_x * (halo ? (d.Ho + 15) / 16 : (d.Ho + kTileH - 1) / kTileH);
    const int total_tiles = tiles * d.B * n_phases;
    // persistent grid over the SMs of the current device
    int dev = 0, sms = 0;
    MR_CUDA(cudaGetDevice(&dev));
    MR_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    // resident CTAs per SM: bounded by the accumulator registers and capped at 4; with MMA N = 32..64 one CTA cannot keep the
    // tensor pipe busy, so several CTAs interleave their MMA chains
    const int reg_ctas = resident_ctas(kern.tap);
    mr_tc_plan p{};
    p.n_pad = n_pad; p.kc = kc; p.row_bytes = row_bytes;
    p.total_tiles = total_tiles; p.tiles_x = tiles_x;
    p.tap_reg_ctas = reg_ctas; p.halo_reg_ctas = halo_reg_ctas; p.halo_shape = halo_shape ? 1 : 0;
    if (halo) {
        p.kernel = b_stream ? MR_TC_KERNEL_HALO_STREAM : MR_TC_KERNEL_HALO;
        p.ctas_per_sm = halo_ctas;
        p.stages = b_stream ? stream_stages : halo_fit(halo_ctas);
        p.b_stream = b_stream;
        p.halo_pitch = halo_pitch;
        const size_t halo_front = b_stream ? (size_t)b_stream * b_slice : bres_al;   // bytes in front of the input stages
        p.smem_bytes = (int)(halo_front + (size_t)p.stages * halo_a_bytes + 1024);
    } else {
        const int ctas_per_sm = reg_ctas > 4 ? 4 : reg_ctas;
        const size_t stage_bytes = (size_t)(128 + n_pad) * row_bytes;
        const size_t budget = (size_t)(200 * 1024) / ctas_per_sm - 2 * 1024;
        int stages = (int)(budget / stage_bytes);
        if (stages > 8) stages = 8;
        if (stages < 2) stages = 2;
        p.kernel = MR_TC_KERNEL_TAP;
        p.ctas_per_sm = ctas_per_sm;
        p.stages = stages;
        p.smem_bytes = (int)((size_t)stages * stage_bytes + 1024);
    }
    p.grid = sms * p.ctas_per_sm;
    if (p.grid > total_tiles) p.grid = total_tiles;
    *out = p;
    return MR_OK;
}

}  // namespace

extern "C" int mr_conv2d_nhwc_tc_plan(const mr_conv_desc* descs, int n_phases, int n_pad, int k_pad, mr_tc_plan* out) {
    MR_REQUIRE(out != nullptr, "mr_conv2d_nhwc_tc_plan: null out");
    int kc = 0;
    const int rc = tc_validate(descs, n_phases, n_pad, k_pad, &kc);
    if (rc != MR_OK) return rc;
    return tc_plan(descs, n_phases, n_pad, kc, out);
}

static int conv2d_nhwc_tc_impl(const mr_conv_desc* desc, int n_phases, int n_pad, int k_pad, int round_out, void* stream) {
    int kc = 0;
    int rc = tc_validate(desc, n_phases, n_pad, k_pad, &kc);
    if (rc != MR_OK) return rc;
    EncodeTiledFn encode = get_encode_fn();
    if (encode == nullptr) {
        mr::set_error("mr_conv2d_nhwc_tc: cuTensorMapEncodeTiled is not available from this driver");
        return MR_ENOSUPPORT;
    }
    mr_tc_plan plan;
    rc = tc_plan(desc, n_phases, n_pad, kc, &plan);
    if (rc != MR_OK) return rc;
    const mr_conv_desc& d = desc[0];
    const bool f16 = d.src_dtype == MR_DT_F16;
    const bool halo = plan.kernel != MR_TC_KERNEL_TAP;
    const int esize = f16 ? 2 : 4;
    TcArgs a{};
    a.n_src = d.n_src;
    a.row_bytes = plan.row_bytes;
    a.kc = kc; a.out_f16 = (d.dst_dtype == MR_DT_F16) ? 1 : 0;
    CUtensorMap tmA[MR_CONV_MAX_SRC];
    for (int s = 0; s < d.n_src; ++s) {
        const int C = d.src_c[s];
        a.chunks[s] = (C + kc - 1) / kc;
        a.tail_ksteps[s] = ((C - (a.chunks[s] - 1) * kc) * esize + 31) / 32;
        const cuuint64_t gdim[4] = {(cuuint64_t)C, (cuuint64_t)d.Ws, (cuuint64_t)d.Hs, (cuuint64_t)d.B};
        const cuuint64_t gstr[3] = {(cuuint64_t)C * esize, (cuuint64_t)d.Ws * C * esize, (cuuint64_t)d.Hs * d.Ws * C * esize};
        // with a traversal stride s the box spans box/s loaded elements: 16 (8) output pixels need a span of 16*s (8*s)
        cuuint32_t box[4] = {(cuuint32_t)kc, (cuuint32_t)(kTileW * d.sx), (cuuint32_t)(kTileH * d.sy), 1};
        if (halo) { box[1] = (cuuint32_t)plan.halo_pitch; box[2] = (cuuint32_t)(16 + d.kh - 1); }
        const cuuint32_t estr[4] = {1, (cuuint32_t)d.sx, (cuuint32_t)d.sy, 1};
        CUresult r = encode(&tmA[s], f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float*>(d.src[s]), gdim, gstr, box, estr,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, a.row_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                            CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) {
            mr::set_error("mr_conv2d_nhwc_tc: cuTensorMapEncodeTiled(A%d) failed with CUresult %d", s, (int)r);
            return MR_EINVAL;
        }
    }
    for (int s = d.n_src; s < MR_CONV_MAX_SRC; ++s) tmA[s] = tmA[0];
    CUtensorMap tmBs[4];
    for (int p = 0; p < n_phases; ++p) {
        const mr_conv_desc& e = desc[p];
        const cuuint64_t gdim[2] = {(cuuint64_t)k_pad, (cuuint64_t)e.kh * e.kw * n_pad};
        const cuuint64_t gstr[1] = {(cuuint64_t)k_pad * esize};
        const cuuint32_t box[2] = {(cuuint32_t)kc, (cuuint32_t)n_pad};
        const cuuint32_t estr[2] = {1, 1};
        CUresult r = encode(&tmBs[p], f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(e.weight), gdim, gstr, box, estr,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, a.row_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                            CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) {
            mr::set_error("mr_conv2d_nhwc_tc: cuTensorMapEncodeTiled(B) failed with CUresult %d", (int)r);
            return MR_EINVAL;
        }
    }
    for (int p = n_phases; p < 4; ++p) tmBs[p] = tmBs[0];
    a.n_phase = n_phases;
    for (int p = 0; p < 4; ++p) {
        const mr_conv_desc& e = desc[p < n_phases ? p : 0];
        a.ph_kh[p] = e.kh; a.ph_kw[p] = e.kw; a.ph_pad_t[p] = e.pad_t; a.ph_pad_l[p] = e.pad_l; a.ph_oy_off[p] = e.oy_off; a.ph_ox_off[p] = e.ox_off;
    }
    a.kh = d.kh; a.kw = d.kw; a.sy = d.sy; a.sx = d.sx; a.pad_t = d.pad_t; a.pad_l = d.pad_l;
    a.Ho = d.Ho; a.Wo = d.Wo; a.Cout = d.Cout; a.n_pad = n_pad;
    a.tiles_x = plan.tiles_x;
    a.tiles_per_img = plan.total_tiles / (d.B * n_phases);
    a.total_tiles = plan.total_tiles;
    a.stages = plan.stages;
    a.bias = d.bias; a.dst = d.dst;
    a.dst_H = d.dst_H; a.dst_W = d.dst_W; a.dst_c = d.dst_c; a.dst_coff = d.dst_coff;
    a.oy_step = d.oy_step; a.ox_step = d.ox_step; a.oy_off = d.oy_off; a.ox_off = d.ox_off;
    a.act = d.act; a.act_a = d.act_a; a.act_b = d.act_b; a.round_out = round_out;
    const TcKernels kern = tc_kernels(n_pad, f16);
    if (halo) {
        a.halo_pitch = plan.halo_pitch;
        a.halo_a_bytes = (uint32_t)halo_box_bytes(d.kh, plan.halo_pitch, plan.row_bytes);
        a.b_stream = plan.b_stream;
        void* args[] = {&tmA[0], &tmA[1], &tmA[2], &tmBs[0], &a};
        MR_CUDA(cudaFuncSetAttribute(kern.halo, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(212 * 1024)));
        MR_CUDA(cudaLaunchKernel(kern.halo, dim3(plan.grid), dim3(kTcThreads), args, (size_t)plan.smem_bytes, (cudaStream_t)stream));
        MR_LAUNCH_CHECK("conv_tc_halo_kernel");
        return MR_OK;
    }
    void* args[] = {&tmA[0], &tmA[1], &tmA[2], &tmBs[0], &tmBs[1], &tmBs[2], &tmBs[3], &a};
    MR_CUDA(cudaFuncSetAttribute(kern.tap, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(212 * 1024)));
    MR_CUDA(cudaLaunchKernel(kern.tap, dim3(plan.grid), dim3(kTcThreads), args, (size_t)plan.smem_bytes, (cudaStream_t)stream));
    MR_LAUNCH_CHECK("conv_tc_kernel");
    return MR_OK;
}

extern "C" int mr_conv2d_nhwc_tc(const mr_conv_desc* desc, int n_pad, int k_pad, int round_out, void* stream) {
    return conv2d_nhwc_tc_impl(desc, 1, n_pad, k_pad, round_out, stream);
}

extern "C" int mr_conv2d_nhwc_tc_phases(const mr_conv_desc* descs, int n_phases, int n_pad, int k_pad, int round_out, void* stream) {
    return conv2d_nhwc_tc_impl(descs, n_phases, n_pad, k_pad, round_out, stream);
}
