// Host-buffer entries of the cost-volume path (include/monorec_b200.h: mr_cost_volume_host, and mr_cost_volume_host_f16 with
// half volumes).
// Batch elements are pipelined over a small ring of internal streams: the H2D copy of element b+1 and the D2H copy
// of element b-1 overlap the kernel of element b.  The caller owns the device workspace; the streams and the event are
// created once per host thread and device and reused by later calls.
#include "mr_common.cuh"
#include <cstdint>

namespace {

struct HostPlan {
    size_t img, mats, proj, depths, cv, sfcv, total;  // byte offsets into the workspace
};

// vb: bytes per volume element (4: fp32, 2: half)
HostPlan plan(int B, int F, int D, int H, int W, int vb = 4) {
    auto al = [](size_t x) { return (x + 255) & ~size_t(255); };
    HostPlan p;
    size_t off = 0;
    p.img = off;    off = al(off + (size_t)(1 + F) * B * 3 * H * W * 4);
    p.mats = off;   off = al(off + (size_t)(2 + 2 * F) * B * 16 * 4);
    p.proj = off;   off = al(off + (size_t)B * F * 12 * 4);
    p.depths = off; off = al(off + (size_t)D * 4);
    p.cv = off;     off = al(off + (size_t)B * D * H * W * vb);
    p.sfcv = off;   off = al(off + (size_t)F * B * D * H * W * vb);
    p.total = off;
    return p;
}

constexpr int kStreams = 3;

struct StreamRing {
    cudaStream_t st[kStreams] = {};
    cudaEvent_t ready = nullptr;
    int n = 0, device = -1;
    int init() {   // idempotent: re-created only when the calling thread has switched devices
        int dev = 0;
        MR_CUDA(cudaGetDevice(&dev));
        if (dev == device && n == kStreams && ready != nullptr) return MR_OK;
        release();
        for (; n < kStreams; ++n) MR_CUDA(cudaStreamCreateWithFlags(&st[n], cudaStreamNonBlocking));
        MR_CUDA(cudaEventCreateWithFlags(&ready, cudaEventDisableTiming));
        device = dev;
        return MR_OK;
    }
    void release() {
        for (int i = 0; i < n; ++i) cudaStreamDestroy(st[i]);
        if (ready) cudaEventDestroy(ready);
        n = 0; ready = nullptr; device = -1;
    }
    ~StreamRing() { release(); }   // at thread exit (errors after context teardown are ignored)
};

thread_local StreamRing g_ring;

}  // namespace

extern "C" long long mr_cost_volume_host_workspace(int B, int F, int D, int H, int W) {
    if (B < 1 || F < 1 || D < 2 || H < 5 || W < 5) return 0;
    return (long long)plan(B, F, D, H, W).total;
}

extern "C" long long mr_cost_volume_host_sfcv_offset(int B, int F, int D, int H, int W) {
    if (B < 1 || F < 1 || D < 2 || H < 5 || W < 5) return -1;
    return (long long)plan(B, F, D, H, W).sfcv;
}

extern "C" long long mr_cost_volume_host_f16_workspace(int B, int F, int D, int H, int W) {
    if (B < 1 || F < 1 || D < 2 || H < 5 || W < 5) return 0;
    return (long long)plan(B, F, D, H, W, 2).total;
}

extern "C" long long mr_cost_volume_host_f16_sfcv_offset(int B, int F, int D, int H, int W) {
    if (B < 1 || F < 1 || D < 2 || H < 5 || W < 5) return -1;
    return (long long)plan(B, F, D, H, W, 2).sfcv;
}

namespace {

// both host entries; out_dtype MR_DT_F32 / MR_DT_F16 is the type of the volumes on the device and in the host buffers
int cost_volume_host(const char* fn, const float* h_keyframe, const float* h_frames, const float* h_keyframe_pose,
                     const float* h_keyframe_K, const float* h_poses, const float* h_intrinsics, void* h_out_cv,
                     void* h_out_sfcv, int B, int F, int D, int H, int W, float inv_depth_lo, float inv_depth_hi, float alpha,
                     void* workspace, long long workspace_bytes, int out_dtype) {
    MR_REQUIRE(h_keyframe && h_frames && h_keyframe_pose && h_keyframe_K && h_poses && h_intrinsics && h_out_cv && workspace,
               "%s: null pointer", fn);
    MR_REQUIRE(B >= 1 && F >= 1 && F <= MR_MAX_FRAMES && D >= 2 && D <= 128 && H >= 5 && W >= 5,
               "%s: bad shape B=%d F=%d D=%d H=%d W=%d", fn, B, F, D, H, W);
    const int vb = out_dtype == MR_DT_F16 ? 2 : 4;
    const HostPlan p = plan(B, F, D, H, W, vb);
    if ((long long)p.total > workspace_bytes) {
        mr::set_error("%s: workspace too small (%lld < %zu bytes)", fn, workspace_bytes, p.total);
        return MR_ENOMEM;
    }
    char* ws = static_cast<char*>(workspace);
    const size_t img1 = (size_t)3 * H * W;  // floats per image
    const size_t vol1 = (size_t)D * H * W;  // elements per volume
    float* d_key = reinterpret_cast<float*>(ws + p.img);     // [B,3,H,W]
    float* d_frames = d_key + (size_t)B * img1;              // [F,B,3,H,W]
    float* d_kpose = reinterpret_cast<float*>(ws + p.mats);  // [B,16]
    float* d_kK = d_kpose + (size_t)B * 16;                  // [B,16]
    float* d_poses = d_kK + (size_t)B * 16;                  // [F,B,16]
    float* d_intr = d_poses + (size_t)F * B * 16;            // [F,B,16]
    float* d_proj = reinterpret_cast<float*>(ws + p.proj);
    float* d_depths = reinterpret_cast<float*>(ws + p.depths);
    char* d_cv = ws + p.cv;
    char* d_sfcv = ws + p.sfcv;
    char* o_cv = static_cast<char*>(h_out_cv);
    char* o_sfcv = static_cast<char*>(h_out_sfcv);

    StreamRing& ring = g_ring;
    int rc = ring.init();
    if (rc != MR_OK) return rc;
    // everything below only enqueues work; whatever happens, the internal streams are drained before returning so that no
    // copy into the caller's buffers is still in flight (and the first error, if any, is the one reported)
    auto enqueue = [&]() -> int {
        cudaStream_t s0 = ring.st[0];
        MR_CUDA(cudaMemcpyAsync(d_kpose, h_keyframe_pose, (size_t)B * 64, cudaMemcpyHostToDevice, s0));
        MR_CUDA(cudaMemcpyAsync(d_kK, h_keyframe_K, (size_t)B * 64, cudaMemcpyHostToDevice, s0));
        MR_CUDA(cudaMemcpyAsync(d_poses, h_poses, (size_t)F * B * 64, cudaMemcpyHostToDevice, s0));
        MR_CUDA(cudaMemcpyAsync(d_intr, h_intrinsics, (size_t)F * B * 64, cudaMemcpyHostToDevice, s0));
        const float* pp[MR_MAX_FRAMES];
        const float* ip[MR_MAX_FRAMES];
        const float* fp[MR_MAX_FRAMES];
        for (int f = 0; f < F; ++f) {
            pp[f] = d_poses + (size_t)f * B * 16;
            ip[f] = d_intr + (size_t)f * B * 16;
            fp[f] = d_frames + (size_t)f * B * img1;
        }
        rc = mr_projection_tables(d_kpose, d_kK, pp, ip, B, F, H, W, d_proj, d_depths, D, inv_depth_lo, inv_depth_hi, s0);
        if (rc != MR_OK) return rc;
        MR_CUDA(cudaEventRecord(ring.ready, s0));
        for (int b = 0; b < B; ++b) {
            cudaStream_t s = ring.st[b % kStreams];
            MR_CUDA(cudaMemcpyAsync(d_key + b * img1, h_keyframe + b * img1, img1 * 4, cudaMemcpyHostToDevice, s));
            for (int f = 0; f < F; ++f) {
                size_t o = ((size_t)f * B + b) * img1;
                MR_CUDA(cudaMemcpyAsync(d_frames + o, h_frames + o, img1 * 4, cudaMemcpyHostToDevice, s));
            }
            MR_CUDA(cudaStreamWaitEvent(s, ring.ready, 0));
            rc = mr::launch_cost_volume(d_key, fp, d_proj, d_depths, d_cv, d_sfcv, B, F, D, H, W, alpha, nullptr, b, 1, 0, s,
                                        nullptr, 0, 0, MR_CV_SSIM, 1, out_dtype);
            if (rc != MR_OK) return rc;
            const size_t vbytes = vol1 * vb;
            MR_CUDA(cudaMemcpyAsync(o_cv + b * vbytes, d_cv + b * vbytes, vbytes, cudaMemcpyDeviceToHost, s));
            for (int f = 0; f < F && o_sfcv != nullptr; ++f) {
                size_t o = ((size_t)f * B + b) * vbytes;
                MR_CUDA(cudaMemcpyAsync(o_sfcv + o, d_sfcv + o, vbytes, cudaMemcpyDeviceToHost, s));
            }
        }
        return MR_OK;
    };
    rc = enqueue();
    for (int i = 0; i < ring.n; ++i) {
        const cudaError_t e = cudaStreamSynchronize(ring.st[i]);
        if (rc == MR_OK && e != cudaSuccess) rc = mr::check_cuda(e, out_dtype == MR_DT_F16 ? "mr_cost_volume_host_f16: cudaStreamSynchronize"
                                                                                  : "mr_cost_volume_host: cudaStreamSynchronize");
    }
    return rc;
}

}  // namespace

extern "C" int mr_cost_volume_host(const float* h_keyframe, const float* h_frames, const float* h_keyframe_pose,
                                   const float* h_keyframe_K, const float* h_poses, const float* h_intrinsics,
                                   float* h_out_cv, float* h_out_sfcv, int B, int F, int D, int H, int W,
                                   float inv_depth_lo, float inv_depth_hi, float alpha, void* workspace,
                                   long long workspace_bytes) {
    return cost_volume_host("mr_cost_volume_host", h_keyframe, h_frames, h_keyframe_pose, h_keyframe_K, h_poses, h_intrinsics,
                            h_out_cv, h_out_sfcv, B, F, D, H, W, inv_depth_lo, inv_depth_hi, alpha, workspace, workspace_bytes,
                            MR_DT_F32);
}

extern "C" int mr_cost_volume_host_f16(const float* h_keyframe, const float* h_frames, const float* h_keyframe_pose,
                                       const float* h_keyframe_K, const float* h_poses, const float* h_intrinsics,
                                       void* h_out_cv, void* h_out_sfcv, int B, int F, int D, int H, int W,
                                       float inv_depth_lo, float inv_depth_hi, float alpha, void* workspace,
                                       long long workspace_bytes) {
    return cost_volume_host("mr_cost_volume_host_f16", h_keyframe, h_frames, h_keyframe_pose, h_keyframe_K, h_poses,
                            h_intrinsics, h_out_cv, h_out_sfcv, B, F, D, H, W, inv_depth_lo, inv_depth_hi, alpha, workspace,
                            workspace_bytes, MR_DT_F16);
}
