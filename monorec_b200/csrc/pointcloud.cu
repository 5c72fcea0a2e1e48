// Point-cloud side of SURVEY.md section 8f row 3 (include/monorec_b200.h: mr_pointcloud_keep_mask, mr_pointcloud_add).
//
// Reference: create_pointcloud.py:65-105 (moving-object mask dilated by a 33x33 box, votes over a sliding window of frames,
// depth *= mask) and utils/ply_utils.py:34-53 PLYSaver.add_depthmap (1/x, distance / roi / dropout filter, Backprojection
// (model/layers.py:43-58) with inv(K), pose transform, boolean-mask compaction, .cpu().tolist() per frame).  Here the
// vertices stay on the device in one growing buffer, in the reference's order (batch element, then pixel, row-major).
// mr_pointcloud_add_windows runs the same vote for a batch of consecutive key frames of a sequence, each with its own window
// of keep masks in a device ring (create_pointcloud.py's sliding window, which crosses batch boundaries).
#include "mr_common.cuh"
#include <cstdint>

namespace {

constexpr int kBlk = 256;          // pixels per block of the compaction kernels

// keep[b,p] = 1 iff no pixel with cv_mask >= thresh lies in the (fill+1) x (fill+1) window centred on p
// (create_pointcloud.py:77-78: conv2d(mask, ones(fill+1), padding = fill // 2) < 1; zero padding outside the image)
__global__ void keep_mask_kernel(const float* __restrict__ cv_mask, float* __restrict__ keep, int H, int W, int rad, float thresh) {
    // separable box test: a block handles one image row segment; rows are scanned directly (the mask is small and L2-resident)
    const int b = blockIdx.z, y = blockIdx.y, x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= W) return;
    const float* m = cv_mask + (size_t)b * H * W;
    bool hit = false;
    const int y0 = max(y - rad, 0), y1 = min(y + rad, H - 1), x0 = max(x - rad, 0), x1 = min(x + rad, W - 1);
    for (int yy = y0; yy <= y1 && !hit; ++yy) {
        const float* row = m + (size_t)yy * W;
        for (int xx = x0; xx <= x1; ++xx)
            if (__ldg(row + xx) >= thresh) { hit = true; break; }
    }
    keep[((size_t)b * H + y) * W + x] = hit ? 0.f : 1.f;
}

constexpr int kMaxWindows = 256;   // key frames per mr_pointcloud_add_windows call (their window starts are kernel arguments)

struct PtrPackPC {
    const float* p[16];
};

// mr_pointcloud_add: n_masks keep masks [B,1,H,W] (sliding window), the same window for every batch element; may be empty
struct ListVote {
    PtrPackPC keeps;
    int n_masks;
    __device__ __forceinline__ float sum(int b, int i, size_t hw) const {
        float s = 0.f;
        for (int k = 0; k < n_masks; ++k) s += __ldg(keeps.p[k] + b * hw + i);
        return s;
    }
};

// mr_pointcloud_add_windows: batch element b votes with ring slots start[b], start[b] + 1, ... (mod ring_len), n_masks of them
struct RingVote {
    const float* ring;        // [ring_len,1,H,W]
    int ring_len, n_masks;
    int start[kMaxWindows];
    __device__ __forceinline__ float sum(int b, int i, size_t hw) const {
        float s = 0.f;
        int slot = start[b];
        for (int k = 0; k < n_masks; ++k) {
            s += __ldg(ring + slot * hw + i);
            if (++slot == ring_len) slot = 0;
        }
        return s;
    }
};

template <class Vote>
struct PcArgs {
    const float* inv_depth;   // [B,1,H,W] data_dict["result"]
    const float* image;       // [B,3,H,W] keyframe in [-0.5, 0.5]
    const float* K;           // [B,4,4] keyframe intrinsics
    const float* pose;        // [B,4,4] keyframe pose (camera -> world)
    Vote vote;
    int min_hits;
    const float* rnd;         // [B,1,H,W] uniform numbers for the dropout, or nullptr
    float dropout, min_d, max_d;
    int B, H, W, r0, r1, c0, c1;      // region of interest [r0, r1) x [c0, c1), clipped (the whole image without a roi)
    int* counts;              // [B * blocks_per_image] kept vertices per block, then exclusive offsets (in place)
    float* out;               // [capacity][6]
    long long capacity;
    long long* base;          // device: the buffer position of this call's first vertex (set by pc_scan_kernel)
    long long* total;         // device: number of vertices in the buffer after this call
};

template <class Vote>
__device__ __forceinline__ bool keep_vertex(const PcArgs<Vote>& a, int b, int i, float& depth) {
    const size_t o = (size_t)b * a.H * a.W + i;
    float inv = __ldg(a.inv_depth + o);
    if (a.vote.n_masks > 0) {   // mask = sum(mask_buffer) > buffer_length - min_hits; depth *= mask  (create_pointcloud.py:93-95)
        const float s = a.vote.sum(b, i, (size_t)a.H * a.W);
        inv *= (s > (float)(a.vote.n_masks - a.min_hits)) ? 1.f : 0.f;
    }
    depth = __fdiv_rn(1.0f, inv);                           // ply_utils.py:36 (1 / 0 = inf fails the range test below)
    const int y = i / a.W, x = i - y * a.W;
    bool ok = (a.min_d <= depth) && (depth <= a.max_d);     // :38
    ok = ok && y >= a.r0 && y < a.r1 && x >= a.c0 && x < a.c1;   // :39-43
    if (a.rnd != nullptr && a.dropout > 0.f) ok = ok && (__ldg(a.rnd + o) > a.dropout);   // :44-45
    return ok;
}

template <class Vote>
__global__ void pc_count_kernel(const __grid_constant__ PcArgs<Vote> a) {
    const int b = blockIdx.y, i = blockIdx.x * kBlk + threadIdx.x;
    float depth;
    const bool ok = (i < a.H * a.W) && keep_vertex(a, b, i, depth);
    const int n = __syncthreads_count(ok ? 1 : 0);
    if (threadIdx.x == 0) a.counts[b * gridDim.x + blockIdx.x] = n;
}

// exclusive scan of the per-block counts (a few thousand entries: one block, sequential chunks per thread + block scan).
// The batch's position is n_before, or (n_before < 0) the count *total left by the previous call on the stream; a negative
// count (an earlier call overflowed) stays negative and grows by this batch, so nothing more is written.
__global__ void pc_scan_kernel(int* counts, int n, long long n_before, long long capacity, long long* base_out,
                               long long* total) {
    __shared__ long long part[1024];
    const int t = threadIdx.x, per = (n + blockDim.x - 1) / blockDim.x;
    const int lo = min(t * per, n), hi = min(lo + per, n);
    long long s = 0;
    for (int i = lo; i < hi; ++i) s += counts[i];
    part[t] = s;
    __syncthreads();
    if (t == 0) {
        long long run = 0;
        for (int k = 0; k < (int)blockDim.x; ++k) { const long long v = part[k]; part[k] = run; run += v; }
        const long long base = n_before >= 0 ? n_before : *total;
        *base_out = base;
        if (base < 0) *total = base - run;
        else *total = (base + run <= capacity) ? base + run : -(base + run);   // negative: the buffer is too small (nothing is written)
    }
    __syncthreads();
    long long run = part[t];
    for (int i = lo; i < hi; ++i) { const int v = counts[i]; counts[i] = (int)run; run += v; }
}

__device__ bool invert4d(const float* src, double* out) {
    double m[4][8];
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) { m[i][j] = (double)src[i * 4 + j]; m[i][4 + j] = (i == j) ? 1.0 : 0.0; }
    for (int c = 0; c < 4; ++c) {
        int piv = c;
        double best = fabs(m[c][c]);
        for (int r = c + 1; r < 4; ++r)
            if (fabs(m[r][c]) > best) { best = fabs(m[r][c]); piv = r; }
        if (best == 0.0) return false;
        if (piv != c)
            for (int j = 0; j < 8; ++j) { double tmp = m[c][j]; m[c][j] = m[piv][j]; m[piv][j] = tmp; }
        const double inv = 1.0 / m[c][c];
        for (int j = 0; j < 8; ++j) m[c][j] *= inv;
        for (int r = 0; r < 4; ++r)
            if (r != c) { const double f = m[r][c]; for (int j = 0; j < 8; ++j) m[r][j] -= f * m[c][j]; }
    }
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) out[i * 4 + j] = m[i][4 + j];
    return true;
}

template <class Vote>
__global__ void pc_write_kernel(const __grid_constant__ PcArgs<Vote> a) {
    __shared__ float kinv[9], pose[12];
    __shared__ int wsum[kBlk / 32];
    const int b = blockIdx.y, i = blockIdx.x * kBlk + threadIdx.x;
    if (*a.total < 0) return;                    // capacity exceeded: reported through *total, nothing written
    if (threadIdx.x == 0) {
        double inv[16];
        const bool okk = invert4d(a.K + b * 16, inv);
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) kinv[r * 3 + c] = okk ? (float)inv[r * 4 + c] : __int_as_float(0x7fc00000);
        for (int k = 0; k < 12; ++k) pose[k] = a.pose[b * 16 + k];
    }
    float depth = 0.f;
    const bool ok = (i < a.H * a.W) && keep_vertex(a, b, i, depth);
    const unsigned bal = __ballot_sync(0xffffffffu, ok);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) wsum[warp] = __popc(bal);
    __syncthreads();
    if (!ok) return;
    int rank = __popc(bal & ((1u << lane) - 1));
    for (int w = 0; w < warp; ++w) rank += wsum[w];
    const long long at = *a.base + a.counts[b * gridDim.x + blockIdx.x] + rank;
    const int y = i / a.W, x = i - y * a.W;
    const float fx = (float)x, fy = (float)y;
    // Backprojection (layers.py:56-58): inv(K)[:3,:3] . (x, y, 1) * depth; then pose . (X, 1)   (ply_utils.py:47-49)
    const float cx = (kinv[0] * fx + kinv[1] * fy + kinv[2]) * depth;
    const float cy = (kinv[3] * fx + kinv[4] * fy + kinv[5]) * depth;
    const float cz = (kinv[6] * fx + kinv[7] * fy + kinv[8]) * depth;
    float* o = a.out + at * 6;
    o[0] = pose[0] * cx + pose[1] * cy + pose[2] * cz + pose[3];
    o[1] = pose[4] * cx + pose[5] * cy + pose[6] * cz + pose[7];
    o[2] = pose[8] * cx + pose[9] * cy + pose[10] * cz + pose[11];
    const size_t hw = (size_t)a.H * a.W;
    const float* im = a.image + (size_t)b * 3 * hw + i;
    o[3] = (__ldg(im) + 0.5f) * 255.0f;           // ply_utils.py:37
    o[4] = (__ldg(im + hw) + 0.5f) * 255.0f;
    o[5] = (__ldg(im + 2 * hw) + 0.5f) * 255.0f;
}

}  // namespace

extern "C" int mr_pointcloud_keep_mask(const float* cv_mask, float* keep, int B, int H, int W, int mask_fill, float thresh,
                                       void* stream) {
    MR_REQUIRE(cv_mask && keep, "mr_pointcloud_keep_mask: null pointer");
    MR_REQUIRE(B >= 1 && B <= 65535 && H >= 1 && H <= 65535 && W >= 1 && mask_fill >= 0 && (mask_fill % 2) == 0,
               "mr_pointcloud_keep_mask: bad shape / mask_fill must be even (the reference's conv2d keeps the size only then)");
    keep_mask_kernel<<<dim3((W + 127) / 128, H, B), 128, 0, (cudaStream_t)stream>>>(cv_mask, keep, H, W, mask_fill / 2, thresh);
    MR_LAUNCH_CHECK("keep_mask_kernel");
    return MR_OK;
}

// workspace: the batch's buffer position (one long long), then the per-block counts
extern "C" long long mr_pointcloud_workspace(int B, int H, int W) {
    if (B < 1 || H < 1 || W < 1) return 0;
    return (long long)sizeof(long long) + (long long)B * ((H * W + kBlk - 1) / kBlk) * (long long)sizeof(int);
}

namespace {

// the arguments both entries share, then count -> scan -> write
template <class Vote>
int add_vertices(PcArgs<Vote>& a, const float* inv_depth, const float* keyframe, const float* K, const float* pose,
                 int min_hits, int B, int H, int W, float min_d, float max_d, const int* roi, const float* dropout_rand,
                 float dropout, float* vertices, long long capacity, long long n_before, long long* n_after, void* workspace,
                 cudaStream_t st) {
    a.inv_depth = inv_depth; a.image = keyframe; a.K = K; a.pose = pose;
    a.min_hits = min_hits;
    a.rnd = dropout_rand; a.dropout = dropout; a.min_d = min_d; a.max_d = max_d;
    a.B = B; a.H = H; a.W = W;
    mr::clip_roi(roi, H, W, a.r0, a.r1, a.c0, a.c1);       // python slices, as PLYSaver masks; an empty roi keeps nothing
    a.base = static_cast<long long*>(workspace);
    a.counts = reinterpret_cast<int*>(a.base + 1);
    a.out = vertices; a.capacity = capacity; a.total = n_after;
    const int nb = (H * W + kBlk - 1) / kBlk;
    pc_count_kernel<<<dim3(nb, B), kBlk, 0, st>>>(a);
    MR_LAUNCH_CHECK("pc_count_kernel");
    pc_scan_kernel<<<1, 1024, 0, st>>>(a.counts, nb * B, n_before, capacity, a.base, n_after);
    MR_LAUNCH_CHECK("pc_scan_kernel");
    pc_write_kernel<<<dim3(nb, B), kBlk, 0, st>>>(a);
    MR_LAUNCH_CHECK("pc_write_kernel");
    return MR_OK;
}

}  // namespace

extern "C" int mr_pointcloud_add(const float* inv_depth, const float* keyframe, const float* K, const float* pose,
                                 const float* const* keep_masks, int n_masks, int min_hits, int B, int H, int W, float min_d,
                                 float max_d, const int* roi, const float* dropout_rand, float dropout, float* vertices,
                                 long long capacity, long long n_before, long long* n_after, void* workspace,
                                 long long workspace_bytes, void* stream) {
    MR_REQUIRE(inv_depth && keyframe && K && pose && vertices && n_after && workspace, "mr_pointcloud_add: null pointer");
    MR_REQUIRE(B >= 1 && B <= 65535 && H >= 1 && W >= 1 && n_masks >= 0 && n_masks <= 16 && (n_masks == 0 || keep_masks != nullptr),
               "mr_pointcloud_add: bad shape or more than 16 masks");
    MR_REQUIRE(capacity >= 0 && n_before <= capacity, "mr_pointcloud_add: bad buffer position");
    if (workspace_bytes < mr_pointcloud_workspace(B, H, W)) {
        mr::set_error("mr_pointcloud_add: workspace too small (%lld < %lld bytes)", workspace_bytes, mr_pointcloud_workspace(B, H, W));
        return MR_ENOMEM;
    }
    PcArgs<ListVote> a{};
    for (int k = 0; k < n_masks; ++k) {
        MR_REQUIRE(keep_masks[k] != nullptr, "mr_pointcloud_add: null mask %d", k);
        a.vote.keeps.p[k] = keep_masks[k];
    }
    a.vote.n_masks = n_masks;
    return add_vertices(a, inv_depth, keyframe, K, pose, min_hits, B, H, W, min_d, max_d, roi, dropout_rand, dropout, vertices,
                        capacity, n_before, n_after, workspace, (cudaStream_t)stream);
}

extern "C" int mr_pointcloud_add_windows(const float* inv_depth, const float* keyframe, const float* K, const float* pose,
                                         const float* keep_ring, int ring_len, const int* window_start, int n_masks,
                                         int min_hits, int B, int H, int W, float min_d, float max_d, const int* roi,
                                         const float* dropout_rand, float dropout, float* vertices, long long capacity,
                                         long long n_before, long long* n_after, void* workspace, long long workspace_bytes,
                                         void* stream) {
    MR_REQUIRE(inv_depth, "mr_pointcloud_add_windows: null pointer inv_depth");
    MR_REQUIRE(keyframe, "mr_pointcloud_add_windows: null pointer keyframe");
    MR_REQUIRE(K, "mr_pointcloud_add_windows: null pointer K");
    MR_REQUIRE(pose, "mr_pointcloud_add_windows: null pointer pose");
    MR_REQUIRE(keep_ring, "mr_pointcloud_add_windows: null pointer keep_ring");
    MR_REQUIRE(window_start, "mr_pointcloud_add_windows: null pointer window_start");
    MR_REQUIRE(vertices, "mr_pointcloud_add_windows: null pointer vertices");
    MR_REQUIRE(n_after, "mr_pointcloud_add_windows: null pointer n_after");
    MR_REQUIRE(workspace, "mr_pointcloud_add_windows: null pointer workspace");
    MR_REQUIRE(B >= 1 && B <= kMaxWindows, "mr_pointcloud_add_windows: B = %d outside [1, %d]", B, kMaxWindows);
    MR_REQUIRE(H >= 1 && W >= 1, "mr_pointcloud_add_windows: bad image size H = %d, W = %d", H, W);
    MR_REQUIRE(ring_len >= 1 && ring_len <= 65535, "mr_pointcloud_add_windows: ring_len = %d outside [1, 65535]", ring_len);
    MR_REQUIRE(n_masks >= 1 && n_masks <= ring_len, "mr_pointcloud_add_windows: n_masks = %d outside [1, ring_len = %d]",
               n_masks, ring_len);
    MR_REQUIRE(min_hits >= 1 && min_hits <= n_masks, "mr_pointcloud_add_windows: min_hits = %d outside [1, n_masks = %d]",
               min_hits, n_masks);
    for (int b = 0; b < B; ++b)
        MR_REQUIRE(window_start[b] >= 0 && window_start[b] < ring_len,
                   "mr_pointcloud_add_windows: window_start[%d] = %d outside the ring [0, %d)", b, window_start[b], ring_len);
    MR_REQUIRE(capacity >= 0 && n_before <= capacity,
               "mr_pointcloud_add_windows: bad buffer position n_before = %lld, capacity = %lld", n_before, capacity);
    if (workspace_bytes < mr_pointcloud_workspace(B, H, W)) {
        mr::set_error("mr_pointcloud_add_windows: workspace too small (%lld < %lld bytes)", workspace_bytes,
                      mr_pointcloud_workspace(B, H, W));
        return MR_ENOMEM;
    }
    PcArgs<RingVote> a{};
    a.vote.ring = keep_ring; a.vote.ring_len = ring_len; a.vote.n_masks = n_masks;
    for (int b = 0; b < B; ++b) a.vote.start[b] = window_start[b];
    return add_vertices(a, inv_depth, keyframe, K, pose, min_hits, B, H, W, min_d, max_d, roi, dropout_rand, dropout, vertices,
                        capacity, n_before, n_after, workspace, (cudaStream_t)stream);
}
