// Oxford RobotCar lidar depth targets for sm_90a: OxfordRobotCarDataset.get_depth (reference:
// data_loader/oxford_robotcar_dataset.py:121-144) with the SDK's pinhole CameraModel.project.
//
// The loader re-reads and re-transforms every LD-MRS scan within +-lidar_timestamp_range of each key frame, projects the
// points, argsorts them by inverse depth and scatters them into a full-size float64 array (last write wins: the largest
// inverse depth, the nearest point), crops it and rounds it to float32.  Here:
//   mr_lidar_to_world  one launch per scan: (lidar_pose @ lidar_transform) @ [x y z 1]^T into a device ring of world points,
//                      once per scan rather than once per key frame;
//   mr_lidar_depth     K key frames per launch: each thread takes one world point of one key frame's window, applies the
//                      key frame's camera matrix, G_camera_image and the pinhole projection, filters, scales, truncates and
//                      stores 1/z, rounded to float32, with atomicMax on the bit pattern.  Positive floats order as their bits
//                      and rounding is monotone, so the maximum of the rounded values is the rounded maximum: the loader's
//                      last-write-wins scatter after its ascending sort, without a sort and independent of the point order.
// All arithmetic is float64, op by op in the loader's order (naive left-to-right sums, no contracted FMAs), so each point's
// pixel and value equal the numpy restatement's bit for bit; numpy's BLAS products may differ from it in the last bit.
#include "mr_common.cuh"
#include <cmath>
#include <cstdint>

namespace {

constexpr int kThreads = 256;
constexpr int kKeysPerLaunch = 16;    // per-key data rides in the kernel parameters (16 x 144 B + the common part < 4 KB)

struct WorldArgs {
    const double* scan;   // [n,3]
    double* ring;         // [capacity,4]
    double M[16];         // row-major 4x4
    long long n, capacity, first;
};

// ((m0 x + m1 y) + m2 z) + m3 w, each product and sum rounded on its own: numpy's 4x4 @ [4,n] in the naive order
__device__ __forceinline__ double dot4(const double* m, double x, double y, double z, double w) {
    return __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(m[0], x), __dmul_rn(m[1], y)), __dmul_rn(m[2], z)), __dmul_rn(m[3], w));
}

__global__ void __launch_bounds__(kThreads) lidar_to_world_kernel(const WorldArgs a) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i >= a.n) return;
    const double x = a.scan[3 * i], y = a.scan[3 * i + 1], z = a.scan[3 * i + 2];
    long long r = a.first + i;
    if (r >= a.capacity) r -= a.capacity;
    double* o = a.ring + 4 * r;
    const double2 lo = make_double2(dot4(a.M, x, y, z, 1.0), dot4(a.M + 4, x, y, z, 1.0));
    const double2 hi = make_double2(dot4(a.M + 8, x, y, z, 1.0), dot4(a.M + 12, x, y, z, 1.0));
    reinterpret_cast<double2*>(o)[0] = lo;
    reinterpret_cast<double2*>(o)[1] = hi;
}

struct KeyArgs {
    double C[16];               // camera_transform @ inv(pose @ swapaxes_), row-major
    long long first, count;     // window: ring rows first, first + 1, ... (mod capacity), count of them
};

struct DepthArgs {
    const double* ring;         // [capacity,4]
    float* out;                 // [K,1,r1-r0,c1-c0]
    int* oob;                   // [K] points whose truncated pixel lies outside the Hd x Wd array
    double G[16];               // G_camera_image, row-major
    double fx, fy, cx, cy, lo, u_hi, v_hi, scale;
    long long capacity;
    int Hd, Wd, r0, r1, c0, c1;
    int k0;                     // index of keys[0] in the K key frames of the call
    KeyArgs keys[kKeysPerLaunch];
};

__global__ void __launch_bounds__(kThreads) lidar_depth_kernel(const DepthArgs a) {
    __shared__ double sC[16];
    __shared__ long long sWin[2];
    const int k = blockIdx.y;
    if (threadIdx.x == 0) {
        // constant indices only: a dynamic index into the parameter struct would copy it to the stack
#pragma unroll
        for (int j = 0; j < kKeysPerLaunch; ++j)
            if (j == k) {
#pragma unroll
                for (int e = 0; e < 16; ++e) sC[e] = a.keys[j].C[e];
                sWin[0] = a.keys[j].first;
                sWin[1] = a.keys[j].count;
            }
    }
    __syncthreads();
    double C[16];
#pragma unroll
    for (int e = 0; e < 16; ++e) C[e] = sC[e];
    const long long first = sWin[0], count = sWin[1];
    const int kk = a.k0 + k, ho = a.r1 - a.r0, wo = a.c1 - a.c0;
    int* plane = reinterpret_cast<int*>(a.out) + (size_t)kk * ho * wo;
    int oob = 0;
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < count; i += (long long)gridDim.x * kThreads) {
        long long r = first + i;
        if (r >= a.capacity) r -= a.capacity;
        const double2 p01 = __ldg(reinterpret_cast<const double2*>(a.ring + 4 * r));
        const double2 p23 = __ldg(reinterpret_cast<const double2*>(a.ring + 4 * r) + 1);
        // world -> camera (step 3), then G_camera_image (the SDK's projection)
        const double q0 = dot4(C, p01.x, p01.y, p23.x, p23.y), q1 = dot4(C + 4, p01.x, p01.y, p23.x, p23.y);
        const double q2 = dot4(C + 8, p01.x, p01.y, p23.x, p23.y), q3 = dot4(C + 12, p01.x, p01.y, p23.x, p23.y);
        const double x = dot4(a.G, q0, q1, q2, q3), y = dot4(a.G + 4, q0, q1, q2, q3), z = dot4(a.G + 8, q0, q1, q2, q3);
        if (!(z > 0.0)) continue;
        // uv = f * xy / z + principal_point; kept iff 0.5 <= u <= W and 0.5 <= v <= H (NaN compares false)
        const double u = __dadd_rn(__ddiv_rn(__dmul_rn(a.fx, x), z), a.cx);
        const double v = __dadd_rn(__ddiv_rn(__dmul_rn(a.fy, y), z), a.cy);
        if (!(a.lo <= u && u <= a.u_hi && a.lo <= v && v <= a.v_hi)) continue;
        // uv *= scale; astype(int) truncates toward zero
        const long long iu = __double2ll_rz(__dmul_rn(u, a.scale)), iv = __double2ll_rz(__dmul_rn(v, a.scale));
        if (iu < 0 || iu >= a.Wd || iv < 0 || iv >= a.Hd) { ++oob; continue; }    // numpy raises IndexError
        if (iv < a.r0 || iv >= a.r1 || iu < a.c0 || iu >= a.c1) continue;           // cropped away
        const float d = __double2float_rn(__ddiv_rn(1.0, z));
        atomicMax(plane + (size_t)(iv - a.r0) * wo + (iu - a.c0), __float_as_int(d));
    }
    if (oob) atomicAdd(a.oob + kk, oob);
}

}  // namespace

extern "C" int mr_lidar_to_world(const double* scan, long long n, const double* M, double* ring, long long capacity,
                                 long long first, void* stream) {
    const char* who = "mr_lidar_to_world";
    MR_REQUIRE(M && ring && (scan || n == 0), "%s: null pointer", who);
    MR_REQUIRE(capacity >= 1 && capacity <= (1LL << 40), "%s: capacity %lld out of range (1 .. 2^40)", who, capacity);
    MR_REQUIRE(n >= 0 && n <= capacity, "%s: point count %lld out of range (0 .. capacity %lld)", who, n, capacity);
    MR_REQUIRE(first >= 0 && first < capacity, "%s: first row %lld out of range (0 .. capacity %lld)", who, first, capacity);
    MR_REQUIRE((reinterpret_cast<uintptr_t>(scan) & 7) == 0 && (reinterpret_cast<uintptr_t>(ring) & 15) == 0,
               "%s: scan must be 8-byte and ring 16-byte aligned", who);
    for (int e = 0; e < 16; ++e) MR_REQUIRE(std::isfinite(M[e]), "%s: M[%d] is not finite", who, e);
    if (n == 0) return MR_OK;
    WorldArgs a{};
    a.scan = scan; a.ring = ring; a.n = n; a.capacity = capacity; a.first = first;
    for (int e = 0; e < 16; ++e) a.M[e] = M[e];
    lidar_to_world_kernel<<<(unsigned)((n + kThreads - 1) / kThreads), kThreads, 0, (cudaStream_t)stream>>>(a);
    MR_LAUNCH_CHECK("lidar_to_world_kernel");
    return MR_OK;
}

extern "C" int mr_lidar_depth(const double* ring, long long capacity, int K, const long long* first, const long long* count,
                              const double* cam, const double* G, const double* proj, int Hd, int Wd, const int* crop,
                              float* out, int* out_of_array, void* stream) {
    const char* who = "mr_lidar_depth";
    MR_REQUIRE(ring && first && count && cam && G && proj && crop && out && out_of_array, "%s: null pointer", who);
    MR_REQUIRE(capacity >= 1 && capacity <= (1LL << 40), "%s: capacity %lld out of range (1 .. 2^40)", who, capacity);
    MR_REQUIRE(K >= 1 && K <= 65535, "%s: key-frame count %d out of range (1 .. 65535)", who, K);
    MR_REQUIRE(Hd >= 1 && Wd >= 1 && Hd <= 65535 && Wd <= 65535, "%s: depth array %dx%d out of range (1 .. 65535)", who, Hd, Wd);
    MR_REQUIRE(crop[0] >= 0 && crop[0] < crop[1] && crop[1] <= Hd && crop[2] >= 0 && crop[2] < crop[3] && crop[3] <= Wd,
               "%s: crop [%d:%d, %d:%d] is not a non-empty window of the %dx%d array", who, crop[0], crop[1], crop[2],
               crop[3], Hd, Wd);
    for (int e = 0; e < 16; ++e) MR_REQUIRE(std::isfinite(G[e]), "%s: G[%d] is not finite", who, e);
    for (int e = 0; e < 8; ++e) MR_REQUIRE(std::isfinite(proj[e]), "%s: proj[%d] is not finite", who, e);
    MR_REQUIRE(proj[7] > 0.0, "%s: scale (%g) must be > 0", who, proj[7]);
    long long most = 0;
    for (int k = 0; k < K; ++k) {
        MR_REQUIRE(count[k] >= 0 && count[k] <= capacity, "%s: key frame %d: count %lld out of range (0 .. %lld)", who, k,
                   count[k], capacity);
        MR_REQUIRE(first[k] >= 0 && first[k] < capacity, "%s: key frame %d: first row %lld out of range (0 .. %lld)", who, k,
                   first[k], capacity);
        for (int e = 0; e < 16; ++e)
            MR_REQUIRE(std::isfinite(cam[16 * k + e]), "%s: key frame %d: camera matrix entry %d is not finite", who, k, e);
        most = count[k] > most ? count[k] : most;
    }
    MR_REQUIRE((reinterpret_cast<uintptr_t>(ring) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 3) == 0 &&
               (reinterpret_cast<uintptr_t>(out_of_array) & 3) == 0,
               "%s: ring must be 16-byte, out and out_of_array 4-byte aligned", who);
    const size_t plane = (size_t)(crop[1] - crop[0]) * (crop[3] - crop[2]);
    cudaStream_t s = (cudaStream_t)stream;
    MR_CUDA(cudaMemsetAsync(out, 0, (size_t)K * plane * sizeof(float), s));
    MR_CUDA(cudaMemsetAsync(out_of_array, 0, (size_t)K * sizeof(int), s));
    if (most == 0) return MR_OK;
    DepthArgs a{};
    a.ring = ring; a.out = out; a.oob = out_of_array; a.capacity = capacity;
    for (int e = 0; e < 16; ++e) a.G[e] = G[e];
    a.fx = proj[0]; a.fy = proj[1]; a.cx = proj[2]; a.cy = proj[3]; a.lo = proj[4]; a.u_hi = proj[5]; a.v_hi = proj[6];
    a.scale = proj[7];
    a.Hd = Hd; a.Wd = Wd; a.r0 = crop[0]; a.r1 = crop[1]; a.c0 = crop[2]; a.c1 = crop[3];
    // enough CTAs per key frame to fill the SMs; each walks its window with a grid stride
    const long long blocks = (most + kThreads - 1) / kThreads;
    for (int k0 = 0; k0 < K; k0 += kKeysPerLaunch) {
        const int nk = K - k0 < kKeysPerLaunch ? K - k0 : kKeysPerLaunch;
        a.k0 = k0;
        for (int j = 0; j < nk; ++j) {
            for (int e = 0; e < 16; ++e) a.keys[j].C[e] = cam[16 * (k0 + j) + e];
            a.keys[j].first = first[k0 + j];
            a.keys[j].count = count[k0 + j];
        }
        dim3 grid((unsigned)(blocks < 1024 ? blocks : 1024), nk);
        lidar_depth_kernel<<<grid, kThreads, 0, s>>>(a);
        MR_LAUNCH_CHECK("lidar_depth_kernel");
    }
    return MR_OK;
}
