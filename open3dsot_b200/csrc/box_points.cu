// Evidence of the live tracker (tracking/multi_tracker.py): how many points of the scan a target advanced on lie in the box it
// was just given.  nuscenes points_in_box(box, points, wlh_factor) restated as the inclusive test in the box frame:
//
//   n_in[k] = #{ i < count[frame[k]] :  |R[k]^T (scans[frame[k], i] - center[k])| <= half[k] per axis }
//
// The box-frame coordinates are tracking/boxes.py box_point_counts' fp32 arithmetic, operation by operation:
//   d = p - c;  local_j = (d_x R[0][j] + d_y R[1][j]) + d_z R[2][j]
// every operation an explicit round-to-nearest intrinsic, since the build contracts a*b+c into FMAs by default and the tensor
// formulation does not.  So the counts equal that formulation's exactly.
//
// One launch sequence: a memset of n_in, then a (gx, K) grid; block (x, k) walks a grid-stride share of row k's scan, reduces
// its count over warps and adds it to n_in[k] with one integer atomic.  Integer sums do not depend on the order the blocks
// arrive in, so the counts are identical run to run.  Rows that read the same scan find it in L2 (a 120,000-point scan is
// 1.44 MB).
#include "common.cuh"
#include "../../include/o3d_b200.h"

namespace {

constexpr int BP_THREADS = 256;
constexpr int BP_POINTS_PER_THREAD = 8;        // points a thread tests before the grid is capped

__global__ void __launch_bounds__(BP_THREADS)
    box_points_kernel(const float* __restrict__ scans, const long long* __restrict__ count, const long long* __restrict__ frame,
                      const float* __restrict__ center, const float* __restrict__ rot, const float* __restrict__ half, int N,
                      int* __restrict__ n_in) {
    __shared__ int s_warp[BP_THREADS / 32];
    const int k = blockIdx.y;
    const long long f = frame[k];
    const long long c = count ? count[f] : (long long)N;
    const int n_valid = (int)max(0LL, min((long long)N, c));
    const float cx = center[k * 3 + 0], cy = center[k * 3 + 1], cz = center[k * 3 + 2];
    float R[9];
#pragma unroll
    for (int j = 0; j < 9; ++j) R[j] = rot[k * 9 + j];
    const float hx = half[k * 3 + 0], hy = half[k * 3 + 1], hz = half[k * 3 + 2];
    const float* __restrict__ src = scans + (size_t)f * N * 3;
    int n = 0;
    for (int i = blockIdx.x * BP_THREADS + threadIdx.x; i < n_valid; i += gridDim.x * BP_THREADS) {
        const float dx = __fsub_rn(src[i * 3 + 0], cx);
        const float dy = __fsub_rn(src[i * 3 + 1], cy);
        const float dz = __fsub_rn(src[i * 3 + 2], cz);
        const float x = __fadd_rn(__fadd_rn(__fmul_rn(dx, R[0]), __fmul_rn(dy, R[3])), __fmul_rn(dz, R[6]));
        const float y = __fadd_rn(__fadd_rn(__fmul_rn(dx, R[1]), __fmul_rn(dy, R[4])), __fmul_rn(dz, R[7]));
        const float z = __fadd_rn(__fadd_rn(__fmul_rn(dx, R[2]), __fmul_rn(dy, R[5])), __fmul_rn(dz, R[8]));
        n += (fabsf(x) <= hx && fabsf(y) <= hy && fabsf(z) <= hz) ? 1 : 0;
    }
    n = __reduce_add_sync(0xffffffffu, n);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) s_warp[warp] = n;
    __syncthreads();
    if (warp == 0) {
        n = lane < BP_THREADS / 32 ? s_warp[lane] : 0;
        n = __reduce_add_sync(0xffffffffu, n);
        if (lane == 0 && n != 0) atomicAdd(n_in + k, n);
    }
}

}  // namespace

extern "C" int o3d_box_points(const float* scans, const long long* count, const long long* frame, const float* center,
                              const float* rot, const float* half, int N, int K, int* n_in, void* stream) {
    O3D_REQUIRE(scans && frame && center && rot && half && n_in, O3D_ERR_ARG, "o3d_box_points: null pointer");
    O3D_REQUIRE(K >= 0 && K <= 65535 && N >= 0, O3D_ERR_ARG, "o3d_box_points: bad sizes K=%d N=%d", K, N);
    if (K == 0) return O3D_OK;
    const cudaStream_t s = (cudaStream_t)stream;
    O3D_CUDA(cudaMemsetAsync(n_in, 0, (size_t)K * sizeof(int), s), "o3d_box_points");
    if (N == 0) return O3D_OK;
    int gx = (N + BP_THREADS * BP_POINTS_PER_THREAD - 1) / (BP_THREADS * BP_POINTS_PER_THREAD);
    const int cap = (16 * o3d_num_sms() + K - 1) / K;       // ~16 blocks per SM over all rows
    if (gx > cap) gx = cap < 1 ? 1 : cap;
    box_points_kernel<<<dim3(gx, K), BP_THREADS, 0, s>>>(scans, count, frame, center, rot, half, N, n_in);
    O3D_CHECK_LAUNCH("o3d_box_points");
    return O3D_OK;
}
