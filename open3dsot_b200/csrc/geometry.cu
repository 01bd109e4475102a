// Box-frame crop of LiDAR scans — the per-frame / per-pair geometry of the tracking loop and of the training sampler
// (reference: datasets/points_utils.py generate_subwindow :223-254, cropAndCenterPC :102-124, crop_pc_axis_aligned :147-173).
//
//   local[b, i, :] = R[b]^T (scan[frame[b], i, :] - c[b])            points of sample b's scan in the frame of its box
//   keep[b, i]     = i < count[frame[b]]  &&  |local| < half[b]      strictly inside the scaled + padded box, per axis
//
// o3d_crop_box_frame: one pass over the scans: the frame gather, the rigid transform, the three comparisons and the padding
// mask that the tensor formulation spreads over a batched 3x3 GEMM and a dozen elementwise kernels.  HBM-bound: 12 B read,
// 13 B written per point; thread = point, a warp reads 384 contiguous bytes.
//
// o3d_crop_append: the same crop, compacted: the kept points of every slot are appended, in scan order, to the slot's
// history (the template of shape_aggregation 'all', getModel over every past frame, points_utils.py:88-100).  One CTA per
// slot walks its scan in tiles of 4096 points (4 consecutive points per thread: a warp reads 1.5 KB contiguously), one block
// scan per tile orders the kept points, and a warp's kept points land at consecutive history positions.
#include "common.cuh"
#include "../../include/o3d_b200.h"

namespace {

__global__ void __launch_bounds__(256)
    crop_box_frame_kernel(const float* __restrict__ scans, const long long* __restrict__ count, const long long* __restrict__ frame,
                          const float* __restrict__ center, const float* __restrict__ rot, const float* __restrict__ half, int N,
                          float* __restrict__ local, uint8_t* __restrict__ keep) {
    const int b = blockIdx.y;
    const long long f = frame ? frame[b] : b;
    const int n_valid = count ? (int)min((long long)N, count[f]) : N;
    const float cx = center[b * 3 + 0], cy = center[b * 3 + 1], cz = center[b * 3 + 2];
    float R[9];
#pragma unroll
    for (int j = 0; j < 9; ++j) R[j] = rot[b * 9 + j];
    const float hx = half[b * 3 + 0], hy = half[b * 3 + 1], hz = half[b * 3 + 2];
    const float* __restrict__ src = scans + (size_t)f * N * 3;
    float* __restrict__ dst = local + (size_t)b * N * 3;
    uint8_t* __restrict__ k = keep + (size_t)b * N;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < N; i += gridDim.x * blockDim.x) {
        float x, y, z;
        o3d_to_box_frame(src[i * 3 + 0] - cx, src[i * 3 + 1] - cy, src[i * 3 + 2] - cz, R, x, y, z);
        dst[i * 3 + 0] = x;
        dst[i * 3 + 1] = y;
        dst[i * 3 + 2] = z;
        k[i] = (uint8_t)(i < n_valid && fabsf(x) < hx && fabsf(y) < hy && fabsf(z) < hz);
    }
}

constexpr int CA_THREADS = 1024;           // o3d_block_exscan1024
constexpr int CA_PER = 4;                  // consecutive points per thread and tile
constexpr int CA_TILE = CA_THREADS * CA_PER;

__global__ void __launch_bounds__(CA_THREADS)
    crop_append_kernel(const float* __restrict__ scans, const long long* __restrict__ count, const long long* __restrict__ frame,
                       const float* __restrict__ center, const float* __restrict__ rot, const float* __restrict__ half, int N,
                       int H, float* __restrict__ hist, uint8_t* __restrict__ hist_keep, long long* __restrict__ hist_count) {
    __shared__ uint32_t s_warp[32];
    const int b = blockIdx.x, tid = threadIdx.x;
    const long long f = frame[b];
    if (f < 0) return;                                     // idle slot
    const int n_valid = count ? (int)min((long long)N, count[f]) : N;
    const float cx = center[b * 3 + 0], cy = center[b * 3 + 1], cz = center[b * 3 + 2];
    float R[9];
#pragma unroll
    for (int j = 0; j < 9; ++j) R[j] = rot[b * 9 + j];
    const float hx = half[b * 3 + 0], hy = half[b * 3 + 1], hz = half[b * 3 + 2];
    const float* __restrict__ src = scans + (size_t)f * N * 3;
    float* __restrict__ dst = hist + (size_t)b * H * 3;
    uint8_t* __restrict__ dk = hist_keep + (size_t)b * H;
    // every thread reads the count before the first barrier; thread 0 writes it back after the last one
    long long base = hist_count[b];
    for (int t0 = 0; t0 < n_valid; t0 += CA_TILE) {
        const int i0 = t0 + tid * CA_PER;
        float p[CA_PER][3];
        uint32_t m = 0;
#pragma unroll
        for (int j = 0; j < CA_PER; ++j) {
            const int i = i0 + j;
            if (i < n_valid) {
                o3d_to_box_frame(src[i * 3 + 0] - cx, src[i * 3 + 1] - cy, src[i * 3 + 2] - cz, R, p[j][0], p[j][1], p[j][2]);
                if (fabsf(p[j][0]) < hx && fabsf(p[j][1]) < hy && fabsf(p[j][2]) < hz) m |= 1u << j;
            }
        }
        uint32_t total;
        long long pos = base + o3d_block_exscan1024(__popc(m), s_warp, total);
#pragma unroll
        for (int j = 0; j < CA_PER; ++j) {
            if (m & (1u << j)) {
                if (pos < H) {
                    dst[pos * 3 + 0] = p[j][0];
                    dst[pos * 3 + 1] = p[j][1];
                    dst[pos * 3 + 2] = p[j][2];
                    dk[pos] = 1;
                }
                ++pos;
            }
        }
        base += total;
    }
    if (tid == 0) hist_count[b] = base;                    // the true count, including points past H
}

}  // namespace

extern "C" int o3d_crop_box_frame(const float* scans, const long long* count, const long long* frame, const float* center,
                                  const float* rot, const float* half, int B, int N, float* local, unsigned char* keep,
                                  void* stream) {
    O3D_REQUIRE(scans && center && rot && half && local && keep, O3D_ERR_ARG, "o3d_crop_box_frame: null pointer");
    O3D_REQUIRE(B >= 0 && N >= 0 && B <= 65535, O3D_ERR_ARG, "o3d_crop_box_frame: bad sizes B=%d N=%d", B, N);
    if (B == 0 || N == 0) return O3D_OK;
    int gx = (N + 255) / 256;
    const int cap = (8 * o3d_num_sms() + B - 1) / B;          // ~8 blocks per SM over the whole batch
    if (gx > cap) gx = cap < 1 ? 1 : cap;
    crop_box_frame_kernel<<<dim3(gx, B), 256, 0, (cudaStream_t)stream>>>(scans, count, frame, center, rot, half, N, local, keep);
    O3D_CHECK_LAUNCH("o3d_crop_box_frame");
    return O3D_OK;
}

extern "C" int o3d_crop_append(const float* scans, const long long* count, const long long* frame, const float* center,
                               const float* rot, const float* half, int B, int N, int H, float* hist, unsigned char* hist_keep,
                               long long* hist_count, void* stream) {
    O3D_REQUIRE(scans && frame && center && rot && half && hist && hist_keep && hist_count, O3D_ERR_ARG,
                "o3d_crop_append: null pointer");
    O3D_REQUIRE(B >= 0 && N >= 0 && H >= 0 && B <= 65535, O3D_ERR_ARG, "o3d_crop_append: bad sizes B=%d N=%d H=%d", B, N, H);
    if (B == 0 || N == 0) return O3D_OK;
    crop_append_kernel<<<B, CA_THREADS, 0, (cudaStream_t)stream>>>(scans, count, frame, center, rot, half, N, H, hist, hist_keep,
                                                                   hist_count);
    O3D_CHECK_LAUNCH("o3d_crop_append");
    return O3D_OK;
}
