// Ball query, and ball query fused with grouping, for sm_90a.
//
// Replaces `_ext.ball_query` (pointnet2/utils/pointnet2_utils.py:268) and the whole of
// QueryAndGroup.forward (pointnet2/utils/pointnet2_utils.py:299-339: ball_query, 2x group_points,
// centre subtraction, optional /radius, cat).
//
// Design: a CTA serves CENTRES_PER_CTA centres of ONE cloud; the cloud's xyz (N*12 bytes) is staged into
// shared memory with a single 1-D bulk copy (cp.async.bulk -> UBLKCP, completion on an mbarrier) so the
// N-scan of every centre reads SMEM instead of re-reading global memory per thread as upstream does.
// One warp owns one centre: the 32 lanes test 32 consecutive points, `ballot` + `popc` compacts the hits in
// ascending index order (upstream's order), and the scan stops as soon as nsample hits exist.
// Grid = (ceil(M / CENTRES_PER_CTA), B)  -> hundreds of CTAs at the reference sizes instead of B blocks.
//
// In the fused kernel the same warp then emits the grouped rows: for each of its nsample neighbours it
// copies the neighbour's channels-last feature row with one float4 per lane (fully coalesced, 16-byte
// vectors) and appends (dx,dy,dz,0).  Output row = [features(C) | dx dy dz 0]  (C+4 floats, 16 B aligned).
//
// Exact semantics kept from upstream: d2 = fma(dz,dz,fma(dy,dy,dx*dx)) with centre-minus-point operands,
// strict d2 < r*r with r*r rounded in fp32, first hit replicated into unused slots, zeros when no hit.
#include "common.cuh"
#include "ball_query.cuh"
#include "../../include/o3d_b200.h"

namespace {

constexpr int BQ_WARPS = 8;
constexpr int BQ_THREADS = BQ_WARPS * 32;
constexpr int BQ_CENTRES_PER_WARP = 4;
constexpr int BQ_CENTRES_PER_CTA = BQ_WARPS * BQ_CENTRES_PER_WARP;

// Stage one cloud (N*3 floats) into shared memory.  Uses the bulk-copy engine when the source is 16-byte
// aligned and N*12 is a multiple of 16, otherwise a plain cooperative copy.
__device__ __forceinline__ void stage_cloud(float* s_xyz, const float* __restrict__ g, int N, uint64_t* bar) {
    const uint32_t bytes = (uint32_t)N * 12u;
    const bool bulk = ((bytes & 15u) == 0u) && ((reinterpret_cast<uintptr_t>(g) & 15u) == 0u);
    if (bulk) {
        if (threadIdx.x == 0) {
            o3d_mbar_init(bar, 1);
            o3d_fence_mbar_init();
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            o3d_mbar_expect_tx(bar, bytes);
            o3d_bulk_g2s(s_xyz, g, bytes, bar);
        }
        o3d_mbar_wait(bar, 0);
    } else {
        for (int i = threadIdx.x; i < 3 * N; i += blockDim.x) s_xyz[i] = g[i];
        __syncthreads();
    }
}

__global__ void __launch_bounds__(BQ_THREADS) ball_query_kernel(const float* __restrict__ new_xyz,
                                                                const float* __restrict__ xyz, int N, int M,
                                                                float radius2, int nsample, int32_t* __restrict__ idx) {
    extern __shared__ __align__(16) float s_xyz[];
    __shared__ __align__(8) uint64_t bar;
    const int b = blockIdx.y;
    stage_cloud(s_xyz, xyz + (size_t)b * N * 3, N, &bar);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int c_end = min(M, (int)(blockIdx.x + 1) * BQ_CENTRES_PER_CTA);
    for (int j = blockIdx.x * BQ_CENTRES_PER_CTA + warp; j < c_end; j += BQ_WARPS) {
        const float* c = new_xyz + ((size_t)b * M + j) * 3;
        warp_ball_query(s_xyz, N, c[0], c[1], c[2], radius2, nsample, idx + ((size_t)b * M + j) * nsample, lane);
    }
}

// Fused: ball query + grouping (+ centre subtraction, optional 1/radius) into channels-last rows.
__global__ void __launch_bounds__(BQ_THREADS)
    ballquery_group_kernel(const float* __restrict__ xyz, const float* __restrict__ new_xyz,
                           const float* __restrict__ feat_cl, int N, int M, int C, float radius, float radius2,
                           int nsample, int normalize, int32_t* __restrict__ idx, float* __restrict__ grouped) {
    extern __shared__ __align__(16) float s_xyz[];  // 3*N floats, then BQ_WARPS*nsample ints
    __shared__ __align__(8) uint64_t bar;
    const int b = blockIdx.y;
    int32_t* s_idx_all = reinterpret_cast<int32_t*>(s_xyz + ((3 * N + 3) & ~3));
    stage_cloud(s_xyz, xyz + (size_t)b * N * 3, N, &bar);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int32_t* s_idx = s_idx_all + warp * nsample;
    const int row = C + 4;
    const int c_end = min(M, (int)(blockIdx.x + 1) * BQ_CENTRES_PER_CTA);
    const float* __restrict__ fbase = feat_cl ? feat_cl + (size_t)b * N * C : nullptr;
    for (int j = blockIdx.x * BQ_CENTRES_PER_CTA + warp; j < c_end; j += BQ_WARPS) {
        const float* c = new_xyz + ((size_t)b * M + j) * 3;
        const float cx = c[0], cy = c[1], cz = c[2];
        warp_ball_query(s_xyz, N, cx, cy, cz, radius2, nsample, s_idx, lane);
        __syncwarp();
        float* __restrict__ obase = grouped + ((size_t)b * M + j) * nsample * row;
        if (idx) {
            int32_t* oi = idx + ((size_t)b * M + j) * nsample;
            for (int l = lane; l < nsample; l += 32) oi[l] = s_idx[l];
        }
        // relative coordinates: one lane per sample
        for (int l = lane; l < nsample; l += 32) {
            const int k = s_idx[l];
            float dx = __fsub_rn(s_xyz[k * 3 + 0], cx), dy = __fsub_rn(s_xyz[k * 3 + 1], cy),
                  dz = __fsub_rn(s_xyz[k * 3 + 2], cz);
            if (normalize) {
                dx = __fdiv_rn(dx, radius);
                dy = __fdiv_rn(dy, radius);
                dz = __fdiv_rn(dz, radius);
            }
            *reinterpret_cast<float4*>(obase + (size_t)l * row + C) = make_float4(dx, dy, dz, 0.f);
        }
        // feature rows: C/4 float4 per row, lanes stride the row
        if (fbase) {
            const int c4 = C >> 2;
            for (int l = 0; l < nsample; ++l) {
                const float4* __restrict__ src = reinterpret_cast<const float4*>(fbase + (size_t)s_idx[l] * C);
                float4* __restrict__ dst = reinterpret_cast<float4*>(obase + (size_t)l * row);
                for (int v = lane; v < c4; v += 32) dst[v] = __ldg(src + v);
            }
        }
        __syncwarp();
    }
}

// Backward of the fused grouping: scatter-add rows back to the source points.
//   grid = (ceil(M*S / rows_per_cta), B); a warp handles one grouped row at a time.
__global__ void __launch_bounds__(256)
    ballquery_group_grad_kernel(const float* __restrict__ gg, const int32_t* __restrict__ idx, int N, int M, int C,
                                int S, float inv_scale, float* __restrict__ gfeat, float* __restrict__ gxyz,
                                float* __restrict__ gnew) {
    const int b = blockIdx.y;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int rows = M * S;
    const int row = C + 4;
    for (int r = blockIdx.x * 8 + warp; r < rows; r += gridDim.x * 8) {
        const int k = idx[(size_t)b * rows + r];
        const float* __restrict__ g = gg + ((size_t)b * rows + r) * row;
        if (gfeat) {
            float* __restrict__ dst = gfeat + ((size_t)b * N + k) * C;
            for (int v = lane * 4; v < C; v += 128) {
                const float4 x = *reinterpret_cast<const float4*>(g + v);
                atomicAdd(reinterpret_cast<float4*>(dst + v), x);  // sm_90+: one vector RED per 16 bytes
            }
        }
        if ((gxyz || gnew) && lane < 3) {
            const float v = g[C + lane] * inv_scale;
            if (gxyz) atomicAdd(gxyz + ((size_t)b * N + k) * 3 + lane, v);
            if (gnew) atomicAdd(gnew + ((size_t)b * M + r / S) * 3 + lane, -v);
        }
    }
}

// Channels-last row gather by an explicit index list (BoxAware top-k grouping, xcorr.py:87-90):
//   out[b, j, s, :] = feat[b, idx[b,j,s], :]      one warp per output row, float4 per lane.
__global__ void __launch_bounds__(256)
    group_rows_kernel(const float* __restrict__ feat, const int32_t* __restrict__ idx, int N, int L, int C,
                      float* __restrict__ out) {
    const int b = blockIdx.y;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int c4 = C >> 2;
    for (int r = blockIdx.x * 8 + warp; r < L; r += gridDim.x * 8) {
        const int k = idx[(size_t)b * L + r];
        const float4* __restrict__ src = reinterpret_cast<const float4*>(feat + ((size_t)b * N + k) * C);
        float4* __restrict__ dst = reinterpret_cast<float4*>(out + ((size_t)b * L + r) * C);
        for (int v = lane; v < c4; v += 32) dst[v] = __ldg(src + v);
    }
}

__global__ void __launch_bounds__(256)
    group_rows_grad_kernel(const float* __restrict__ gout, const int32_t* __restrict__ idx, int N, int L, int C,
                           float* __restrict__ gfeat) {
    const int b = blockIdx.y;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int r = blockIdx.x * 8 + warp; r < L; r += gridDim.x * 8) {
        const int k = idx[(size_t)b * L + r];
        const float* __restrict__ g = gout + ((size_t)b * L + r) * C;
        float* __restrict__ dst = gfeat + ((size_t)b * N + k) * C;
        for (int v = lane * 4; v < C; v += 128) atomicAdd(reinterpret_cast<float4*>(dst + v), *reinterpret_cast<const float4*>(g + v));
    }
}

}  // namespace

extern "C" int o3d_ball_query(const float* new_xyz, const float* xyz, int B, int N, int M, float radius, int nsample,
                              int32_t* idx, void* stream) {
    O3D_REQUIRE(new_xyz && xyz && idx, O3D_ERR_ARG, "o3d_ball_query: null pointer");
    O3D_REQUIRE(B >= 0 && N >= 1 && M >= 0 && nsample >= 1, O3D_ERR_ARG, "o3d_ball_query: bad sizes");
    const size_t smem = (size_t)N * 12;
    O3D_REQUIRE(smem <= 200 * 1024, O3D_ERR_ARG, "o3d_ball_query: N=%d too large for the shared-memory tile", N);
    if (B == 0 || M == 0) return O3D_OK;
    if (smem > 48 * 1024)
        O3D_CUDA(cudaFuncSetAttribute(ball_query_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem),
                 "o3d_ball_query: smem attribute");
    dim3 grid((M + BQ_CENTRES_PER_CTA - 1) / BQ_CENTRES_PER_CTA, B);
    ball_query_kernel<<<grid, BQ_THREADS, smem, (cudaStream_t)stream>>>(new_xyz, xyz, N, M, radius * radius, nsample,
                                                                         idx);
    O3D_CHECK_LAUNCH("o3d_ball_query");
    return O3D_OK;
}

extern "C" int o3d_ballquery_group(const float* xyz, const float* new_xyz, const float* feat_cl, int B, int N, int M,
                                   int C, float radius, int nsample, int normalize_xyz, int32_t* idx,
                                   float* grouped_cl, void* stream) {
    O3D_REQUIRE(xyz && new_xyz && grouped_cl, O3D_ERR_ARG, "o3d_ballquery_group: null pointer");
    O3D_REQUIRE(B >= 0 && N >= 1 && M >= 0 && nsample >= 1 && C >= 0, O3D_ERR_ARG, "o3d_ballquery_group: bad sizes");
    O3D_REQUIRE((C & 3) == 0, O3D_ERR_ARG, "o3d_ballquery_group: C=%d must be a multiple of 4", C);
    O3D_REQUIRE(feat_cl || C == 0, O3D_ERR_ARG, "o3d_ballquery_group: C>0 needs features");
    O3D_REQUIRE(((uintptr_t)grouped_cl & 15) == 0 && ((uintptr_t)feat_cl & 15) == 0, O3D_ERR_ALIGN,
                "o3d_ballquery_group: feature/grouped pointers must be 16-byte aligned");
    const size_t smem = (size_t)((3 * N + 3) & ~3) * 4 + (size_t)BQ_WARPS * nsample * 4;
    O3D_REQUIRE(smem <= 200 * 1024, O3D_ERR_ARG, "o3d_ballquery_group: N=%d too large", N);
    if (B == 0 || M == 0) return O3D_OK;
    if (smem > 48 * 1024)
        O3D_CUDA(cudaFuncSetAttribute(ballquery_group_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem),
                 "o3d_ballquery_group: smem attribute");
    dim3 grid((M + BQ_CENTRES_PER_CTA - 1) / BQ_CENTRES_PER_CTA, B);
    ballquery_group_kernel<<<grid, BQ_THREADS, smem, (cudaStream_t)stream>>>(
        xyz, new_xyz, feat_cl, N, M, C, radius, radius * radius, nsample, normalize_xyz, idx, grouped_cl);
    O3D_CHECK_LAUNCH("o3d_ballquery_group");
    return O3D_OK;
}

extern "C" int o3d_ballquery_group_grad(const float* grad_grouped_cl, const int32_t* idx, int B, int N, int M, int C,
                                        int S, float radius, int normalize_xyz, float* grad_feat_cl, float* grad_xyz,
                                        float* grad_new_xyz, void* stream) {
    O3D_REQUIRE(grad_grouped_cl && idx, O3D_ERR_ARG, "o3d_ballquery_group_grad: null pointer");
    O3D_REQUIRE((C & 3) == 0, O3D_ERR_ARG, "o3d_ballquery_group_grad: C must be a multiple of 4");
    O3D_REQUIRE(((uintptr_t)grad_grouped_cl & 15) == 0 && ((uintptr_t)grad_feat_cl & 15) == 0, O3D_ERR_ALIGN,
                "o3d_ballquery_group_grad: pointers must be 16-byte aligned");
    if (B == 0 || M == 0 || S == 0) return O3D_OK;
    const int rows = M * S;
    int gx = (rows + 7) / 8;
    const int cap = o3d_num_sms() * 8;
    if (gx > cap) gx = cap;
    dim3 grid(gx, B);
    ballquery_group_grad_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(grad_grouped_cl, idx, N, M, C, S,
                                                                         normalize_xyz ? 1.0f / radius : 1.0f,
                                                                         grad_feat_cl, grad_xyz, grad_new_xyz);
    O3D_CHECK_LAUNCH("o3d_ballquery_group_grad");
    return O3D_OK;
}

extern "C" int o3d_group_rows(const float* feat_cl, const int32_t* idx, int B, int N, int L, int C, float* out_cl,
                              void* stream) {
    O3D_REQUIRE(feat_cl && idx && out_cl, O3D_ERR_ARG, "o3d_group_rows: null pointer");
    O3D_REQUIRE((C & 3) == 0, O3D_ERR_ARG, "o3d_group_rows: C must be a multiple of 4");
    O3D_REQUIRE(((uintptr_t)feat_cl & 15) == 0 && ((uintptr_t)out_cl & 15) == 0, O3D_ERR_ALIGN,
                "o3d_group_rows: pointers must be 16-byte aligned");
    if (B == 0 || L == 0 || C == 0) return O3D_OK;
    int gx = (L + 7) / 8;
    const int cap = o3d_num_sms() * 8;
    if (gx > cap) gx = cap;
    group_rows_kernel<<<dim3(gx, B), 256, 0, (cudaStream_t)stream>>>(feat_cl, idx, N, L, C, out_cl);
    O3D_CHECK_LAUNCH("o3d_group_rows");
    return O3D_OK;
}

extern "C" int o3d_group_rows_grad(const float* grad_out_cl, const int32_t* idx, int B, int N, int L, int C,
                                   float* grad_feat_cl, void* stream) {
    O3D_REQUIRE(grad_out_cl && idx && grad_feat_cl, O3D_ERR_ARG, "o3d_group_rows_grad: null pointer");
    O3D_REQUIRE((C & 3) == 0, O3D_ERR_ARG, "o3d_group_rows_grad: C must be a multiple of 4");
    if (B == 0 || L == 0 || C == 0) return O3D_OK;
    int gx = (L + 7) / 8;
    const int cap = o3d_num_sms() * 8;
    if (gx > cap) gx = cap;
    group_rows_grad_kernel<<<dim3(gx, B), 256, 0, (cudaStream_t)stream>>>(grad_out_cl, idx, N, L, C, grad_feat_cl);
    O3D_CHECK_LAUNCH("o3d_group_rows_grad");
    return O3D_OK;
}
