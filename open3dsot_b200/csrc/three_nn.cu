// three_nn / three_interpolate (+grad) and the fused three_nn+interpolate, for sm_90a.
//
// Replaces `_ext.three_nn` (pointnet2/utils/pointnet2_utils.py:125), `_ext.three_interpolate(_grad)`
// (:162,:184) and — fused — the body of PointnetFPModule.forward (pointnet2/utils/pointnet2_modules.py:187-195).
//
// Design: one WARP per unknown point.  The known cloud is staged in shared memory per CTA; each lane scans
// k = lane, lane+32, ... keeping its private top-3 (strict '<' insertion, ascending k, exactly upstream's
// rule), then three REDUX rounds pop the warp-wide minimum of the lane heads ordered by (d2, k) — the same
// total order upstream's single ascending scan produces (ties -> lower index first).  The fused kernel goes
// on to compute the inverse-distance weights and writes the interpolated channels-last row with coalesced
// float4 stores, so the (B,c,n) gather of upstream (stride-m reads, one block per batch) disappears.
#include "common.cuh"
#include "../../include/o3d_b200.h"

namespace {

constexpr int NN_WARPS = 8;
constexpr int NN_THREADS = NN_WARPS * 32;
constexpr uint32_t NN_INF = 0x7f800000u;  // +inf: upstream's 1e40 sentinel after the cast to float

struct Top3 {
    uint32_t d[3];  // float bit patterns of squared distances (>= +0 -> monotone as unsigned)
    int k[3];
};

__device__ __forceinline__ void top3_insert(Top3& t, uint32_t d, int k) {
    if (d < t.d[0]) {
        t.d[2] = t.d[1]; t.k[2] = t.k[1]; t.d[1] = t.d[0]; t.k[1] = t.k[0]; t.d[0] = d; t.k[0] = k;
    } else if (d < t.d[1]) {
        t.d[2] = t.d[1]; t.k[2] = t.k[1]; t.d[1] = d; t.k[1] = k;
    } else if (d < t.d[2]) {
        t.d[2] = d; t.k[2] = k;
    }
}

// Warp-wide 3 nearest of `m` staged points to (ux,uy,uz); result identical on all lanes.
__device__ __forceinline__ Top3 warp_three_nn(const float* s_known, int m, float ux, float uy, float uz, int lane) {
    Top3 t;
    t.d[0] = t.d[1] = t.d[2] = NN_INF;
    t.k[0] = t.k[1] = t.k[2] = 0;
    for (int k = lane; k < m; k += 32) {
        const float d = o3d_dist2(ux, uy, uz, s_known[k * 3 + 0], s_known[k * 3 + 1], s_known[k * 3 + 2]);
        top3_insert(t, __float_as_uint(d), k);
    }
    Top3 r;
#pragma unroll
    for (int round = 0; round < 3; ++round) {
        const uint32_t md = __reduce_min_sync(0xFFFFFFFFu, t.d[0]);
        // among lanes whose head equals md, the lowest index wins; a head of +inf means "empty"
        const uint32_t cand = (t.d[0] == md && md != NN_INF) ? (uint32_t)t.k[0] : 0xFFFFFFFFu;
        const uint32_t mk = __reduce_min_sync(0xFFFFFFFFu, cand);
        r.d[round] = md;
        r.k[round] = (mk == 0xFFFFFFFFu) ? 0 : (int)mk;
        if (cand == mk && mk != 0xFFFFFFFFu) {  // pop this lane's head
            t.d[0] = t.d[1]; t.k[0] = t.k[1]; t.d[1] = t.d[2]; t.k[1] = t.k[2]; t.d[2] = NN_INF; t.k[2] = 0;
        }
    }
    return r;
}

__device__ __forceinline__ void stage_known(float* s, const float* __restrict__ g, int m) {
    for (int i = threadIdx.x; i < 3 * m; i += blockDim.x) s[i] = g[i];
    __syncthreads();
}

__global__ void __launch_bounds__(NN_THREADS)
    three_nn_kernel(const float* __restrict__ unknown, const float* __restrict__ known, int n, int m,
                    float* __restrict__ dist2, int32_t* __restrict__ idx) {
    extern __shared__ __align__(16) float s_known[];
    const int b = blockIdx.y;
    stage_known(s_known, known + (size_t)b * m * 3, m);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int j = blockIdx.x * NN_WARPS + warp; j < n; j += gridDim.x * NN_WARPS) {
        const float* u = unknown + ((size_t)b * n + j) * 3;
        const Top3 r = warp_three_nn(s_known, m, u[0], u[1], u[2], lane);
        if (lane < 3) {
            dist2[((size_t)b * n + j) * 3 + lane] = __uint_as_float(lane == 0 ? r.d[0] : lane == 1 ? r.d[1] : r.d[2]);
            idx[((size_t)b * n + j) * 3 + lane] = lane == 0 ? r.k[0] : lane == 1 ? r.k[1] : r.k[2];
        }
    }
}

// (B,c,m) layout interpolation, reference-compatible.
__global__ void __launch_bounds__(256)
    three_interpolate_kernel(const float* __restrict__ feat, const int32_t* __restrict__ idx,
                             const float* __restrict__ w, int c, int m, int n, float* __restrict__ out) {
    const int b = blockIdx.z, l = blockIdx.y;
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const int32_t* i3 = idx + ((size_t)b * n + j) * 3;
    const float* w3 = w + ((size_t)b * n + j) * 3;
    const float* __restrict__ f = feat + ((size_t)b * c + l) * m;
    out[((size_t)b * c + l) * n + j] =
        __fmaf_rn(__ldg(f + i3[2]), w3[2], __fmaf_rn(__ldg(f + i3[1]), w3[1], __fmul_rn(__ldg(f + i3[0]), w3[0])));
}

__global__ void __launch_bounds__(256)
    three_interpolate_grad_kernel(const float* __restrict__ gout, const int32_t* __restrict__ idx,
                                  const float* __restrict__ w, int c, int n, int m, float* __restrict__ gfeat) {
    const int b = blockIdx.z, l = blockIdx.y;
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const int32_t* i3 = idx + ((size_t)b * n + j) * 3;
    const float* w3 = w + ((size_t)b * n + j) * 3;
    const float g = gout[((size_t)b * c + l) * n + j];
    float* gf = gfeat + ((size_t)b * c + l) * m;
    atomicAdd(gf + i3[0], g * w3[0]);
    atomicAdd(gf + i3[1], g * w3[1]);
    atomicAdd(gf + i3[2], g * w3[2]);
}

// Fused FP-module front end, channels-last.
__global__ void __launch_bounds__(NN_THREADS)
    three_nn_interpolate_kernel(const float* __restrict__ unknown, const float* __restrict__ known,
                                const float* __restrict__ kfeat, int n, int m, int c, float* __restrict__ out,
                                int32_t* __restrict__ idx, float* __restrict__ weight) {
    extern __shared__ __align__(16) float s_known[];
    const int b = blockIdx.y;
    stage_known(s_known, known + (size_t)b * m * 3, m);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int c4 = c >> 2;
    for (int j = blockIdx.x * NN_WARPS + warp; j < n; j += gridDim.x * NN_WARPS) {
        const float* u = unknown + ((size_t)b * n + j) * 3;
        const Top3 r = warp_three_nn(s_known, m, u[0], u[1], u[2], lane);
        // weights as the reference computes them with torch ops (pointnet2_modules.py:188-191)
        const float r0 = __fdiv_rn(1.0f, __fadd_rn(__fsqrt_rn(__uint_as_float(r.d[0])), 1e-8f));
        const float r1 = __fdiv_rn(1.0f, __fadd_rn(__fsqrt_rn(__uint_as_float(r.d[1])), 1e-8f));
        const float r2 = __fdiv_rn(1.0f, __fadd_rn(__fsqrt_rn(__uint_as_float(r.d[2])), 1e-8f));
        const float norm = __fadd_rn(__fadd_rn(r0, r1), r2);
        const float w0 = __fdiv_rn(r0, norm), w1 = __fdiv_rn(r1, norm), w2 = __fdiv_rn(r2, norm);
        if (lane < 3) {
            idx[((size_t)b * n + j) * 3 + lane] = lane == 0 ? r.k[0] : lane == 1 ? r.k[1] : r.k[2];
            weight[((size_t)b * n + j) * 3 + lane] = lane == 0 ? w0 : lane == 1 ? w1 : w2;
        }
        const float4* __restrict__ f0 = reinterpret_cast<const float4*>(kfeat + ((size_t)b * m + r.k[0]) * c);
        const float4* __restrict__ f1 = reinterpret_cast<const float4*>(kfeat + ((size_t)b * m + r.k[1]) * c);
        const float4* __restrict__ f2 = reinterpret_cast<const float4*>(kfeat + ((size_t)b * m + r.k[2]) * c);
        float4* __restrict__ o = reinterpret_cast<float4*>(out + ((size_t)b * n + j) * c);
        for (int v = lane; v < c4; v += 32) {
            const float4 a = __ldg(f0 + v), bb = __ldg(f1 + v), cc = __ldg(f2 + v);
            float4 y;
            y.x = __fmaf_rn(cc.x, w2, __fmaf_rn(bb.x, w1, __fmul_rn(a.x, w0)));
            y.y = __fmaf_rn(cc.y, w2, __fmaf_rn(bb.y, w1, __fmul_rn(a.y, w0)));
            y.z = __fmaf_rn(cc.z, w2, __fmaf_rn(bb.z, w1, __fmul_rn(a.z, w0)));
            y.w = __fmaf_rn(cc.w, w2, __fmaf_rn(bb.w, w1, __fmul_rn(a.w, w0)));
            o[v] = y;
        }
    }
}

__global__ void __launch_bounds__(NN_THREADS)
    three_nn_interpolate_grad_kernel(const float* __restrict__ gout, const int32_t* __restrict__ idx,
                                     const float* __restrict__ weight, int n, int m, int c,
                                     float* __restrict__ gfeat) {
    const int b = blockIdx.y;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int j = blockIdx.x * NN_WARPS + warp; j < n; j += gridDim.x * NN_WARPS) {
        const int32_t* i3 = idx + ((size_t)b * n + j) * 3;
        const float* w3 = weight + ((size_t)b * n + j) * 3;
        const float* __restrict__ g = gout + ((size_t)b * n + j) * c;
        for (int t = 0; t < 3; ++t) {
            float* dst = gfeat + ((size_t)b * m + i3[t]) * c;
            const float w = w3[t];
            for (int v = lane * 4; v < c; v += 128) {
                float4 x = *reinterpret_cast<const float4*>(g + v);
                x.x *= w; x.y *= w; x.z *= w; x.w *= w;
                atomicAdd(reinterpret_cast<float4*>(dst + v), x);
            }
        }
    }
}

}  // namespace

extern "C" int o3d_three_nn(const float* unknown, const float* known, int B, int n, int m, float* dist2, int32_t* idx,
                            void* stream) {
    O3D_REQUIRE(unknown && known && dist2 && idx, O3D_ERR_ARG, "o3d_three_nn: null pointer");
    O3D_REQUIRE(B >= 0 && n >= 0 && m >= 0, O3D_ERR_ARG, "o3d_three_nn: bad sizes");
    const size_t smem = (size_t)m * 12;
    O3D_REQUIRE(smem <= 200 * 1024, O3D_ERR_ARG, "o3d_three_nn: m=%d too large", m);
    if (B == 0 || n == 0) return O3D_OK;
    if (smem > 48 * 1024)
        O3D_CUDA(cudaFuncSetAttribute(three_nn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem),
                 "o3d_three_nn: smem attribute");
    dim3 grid((n + NN_WARPS * 4 - 1) / (NN_WARPS * 4), B);
    three_nn_kernel<<<grid, NN_THREADS, smem, (cudaStream_t)stream>>>(unknown, known, n, m, dist2, idx);
    O3D_CHECK_LAUNCH("o3d_three_nn");
    return O3D_OK;
}

extern "C" int o3d_three_interpolate(const float* features, const int32_t* idx, const float* weight, int B, int c,
                                     int m, int n, float* out, void* stream) {
    O3D_REQUIRE(features && idx && weight && out, O3D_ERR_ARG, "o3d_three_interpolate: null pointer");
    if (B == 0 || c == 0 || n == 0) return O3D_OK;
    O3D_REQUIRE(c <= 65535 && B <= 65535, O3D_ERR_ARG, "o3d_three_interpolate: B or c too large");
    dim3 grid((n + 255) / 256, c, B);
    three_interpolate_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(features, idx, weight, c, m, n, out);
    O3D_CHECK_LAUNCH("o3d_three_interpolate");
    return O3D_OK;
}

extern "C" int o3d_three_interpolate_grad(const float* grad_out, const int32_t* idx, const float* weight, int B, int c,
                                          int n, int m, float* grad_features, void* stream) {
    O3D_REQUIRE(grad_out && idx && weight && grad_features, O3D_ERR_ARG, "o3d_three_interpolate_grad: null pointer");
    if (B == 0 || c == 0 || n == 0) return O3D_OK;
    O3D_REQUIRE(c <= 65535 && B <= 65535, O3D_ERR_ARG, "o3d_three_interpolate_grad: B or c too large");
    dim3 grid((n + 255) / 256, c, B);
    three_interpolate_grad_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(grad_out, idx, weight, c, n, m,
                                                                           grad_features);
    O3D_CHECK_LAUNCH("o3d_three_interpolate_grad");
    return O3D_OK;
}

extern "C" int o3d_three_nn_interpolate(const float* unknown, const float* known, const float* known_feat_cl, int B,
                                        int n, int m, int c, float* out_cl, int32_t* idx, float* weight,
                                        void* stream) {
    O3D_REQUIRE(unknown && known && known_feat_cl && out_cl && idx && weight, O3D_ERR_ARG,
                "o3d_three_nn_interpolate: null pointer");
    // every unknown point reads the feature rows of its three neighbours (row 0 stands in for a missing one): an empty known
    // cloud has no row to read
    O3D_REQUIRE(B >= 0 && n >= 0 && m >= 1, O3D_ERR_ARG, "o3d_three_nn_interpolate: bad sizes B=%d n=%d m=%d (m >= 1)", B, n,
                m);
    O3D_REQUIRE((c & 3) == 0, O3D_ERR_ARG, "o3d_three_nn_interpolate: c must be a multiple of 4");
    O3D_REQUIRE(((uintptr_t)known_feat_cl & 15) == 0 && ((uintptr_t)out_cl & 15) == 0, O3D_ERR_ALIGN,
                "o3d_three_nn_interpolate: feature pointers must be 16-byte aligned");
    const size_t smem = (size_t)m * 12;
    O3D_REQUIRE(smem <= 200 * 1024, O3D_ERR_ARG, "o3d_three_nn_interpolate: m too large");
    if (B == 0 || n == 0) return O3D_OK;
    if (smem > 48 * 1024)
        O3D_CUDA(cudaFuncSetAttribute(three_nn_interpolate_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)smem),
                 "o3d_three_nn_interpolate: smem attribute");
    dim3 grid((n + NN_WARPS * 4 - 1) / (NN_WARPS * 4), B);
    three_nn_interpolate_kernel<<<grid, NN_THREADS, smem, (cudaStream_t)stream>>>(unknown, known, known_feat_cl, n, m,
                                                                                  c, out_cl, idx, weight);
    O3D_CHECK_LAUNCH("o3d_three_nn_interpolate");
    return O3D_OK;
}

extern "C" int o3d_three_nn_interpolate_grad(const float* grad_out_cl, const int32_t* idx, const float* weight, int B,
                                             int n, int m, int c, float* grad_known_feat_cl, void* stream) {
    O3D_REQUIRE(grad_out_cl && idx && weight && grad_known_feat_cl, O3D_ERR_ARG,
                "o3d_three_nn_interpolate_grad: null pointer");
    O3D_REQUIRE((c & 3) == 0, O3D_ERR_ARG, "o3d_three_nn_interpolate_grad: c must be a multiple of 4");
    if (B == 0 || n == 0) return O3D_OK;
    dim3 grid((n + NN_WARPS * 4 - 1) / (NN_WARPS * 4), B);
    three_nn_interpolate_grad_kernel<<<grid, NN_THREADS, 0, (cudaStream_t)stream>>>(grad_out_cl, idx, weight, n, m, c,
                                                                                    grad_known_feat_cl);
    O3D_CHECK_LAUNCH("o3d_three_nn_interpolate_grad");
    return O3D_OK;
}
