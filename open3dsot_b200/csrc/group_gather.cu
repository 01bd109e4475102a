// gather_points / group_points and their gradients in the reference's (B,C,N) layout, for sm_90a.
//
// Replaces `_ext.gather_points(_grad)` (pointnet2/utils/pointnet2_utils.py:92,98) and
// `_ext.group_points(_grad)` (:217,:237).  These keep the reference tensor layout so that the
// reference's own autograd Functions work unchanged on top of them (INTEGRATION.md); the native
// modules use the channels-last fused kernels in ball_query.cu / pwmlp.cu instead.
//
// Design: the output is a dense (B*C, M*S) matrix whose rows are gathered from rows of N floats.
// One CTA handles one (b, c-slab) and streams the index list once per slab: indices and outputs are
// contiguous along the thread index (coalesced), the gathered source row (<= a few KB) stays in L1.
// Grid = (ceil(M*S / 1024), ceil(C / CH_PER_CTA), B) — thousands of CTAs rather than upstream's B blocks.
// Backward uses fp32 RED (atomicAdd without return), like upstream's atomicAdd.
#include "common.cuh"
#include "../../include/o3d_b200.h"

namespace {

constexpr int GG_THREADS = 256;
constexpr int GG_PER_THREAD = 4;
constexpr int GG_CH_PER_CTA = 8;

__global__ void __launch_bounds__(GG_THREADS)
    group_kernel(const float* __restrict__ feat, const int32_t* __restrict__ idx, int C, int N, int L /*M*S*/,
                 float* __restrict__ out) {
    const int b = blockIdx.z;
    const int c0 = blockIdx.y * GG_CH_PER_CTA;
    const int c1 = min(C, c0 + GG_CH_PER_CTA);
    const int base = (blockIdx.x * GG_THREADS + threadIdx.x) * GG_PER_THREAD;
    int32_t k[GG_PER_THREAD];
    const int32_t* __restrict__ ib = idx + (size_t)b * L;
    if (base + GG_PER_THREAD <= L && (L & 3) == 0) {
        const int4 v = *reinterpret_cast<const int4*>(ib + base);
        k[0] = v.x; k[1] = v.y; k[2] = v.z; k[3] = v.w;
        for (int c = c0; c < c1; ++c) {
            const float* __restrict__ f = feat + ((size_t)b * C + c) * N;
            float4 o = make_float4(__ldg(f + k[0]), __ldg(f + k[1]), __ldg(f + k[2]), __ldg(f + k[3]));
            *reinterpret_cast<float4*>(out + ((size_t)b * C + c) * L + base) = o;
        }
    } else {
        for (int i = 0; i < GG_PER_THREAD; ++i) k[i] = (base + i < L) ? ib[base + i] : 0;
        for (int c = c0; c < c1; ++c) {
            const float* __restrict__ f = feat + ((size_t)b * C + c) * N;
            for (int i = 0; i < GG_PER_THREAD; ++i)
                if (base + i < L) out[((size_t)b * C + c) * L + base + i] = __ldg(f + k[i]);
        }
    }
}

__global__ void __launch_bounds__(GG_THREADS)
    group_grad_kernel(const float* __restrict__ gout, const int32_t* __restrict__ idx, int C, int N, int L,
                      float* __restrict__ gfeat) {
    const int b = blockIdx.z;
    const int c0 = blockIdx.y * GG_CH_PER_CTA;
    const int c1 = min(C, c0 + GG_CH_PER_CTA);
    const int base = (blockIdx.x * GG_THREADS + threadIdx.x) * GG_PER_THREAD;
    const int32_t* __restrict__ ib = idx + (size_t)b * L;
    for (int i = 0; i < GG_PER_THREAD; ++i) {
        if (base + i >= L) break;
        const int k = ib[base + i];
        for (int c = c0; c < c1; ++c)
            atomicAdd(gfeat + ((size_t)b * C + c) * N + k, gout[((size_t)b * C + c) * L + base + i]);
    }
}

int launch_group(const float* feat, const int32_t* idx, int B, int C, int N, int L, float* out, cudaStream_t st,
                 const char* name) {
    if (B == 0 || C == 0 || L == 0) return O3D_OK;
    dim3 grid((L + GG_THREADS * GG_PER_THREAD - 1) / (GG_THREADS * GG_PER_THREAD),
              (C + GG_CH_PER_CTA - 1) / GG_CH_PER_CTA, B);
    O3D_REQUIRE(grid.y <= 65535 && grid.z <= 65535, O3D_ERR_ARG, "%s: B or C too large for the launch grid", name);
    group_kernel<<<grid, GG_THREADS, 0, st>>>(feat, idx, C, N, L, out);
    O3D_CHECK_LAUNCH(name);
    return O3D_OK;
}

int launch_group_grad(const float* gout, const int32_t* idx, int B, int C, int N, int L, float* gfeat, cudaStream_t st,
                      const char* name) {
    if (B == 0 || C == 0 || L == 0) return O3D_OK;
    dim3 grid((L + GG_THREADS * GG_PER_THREAD - 1) / (GG_THREADS * GG_PER_THREAD),
              (C + GG_CH_PER_CTA - 1) / GG_CH_PER_CTA, B);
    O3D_REQUIRE(grid.y <= 65535 && grid.z <= 65535, O3D_ERR_ARG, "%s: B or C too large for the launch grid", name);
    group_grad_kernel<<<grid, GG_THREADS, 0, st>>>(gout, idx, C, N, L, gfeat);
    O3D_CHECK_LAUNCH(name);
    return O3D_OK;
}

}  // namespace

extern "C" int o3d_gather(const float* features, const int32_t* idx, int B, int C, int N, int M, float* out,
                          void* stream) {
    O3D_REQUIRE(features && idx && out, O3D_ERR_ARG, "o3d_gather: null pointer");
    return launch_group(features, idx, B, C, N, M, out, (cudaStream_t)stream, "o3d_gather");
}
extern "C" int o3d_gather_grad(const float* grad_out, const int32_t* idx, int B, int C, int N, int M,
                               float* grad_features, void* stream) {
    O3D_REQUIRE(grad_out && idx && grad_features, O3D_ERR_ARG, "o3d_gather_grad: null pointer");
    return launch_group_grad(grad_out, idx, B, C, N, M, grad_features, (cudaStream_t)stream, "o3d_gather_grad");
}
extern "C" int o3d_group(const float* features, const int32_t* idx, int B, int C, int N, int M, int S, float* out,
                         void* stream) {
    O3D_REQUIRE(features && idx && out, O3D_ERR_ARG, "o3d_group: null pointer");
    return launch_group(features, idx, B, C, N, M * S, out, (cudaStream_t)stream, "o3d_group");
}
extern "C" int o3d_group_grad(const float* grad_out, const int32_t* idx, int B, int C, int N, int M, int S,
                              float* grad_features, void* stream) {
    O3D_REQUIRE(grad_out && idx && grad_features, O3D_ERR_ARG, "o3d_group_grad: null pointer");
    return launch_group_grad(grad_out, idx, B, C, N, M * S, grad_features, (cudaStream_t)stream, "o3d_group_grad");
}
