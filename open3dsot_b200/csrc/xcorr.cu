// Template-search cross-correlation front ends (models/head/xcorr.py), sm_90a.
//
//   o3d_xcorr_boxaware_fwd   BoxAwareXCorr (xcorr.py:81-88): for every search point the k template points whose 9-D box
//                            clouds are nearest.  The reference computes `torch.cdist` (64 x 128 points -> its
//                            |a|^2 + |b|^2 - 2ab matmul formulation), a full `argsort` of the 64 distances per column and
//                            keeps the first k (k = 4).  Here: one thread per search point, the template box cloud in shared
//                            memory, squared distances by direct differences (fma chain, more accurate than the matmul
//                            form) and a k-slot insertion list in registers; ties keep the LOWER template index (the
//                            reference's argsort is not stable: its tie order is unspecified).  Ranking by d^2 equals ranking
//                            by d.  Membership can differ from cdist's only when two candidates are within cdist's own
//                            rounding error of each other.
//   o3d_xcorr_p2b_fwd/bwd    P2B_XCorr's cosine map (xcorr.py:37-38): sim[b,j,i] = <t_i/max(|t_i|,eps), s_j/max(|s_j|,eps)>
//                            (torch >= 1.12 cosine_similarity semantics), laid out (B, n2, n1) = the position order of the
//                            lifted stack that consumes it as its per-position scalar `s` (o3d_lift_t), and its gradient.
//                            Warp-level dot products over the template points: a warp owns two search points, a lane two
//                            template points, operands staged through shared memory in 32-channel chunks.
// The MLP + max-pool that follows either front end is the lifted stack (lift.cu, pwmlp_tc.cu); the gradient of the
// BoxAware grouping is its scatter kernel (indices carry no gradient).
#include "common.cuh"
#include "../../include/o3d_b200.h"

namespace {

constexpr int TOPK_MAX = 8;
constexpr int TOPK_THREADS = 128;

__global__ void __launch_bounds__(TOPK_THREADS)
    boxaware_topk_kernel(const float* __restrict__ tbc, const float* __restrict__ sbc, int M, int N, int D, int k,
                         int32_t* __restrict__ idx) {
    extern __shared__ float s_t[];                    // [M][D]
    const int b = blockIdx.y;
    for (int i = threadIdx.x; i < M * D; i += blockDim.x) s_t[i] = tbc[(size_t)b * M * D + i];
    __syncthreads();
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= N) return;
    float q[16];
    const float* sp = sbc + ((size_t)b * N + j) * D;
#pragma unroll
    for (int d = 0; d < 16; ++d) q[d] = d < D ? sp[d] : 0.f;
    float bd[TOPK_MAX];
    int bi[TOPK_MAX];
#pragma unroll
    for (int t = 0; t < TOPK_MAX; ++t) { bd[t] = INFINITY; bi[t] = 0; }
    for (int i = 0; i < M; ++i) {
        float d2 = 0.f;
#pragma unroll
        for (int d = 0; d < 16; ++d) {
            if (d < D) {
                const float df = s_t[i * D + d] - q[d];
                d2 = fmaf(df, df, d2);
            }
        }
        // insertion: strictly smaller moves ahead, so equal distances keep ascending template order
        float cd = d2;
        int ci = i;
        bool shifting = false;       // once the candidate is placed, everything below it moves down one slot
#pragma unroll
        for (int t = 0; t < TOPK_MAX; ++t) {
            if (t < k && (shifting || cd < bd[t])) {
                shifting = true;
                const float td = bd[t]; const int ti = bi[t];
                bd[t] = cd; bi[t] = ci;
                cd = td; ci = ti;
            }
        }
    }
    int32_t* o = idx + ((size_t)b * N + j) * k;
#pragma unroll
    for (int t = 0; t < TOPK_MAX; ++t)
        if (t < k) o[t] = t < M ? bi[t] : 0;
}

// ---- cosine map --------------------------------------------------------------------------------------------
constexpr int SIM_J = 16;        // search points per block (2 per warp)
constexpr int SIM_CH = 32;       // channels per staged chunk
constexpr int SIM_IMAX = 4;      // template points per lane (n1 <= 128)

__global__ void __launch_bounds__(256)
    p2b_sim_kernel(const float* __restrict__ tf, const float* __restrict__ sf, int n1, int n2, int C, float eps,
                   float* __restrict__ sim, float* __restrict__ tnorm, float* __restrict__ snorm) {
    extern __shared__ float sm[];                     // T chunk [n1][33] | S chunk [SIM_J][33]
    float* st = sm;
    float* ss = sm + n1 * (SIM_CH + 1);
    const int b = blockIdx.y, j0 = blockIdx.x * SIM_J;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float acc[2][SIM_IMAX], tt[SIM_IMAX], sq[2];
#pragma unroll
    for (int a = 0; a < 2; ++a) {
        sq[a] = 0.f;
#pragma unroll
        for (int u = 0; u < SIM_IMAX; ++u) acc[a][u] = 0.f;
    }
#pragma unroll
    for (int u = 0; u < SIM_IMAX; ++u) tt[u] = 0.f;
    for (int c0 = 0; c0 < C; c0 += SIM_CH) {
        __syncthreads();
        for (int e = threadIdx.x; e < n1 * SIM_CH; e += blockDim.x) {
            const int i = e / SIM_CH, c = e % SIM_CH;
            st[i * (SIM_CH + 1) + c] = (c0 + c < C) ? tf[((size_t)b * n1 + i) * C + c0 + c] : 0.f;
        }
        for (int e = threadIdx.x; e < SIM_J * SIM_CH; e += blockDim.x) {
            const int j = e / SIM_CH, c = e % SIM_CH;
            ss[j * (SIM_CH + 1) + c] = (j0 + j < n2 && c0 + c < C) ? sf[((size_t)b * n2 + j0 + j) * C + c0 + c] : 0.f;
        }
        __syncthreads();
#pragma unroll 8
        for (int c = 0; c < SIM_CH; ++c) {
            const float s0 = ss[(2 * warp) * (SIM_CH + 1) + c], s1 = ss[(2 * warp + 1) * (SIM_CH + 1) + c];
            sq[0] = fmaf(s0, s0, sq[0]);
            sq[1] = fmaf(s1, s1, sq[1]);
#pragma unroll
            for (int u = 0; u < SIM_IMAX; ++u) {
                const int i = lane + 32 * u;
                const float t = i < n1 ? st[i * (SIM_CH + 1) + c] : 0.f;
                tt[u] = fmaf(t, t, tt[u]);
                acc[0][u] = fmaf(t, s0, acc[0][u]);
                acc[1][u] = fmaf(t, s1, acc[1][u]);
            }
        }
    }
#pragma unroll
    for (int a = 0; a < 2; ++a) {
        const int j = j0 + 2 * warp + a;
        if (j >= n2) continue;
        const float ns = sqrtf(sq[a]);
        if (lane == 0 && snorm) snorm[(size_t)b * n2 + j] = ns;
        const float is = 1.f / fmaxf(ns, eps);
#pragma unroll
        for (int u = 0; u < SIM_IMAX; ++u) {
            const int i = lane + 32 * u;
            if (i >= n1) continue;
            const float nt = sqrtf(tt[u]);
            if (blockIdx.x == 0 && warp == 0 && a == 0 && tnorm) tnorm[(size_t)b * n1 + i] = nt;
            sim[((size_t)b * n2 + j) * n1 + i] = acc[a][u] * (1.f / fmaxf(nt, eps)) * is;
        }
    }
}

// gradient w.r.t. the rows of X (one block per row r of X) given the rows of the other operand Y:
//   dX[r] = ( sum_q w[q] * Y[q] / max(|Y[q]|, eps)  -  [|X[r]| > eps] * (sum_q w[q] * sim[q]) * X[r] / |X[r]| ) / max(|X[r]|, eps)
// with w[q] = dsim at (r, q).  `stride_q` / `stride_r` address dsim / sim, which are stored (B, n2, n1).
__global__ void __launch_bounds__(256)
    p2b_sim_grad_kernel(const float* __restrict__ dsim, const float* __restrict__ sim, const float* __restrict__ X,
                        const float* __restrict__ Y, const float* __restrict__ xnorm, const float* __restrict__ ynorm,
                        int nx, int ny, int C, float eps, long long stride_r, long long stride_q, float* __restrict__ dX) {
    extern __shared__ float w[];                      // [ny] weights, then [1] the sim-weighted sum
    const int b = blockIdx.y, r = blockIdx.x;
    const float* ds = dsim + (size_t)b * nx * ny + (size_t)r * stride_r;
    const float* si = sim + (size_t)b * nx * ny + (size_t)r * stride_r;
    float part = 0.f;
    for (int q = threadIdx.x; q < ny; q += blockDim.x) {
        const float g = ds[(size_t)q * stride_q];
        w[q] = g / fmaxf(ynorm[(size_t)b * ny + q], eps);
        part = fmaf(g, si[(size_t)q * stride_q], part);
    }
    __shared__ float red[8];
    for (int o = 16; o >= 1; o >>= 1) part += __shfl_xor_sync(0xFFFFFFFFu, part, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = part;
    __syncthreads();
    float rs = 0.f;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) rs += red[i];
    const float nx_ = xnorm[(size_t)b * nx + r];
    const float im = 1.f / fmaxf(nx_, eps);
    const float proj = nx_ > eps ? rs / nx_ : 0.f;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        float a = 0.f;
        for (int q = 0; q < ny; ++q) a = fmaf(w[q], Y[((size_t)b * ny + q) * C + c], a);
        const float x = X[((size_t)b * nx + r) * C + c];
        dX[((size_t)b * nx + r) * C + c] = (a - proj * x) * im;
    }
}

}  // namespace

extern "C" int o3d_xcorr_boxaware_fwd(const float* template_bc, const float* search_bc, int B, int M, int N, int D, int k,
                                      int32_t* idx, void* stream) {
    O3D_REQUIRE(template_bc && search_bc && idx, O3D_ERR_ARG, "o3d_xcorr_boxaware_fwd: null pointer");
    O3D_REQUIRE(B >= 0 && M >= 1 && N >= 0 && D >= 1 && D <= 16 && k >= 1 && k <= TOPK_MAX && k <= M, O3D_ERR_ARG,
                "o3d_xcorr_boxaware_fwd: need 1 <= D <= 16, 1 <= k <= min(%d, M); got M=%d D=%d k=%d", TOPK_MAX, M, D, k);
    O3D_REQUIRE((size_t)M * D * sizeof(float) <= 48 * 1024, O3D_ERR_ARG, "o3d_xcorr_boxaware_fwd: template box cloud too large");
    if (B == 0 || N == 0) return O3D_OK;
    dim3 grid((N + TOPK_THREADS - 1) / TOPK_THREADS, B);
    boxaware_topk_kernel<<<grid, TOPK_THREADS, sizeof(float) * M * D, (cudaStream_t)stream>>>(template_bc, search_bc, M, N, D, k, idx);
    O3D_CHECK_LAUNCH("o3d_xcorr_boxaware_fwd");
    return O3D_OK;
}

extern "C" int o3d_xcorr_p2b_fwd(const float* tfeat_cl, const float* sfeat_cl, int B, int n1, int n2, int C, float eps,
                                 float* sim, float* tnorm, float* snorm, void* stream) {
    O3D_REQUIRE(tfeat_cl && sfeat_cl && sim, O3D_ERR_ARG, "o3d_xcorr_p2b_fwd: null pointer");
    O3D_REQUIRE(n1 >= 1 && n1 <= 32 * SIM_IMAX && n2 >= 1 && C >= 1, O3D_ERR_ARG, "o3d_xcorr_p2b_fwd: n1 must be in 1..%d", 32 * SIM_IMAX);
    if (B == 0) return O3D_OK;
    const size_t smem = sizeof(float) * (size_t)(n1 + SIM_J) * (SIM_CH + 1);
    dim3 grid((n2 + SIM_J - 1) / SIM_J, B);
    p2b_sim_kernel<<<grid, 256, smem, (cudaStream_t)stream>>>(tfeat_cl, sfeat_cl, n1, n2, C, eps, sim, tnorm, snorm);
    O3D_CHECK_LAUNCH("o3d_xcorr_p2b_fwd");
    return O3D_OK;
}

extern "C" int o3d_xcorr_p2b_bwd(const float* dsim, const float* sim, const float* tfeat_cl, const float* sfeat_cl,
                                 const float* tnorm, const float* snorm, int B, int n1, int n2, int C, float eps,
                                 float* d_tfeat_cl, float* d_sfeat_cl, void* stream) {
    O3D_REQUIRE(dsim && sim && tfeat_cl && sfeat_cl && tnorm && snorm, O3D_ERR_ARG, "o3d_xcorr_p2b_bwd: null pointer");
    if (B == 0) return O3D_OK;
    cudaStream_t st = (cudaStream_t)stream;
    // sim / dsim are (B, n2, n1): template row i walks j with stride n1; search row j walks i with stride 1
    if (d_tfeat_cl) {
        p2b_sim_grad_kernel<<<dim3(n1, B), 256, sizeof(float) * n2, st>>>(dsim, sim, tfeat_cl, sfeat_cl, tnorm, snorm, n1, n2, C, eps,
                                                                        1, n1, d_tfeat_cl);
        O3D_CHECK_LAUNCH("o3d_xcorr_p2b_bwd: template");
    }
    if (d_sfeat_cl) {
        p2b_sim_grad_kernel<<<dim3(n2, B), 256, sizeof(float) * n1, st>>>(dsim, sim, sfeat_cl, tfeat_cl, snorm, tnorm, n2, n1, C, eps,
                                                                        n1, 1, d_sfeat_cl);
        O3D_CHECK_LAUNCH("o3d_xcorr_p2b_bwd: search");
    }
    return O3D_OK;
}
