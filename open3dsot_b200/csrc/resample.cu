// Fixed-shape resampling of a masked point set in one kernel — the device-side form of points_utils.regularize_pc
// (datasets/points_utils.py:24-40: `rng.choice(n, size, replace=size > n)` on the survivors of a crop), used per frame by the
// tracking loop (crop -> resample -> network) and per pair by the device-side batch construction.
//
// Semantics (identical to open3dsot_b200/tracking/sampling.py, which it replaces on the device):
//   n = number of kept candidates
//   n >= size     : the `size` kept candidates with the smallest random keys u_perm (a uniform draw without replacement),
//                   emitted in ascending key order (= a uniformly random order, as numpy's choice returns);
//   2 < n < size  : size draws with replacement, draw i = the floor(u_pick[i] * n)-th kept candidate (index order);
//   n <= 2        : an all-zero cloud (the reference's "too few points" placeholder).
// The torch formulation costs ~25 launches (radix top-k over all candidates, cumsum, searchsorted, where / gather glue) —
// 170 us of a 0.86 ms tracking frame; this is one CTA per cloud:
//   A. ordered compaction of the kept indices (a contiguous run of candidates per thread, one block scan),
//   B. 3-pass radix select (11 / 11 / 10 bits, shared-memory histograms) of the size-th smallest key over the survivors,
//   C. collection of the keys below the threshold (+ ties in index order), bitonic sort of the <= 2048 (key, index) pairs,
//   D. gather of the selected points.
#include "resample_core.cuh"
#include "../../include/o3d_b200.h"

namespace {

constexpr int RS_THREADS = O3D_RS_THREADS;
constexpr int RS_MAX_SIZE = O3D_RS_MAX_SIZE;

__global__ void __launch_bounds__(RS_THREADS)
    resample_kernel(const float* __restrict__ points, const uint8_t* __restrict__ keep, const float* __restrict__ u_perm,
                    const float* __restrict__ u_pick, int N, int size, int32_t* __restrict__ scratch, float* __restrict__ out,
                    long long* __restrict__ src, long long* __restrict__ n_out) {
    __shared__ O3dResampleSmem sm;

    const int b = blockIdx.x, tid = threadIdx.x;
    const float* __restrict__ P = points + (size_t)b * N * 3;
    const uint8_t* __restrict__ K = keep + (size_t)b * N;
    const float* __restrict__ U = u_perm + (size_t)b * N;
    const float* __restrict__ UP = u_pick + (size_t)b * size;
    int32_t* __restrict__ S = scratch + (size_t)b * N;
    float* __restrict__ O = out + (size_t)b * size * 3;
    long long* __restrict__ SRC = src + (size_t)b * size;

    // ---- A. ordered compaction of the kept indices: every thread owns a CONTIGUOUS run of candidates (one block scan in all;
    //         the flags are read twice — count, then write — the second time from L1)
    const int L = (((N + RS_THREADS - 1) / RS_THREADS) + 3) & ~3;
    const int beg = tid * L, end = min(N, beg + L);
    const bool vec = (reinterpret_cast<uintptr_t>(K) & 3) == 0;
    auto flags4 = [&](int i) -> uint32_t {             // bit j set = candidate i + j is kept
        uint32_t f = 0;
        if (vec && i + 4 <= N) {
            const uint32_t w = *reinterpret_cast<const uint32_t*>(K + i);
#pragma unroll
            for (int j = 0; j < 4; ++j) f |= ((w >> (8 * j)) & 0xFFu) ? 1u << j : 0u;
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (i + j < N && K[i + j]) f |= 1u << j;
        }
        return f;
    };
    uint32_t cnt = 0;
    for (int i = beg; i < end; i += 4) cnt += __popc(flags4(i));
    uint32_t n;
    uint32_t pos = o3d_block_exscan1024(cnt, sm.warp, n);
    for (int i = beg; i < end; i += 4) {
        const uint32_t f = flags4(i);
#pragma unroll
        for (int j = 0; j < 4; ++j)
            if (f & (1u << j)) S[pos++] = i + j;
    }
    __syncthreads();                       // S (global) written by this block, read below by other threads of it
    if (tid == 0 && n_out) n_out[b] = n;

    if ((int)n < size || n <= 2) {
        // ---- with replacement (2 < n < size) / placeholder (n <= 2)
        for (int i = tid; i < size; i += RS_THREADS) {
            const long long w = n == 0 ? N - 1 : S[o3d_pick_rank(UP[i], n)];
            SRC[i] = w;
            const bool zero = n <= 2;
            O[i * 3 + 0] = zero ? 0.f : P[w * 3 + 0];
            O[i * 3 + 1] = zero ? 0.f : P[w * 3 + 1];
            O[i * 3 + 2] = zero ? 0.f : P[w * 3 + 2];
        }
        return;
    }
    // ---- B-D. select the `size` smallest keys, sort them, gather (resample_core.cuh)
    o3d_resample_select(
        n, size, S, [&](uint32_t s) { return __float_as_uint(U[S[s]]); },
        [&](int i, uint32_t idx) {
            SRC[i] = idx;
            O[i * 3 + 0] = P[(size_t)idx * 3 + 0];
            O[i * 3 + 1] = P[(size_t)idx * 3 + 1];
            O[i * 3 + 2] = P[(size_t)idx * 3 + 2];
        },
        sm);
}

}  // namespace

extern "C" int o3d_resample(const float* points, const unsigned char* keep, const float* u_perm, const float* u_pick, int B, int N,
                            int size, int32_t* scratch, float* out, long long* src, long long* n_out, void* stream) {
    O3D_REQUIRE(points && keep && u_perm && u_pick && scratch && out && src, O3D_ERR_ARG, "o3d_resample: null pointer");
    O3D_REQUIRE(B >= 0 && N >= 1 && size >= 1 && size <= RS_MAX_SIZE, O3D_ERR_ARG, "o3d_resample: bad sizes B=%d N=%d size=%d (size <= %d)",
                B, N, size, RS_MAX_SIZE);
    if (B == 0) return O3D_OK;
    resample_kernel<<<B, RS_THREADS, 0, (cudaStream_t)stream>>>(points, keep, u_perm, u_pick, N, size, scratch, out, src, n_out);
    O3D_CHECK_LAUNCH("o3d_resample");
    return O3D_OK;
}
