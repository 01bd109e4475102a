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
#include "common.cuh"
#include "../../include/o3d_b200.h"

namespace {

constexpr int RS_THREADS = 1024;
constexpr int RS_MAX_SIZE = 2048;
static_assert(RS_THREADS == 1024, "o3d_block_exscan1024 scans exactly 32 warps");

__global__ void __launch_bounds__(RS_THREADS)
    resample_kernel(const float* __restrict__ points, const uint8_t* __restrict__ keep, const float* __restrict__ u_perm,
                    const float* __restrict__ u_pick, int N, int size, int32_t* __restrict__ scratch, float* __restrict__ out,
                    long long* __restrict__ src, long long* __restrict__ n_out) {
    __shared__ unsigned long long s_sel[RS_MAX_SIZE];
    __shared__ uint32_t s_hist[2048];
    __shared__ uint32_t s_warp[32];
    __shared__ uint32_t s_digit, s_krem, s_eq, s_cnt;

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
    uint32_t pos = o3d_block_exscan1024(cnt, s_warp, n);
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
            long long w;
            if (n == 0) {
                w = N - 1;
            } else {
                long long r = (long long)(UP[i] * (float)n);
                if (r > (long long)n - 1) r = (long long)n - 1;
                if (r < 0) r = 0;
                w = S[r];
            }
            SRC[i] = w;
            const bool zero = n <= 2;
            O[i * 3 + 0] = zero ? 0.f : P[w * 3 + 0];
            O[i * 3 + 1] = zero ? 0.f : P[w * 3 + 1];
            O[i * 3 + 2] = zero ? 0.f : P[w * 3 + 2];
        }
        return;
    }

    // ---- B. radix select: the size-th smallest key among the n survivors (keys are floats in [0, 1): bit patterns are monotone)
    uint32_t prefix = 0, krem = (uint32_t)size, eq_total = 0;
    if ((int)n > size) {
        const int shifts[3] = {21, 10, 0}, bits[3] = {11, 11, 10};
        for (int pass = 0; pass < 3; ++pass) {
            const int sh = shifts[pass], nb = bits[pass];
            for (int i = tid; i < 2048; i += RS_THREADS) s_hist[i] = 0;
            __syncthreads();
            for (uint32_t s = tid; s < n; s += RS_THREADS) {
                const uint32_t key = __float_as_uint(U[S[s]]);
                if (pass == 0 || (key >> (sh + nb)) == prefix) atomicAdd(&s_hist[(key >> sh) & ((1u << nb) - 1u)], 1u);
            }
            __syncthreads();
            const uint32_t h0 = s_hist[2 * tid], h1 = s_hist[2 * tid + 1];
            uint32_t total;
            const uint32_t ex = o3d_block_exscan1024(h0 + h1, s_warp, total);
            if (ex < krem && krem <= ex + h0) {
                s_digit = 2 * tid; s_krem = krem - ex; s_eq = h0;
            } else if (ex + h0 < krem && krem <= ex + h0 + h1) {
                s_digit = 2 * tid + 1; s_krem = krem - ex - h0; s_eq = h1;
            }
            __syncthreads();
            prefix = (prefix << nb) | s_digit;
            krem = s_krem;
            eq_total = s_eq;
            __syncthreads();
        }
    }
    // ---- C. collect: keys below the threshold, then `krem` of the keys equal to it (index order when there are more)
    const bool all = (int)n == size;
    if (tid == 0) s_cnt = 0;
    __syncthreads();
    const uint32_t n_less = all ? n : (uint32_t)size - krem;
    for (uint32_t s = tid; s < n; s += RS_THREADS) {
        const uint32_t idx = (uint32_t)S[s];
        const uint32_t key = __float_as_uint(U[idx]);
        if (all || key < prefix) {
            const uint32_t p = atomicAdd(&s_cnt, 1u);
            s_sel[p] = ((unsigned long long)key << 32) | idx;
        }
    }
    if (!all) {
        if (eq_total == krem) {
            for (uint32_t s = tid; s < n; s += RS_THREADS) {
                const uint32_t idx = (uint32_t)S[s];
                const uint32_t key = __float_as_uint(U[idx]);
                if (key == prefix) {
                    const uint32_t p = atomicAdd(&s_cnt, 1u);
                    s_sel[p] = ((unsigned long long)key << 32) | idx;
                }
            }
        } else {
            // more equal keys than places: the first `krem` in index order (ordered block scan over the survivors)
            uint32_t taken = 0;
            for (uint32_t s0 = 0; s0 < n && taken < krem; s0 += RS_THREADS) {
                const uint32_t s = s0 + tid;
                uint32_t idx = 0, hit = 0;
                if (s < n) {
                    idx = (uint32_t)S[s];
                    hit = __float_as_uint(U[idx]) == prefix;
                }
                uint32_t total;
                const uint32_t r = taken + o3d_block_exscan1024(hit, s_warp, total);
                if (hit && r < krem) s_sel[n_less + r] = ((unsigned long long)prefix << 32) | idx;
                taken += total;
            }
        }
    }
    int P2 = 1;
    while (P2 < size) P2 <<= 1;
    for (int i = size + tid; i < P2; i += RS_THREADS) s_sel[i] = ~0ull;
    __syncthreads();
    // bitonic sort, ascending (key, index)
    for (int k = 2; k <= P2; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = tid; i < P2; i += RS_THREADS) {
                const int x = i ^ j;
                if (x > i) {
                    const unsigned long long a = s_sel[i], c = s_sel[x];
                    const bool up = (i & k) == 0;
                    if ((a > c) == up) { s_sel[i] = c; s_sel[x] = a; }
                }
            }
            __syncthreads();
        }
    }
    // ---- D. gather
    for (int i = tid; i < size; i += RS_THREADS) {
        const uint32_t idx = (uint32_t)(s_sel[i] & 0xFFFFFFFFull);
        SRC[i] = idx;
        O[i * 3 + 0] = P[(size_t)idx * 3 + 0];
        O[i * 3 + 1] = P[(size_t)idx * 3 + 1];
        O[i * 3 + 2] = P[(size_t)idx * 3 + 2];
    }
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
