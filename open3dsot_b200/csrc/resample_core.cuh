// The pieces of the fixed-shape resampling shared by resample_kernel (resample.cu: a candidate array + keep mask + draw arrays)
// and crop_resample_kernel (crop_resample.cu: the crop and the keyed draws computed in place), so that both select, order and
// gather through the same instructions:
//   * the Philox4x32-10 block of o3d_keyed_uniform (track_eval.cu) and its word -> uniform mapping;
//   * the rank of a with-replacement draw;
//   * stages B-D of the resampling: radix select of the size-th smallest key over the n compacted survivors, collection of the
//     keys below it (+ ties in index order), bitonic sort of the (key, index) pairs, gather.
// The survivors are given as S[0 .. n-1] (candidate indices in ascending order) and key(s) = the key bits of survivor s (the
// float bit pattern of its uniform draw in [0, 1): monotone in the value).
#pragma once
#include "common.cuh"

constexpr int O3D_RS_THREADS = 1024;
constexpr int O3D_RS_MAX_SIZE = 2048;
static_assert(O3D_RS_THREADS == 1024, "o3d_block_exscan1024 scans exactly 32 warps");

constexpr uint32_t kO3dPhiloxM0 = 0xD2511F53u, kO3dPhiloxM1 = 0xCD9E8D57u;
constexpr uint32_t kO3dPhiloxW0 = 0x9E3779B9u, kO3dPhiloxW1 = 0xBB67AE85u;

__device__ __forceinline__ uint4 o3d_philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        if (r) {
            k0 += kO3dPhiloxW0;
            k1 += kO3dPhiloxW1;
        }
        const uint32_t hi0 = __umulhi(kO3dPhiloxM0, c.x), lo0 = kO3dPhiloxM0 * c.x;
        const uint32_t hi1 = __umulhi(kO3dPhiloxM1, c.z), lo1 = kO3dPhiloxM1 * c.z;
        c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
    }
    return c;
}

__device__ __forceinline__ float o3d_word_to_uniform(uint32_t w) { return (float)(w >> 8) * 5.9604644775390625e-8f; }  // 2^-24

// Element e of a keyed stream: word e % 4 of the block at counter (e / 4, frame, stream, 0), key (seed, id).
__device__ __forceinline__ float o3d_keyed_element(uint32_t seed, uint32_t id, uint32_t frame, uint32_t stream, uint32_t e) {
    const uint4 w = o3d_philox4x32_10(make_uint4(e >> 2, frame, stream, 0u), seed, id);
    const uint32_t j = e & 3u;
    return o3d_word_to_uniform(j == 0 ? w.x : j == 1 ? w.y : j == 2 ? w.z : w.w);
}

// With replacement (2 < n < size): draw u -> the floor(u * n)-th survivor, clamped to [0, n - 1].
__device__ __forceinline__ long long o3d_pick_rank(float u, uint32_t n) {
    long long r = (long long)(u * (float)n);
    if (r > (long long)n - 1) r = (long long)n - 1;
    if (r < 0) r = 0;
    return r;
}

struct O3dResampleSmem {
    unsigned long long sel[O3D_RS_MAX_SIZE];
    uint32_t hist[2048];
    uint32_t warp[32];
    uint32_t digit, krem, eq, cnt;
};

// Stages B-D for n >= size (and n > 2): emit(i, idx) receives the i-th selected candidate index, i in [0, size), in ascending
// (key, index) order.  Every thread of the block must call it.
template <class KeyAt, class Emit>
__device__ __forceinline__ void o3d_resample_select(uint32_t n, int size, const int32_t* __restrict__ S, KeyAt key, Emit emit,
                                                    O3dResampleSmem& sm) {
    const int tid = threadIdx.x;
    // ---- B. radix select: the size-th smallest key among the n survivors
    uint32_t prefix = 0, krem = (uint32_t)size, eq_total = 0;
    if ((int)n > size) {
        const int shifts[3] = {21, 10, 0}, bits[3] = {11, 11, 10};
        for (int pass = 0; pass < 3; ++pass) {
            const int sh = shifts[pass], nb = bits[pass];
            for (int i = tid; i < 2048; i += O3D_RS_THREADS) sm.hist[i] = 0;
            __syncthreads();
            for (uint32_t s = tid; s < n; s += O3D_RS_THREADS) {
                const uint32_t k = key(s);
                if (pass == 0 || (k >> (sh + nb)) == prefix) atomicAdd(&sm.hist[(k >> sh) & ((1u << nb) - 1u)], 1u);
            }
            __syncthreads();
            const uint32_t h0 = sm.hist[2 * tid], h1 = sm.hist[2 * tid + 1];
            uint32_t total;
            const uint32_t ex = o3d_block_exscan1024(h0 + h1, sm.warp, total);
            if (ex < krem && krem <= ex + h0) {
                sm.digit = 2 * tid; sm.krem = krem - ex; sm.eq = h0;
            } else if (ex + h0 < krem && krem <= ex + h0 + h1) {
                sm.digit = 2 * tid + 1; sm.krem = krem - ex - h0; sm.eq = h1;
            }
            __syncthreads();
            prefix = (prefix << nb) | sm.digit;
            krem = sm.krem;
            eq_total = sm.eq;
            __syncthreads();
        }
    }
    // ---- C. collect: keys below the threshold, then `krem` of the keys equal to it (index order when there are more)
    const bool all = (int)n == size;
    if (tid == 0) sm.cnt = 0;
    __syncthreads();
    const uint32_t n_less = all ? n : (uint32_t)size - krem;
    for (uint32_t s = tid; s < n; s += O3D_RS_THREADS) {
        const uint32_t idx = (uint32_t)S[s];
        const uint32_t k = key(s);
        if (all || k < prefix) {
            const uint32_t p = atomicAdd(&sm.cnt, 1u);
            sm.sel[p] = ((unsigned long long)k << 32) | idx;
        }
    }
    if (!all) {
        if (eq_total == krem) {
            for (uint32_t s = tid; s < n; s += O3D_RS_THREADS) {
                const uint32_t idx = (uint32_t)S[s];
                const uint32_t k = key(s);
                if (k == prefix) {
                    const uint32_t p = atomicAdd(&sm.cnt, 1u);
                    sm.sel[p] = ((unsigned long long)k << 32) | idx;
                }
            }
        } else {
            // more equal keys than places: the first `krem` in index order (ordered block scan over the survivors)
            uint32_t taken = 0;
            for (uint32_t s0 = 0; s0 < n && taken < krem; s0 += O3D_RS_THREADS) {
                const uint32_t s = s0 + tid;
                uint32_t idx = 0, hit = 0;
                if (s < n) {
                    idx = (uint32_t)S[s];
                    hit = key(s) == prefix;
                }
                uint32_t total;
                const uint32_t r = taken + o3d_block_exscan1024(hit, sm.warp, total);
                if (hit && r < krem) sm.sel[n_less + r] = ((unsigned long long)prefix << 32) | idx;
                taken += total;
            }
        }
    }
    int P2 = 1;
    while (P2 < size) P2 <<= 1;
    for (int i = size + tid; i < P2; i += O3D_RS_THREADS) sm.sel[i] = ~0ull;
    __syncthreads();
    // bitonic sort, ascending (key, index)
    for (int k = 2; k <= P2; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = tid; i < P2; i += O3D_RS_THREADS) {
                const int x = i ^ j;
                if (x > i) {
                    const unsigned long long a = sm.sel[i], c = sm.sel[x];
                    const bool up = (i & k) == 0;
                    if ((a > c) == up) { sm.sel[i] = c; sm.sel[x] = a; }
                }
            }
            __syncthreads();
        }
    }
    // ---- D. gather
    for (int i = tid; i < size; i += O3D_RS_THREADS) emit(i, (uint32_t)(sm.sel[i] & 0xFFFFFFFFull));
}
