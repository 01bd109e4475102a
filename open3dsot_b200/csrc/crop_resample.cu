// Crop a shared scan in each target's box and resample the crop to a fixed size, one CTA per target, without any (K, N)
// intermediate — the live multi-target tracker's every crop (tracking/multi_tracker.py).
//
// Bitwise the same as the three-kernel path on the candidate set [prefix, crop of scan] (element e < Np: prefix point e, element
// Np + i: point i of the scan in the frame of the target's box):
//   o3d_crop_box_frame -> o3d_keyed_uniform (perm stream over Np + N elements, pick stream over size) -> o3d_resample
// which writes a (K, N) local-coordinate array, a keep mask and a draw array only to read them back for a few thousand points.
//   A. ordered compaction, tiled as o3d_crop_append walks its scan (4096 elements per tile, 4 consecutive per thread, one block
//      scan per tile): the crop test is done here, with o3d_to_box_frame (bit-identical local coordinates), and the perm key of
//      every survivor is evaluated from its Philox block (4 consecutive elements = one block: one evaluation per thread and tile)
//      and stashed next to its index.  Scratch is written for survivors only.
//   B-D. resample_core.cuh, as resample_kernel; the gather recomputes the local coordinates of the selected points.
#include "resample_core.cuh"
#include "../../include/o3d_b200.h"

namespace {

constexpr int CR_PER = 4;                                  // consecutive elements per thread and tile = one Philox block
constexpr int CR_TILE = O3D_RS_THREADS * CR_PER;

__global__ void __launch_bounds__(O3D_RS_THREADS)
    crop_resample_kernel(const float* __restrict__ scans, const long long* __restrict__ count, const long long* __restrict__ frame,
                         const float* __restrict__ center, const float* __restrict__ rot, const float* __restrict__ half, int N,
                         const float* __restrict__ prefix, const uint8_t* __restrict__ prefix_keep, int Np, uint32_t seed,
                         const long long* __restrict__ key, const long long* __restrict__ key_frame, uint32_t perm_stream,
                         uint32_t pick_stream, int size, int32_t* __restrict__ scratch, float* __restrict__ out,
                         long long* __restrict__ n_out) {
    __shared__ O3dResampleSmem sm;
    const int b = blockIdx.x, tid = threadIdx.x;
    const int M = Np + N;
    const uint32_t id = (uint32_t)key[b], fr = (uint32_t)key_frame[b];
    int n_valid = 0;
    const float* __restrict__ src = scans;
    float cx = 0.f, cy = 0.f, cz = 0.f, hx = 0.f, hy = 0.f, hz = 0.f;
    float R[9];
#pragma unroll
    for (int j = 0; j < 9; ++j) R[j] = 0.f;
    if (N > 0) {
        const long long f = frame[b];
        n_valid = count ? (int)min((long long)N, count[f]) : N;
        src = scans + (size_t)f * N * 3;
        cx = center[b * 3 + 0]; cy = center[b * 3 + 1]; cz = center[b * 3 + 2];
#pragma unroll
        for (int j = 0; j < 9; ++j) R[j] = rot[b * 9 + j];
        hx = half[b * 3 + 0]; hy = half[b * 3 + 1]; hz = half[b * 3 + 2];
    }
    const float* __restrict__ PF = prefix + (size_t)b * Np * 3;
    const uint8_t* __restrict__ PK = prefix_keep + (size_t)b * Np;
    int32_t* __restrict__ SI = scratch + (size_t)b * 2 * M;
    uint32_t* __restrict__ SK = reinterpret_cast<uint32_t*>(SI + M);
    float* __restrict__ O = out + (size_t)b * size * 3;

    // candidate e in the frame of the box: a prefix point as given, a scan point transformed exactly as crop_box_frame_kernel does
    auto local = [&](uint32_t e, float& x, float& y, float& z) {
        if ((int)e < Np) {
            x = PF[(size_t)e * 3 + 0]; y = PF[(size_t)e * 3 + 1]; z = PF[(size_t)e * 3 + 2];
        } else {
            const size_t i = e - (uint32_t)Np;
            o3d_to_box_frame(src[i * 3 + 0] - cx, src[i * 3 + 1] - cy, src[i * 3 + 2] - cz, R, x, y, z);
        }
    };

    // ---- A. ordered compaction with the crop test; elements past Np + n_valid are never kept
    const int Mv = Np + n_valid;
    uint32_t n = 0;
    for (int t0 = 0; t0 < Mv; t0 += CR_TILE) {
        const int e0 = t0 + tid * CR_PER;
        uint32_t m = 0;
#pragma unroll
        for (int j = 0; j < CR_PER; ++j) {
            const int e = e0 + j;
            if (e < Np) {
                if (PK[e]) m |= 1u << j;
            } else if (e < Mv) {
                float x, y, z;
                local((uint32_t)e, x, y, z);
                if (fabsf(x) < hx && fabsf(y) < hy && fabsf(z) < hz) m |= 1u << j;
            }
        }
        uint4 w = make_uint4(0u, 0u, 0u, 0u);
        if (m) w = o3d_philox4x32_10(make_uint4((uint32_t)e0 >> 2, fr, perm_stream, 0u), seed, id);
        const uint32_t ws[4] = {w.x, w.y, w.z, w.w};
        uint32_t total;
        uint32_t pos = n + o3d_block_exscan1024(__popc(m), sm.warp, total);
#pragma unroll
        for (int j = 0; j < CR_PER; ++j) {
            if (m & (1u << j)) {
                SI[pos] = e0 + j;
                SK[pos] = __float_as_uint(o3d_word_to_uniform(ws[j]));
                ++pos;
            }
        }
        n += total;
    }
    __syncthreads();                       // SI / SK (global) written by this block, read below by other threads of it
    if (tid == 0 && n_out) n_out[b] = n;

    if ((int)n < size || n <= 2) {
        // ---- with replacement (2 < n < size) / placeholder (n <= 2)
        for (int i = tid; i < size; i += O3D_RS_THREADS) {
            float x = 0.f, y = 0.f, z = 0.f;
            if (n > 2) local((uint32_t)SI[o3d_pick_rank(o3d_keyed_element(seed, id, fr, pick_stream, (uint32_t)i), n)], x, y, z);
            O[i * 3 + 0] = x;
            O[i * 3 + 1] = y;
            O[i * 3 + 2] = z;
        }
        return;
    }
    // ---- B-D. select the `size` smallest keys, sort them, gather (resample_core.cuh)
    o3d_resample_select(
        n, size, SI, [&](uint32_t s) { return SK[s]; },
        [&](int i, uint32_t idx) {
            float x, y, z;
            local(idx, x, y, z);
            O[i * 3 + 0] = x;
            O[i * 3 + 1] = y;
            O[i * 3 + 2] = z;
        },
        sm);
}

}  // namespace

extern "C" int o3d_crop_resample(const float* scans, const long long* count, const long long* frame, const float* center,
                                 const float* rot, const float* half, int N, const float* prefix, const unsigned char* prefix_keep,
                                 int Np, unsigned int seed, const long long* key, const long long* key_frame, int perm_stream,
                                 int pick_stream, int K, int size, int32_t* scratch, float* out, long long* n_out, void* stream) {
    O3D_REQUIRE(key && key_frame && scratch && out, O3D_ERR_ARG, "o3d_crop_resample: null pointer");
    O3D_REQUIRE(N <= 0 || (scans && frame && center && rot && half), O3D_ERR_ARG, "o3d_crop_resample: null pointer (scan crop)");
    O3D_REQUIRE(Np <= 0 || (prefix && prefix_keep), O3D_ERR_ARG, "o3d_crop_resample: null pointer (prefix)");
    O3D_REQUIRE(K >= 0 && K <= 65535 && N >= 0 && Np >= 0 && (long long)N + Np <= (1LL << 30), O3D_ERR_ARG,
                "o3d_crop_resample: bad sizes K=%d N=%d Np=%d", K, N, Np);
    O3D_REQUIRE(size >= 1 && size <= O3D_RS_MAX_SIZE, O3D_ERR_ARG, "o3d_crop_resample: size=%d out of [1, %d]", size,
                O3D_RS_MAX_SIZE);
    O3D_REQUIRE(perm_stream >= 0 && pick_stream >= 0, O3D_ERR_ARG, "o3d_crop_resample: negative stream %d / %d", perm_stream,
                pick_stream);
    if (K == 0) return O3D_OK;
    crop_resample_kernel<<<K, O3D_RS_THREADS, 0, (cudaStream_t)stream>>>(scans, count, frame, center, rot, half, N, prefix,
                                                                         prefix_keep, Np, seed, key, key_frame,
                                                                         (uint32_t)perm_stream, (uint32_t)pick_stream, size,
                                                                         scratch, out, n_out);
    O3D_CHECK_LAUNCH("o3d_crop_resample");
    return O3D_OK;
}
