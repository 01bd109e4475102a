// Detection matching of the live tracker (tracking/multi_tracker.py associate_tensors): per feed, the rows that advance are
// matched to the feed's detections greedily in ascending (squared plane distance, row, detection) order.  One CTA per feed.
//
// The greedy assignment is found in rounds.  A pair that is each other's best among the free rows and free detections (its key
// is the smallest of every pair of its row and of every pair of its detection) is accepted by the sequential greedy loop too:
// no pair with a smaller key can take its row or its detection first.  Each round takes every such pair out at once; the
// smallest remaining pair is always one of them, so every round takes at least one, and most scenes need one or two rounds.
//   phase 1: every free detection finds its best free row (a warp per detection, lanes over rows);
//   phase 2: every free row finds its best free detection (a warp per row, lanes over detections), and takes it when the
//            detection's best row is this row;
//   phase 3: the taken rows and detections leave the free sets.
// Keys are (d2 bits << 32 | index): d2 >= 0 is never NaN once gated, so its bits order as the values do.  Rows are tracked in a
// shared bitmask (b <= 65535), detections in shared arrays (D <= 1024).  No atomics: each detection is claimed by at most the one
// row that is its best, and each bitmask word is rewritten by one thread.
#include "common.cuh"
#include "track_predict.cuh"
#include "../../include/o3d_b200.h"

namespace {

constexpr int AS_THREADS = 256;
constexpr int AS_WARPS = AS_THREADS / 32;
constexpr int AS_MAX_D = 1024;
constexpr int AS_MAX_WORDS = 65536 / 32;
constexpr unsigned long long AS_NONE = ~0ull;

__device__ __forceinline__ unsigned long long as_key(float d2, int index) {
    return ((unsigned long long)__float_as_uint(d2) << 32) | (unsigned)index;
}

__device__ __forceinline__ unsigned long long as_warp_min(unsigned long long v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long w = __shfl_xor_sync(0xffffffffu, v, o);
        v = w < v ? w : v;
    }
    return v;
}

// d2 = dx*dx + dy*dy, every operation rounded on its own (associate_tensors' expression)
__device__ __forceinline__ float as_d2(float px, float py, float2 q) {
    const float dx = __fsub_rn(px, q.x), dy = __fsub_rn(py, q.y);
    return __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy));
}

__global__ void __launch_bounds__(AS_THREADS) associate_kernel(const o3d_box_associate_t p) {
    __shared__ float2 s_det[AS_MAX_D];                // detections' plane coordinates
    __shared__ unsigned long long s_best[AS_MAX_D];   // phase 1: the detection's best free row
    __shared__ int s_stake[AS_MAX_D];                 // phase 2: the row that took the detection this round, or -1
    __shared__ int s_drow[AS_MAX_D];                  // the row the detection is matched to, or -1
    __shared__ unsigned char s_free[AS_MAX_D];
    __shared__ uint32_t s_rows[AS_MAX_WORDS];         // bit i: row i takes part and is free

    const int f = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int b = p.b;
    const bool fed = p.fed[f] != 0;
    const int nd = fed ? p.count[f] : 0;
    const long long D = p.D;
    const float* det = p.det + (long long)f * D * 16;

    // the rows of this feed: the centre each is matched against (NaN when it does not take part), no match yet
    for (int i = tid; i < b; i += AS_THREADS) {
        if (p.feed[i] != f) continue;
        float c[3] = {__int_as_float(0x7fc00000), __int_as_float(0x7fc00000), __int_as_float(0x7fc00000)};
        if (p.adv[i]) {
            const long long s = p.src[i];
            const bool hit = !p.rule || p.points[i] >= p.min_points;
            float pc[3], hc[3], v[3];
#pragma unroll
            for (int j = 0; j < 3; ++j) {
                pc[j] = p.center[i * 3 + j];
                hc[j] = p.hit_c[s * 3 + j];
                v[j] = p.vel[s * 3 + j];
            }
            o3d_predicted_centre(pc, hit, p.coast != 0, hc, v, (float)(p.t[s] + 1 - p.hit_t[s]), c);
        }
#pragma unroll
        for (int j = 0; j < 3; ++j) p.pred[i * 3 + j] = c[j];
        p.match[i] = -1;
#pragma unroll
        for (int j = 0; j < 12; ++j) p.match_box[i * 12 + j] = 0.0f;
    }
    const int words = (b + 31) >> 5;
    for (int w = tid; w < words; w += AS_THREADS) {
        uint32_t bits = 0;
        if (nd > 0) {
            for (int k = 0; k < 32; ++k) {
                const int i = w * 32 + k;
                if (i < b && p.feed[i] == f && p.adv[i]) bits |= 1u << k;
            }
        }
        s_rows[w] = bits;
    }
    for (int d = tid; d < nd; d += AS_THREADS) {
        s_det[d] = make_float2(det[d * 16 + p.axis0], det[d * 16 + p.axis1]);
        s_free[d] = 1;
        s_stake[d] = -1;
        s_drow[d] = -1;
    }
    __syncthreads();

    for (;;) {
        // phase 1: each free detection's best free row
        bool found = false;
        for (int d = warp; d < nd; d += AS_WARPS) {
            if (!s_free[d]) continue;
            const float2 q = s_det[d];
            unsigned long long best = AS_NONE;
            for (int i = lane; i < b; i += 32) {
                if (!((s_rows[i >> 5] >> (i & 31)) & 1u)) continue;
                const float d2 = as_d2(p.pred[i * 3 + p.axis0], p.pred[i * 3 + p.axis1], q);
                if (d2 <= p.gate2) {
                    const unsigned long long k = as_key(d2, i);
                    best = k < best ? k : best;
                }
            }
            best = as_warp_min(best);
            if (lane == 0) s_best[d] = best;
            found = found || best != AS_NONE;
        }
        if (!__syncthreads_or(found)) break;
        // phase 2: each free row's best free detection, taken when the row is that detection's best too
        for (int i = warp; i < b; i += AS_WARPS) {
            if (!((s_rows[i >> 5] >> (i & 31)) & 1u)) continue;
            const float px = p.pred[i * 3 + p.axis0], py = p.pred[i * 3 + p.axis1];
            unsigned long long best = AS_NONE;
            for (int d = lane; d < nd; d += 32) {
                if (!s_free[d]) continue;
                const float d2 = as_d2(px, py, s_det[d]);
                if (d2 <= p.gate2) {
                    const unsigned long long k = as_key(d2, d);
                    best = k < best ? k : best;
                }
            }
            best = as_warp_min(best);
            if (best == AS_NONE) continue;
            const int d = (int)(best & 0xffffffffu);
            if ((int)(s_best[d] & 0xffffffffu) != i) continue;
            if (lane == 0) {
                s_stake[d] = i;
                p.match[i] = d;
            }
            if (lane < 12) p.match_box[i * 12 + lane] = det[d * 16 + (lane < 3 ? lane : lane + 3)];   // centre, rotation
        }
        __syncthreads();
        // phase 3: the pairs taken leave the free sets
        for (int d = tid; d < nd; d += AS_THREADS) {
            if (s_stake[d] >= 0) {
                s_free[d] = 0;
                s_drow[d] = s_stake[d];
                s_stake[d] = -1;
            }
        }
        for (int w = tid; w < words; w += AS_THREADS) {
            uint32_t bits = s_rows[w];
            for (uint32_t m = bits; m; m &= m - 1) {
                const int k = __ffs(m) - 1;
                if (p.match[w * 32 + k] >= 0) bits &= ~(1u << k);
            }
            s_rows[w] = bits;
        }
        __syncthreads();
    }

    // the feed's records: its detections of this advance and the slot each matched
    if (fed) {
        float* rec = p.rec_det + (long long)f * D * 16;
        for (long long e = tid; e < (long long)nd * 16; e += AS_THREADS) rec[e] = det[e];
        for (int d = tid; d < nd; d += AS_THREADS) p.rec_slot[f * D + d] = s_drow[d] >= 0 ? (int)p.src[s_drow[d]] : -1;
        if (tid == 0) p.rec_count[f] = nd;
    }
}

}  // namespace

extern "C" int o3d_box_associate(const o3d_box_associate_t* p, void* stream) {
    O3D_REQUIRE(p, O3D_ERR_ARG, "o3d_box_associate: null pointer (descriptor)");
    O3D_REQUIRE(p->b >= 0 && p->b <= 65535 && p->F >= 1 && p->D >= 1 && p->D <= AS_MAX_D, O3D_ERR_ARG,
                "o3d_box_associate: bad sizes b=%d F=%d D=%d", p->b, p->F, p->D);
    O3D_REQUIRE(p->src && p->feed && p->adv && p->center && p->points && p->t && p->hit_t && p->hit_c && p->vel && p->fed &&
                    p->count && p->det && p->pred && p->match && p->match_box && p->rec_det && p->rec_count && p->rec_slot,
                O3D_ERR_ARG, "o3d_box_associate: null pointer");
    O3D_REQUIRE(isfinite(p->gate2) && p->gate2 > 0.0f, O3D_ERR_ARG, "o3d_box_associate: bad gate2=%g", (double)p->gate2);
    O3D_REQUIRE(p->axis0 >= 0 && p->axis0 <= 2 && p->axis1 >= 0 && p->axis1 <= 2 && p->axis0 != p->axis1, O3D_ERR_ARG,
                "o3d_box_associate: bad plane axes %d, %d", p->axis0, p->axis1);
    O3D_REQUIRE((p->rule == 0 || p->rule == 1) && (p->coast == 0 || p->coast == 1) && (!p->coast || p->rule) &&
                    (!p->rule || p->min_points >= 0),
                O3D_ERR_ARG, "o3d_box_associate: bad switches rule=%d min_points=%d coast=%d", p->rule, p->min_points, p->coast);
    if (p->b == 0) return O3D_OK;
    associate_kernel<<<p->F, AS_THREADS, 0, (cudaStream_t)stream>>>(*p);
    O3D_CHECK_LAUNCH("o3d_box_associate");
    return O3D_OK;
}
