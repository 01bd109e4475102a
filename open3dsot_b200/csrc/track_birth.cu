// Target births of the live tracker (tracking/multi_tracker.py birth_tensors): after the detection matching, each fed feed's
// unmatched detections that score at least min_score and lie beyond the gate of every row that took part in the matching are
// ranked by descending score, then ascending index, and walked in that order; a candidate is born into the feed's next reserved
// slot when no candidate born before it in this advance lies within the gate, until the feed's reserved slots run out.
//
// One CTA walks the feeds in ascending order, so the id counter advances in (feed, rank) order whatever the launch.  Per feed:
//   1. every thread marks one detection a candidate or not and builds its key (descending score, ascending index), testing it
//      against the feed's advancing rows, compacted into shared memory 1024 rows of the step at a time;
//   2. a bitonic sort of the keys in shared memory (D <= 1024);
//   3. warp 0 walks the ranked candidates 32 at a time: each lane tests its candidate against the ones born in earlier chunks
//      (at most the feed's reserved slots), then every lane replays the chunk's sequential decisions from the chunk's pairwise
//      conflict masks, so all lanes agree on which are born.
// Scores are normalised with + 0.0f (-0 ranks as +0, as a float comparison does); they are finite (checked on the host).  No
// atomics; every fp32 operation is rounded on its own, as in the formulation.
#include "common.cuh"
#include "../../include/o3d_b200.h"

namespace {

constexpr int TB_THREADS = 1024;
constexpr int TB_MAX_D = 1024;
constexpr unsigned long long TB_NONE = ~0ull;

// d2 = dx*dx + dy*dy with dx = a - b, every operation rounded on its own (birth_tensors' and associate's expression)
__device__ __forceinline__ float tb_d2(float ax, float ay, float bx, float by) {
    const float dx = __fsub_rn(ax, bx), dy = __fsub_rn(ay, by);
    return __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy));
}

// ascending key for (descending score, ascending index)
__device__ __forceinline__ unsigned long long tb_key(float score, int d) {
    const unsigned u = __float_as_uint(__fadd_rn(score, 0.0f));
    const unsigned asc = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
    return ((unsigned long long)(~asc) << 32) | (unsigned)d;
}

// one born detection: the slot state add(id, box, feed) writes, the feed's record and the log entry
__device__ void tb_write(const o3d_track_birth_t& p, int e, long long k, long long id, int f, int d, const float* row) {
    for (int j = 0; j < 3; ++j) {
        p.box_c[k * 3 + j] = row[j];
        p.box_s[k * 3 + j] = row[3 + j];
        p.hit_c[k * 3 + j] = row[j];
        p.vel[k * 3 + j] = 0.0f;
    }
    for (int j = 0; j < 9; ++j) p.box_r[k * 9 + j] = row[6 + j];
    p.first_flag[k] = 1.0f;
    p.active[k] = 1;
    p.key[k] = id;
    p.t[k] = 0;
    p.slot_feed[k] = f;
    p.points[k] = -1;
    p.score[k] = __int_as_float(0x7fc00000);
    p.misses[k] = 0;
    p.lost[k] = 0;
    p.hit_t[k] = 0;
    p.coasting[k] = 0;
    p.detection[k] = -1;
    p.reacquired[k] = 0;
    p.rec_slot[(long long)f * p.D + d] = (int)k;
    p.log[e * 4 + 0] = k;
    p.log[e * 4 + 1] = id;
    p.log[e * 4 + 2] = f;
    p.log[e * 4 + 3] = d;
}

__global__ void __launch_bounds__(TB_THREADS) birth_kernel(const o3d_track_birth_t p) {
    __shared__ unsigned long long s_key[TB_MAX_D];
    __shared__ float2 s_born[TB_MAX_D];               // plane coordinates of the feed's born candidates
    __shared__ float2 s_rows[TB_THREADS];            // the feed's advancing rows' pred centres, one chunk of rows
    __shared__ int s_wcount[TB_THREADS / 32];
    __shared__ long long s_next;
    __shared__ int s_nb;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const long long D = p.D;
    for (int e = tid; e < p.R; e += TB_THREADS) {
#pragma unroll
        for (int j = 0; j < 4; ++j) p.log[e * 4 + j] = -1;
    }
    if (tid == 0) s_next = *p.next;
    __syncthreads();

    for (int f = 0; f < p.F; ++f) {
        // the feed's reserved entries: contiguous, after those of the feeds before it
        int r = 0, start = 0;
        for (int e0 = 0; e0 < p.R; e0 += TB_THREADS) {
            const int e = e0 + tid;
            const long long bf = e < p.R ? p.birth_feed[e] : -1;
            r += __syncthreads_count(bf == f);
            start += __syncthreads_count(bf >= 0 && bf < f);
        }
        const int nd = p.fed[f] != 0 ? p.count[f] : 0;
        if (r == 0 || nd == 0) continue;
        const float* det = p.det + (long long)f * D * 16;

        // 1. candidates and their keys; the feed's advancing rows are compacted into shared memory a chunk at a time
        int P = 1;
        while (P < nd) P <<= 1;
        bool cand = false;
        float qx = 0.0f, qy = 0.0f;
        if (tid < nd) {
            const float* q = det + tid * 16;
            qx = q[p.axis0];
            qy = q[p.axis1];
            cand = p.rec_slot[f * D + tid] < 0 && q[15] >= p.min_score;
        }
        for (int i0 = 0; i0 < p.b; i0 += TB_THREADS) {
            const int i = i0 + tid;
            const bool mine = i < p.b && p.feed[i] == f && p.adv[i];
            const unsigned m = __ballot_sync(0xffffffffu, mine);
            if (lane == 0) s_wcount[warp] = __popc(m);
            __syncthreads();
            int off = 0, n = 0;
            for (int w = 0; w < TB_THREADS / 32; ++w) {
                const int c = s_wcount[w];
                off += w < warp ? c : 0;
                n += c;
            }
            if (mine) s_rows[off + __popc(m & ((1u << lane) - 1u))] = make_float2(p.pred[i * 3 + p.axis0], p.pred[i * 3 + p.axis1]);
            __syncthreads();
            for (int j = 0; cand && j < n; ++j)
                if (tb_d2(s_rows[j].x, s_rows[j].y, qx, qy) <= p.gate2) cand = false;
            __syncthreads();
        }
        if (tid < P) s_key[tid] = cand ? tb_key(det[tid * 16 + 15], tid) : TB_NONE;
        const int n_cand = __syncthreads_count(cand);
        if (n_cand == 0) continue;

        // 2. bitonic sort of the P keys, ascending
        for (int k = 2; k <= P; k <<= 1) {
            for (int j = k >> 1; j > 0; j >>= 1) {
                if (tid < P) {
                    const int o = tid ^ j;
                    if (o > tid) {
                        const unsigned long long a = s_key[tid], c = s_key[o];
                        if (((tid & k) == 0) == (a > c)) {
                            s_key[tid] = c;
                            s_key[o] = a;
                        }
                    }
                }
                __syncthreads();
            }
        }

        // 3. the walk, warp 0
        if (warp == 0) {
            int nb = 0;
            for (int c0 = 0; c0 < n_cand && nb < r; c0 += 32) {
                const int idx = c0 + lane;
                const bool valid = idx < n_cand;
                const int d = valid ? (int)(s_key[idx] & 0xffffffffu) : 0;
                const float qx = valid ? det[d * 16 + p.axis0] : 0.0f, qy = valid ? det[d * 16 + p.axis1] : 0.0f;
                bool alive = valid;
                for (int k = 0; alive && k < nb; ++k)
                    if (tb_d2(qx, qy, s_born[k].x, s_born[k].y) <= p.gate2) alive = false;
                unsigned conflict = 0;                // bit i: earlier chunk candidate i lies within the gate of this one
                for (int i = 0; i < 32; ++i) {
                    const float ix = __shfl_sync(0xffffffffu, qx, i), iy = __shfl_sync(0xffffffffu, qy, i);
                    if (i < lane && tb_d2(qx, qy, ix, iy) <= p.gate2) conflict |= 1u << i;
                }
                const unsigned alive_mask = __ballot_sync(0xffffffffu, alive);
                unsigned born = 0;
                int n = nb;
                for (int j = 0; j < 32; ++j) {
                    const unsigned cj = __shfl_sync(0xffffffffu, conflict, j);
                    if (n < r && ((alive_mask >> j) & 1u) && !(cj & born)) {
                        born |= 1u << j;
                        ++n;
                    }
                }
                if ((born >> lane) & 1u) {
                    const int pos = nb + __popc(born & ((1u << lane) - 1u));
                    s_born[pos] = make_float2(qx, qy);
                    const int e = start + pos;
                    tb_write(p, e, p.birth_slot[e], p.id_base + s_next + pos, f, d, det + d * 16);
                }
                nb = n;
                __syncwarp();
            }
            if (lane == 0) s_nb = nb;
        }
        __syncthreads();
        if (tid == 0) s_next += s_nb;
        __syncthreads();
    }
    if (tid == 0) *p.next = s_next;
}

}  // namespace

extern "C" int o3d_track_birth(const o3d_track_birth_t* p, void* stream) {
    O3D_REQUIRE(p, O3D_ERR_ARG, "o3d_track_birth: null pointer (descriptor)");
    O3D_REQUIRE(p->b >= 0 && p->b <= 65535 && p->F >= 1 && p->D >= 1 && p->D <= TB_MAX_D && p->R >= 1 && p->R <= 65535,
                O3D_ERR_ARG, "o3d_track_birth: bad sizes b=%d F=%d D=%d R=%d", p->b, p->F, p->D, p->R);
    O3D_REQUIRE((p->b == 0 || (p->feed && p->adv && p->pred)) && p->fed && p->count && p->det && p->rec_slot && p->birth_slot &&
                    p->birth_feed && p->next && p->log && p->box_c && p->box_s && p->box_r && p->first_flag && p->active &&
                    p->key && p->t && p->slot_feed && p->points && p->score && p->misses && p->lost && p->vel && p->hit_c &&
                    p->hit_t && p->coasting && p->detection && p->reacquired,
                O3D_ERR_ARG, "o3d_track_birth: null pointer");
    O3D_REQUIRE(isfinite(p->gate2) && p->gate2 > 0.0f, O3D_ERR_ARG, "o3d_track_birth: bad gate2=%g", (double)p->gate2);
    O3D_REQUIRE(isfinite(p->min_score), O3D_ERR_ARG, "o3d_track_birth: bad min_score=%g", (double)p->min_score);
    O3D_REQUIRE(p->axis0 >= 0 && p->axis0 <= 2 && p->axis1 >= 0 && p->axis1 <= 2 && p->axis0 != p->axis1, O3D_ERR_ARG,
                "o3d_track_birth: bad plane axes %d, %d", p->axis0, p->axis1);
    O3D_REQUIRE(p->id_base >= 0, O3D_ERR_ARG, "o3d_track_birth: bad id_base=%lld", p->id_base);
    birth_kernel<<<1, TB_THREADS, 0, (cudaStream_t)stream>>>(*p);
    O3D_CHECK_LAUNCH("o3d_track_birth");
    return O3D_OK;
}
