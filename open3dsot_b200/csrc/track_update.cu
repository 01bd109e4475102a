// The live tracker's per-row write-back (tracking/multi_tracker.py): box, frame counter, first-frame flag, evidence, the
// end-of-track rule, coasting and detection matches, for every row of a bucket step in one launch.  Row i reads its slot's state
// at src[i] and writes it at dst[i]; the rows' slots are distinct, so a thread is the only one to touch its rows and reads them
// before it writes them.  The coast arithmetic is tracking/multi_tracker.py track_update's, one explicitly rounded fp32 operation
// at a time (the build contracts a*b+c into FMAs by default, the tensor formulation does not), so the two agree bit for bit.
#include "common.cuh"
#include "track_predict.cuh"
#include "../../include/o3d_b200.h"

namespace {

constexpr int TU_THREADS = 128;

__global__ void __launch_bounds__(TU_THREADS) track_update_kernel(const o3d_track_update_t p) {
    const int i = blockIdx.x * TU_THREADS + threadIdx.x;
    if (i >= p.b) return;
    const long long s = p.src[i], d = p.dst[i];
    const bool adv = p.adv[i] != 0;
    float c[3], r[9], vel[3], hit_c[3];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        c[j] = p.box_c[s * 3 + j];
        vel[j] = p.vel[s * 3 + j];
        hit_c[j] = p.hit_c[s * 3 + j];
    }
#pragma unroll
    for (int j = 0; j < 9; ++j) r[j] = p.box_r[s * 9 + j];
    long long t = p.t[s], hit_t = p.hit_t[s];
    float first_flag = p.first_flag[s], score = p.slot_score[s];
    int points = p.slot_points[s], misses = p.misses[s];
    bool lost = p.lost[s] != 0, coasting = p.coasting[s] != 0;
    int detection = p.match ? p.slot_detection[s] : -1;
    bool reacquired = p.match ? p.slot_reacquired[s] != 0 : false;
    if (adv) {
        t += 1;
        first_flag = 0.0f;
        points = p.points[i];
        score = p.score[i];
        const bool net_hit = !p.rule || points >= p.min_points;
        // a miss matched to a detection is re-acquired: it counts as a hit on the detection's box
        const int m = p.match ? p.match[i] : -1;
        const bool re = m >= 0 && !net_hit;
        const bool hit = net_hit || re;
        float pc[3];
#pragma unroll
        for (int j = 0; j < 3; ++j) pc[j] = re ? p.match_box[i * 12 + j] : p.center[i * 3 + j];
        if (p.rule) misses = hit ? 0 : misses + 1;
        if (p.rule) lost = lost || misses >= p.patience;
        const float gap = (float)(t - hit_t);
        float nc[3];
        o3d_predicted_centre(pc, hit, p.coast != 0, hit_c, vel, gap, nc);       // before vel / hit_c move
        if (p.coast && hit) {
#pragma unroll
            for (int j = 0; j < 3; ++j) {
                const float v = __fdiv_rn(__fsub_rn(pc[j], hit_c[j]), gap);
                vel[j] = hit_t == 0 ? v : __fadd_rn(__fmul_rn(p.alpha, v), __fmul_rn(p.beta, vel[j]));
                hit_c[j] = pc[j];
            }
            hit_t = t;
        }
#pragma unroll
        for (int j = 0; j < 3; ++j) c[j] = nc[j];
        if (!(p.coast && !hit)) {                                                  // coasted: the previous rotation
#pragma unroll
            for (int j = 0; j < 9; ++j) r[j] = re ? p.match_box[i * 12 + 3 + j] : p.rot[i * 9 + j];
        }
        if (p.coast) coasting = !hit && !lost;
        detection = m;
        reacquired = re;
    } else if (p.rule) {
        lost = lost || misses >= p.patience;
    }
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        p.box_c[d * 3 + j] = c[j];
        p.vel[d * 3 + j] = vel[j];
        p.hit_c[d * 3 + j] = hit_c[j];
    }
#pragma unroll
    for (int j = 0; j < 9; ++j) p.box_r[d * 9 + j] = r[j];
    p.t[d] = t;
    p.hit_t[d] = hit_t;
    p.first_flag[d] = first_flag;
    p.slot_score[d] = score;
    p.slot_points[d] = points;
    p.misses[d] = misses;
    p.lost[d] = lost;
    p.coasting[d] = coasting;
    if (p.match) {
        p.slot_detection[d] = detection;
        p.slot_reacquired[d] = reacquired;
    }
}

}  // namespace

extern "C" int o3d_track_update(const o3d_track_update_t* p, void* stream) {
    O3D_REQUIRE(p, O3D_ERR_ARG, "o3d_track_update: null pointer (descriptor)");
    O3D_REQUIRE(p->b >= 0 && p->b <= 65535, O3D_ERR_ARG, "o3d_track_update: bad sizes b=%d", p->b);
    O3D_REQUIRE(p->src && p->dst && p->adv && p->center && p->rot && p->points && p->score && p->box_c && p->box_r && p->t &&
                    p->first_flag && p->slot_points && p->slot_score && p->misses && p->lost && p->vel && p->hit_c && p->hit_t &&
                    p->coasting,
                O3D_ERR_ARG, "o3d_track_update: null pointer");
    const bool any_match = p->match || p->match_box || p->slot_detection || p->slot_reacquired;
    O3D_REQUIRE(!any_match || (p->match && p->match_box && p->slot_detection && p->slot_reacquired), O3D_ERR_ARG,
                "o3d_track_update: null pointer (the match fields are all set or all null)");
    O3D_REQUIRE((p->rule == 0 || p->rule == 1) && (p->coast == 0 || p->coast == 1), O3D_ERR_ARG,
                "o3d_track_update: bad switches rule=%d coast=%d", p->rule, p->coast);
    O3D_REQUIRE(!p->rule || (p->min_points >= 0 && p->patience >= 1), O3D_ERR_ARG,
                "o3d_track_update: bad rule min_points=%d patience=%d", p->min_points, p->patience);
    O3D_REQUIRE(!p->coast || (p->rule && p->alpha > 0.0f && p->alpha <= 1.0f), O3D_ERR_ARG,
                "o3d_track_update: bad coast (rule=%d alpha=%g): coasting needs the rule and 0 < alpha <= 1", p->rule,
                (double)p->alpha);
    if (p->b == 0) return O3D_OK;
    track_update_kernel<<<(p->b + TU_THREADS - 1) / TU_THREADS, TU_THREADS, 0, (cudaStream_t)stream>>>(*p);
    O3D_CHECK_LAUNCH("o3d_track_update");
    return O3D_OK;
}
