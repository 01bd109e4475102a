// Multi-object tracking scores (tracking/mot.py): the CLEAR MOT events and the identity co-occurrence of many sequences, one
// CTA per sequence walking its frames in order (the events of a frame depend on the matches of the frames before it).
//
// Per frame:
//   load:        each box's footprint, its area and its up-axis interval (IoU) or its centre (distance), once per box;
//   pairs:       one thread per (object, hypothesis): the pair's cost (NaN when not valid) into the CTA's work row, the
//                co-occurrence count of a valid pair (one thread per pair and frame: no atomics), and the object's carry-over
//                candidate (the frame's hypothesis equal to its last match);
//   carry-over:  thread 0, the objects in frame order;
//   assignment:  on the remainder.  When every remaining object and hypothesis has at most one valid partner, the valid pairs
//                are the only maximum matching and are taken as they are.  Otherwise scipy's linear_sum_assignment (shortest
//                augmenting paths, one row at a time) on the remainder with motmetrics' large constant at the invalid pairs:
//                a thread per column of the scan, a block arg-min with scipy's tie rule, thread 0 for the path bookkeeping;
//   events:      a thread per object updates its counts, last match and fragmentation state; thread 0 tallies the frame in
//                object order, so the cost sum has one order whatever the launch.
#include <math.h>

#include "common.cuh"
#include "box_overlap.cuh"
#include "../../include/o3d_b200.h"

namespace {

using namespace o3d_overlap;

constexpr int MOT_THREADS = 256;
constexpr int MOT_WARPS = MOT_THREADS / 32;
constexpr int MOT_MAX = O3D_MOT_MAX_BOXES;
constexpr int BOX_VALUES = 15;      // centre, wlh, row-major rotation
constexpr int PREP = 12;            // per box in shared memory: IoU: footprint (8), area, up centre, height, volume; distance: centre
static_assert(MOT_MAX <= MOT_THREADS, "a thread per column of the assignment scan");

// event codes of an object in a frame
constexpr int EV_MISS = 0, EV_MATCH = 1, EV_SWITCH = 2, EV_FRAG = 4;
// fragmentation walk: 0 = not tracked yet (or no open gap), 1 = tracked on its last frame, 2 = missed since it was tracked
constexpr int FR_NONE = 0, FR_TRACKED = 1, FR_GAP = 2;

struct MotShared {
    double u[MOT_MAX], v[MOT_MAX], spc[MOT_MAX];      // scipy's duals and shortest path costs
    double red_v[MOT_WARPS];
    int red_k[MOT_WARPS];
    int gobj[MOT_MAX], last[MOT_MAX], carry[MOT_MAX], gmatch[MOT_MAX], ev[MOT_MAX];
    int hidx[MOT_MAX], hmatch[MOT_MAX];
    int rows[MOT_MAX], cols[MOT_MAX];                 // the remainder: frame-local object / hypothesis indices
    int path[MOT_MAX], col4row[MOT_MAX], row4col[MOT_MAX], remaining[MOT_MAX];
    unsigned char gnew[MOT_MAX], SR[MOT_MAX], SC[MOT_MAX];
    unsigned long long cmax_bits;
    double min_val, big;
    int nr0, nc0, cur_i, n_rem, sink;
};

// one box of the frame into shared memory
__device__ void prep_box(const double* __restrict__ b, int metric, bool y_up, int u, double* out) {
    double c[3], wlh[3], R[9];
    for (int i = 0; i < 3; ++i) {
        c[i] = b[i];
        wlh[i] = b[3 + i];
    }
    for (int i = 0; i < 9; ++i) R[i] = b[6 + i];
    if (metric == 0) {
        V2* p = reinterpret_cast<V2*>(out);
        footprint(c, wlh, R, y_up, p);
        out[8] = poly_area(p, 4);
        out[9] = c[u];
        out[10] = wlh[2];
        out[11] = __dmul_rn(__dmul_rn(wlh[0], wlh[1]), wlh[2]);
    } else {
        for (int i = 0; i < 3; ++i) out[i] = c[i];
    }
}

// cost of (ground truth a, hypothesis b), NaN when the pair is not valid: o3d_track_metrics' arithmetic with a precomputed
// footprint per box
__device__ double pair_cost(const double* a, const double* b, int metric, int dim, int up_mask, double threshold) {
    if (metric == 0) {
        const double inter = intersection_area(reinterpret_cast<const V2*>(a), reinterpret_cast<const V2*>(b));
        double iou;
        if (dim == 2) {
            const double uni = __dsub_rn(__dadd_rn(a[8], b[8]), inter);
            iou = uni > 0.0 ? __ddiv_rn(inter, uni) : 0.0;
        } else {
            const double up_max = fmin(a[9], b[9]);
            const double up_min = fmax(__dsub_rn(a[9], a[10]), __dsub_rn(b[9], b[10]));
            const double vol = __dmul_rn(inter, fmax(0.0, __dsub_rn(up_max, up_min)));
            iou = __ddiv_rn(vol, __dsub_rn(__dadd_rn(a[11], b[11]), vol));
        }
        return iou >= threshold ? __dsub_rn(1.0, iou) : __longlong_as_double(0x7ff8000000000000ll);
    }
    double d2 = 0.0;
    for (int i = 0; i < 3; ++i) {
        if (dim == 3 || ((up_mask >> i) & 1)) {
            const double d = __dsub_rn(a[i], b[i]);
            d2 = __dadd_rn(d2, __dmul_rn(d, d));
        }
    }
    const double d = __dsqrt_rn(d2);
    return d <= threshold ? d : __longlong_as_double(0x7ff8000000000000ll);
}

__device__ __forceinline__ bool valid(double c) { return c == c; }

// scipy's pick among the columns of the scan: the least shortest-path cost; on a tie the last unassigned column in the scan's
// order, or, when every tied column is assigned, the first.  key: unassigned 256 + it, assigned 255 - it; the larger key wins.
__device__ __forceinline__ void better(double& v, int& k, double v2, int k2) {
    if (v2 < v || (v2 == v && k2 > k)) {
        v = v2;
        k = k2;
    }
}

__global__ void __launch_bounds__(MOT_THREADS) mot_clear_kernel(const o3d_mot_clear_t p) {
    extern __shared__ double s_box[];                 // [max_gt + max_hyp, PREP]
    __shared__ MotShared sh;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const bool y_up = (p.up_mask & 2) != 0;
    const int u_axis = (p.up_mask & 1) ? 0 : ((p.up_mask & 2) ? 1 : 2);
    double* sg = s_box;
    double* shp = s_box + (size_t)p.max_gt * PREP;
    double* W = p.work + (size_t)blockIdx.x * p.max_gt * p.max_hyp;

    for (int s = blockIdx.x; s < p.S; s += gridDim.x) {
        const long long ob = p.obj_off[s], Hs = p.hyp_off[s + 1] - p.hyp_off[s], co = p.cooc_off[s];
        const long long n_obj = p.obj_off[s + 1] - ob;
        for (long long e = tid; e < p.cooc_off[s + 1] - co; e += MOT_THREADS) p.cooc[co + e] = 0;
        for (long long o = tid; o < n_obj; o += MOT_THREADS) {
            int* st = p.obj + (ob + o) * 4;
            st[0] = 0;
            st[1] = 0;
            st[2] = -1;
            st[3] = FR_NONE;
        }
        long long n_gt = 0, n_hyp = 0, n_match = 0, n_switch = 0, n_miss = 0, n_fp = 0, n_frag = 0;
        double cost_sum = 0.0;
        __syncthreads();

        for (long long f = p.seq_frame[s]; f < p.seq_frame[s + 1]; ++f) {
            const long long g0 = p.frame_gt[f], h0 = p.frame_hyp[f];
            const int G = (int)(p.frame_gt[f + 1] - g0), H = (int)(p.frame_hyp[f + 1] - h0);
            // load
            for (int i = tid; i < G + H; i += MOT_THREADS) {
                if (i < G) {
                    prep_box(p.gt_box + (g0 + i) * BOX_VALUES, p.metric, y_up, u_axis, sg + i * PREP);
                    const int o = p.gt_obj[g0 + i];
                    sh.gobj[i] = o;
                    sh.last[i] = p.obj[(ob + o) * 4 + 2];
                    sh.carry[i] = -1;
                    sh.gmatch[i] = -1;
                    sh.gnew[i] = 0;
                } else {
                    const int j = i - G;
                    prep_box(p.hyp_box + (h0 + j) * BOX_VALUES, p.metric, y_up, u_axis, shp + j * PREP);
                    sh.hidx[j] = p.hyp_idx[h0 + j];
                    sh.hmatch[j] = -1;
                }
            }
            __syncthreads();
            // pairs
            for (int q = tid; q < G * H; q += MOT_THREADS) {
                const int o = q / H, h = q - o * H;
                const double c = pair_cost(sg + o * PREP, shp + h * PREP, p.metric, p.dim, p.up_mask, p.threshold);
                W[q] = c;
                if (valid(c)) p.cooc[co + (long long)sh.gobj[o] * Hs + sh.hidx[h]] += 1;
                if (sh.hidx[h] == sh.last[o]) sh.carry[o] = h;
            }
            __syncthreads();
            // carry-over, then the remainder's lists
            if (tid == 0) {
                for (int o = 0; o < G; ++o) {
                    const int h = sh.carry[o];
                    if (h >= 0 && sh.hmatch[h] < 0 && valid(W[o * H + h])) {
                        sh.gmatch[o] = h;
                        sh.hmatch[h] = o;
                    }
                }
                int nr = 0, nc = 0;
                for (int o = 0; o < G; ++o)
                    if (sh.gmatch[o] < 0) sh.rows[nr++] = o;
                for (int h = 0; h < H; ++h)
                    if (sh.hmatch[h] < 0) sh.cols[nc++] = h;
                sh.nr0 = nr;
                sh.nc0 = nc;
                sh.cmax_bits = 0ull;
            }
            __syncthreads();
            const int nr0 = sh.nr0, nc0 = sh.nc0;
            if (nr0 > 0 && nc0 > 0) {
                // valid partners per remaining object and hypothesis, the largest |cost|
                bool multi = false;
                double cmax = 0.0;
                for (int i = tid; i < nr0; i += MOT_THREADS) {
                    const double* row = W + sh.rows[i] * H;
                    int n = 0;
                    for (int j = 0; j < nc0; ++j) {
                        const double c = row[sh.cols[j]];
                        if (valid(c)) {
                            ++n;
                            cmax = fmax(cmax, fabs(c));
                        }
                    }
                    multi = multi || n > 1;
                }
                for (int j = tid; j < nc0; j += MOT_THREADS) {
                    int n = 0;
                    for (int i = 0; i < nr0; ++i) n += valid(W[sh.rows[i] * H + sh.cols[j]]);
                    multi = multi || n > 1;
                }
                atomicMax(&sh.cmax_bits, (unsigned long long)__double_as_longlong(cmax));     // cmax >= 0: its bits order as it
                if (!__syncthreads_or(multi)) {
                    // the valid pairs of the remainder form a matching: take them
                    for (int i = tid; i < nr0; i += MOT_THREADS) {
                        const int o = sh.rows[i];
                        for (int j = 0; j < nc0; ++j) {
                            const int h = sh.cols[j];
                            if (valid(W[o * H + h])) {
                                sh.gmatch[o] = h;
                                sh.hmatch[h] = o;
                                sh.gnew[o] = 1;
                            }
                        }
                    }
                } else {
                    const bool transpose = nc0 < nr0;
                    const int nr = transpose ? nc0 : nr0, nc = transpose ? nr0 : nc0;
                    for (int i = tid; i < MOT_MAX; i += MOT_THREADS) {
                        sh.u[i] = 0.0;
                        sh.v[i] = 0.0;
                        sh.col4row[i] = -1;
                        sh.row4col[i] = -1;
                    }
                    if (tid == 0) {
                        // motmetrics' constant: c = max |valid cost| + 1, l = 2 r c + 1
                        const double c = __dadd_rn(__longlong_as_double((long long)sh.cmax_bits), 1.0);
                        sh.big = __dadd_rn(__dmul_rn((double)(2 * nr), c), 1.0);
                    }
                    __syncthreads();
                    const double big = sh.big;
                    for (int cur = 0; cur < nr; ++cur) {
                        if (tid < nc) {
                            sh.remaining[tid] = nc - tid - 1;
                            sh.SC[tid] = 0;
                            sh.spc[tid] = INFINITY;
                        }
                        if (tid < nr) sh.SR[tid] = 0;
                        if (tid == 0) {
                            sh.cur_i = cur;
                            sh.min_val = 0.0;
                            sh.n_rem = nc;
                            sh.sink = -1;
                        }
                        __syncthreads();
                        for (;;) {
                            const int i = sh.cur_i, n_rem = sh.n_rem;
                            const double min_val = sh.min_val;
                            double bv = INFINITY;
                            int bk = -1;
                            if (tid < n_rem) {
                                const int j = sh.remaining[tid];
                                const int o = transpose ? sh.rows[j] : sh.rows[i];
                                const int h = transpose ? sh.cols[i] : sh.cols[j];
                                double c = W[o * H + h];
                                if (!valid(c)) c = big;
                                const double r = __dsub_rn(__dsub_rn(__dadd_rn(min_val, c), sh.u[i]), sh.v[j]);
                                if (r < sh.spc[j]) {
                                    sh.path[j] = i;
                                    sh.spc[j] = r;
                                }
                                bv = sh.spc[j];
                                bk = sh.row4col[j] == -1 ? MOT_MAX + tid : MOT_MAX - 1 - tid;
                            }
#pragma unroll
                            for (int off = 16; off > 0; off >>= 1) {
                                const double v2 = __shfl_xor_sync(0xffffffffu, bv, off);
                                const int k2 = __shfl_xor_sync(0xffffffffu, bk, off);
                                better(bv, bk, v2, k2);
                            }
                            if (lane == 0) {
                                sh.red_v[warp] = bv;
                                sh.red_k[warp] = bk;
                            }
                            __syncthreads();
                            if (tid == 0) {
                                double lv = sh.red_v[0];
                                int lk = sh.red_k[0];
                                for (int w = 1; w < MOT_WARPS; ++w) better(lv, lk, sh.red_v[w], sh.red_k[w]);
                                const int it = lk >= MOT_MAX ? lk - MOT_MAX : MOT_MAX - 1 - lk;
                                const int j = sh.remaining[it];
                                sh.SR[i] = 1;
                                sh.min_val = lv;
                                if (sh.row4col[j] == -1)
                                    sh.sink = j;
                                else
                                    sh.cur_i = sh.row4col[j];
                                sh.SC[j] = 1;
                                sh.remaining[it] = sh.remaining[--sh.n_rem];
                            }
                            __syncthreads();
                            if (sh.sink >= 0) break;
                        }
                        // duals, then the augmentation along the path
                        const double min_val = sh.min_val;
                        if (tid < nr && tid != cur && sh.SR[tid])
                            sh.u[tid] = __dadd_rn(sh.u[tid], __dsub_rn(min_val, sh.spc[sh.col4row[tid]]));
                        if (tid < nc && sh.SC[tid]) sh.v[tid] = __dsub_rn(sh.v[tid], __dsub_rn(min_val, sh.spc[tid]));
                        __syncthreads();
                        if (tid == 0) {
                            sh.u[cur] = __dadd_rn(sh.u[cur], min_val);
                            int j = sh.sink;
                            for (;;) {
                                const int i = sh.path[j];
                                sh.row4col[j] = i;
                                const int t = sh.col4row[i];
                                sh.col4row[i] = j;
                                j = t;
                                if (i == cur) break;
                            }
                        }
                        __syncthreads();
                    }
                    // the assignment's valid pairs are the frame's new pairs
                    if (tid < nr) {
                        const int j = sh.col4row[tid];
                        const int o = transpose ? sh.rows[j] : sh.rows[tid];
                        const int h = transpose ? sh.cols[tid] : sh.cols[j];
                        if (valid(W[o * H + h])) {
                            sh.gmatch[o] = h;
                            sh.hmatch[h] = o;
                            sh.gnew[o] = 1;
                        }
                    }
                }
            }
            __syncthreads();
            // events
            for (int i = tid; i < G; i += MOT_THREADS) {
                int* st = p.obj + (ob + sh.gobj[i]) * 4;
                const int h = sh.gmatch[i];
                st[0] += 1;
                int ev = EV_MISS;
                if (h >= 0) {
                    const int hh = sh.hidx[h];
                    ev = (sh.gnew[i] && st[2] >= 0 && st[2] != hh) ? EV_SWITCH : EV_MATCH;
                    st[1] += 1;
                    st[2] = hh;
                    if (st[3] == FR_GAP) ev |= EV_FRAG;
                    st[3] = FR_TRACKED;
                } else if (st[3] == FR_TRACKED) {
                    st[3] = FR_GAP;
                }
                sh.ev[i] = ev;
            }
            __syncthreads();
            if (tid == 0) {
                n_gt += G;
                n_hyp += H;
                int matched = 0;
                for (int i = 0; i < G; ++i) {
                    const int ev = sh.ev[i];
                    if ((ev & 3) == EV_MISS) {
                        ++n_miss;
                        continue;
                    }
                    ++matched;
                    n_match += (ev & 3) == EV_MATCH;
                    n_switch += (ev & 3) == EV_SWITCH;
                    n_frag += (ev & EV_FRAG) != 0;
                    cost_sum = __dadd_rn(cost_sum, W[i * H + sh.gmatch[i]]);
                }
                n_fp += H - matched;
            }
            __syncthreads();
        }
        if (tid == 0) {
            long long* c = p.counts + (long long)s * O3D_MOT_COUNTERS;
            c[0] = n_gt;
            c[1] = n_hyp;
            c[2] = n_match;
            c[3] = n_switch;
            c[4] = n_miss;
            c[5] = n_fp;
            c[6] = n_frag;
            p.cost_sum[s] = cost_sum;
        }
    }
}

}  // namespace

extern "C" int o3d_mot_clear(const o3d_mot_clear_t* p, void* stream) {
    O3D_REQUIRE(p, O3D_ERR_ARG, "o3d_mot_clear: null pointer (descriptor)");
    O3D_REQUIRE(p->S >= 0 && p->max_gt >= 0 && p->max_gt <= MOT_MAX && p->max_hyp >= 0 && p->max_hyp <= MOT_MAX &&
                    p->work_rows >= 1,
                O3D_ERR_ARG, "o3d_mot_clear: bad sizes S=%d max_gt=%d max_hyp=%d work_rows=%d (at most %d boxes per frame and side)",
                p->S, p->max_gt, p->max_hyp, p->work_rows, MOT_MAX);
    O3D_REQUIRE(p->seq_frame && p->frame_gt && p->frame_hyp && p->obj_off && p->hyp_off && p->cooc_off && p->gt_obj &&
                    p->hyp_idx && p->gt_box && p->hyp_box && p->counts && p->cost_sum && p->obj && p->cooc && p->work,
                O3D_ERR_ARG, "o3d_mot_clear: null pointer");
    O3D_REQUIRE(p->metric == 0 || p->metric == 1, O3D_ERR_ARG, "o3d_mot_clear: metric must be 0 (IoU) or 1 (distance), got %d",
                p->metric);
    O3D_REQUIRE(p->metric == 0 ? (p->threshold > 0.0 && p->threshold <= 1.0) : (isfinite(p->threshold) && p->threshold > 0.0),
                O3D_ERR_ARG, "o3d_mot_clear: bad threshold %g for metric %d", p->threshold, p->metric);
    O3D_REQUIRE(p->dim == 2 || p->dim == 3, O3D_ERR_ARG, "o3d_mot_clear: dim must be 2 or 3, got %d", p->dim);
    O3D_REQUIRE(p->up_mask > 0 && p->up_mask < 8, O3D_ERR_ARG, "o3d_mot_clear: up_mask must name an axis, got %d", p->up_mask);
    if (p->S == 0) return O3D_OK;
    const int smem = (p->max_gt + p->max_hyp) * PREP * (int)sizeof(double);
    O3D_CUDA(cudaFuncSetAttribute(mot_clear_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem), "o3d_mot_clear");
    const int grid = p->S < p->work_rows ? p->S : p->work_rows;
    mot_clear_kernel<<<grid, MOT_THREADS, smem, (cudaStream_t)stream>>>(*p);
    O3D_CHECK_LAUNCH("o3d_mot_clear");
    return O3D_OK;
}
