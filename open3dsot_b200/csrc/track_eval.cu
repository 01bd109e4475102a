// Split evaluation with many tracklets in flight (tracking/batched_tracker.py): the per-slot random draws and the per-frame
// overlap / centre-distance record, both enqueued inside the captured frame step so that nothing is read back per frame.
//
// o3d_keyed_uniform  — counter-based uniforms: a slot's draws are a pure function of (seed, tracklet id, frame within the
//                      tracklet, stream, element), so a tracklet sees the same numbers whatever slot it runs in and however
//                      many slots run beside it.  Philox4x32-10 with cuRAND's constants, key = (seed, tracklet),
//                      counter = (element / 4, frame, stream, 0); word element % 4 -> (w >> 8) * 2^-24 in [0, 1).
// o3d_track_metrics  — utils/metrics.py estimateOverlap / estimateAccuracy (reference utils/metrics.py:27-60) in fp64 for
//                      one (result box, ground truth) pair per slot.  Every operation is an explicit round-to-nearest
//                      intrinsic: the build contracts a*b+c into FMAs by default, and the host restatement does not.
#include "resample_core.cuh"          // o3d_philox4x32_10, o3d_word_to_uniform
#include "../../include/o3d_b200.h"

namespace {

// thread = one Philox block = four consecutive elements of one slot's stream
__global__ void __launch_bounds__(256)
    keyed_uniform_kernel(const long long* __restrict__ tracklet, const long long* __restrict__ frame, uint32_t seed,
                         uint32_t stream, int n, float* __restrict__ out) {
    const int k = blockIdx.y;
    const uint32_t key1 = (uint32_t)tracklet[k];
    const uint32_t fr = (uint32_t)frame[k];
    float* __restrict__ row = out + (size_t)k * n;
    const int blocks = (n + 3) >> 2;
    for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < blocks; b += gridDim.x * blockDim.x) {
        const uint4 w = o3d_philox4x32_10(make_uint4((uint32_t)b, fr, stream, 0u), seed, key1);
        const int e = b << 2;
        if (e + 3 < n) {
            row[e + 0] = o3d_word_to_uniform(w.x);
            row[e + 1] = o3d_word_to_uniform(w.y);
            row[e + 2] = o3d_word_to_uniform(w.z);
            row[e + 3] = o3d_word_to_uniform(w.w);
        } else {
            const uint32_t ws[4] = {w.x, w.y, w.z, w.w};
            for (int j = 0; e + j < n; ++j) row[e + j] = o3d_word_to_uniform(ws[j]);
        }
    }
}

// ---- metrics ----------------------------------------------------------------------------------------------------------------
constexpr int kMaxPoly = 16;    // a quadrilateral clipped by four half-planes has at most 8 vertices

struct V2 {
    double x, y;
};

// data_classes.Box.corners(): corner = R (l/2 sx, w/2 sy, h/2 sz) + c, corner order of data_classes.py:229-252
__device__ __forceinline__ void corner(const double* c, const double* wlh, const double* R, int i, double* out) {
    const double sx = (i < 4) ? 1.0 : -1.0;
    const double sy = (i == 0 || i == 3 || i == 4 || i == 7) ? 1.0 : -1.0;
    const double sz = (i == 0 || i == 1 || i == 4 || i == 5) ? 1.0 : -1.0;
    const double lx = __dmul_rn(__dmul_rn(wlh[1], 0.5), sx);
    const double ly = __dmul_rn(__dmul_rn(wlh[0], 0.5), sy);
    const double lz = __dmul_rn(__dmul_rn(wlh[2], 0.5), sz);
#pragma unroll
    for (int r = 0; r < 3; ++r)
        out[r] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(lx, R[r * 3 + 0]), __dmul_rn(ly, R[r * 3 + 1])), __dmul_rn(lz, R[r * 3 + 2])),
                           c[r]);
}

// metrics._footprint: y-up -> (x, z) of corners 0, 1, 5, 4; otherwise (x, y) of the bottom corners 2, 3, 7, 6; counter-clockwise
__device__ void footprint(const double* c, const double* wlh, const double* R, bool y_up, V2* p) {
    const int ids_y[4] = {0, 1, 5, 4}, ids_z[4] = {2, 3, 7, 6};
    for (int i = 0; i < 4; ++i) {
        double q[3];
        corner(c, wlh, R, y_up ? ids_y[i] : ids_z[i], q);
        p[i].x = q[0];
        p[i].y = y_up ? q[2] : q[1];
    }
    double a = 0.0, b = 0.0;
    for (int i = 0; i < 4; ++i) {
        a = __dadd_rn(a, __dmul_rn(p[i].x, p[(i + 1) & 3].y));
        b = __dadd_rn(b, __dmul_rn(p[i].y, p[(i + 1) & 3].x));
    }
    if (!(__dsub_rn(a, b) > 0.0)) {
        V2 t = p[0]; p[0] = p[3]; p[3] = t;
        t = p[1]; p[1] = p[2]; p[2] = t;
    }
}

// metrics._poly_area: shoelace
__device__ double poly_area(const V2* p, int n) {
    if (n < 3) return 0.0;
    double a = 0.0, b = 0.0;
    for (int i = 0; i < n; ++i) {
        const int j = (i + 1 == n) ? 0 : i + 1;
        a = __dadd_rn(a, __dmul_rn(p[i].x, p[j].y));
        b = __dadd_rn(b, __dmul_rn(p[i].y, p[j].x));
    }
    return __dmul_rn(0.5, fabs(__dsub_rn(a, b)));
}

// metrics._intersection_area: `pa` clipped by each edge half-plane of `pb` (s >= 0 inside), then the shoelace area
__device__ double intersection_area(const V2* pa, const V2* pb) {
    V2 buf[2][kMaxPoly];
    int n = 4;
    for (int i = 0; i < 4; ++i) buf[0][i] = pa[i];
    int cur = 0;
    for (int e = 0; e < 4; ++e) {
        if (n == 0) return 0.0;
        const V2 a = pb[e], b = pb[(e + 1) & 3];
        const double ex = __dsub_rn(b.x, a.x), ey = __dsub_rn(b.y, a.y);
        const V2* in = buf[cur];
        V2* out = buf[cur ^ 1];
        int m = 0;
        for (int i = 0; i < n; ++i) {
            const V2 p = in[i], q = in[(i + 1 == n) ? 0 : i + 1];
            const double s = __dsub_rn(__dmul_rn(ex, __dsub_rn(p.y, a.y)), __dmul_rn(ey, __dsub_rn(p.x, a.x)));
            const double t = __dsub_rn(__dmul_rn(ex, __dsub_rn(q.y, a.y)), __dmul_rn(ey, __dsub_rn(q.x, a.x)));
            if (s >= 0.0 && m < kMaxPoly) out[m++] = p;
            if ((s >= 0.0) != (t >= 0.0) && m < kMaxPoly) {
                const double r = __ddiv_rn(s, __dsub_rn(s, t));
                out[m++] = V2{__dadd_rn(p.x, __dmul_rn(__dsub_rn(q.x, p.x), r)), __dadd_rn(p.y, __dmul_rn(__dsub_rn(q.y, p.y), r))};
            }
        }
        n = m;
        cur ^= 1;
    }
    return poly_area(buf[cur], n);
}

// thread = slot.  a = ground truth (fp64), b = the slot's result box (fp32 state, widened): estimateOverlap(gt, result) order.
__global__ void track_metrics_kernel(const float* __restrict__ center, const float* __restrict__ rot, const float* __restrict__ wlh,
                                     const double* __restrict__ gt_center, const double* __restrict__ gt_rot,
                                     const double* __restrict__ gt_wlh, const long long* __restrict__ frame, int K, int dim,
                                     int up_mask, double* __restrict__ overlap, double* __restrict__ distance) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= K) return;
    const long long f = frame[k];
    if (f < 0) return;                                        // idle slot: records nothing
    double ca[3], wa[3], Ra[9], cb[3], wb[3], Rb[9];
    for (int i = 0; i < 3; ++i) {
        ca[i] = gt_center[f * 3 + i];
        wa[i] = gt_wlh[f * 3 + i];
        cb[i] = (double)center[k * 3 + i];
        wb[i] = (double)wlh[k * 3 + i];
    }
    for (int i = 0; i < 9; ++i) {
        Ra[i] = gt_rot[f * 9 + i];
        Rb[i] = (double)rot[k * 9 + i];
    }
    const bool y_up = (up_mask & 2) != 0;
    V2 pa[4], pb[4];
    footprint(ca, wa, Ra, y_up, pa);
    footprint(cb, wb, Rb, y_up, pb);
    const double inter = intersection_area(pa, pb);
    double iou;
    if (dim == 2) {
        const double uni = __dsub_rn(__dadd_rn(poly_area(pa, 4), poly_area(pb, 4)), inter);
        iou = uni > 0.0 ? __ddiv_rn(inter, uni) : 0.0;
    } else {
        const int u = (up_mask & 1) ? 0 : ((up_mask & 2) ? 1 : 2);
        const double up_max = fmin(ca[u], cb[u]);
        const double up_min = fmax(__dsub_rn(ca[u], wa[2]), __dsub_rn(cb[u], wb[2]));
        const double vol = __dmul_rn(inter, fmax(0.0, __dsub_rn(up_max, up_min)));
        const double va = __dmul_rn(__dmul_rn(wa[0], wa[1]), wa[2]), vb = __dmul_rn(__dmul_rn(wb[0], wb[1]), wb[2]);
        iou = __ddiv_rn(vol, __dsub_rn(__dadd_rn(va, vb), vol));
    }
    double d2 = 0.0;
    for (int i = 0; i < 3; ++i) {
        if (dim == 3 || ((up_mask >> i) & 1)) {
            const double d = __dsub_rn(ca[i], cb[i]);
            d2 = __dadd_rn(d2, __dmul_rn(d, d));
        }
    }
    overlap[f] = iou;
    distance[f] = __dsqrt_rn(d2);
}

}  // namespace

extern "C" int o3d_keyed_uniform(const long long* tracklet, const long long* frame, int K, unsigned int seed, int stream, int n,
                                 float* out, void* cuda_stream) {
    O3D_REQUIRE(tracklet && frame && out, O3D_ERR_ARG, "o3d_keyed_uniform: null pointer");
    O3D_REQUIRE(K >= 0 && K <= 65535 && n >= 0 && stream >= 0, O3D_ERR_ARG, "o3d_keyed_uniform: bad sizes K=%d n=%d stream=%d", K,
                n, stream);
    if (K == 0 || n == 0) return O3D_OK;
    const int blocks = (n + 3) / 4;
    int gx = (blocks + 255) / 256;
    const int cap = (8 * o3d_num_sms() + K - 1) / K;
    if (gx > cap) gx = cap < 1 ? 1 : cap;
    keyed_uniform_kernel<<<dim3(gx, K), 256, 0, (cudaStream_t)cuda_stream>>>(tracklet, frame, seed, (uint32_t)stream, n, out);
    O3D_CHECK_LAUNCH("o3d_keyed_uniform");
    return O3D_OK;
}

extern "C" int o3d_track_metrics(const float* center, const float* rot, const float* wlh, const double* gt_center,
                                 const double* gt_rot, const double* gt_wlh, const long long* frame, int K, int dim, int up_mask,
                                 double* overlap, double* distance, void* stream) {
    O3D_REQUIRE(center && rot && wlh && gt_center && gt_rot && gt_wlh && frame && overlap && distance, O3D_ERR_ARG,
                "o3d_track_metrics: null pointer");
    O3D_REQUIRE(K >= 0, O3D_ERR_ARG, "o3d_track_metrics: bad K=%d", K);
    O3D_REQUIRE(dim == 2 || dim == 3, O3D_ERR_ARG, "o3d_track_metrics: dim must be 2 or 3, got %d", dim);
    O3D_REQUIRE(up_mask > 0 && up_mask < 8, O3D_ERR_ARG, "o3d_track_metrics: up_mask must name an axis, got %d", up_mask);
    if (K == 0) return O3D_OK;
    track_metrics_kernel<<<(K + 127) / 128, 128, 0, (cudaStream_t)stream>>>(center, rot, wlh, gt_center, gt_rot, gt_wlh, frame, K,
                                                                             dim, up_mask, overlap, distance);
    O3D_CHECK_LAUNCH("o3d_track_metrics");
    return O3D_OK;
}
