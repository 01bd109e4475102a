// utils/metrics.py's box footprint and footprint intersection in fp64 (reference utils/metrics.py:27-60), shared by the
// per-slot overlap of split evaluation (track_eval.cu) and the multi-object scorer (mot_eval.cu).  Every operation is an
// explicit round-to-nearest intrinsic: the build contracts a*b+c into FMAs by default, and the host restatement does not.
#pragma once
#include <cuda_runtime.h>

namespace o3d_overlap {

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
__device__ inline void footprint(const double* c, const double* wlh, const double* R, bool y_up, V2* p) {
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
__device__ inline double poly_area(const V2* p, int n) {
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
__device__ inline double intersection_area(const V2* pa, const V2* pb) {
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

}  // namespace o3d_overlap
