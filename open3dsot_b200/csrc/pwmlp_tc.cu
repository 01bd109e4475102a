// Tensor-core (Hopper wgmma) implementation of the point-wise MLP forward, data-gradient and weight-gradient GEMMs, 3xTF32.
//
// Same contract as pw_fwd_kernel / pw_dgrad_kernel in pwmlp.cu (which remain the exact-fp32 ground truth and
// serve the shapes this kernel does not take: K < 32, ragged channel tails, very small P).
//
//   D[pos, ch] = sum_k  Act[pos, k] * Wmat[ch, k]          pos tile = 128 (2 warpgroups x m64), ch tile = 128 (wgmma N)
//
// with Act produced on the fly from global memory (forward: relu(bn(Y_prev)); dgrad: dY = a*g + b + c*Y) and split
// into a TF32 "hi" part (the fp32 word with its 13 low mantissa bits cleared) and a "lo" part
// (x - hi, exact), so that   Xlo*Whi + Xhi*Wlo + Xhi*Whi   carries ~21 mantissa bits — fp32-grade accuracy, which
// the 1e-4 parity bar needs and a single TF32 pass (10 bits) cannot give.  The role tables are with the kernels below.
#include <type_traits>
#include "common.cuh"
#include "lift.cuh"
#include "tc_ptx.cuh"
#include "../../include/o3d_b200.h"

namespace {

// ---- operand descriptions (same semantics as ActIn / DyIn in pwmlp.cu) --------------------------------------
// `prep(k)` fetches the per-channel coefficients of the thread's 4 channels once per k-block; `row(p)` then costs one
// (forward) or two (dgrad) 16-byte loads.
struct TcAct {
    const float* x; int ld; const float* scale; const float* shift; int relu;
    struct Coef { float4 s, t; bool on; };
    // raw operand rows of one thread for one k-block: rows p0 + i * stride, i < R
    template <int R> struct Batch { float4 v[R]; };
    __device__ __forceinline__ Coef prep(int k, int K) const {
        Coef c;
        c.on = k < K;
        c.s = make_float4(1.f, 1.f, 1.f, 1.f);
        c.t = make_float4(0.f, 0.f, 0.f, 0.f);
        if (c.on && scale) { c.s = ld4g(scale + k); c.t = ld4g(shift + k); }
        return c;
    }
    // unconditional, always-in-range loads (clamped indices): nothing here depends on loaded data, so the whole batch is
    // issued back to back and is in flight together; masking and the transform happen in finish()
    template <int R>
    __device__ __forceinline__ void fetch(Batch<R>& b, int p0, int stride, int P, int k, int K) const {
        const int kk = k < K ? k : 0;
#pragma unroll
        for (int i = 0; i < R; ++i) {
            const int p = p0 + i * stride;
            b.v[i] = ld4g(x + (size_t)(p < P ? p : P - 1) * ld + kk);
        }
    }
    template <int R>
    __device__ __forceinline__ float4 finish(const Batch<R>& b, const Coef& c, int i, int p, int P) const {
        float4 v = b.v[i];
        if (!(c.on && p < P)) return make_float4(0.f, 0.f, 0.f, 0.f);
        if (scale) { v.x = fmaf(v.x, c.s.x, c.t.x); v.y = fmaf(v.y, c.s.y, c.t.y); v.z = fmaf(v.z, c.s.z, c.t.z); v.w = fmaf(v.w, c.s.w, c.t.w); }
        if (relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
        return v;
    }
    __device__ __forceinline__ void prefetch_rows(int p0, int rows, int P) const {   // full rows p0 .. p0+rows-1 -> L2
        if (p0 < P) o3d_prefetch_l2(x + (size_t)p0 * ld, (size_t)min(rows, P - p0) * ld * sizeof(float));
    }
};

// Lifted first layer as an operand (include/o3d_b200.h: o3d_lift_t): row p of the "activation matrix" is
//     relu(bn(Y0[p])),  Y0[p, k] = Z[gidx[p], k] + sum_j s[p][j] * u[j][k]
// gathered from the (L2-resident) source-point matrix Z — the grouped tensor and Y0 itself are never stored.
// Same interface as TcAct; loads stay "raw-first": gidx -> Z row (two dependent loads; the row indices are fetched one call
// ahead), the s.u terms / BN / ReLU happen in finish().
struct TcLift {
    LiftView lv; const float* scale; const float* shift; int relu;
    int la;   // positions between two consecutive fetches of a thread (wgrad: the k-block length; 0: same rows again, next k-block)
    struct Coef { float4 s, t, u0, u1, u2, u3; bool on; };
    // nrow / tag: row indices fetched ahead for the NEXT call (tag = its p0 + 1, 0 = none), so that only a thread's first
    // k-block of a slice / position tile pays the dependent gidx -> Z load chain
    template <int R> struct Batch { float4 v[R]; float4 sv[R]; int nrow[R]; int tag; };
    __device__ __forceinline__ Coef prep(int k, int K) const {
        Coef c;
        c.on = k < K;
        c.s = make_float4(1.f, 1.f, 1.f, 1.f);
        c.t = c.u0 = c.u1 = c.u2 = c.u3 = make_float4(0.f, 0.f, 0.f, 0.f);
        if (c.on && scale) { c.s = ld4g(scale + k); c.t = ld4g(shift + k); }
        if (c.on && lv.u) { c.u0 = ld4g(lv.u + k); c.u1 = ld4g(lv.u + lv.ldz + k); c.u2 = ld4g(lv.u + 2 * lv.ldz + k); c.u3 = ld4g(lv.u + 3 * lv.ldz + k); }
        return c;
    }
    template <int R>
    __device__ __forceinline__ void fetch(Batch<R>& b, int p0, int stride, int P, int k, int K) const {
        const int kk = k < K ? k : 0;
        if (lv.z) {
            int row[R];
            if (b.tag == p0 + 1) {
#pragma unroll
                for (int i = 0; i < R; ++i) row[i] = b.nrow[i];
            } else if (R == 4 && stride == 1 && (p0 & 3) == 0 && p0 + 3 < P) {
                const int4 r4 = __ldg(reinterpret_cast<const int4*>(lv.gidx + p0));
                row[0] = r4.x; row[R > 1 ? 1 : 0] = r4.y; row[R > 2 ? 2 : 0] = r4.z; row[R > 3 ? 3 : 0] = r4.w;
            } else {
#pragma unroll
                for (int i = 0; i < R; ++i) {
                    const int p = p0 + i * stride;
                    row[i] = __ldg(lv.gidx + (p < P ? p : P - 1));
                }
            }
#pragma unroll
            for (int i = 0; i < R; ++i) b.v[i] = ld4g(lv.z + (size_t)row[i] * lv.ldz + kk);
            if (la == 0) {
#pragma unroll
                for (int i = 0; i < R; ++i) b.nrow[i] = row[i];
                b.tag = p0 + 1;
            } else {
                const int pn = p0 + la;
#pragma unroll
                for (int i = 0; i < R; ++i) {
                    const int p = pn + i * stride;
                    b.nrow[i] = __ldg(lv.gidx + (p < P ? p : P - 1));
                }
                b.tag = pn + 1;
            }
        }
        if (lv.s) {
#pragma unroll
            for (int i = 0; i < R; ++i) {
                const int p = p0 + i * stride;
                b.sv[i] = ld4g(lv.s + (size_t)(p < P ? p : P - 1) * 4);
            }
        }
    }
    template <int R>
    __device__ __forceinline__ float4 finish(const Batch<R>& b, const Coef& c, int i, int p, int P) const {
        const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
        if (!(c.on && p < P)) return zero;
        float4 v = lift_val4(lv.z ? b.v[i] : zero, lv.s ? b.sv[i] : zero, c.u0, c.u1, c.u2, c.u3);
        if (scale) { v.x = fmaf(v.x, c.s.x, c.t.x); v.y = fmaf(v.y, c.s.y, c.t.y); v.z = fmaf(v.z, c.s.z, c.t.z); v.w = fmaf(v.w, c.s.w, c.t.w); }
        if (relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
        return v;
    }
    __device__ __forceinline__ void prefetch_rows(int p0, int rows, int P) const {   // index / scalar slices; Z itself lives in L2
        if (p0 >= P) return;
        const size_t n = (size_t)min(rows, P - p0);
        if (lv.z) o3d_prefetch_l2(lv.gidx + p0, n * sizeof(int32_t));
        if (lv.s) o3d_prefetch_l2(lv.s + (size_t)p0 * 4, n * 16);
    }
};

struct TcDy {
    const float* g; int ldg; const float* y; int ldy; const float* a; const float* b; const float* cc;
    const float* dpool; const int32_t* sel; int S; int ldp;
    int sh;   // S == 1 << sh (pooling group sizes are powers of two on this path)
    struct Coef { float4 a, b, c; bool on; };
    // raw operand rows of one thread for one k-block: rows p0 + i * stride, i < R (R >= 2).
    // Pooled gradient: when all R rows fall into one pooling group — the usual case, a thread's rows are neighbours — the
    // two [G, ldp] tables are read ONCE (g[0] = dpool entry, g[1] = bit pattern of sel) and the per-row select moves to
    // finish(); selecting inside fetch() would make every row wait for its own table load before the next row's loads go out.
    template <int R> struct Batch { float4 g[R]; float4 y[R]; bool shared; };
    __device__ __forceinline__ Coef prep(int k, int K) const {
        Coef c;
        c.on = k < K;
        c.a = make_float4(1.f, 1.f, 1.f, 1.f);
        c.b = c.c = make_float4(0.f, 0.f, 0.f, 0.f);
        if (c.on && a) { c.a = ld4g(a + k); c.b = ld4g(b + k); c.c = ld4g(cc + k); }
        return c;
    }
    template <int R>
    __device__ __forceinline__ void fetch(Batch<R>& bt, int p0, int stride, int P, int k, int K) const {
        const int kk = k < K ? k : 0;
        bt.shared = false;
        if (dpool) {
            const int pf = p0 < P ? p0 : P - 1;
            const int pe = p0 + (R - 1) * stride;
            const int pl = pe < P ? pe : P - 1;
            if (R >= 2 && (pf >> sh) == (pl >> sh)) {   // the two tables live in g[0], g[1]
                bt.shared = true;
                const size_t go = (size_t)(pf >> sh) * ldp + kk;
                bt.g[0] = ld4g(dpool + go);
                const int4 sl = __ldg(reinterpret_cast<const int4*>(sel + go));
                bt.g[R >= 2 ? 1 : 0] = make_float4(__int_as_float(sl.x), __int_as_float(sl.y), __int_as_float(sl.z), __int_as_float(sl.w));
            } else {
#pragma unroll
                for (int i = 0; i < R; ++i) {
                    const int p = p0 + i * stride, pp = p < P ? p : P - 1;
                    const int s = pp & (S - 1);
                    const size_t go = (size_t)(pp >> sh) * ldp + kk;
                    const int4 sl = __ldg(reinterpret_cast<const int4*>(sel + go));
                    const float4 d = ld4g(dpool + go);
                    bt.g[i] = make_float4(sl.x == s ? d.x : 0.f, sl.y == s ? d.y : 0.f, sl.z == s ? d.z : 0.f, sl.w == s ? d.w : 0.f);
                }
            }
        } else {
#pragma unroll
            for (int i = 0; i < R; ++i) {
                const int p = p0 + i * stride;
                bt.g[i] = ld4g(g + (size_t)(p < P ? p : P - 1) * ldg + kk);
            }
        }
#pragma unroll
        for (int i = 0; i < R; ++i) {
            const int p = p0 + i * stride;
            bt.y[i] = a ? ld4g(y + (size_t)(p < P ? p : P - 1) * ldy + kk) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    }
    template <int R>
    __device__ __forceinline__ float4 finish(const Batch<R>& bt, const Coef& c, int i, int p, int P) const {
        if (!(c.on && p < P)) return make_float4(0.f, 0.f, 0.f, 0.f);
        float4 v = bt.g[i];
        if (bt.shared) {
            const int s = p & (S - 1);
            const float4 d = bt.g[0], sl = bt.g[R >= 2 ? 1 : 0];
            v = make_float4(__float_as_int(sl.x) == s ? d.x : 0.f, __float_as_int(sl.y) == s ? d.y : 0.f,
                            __float_as_int(sl.z) == s ? d.z : 0.f, __float_as_int(sl.w) == s ? d.w : 0.f);
        }
        if (a) {
            const float4 yy = bt.y[i];
            v.x = fmaf(c.a.x, v.x, fmaf(c.c.x, yy.x, c.b.x)); v.y = fmaf(c.a.y, v.y, fmaf(c.c.y, yy.y, c.b.y));
            v.z = fmaf(c.a.z, v.z, fmaf(c.c.z, yy.z, c.b.z)); v.w = fmaf(c.a.w, v.w, fmaf(c.c.w, yy.w, c.b.w));
        }
        return v;
    }
    __device__ __forceinline__ void prefetch_rows(int p0, int rows, int P) const {
        if (p0 >= P) return;
        const size_t n = (size_t)min(rows, P - p0);
        if (!dpool) o3d_prefetch_l2(g + (size_t)p0 * ldg, n * ldg * sizeof(float));
        if (a) o3d_prefetch_l2(y + (size_t)p0 * ldy, n * ldy * sizeof(float));
        if (dpool) {   // the [G, ldp] tables of the groups these rows belong to: without this every k-block of a tile starts
                       // with a cold miss on a new 128-byte line of each table
            const int g0 = p0 >> sh, g1 = (p0 + (int)n - 1) >> sh;
            const size_t bytes = (size_t)(g1 - g0 + 1) * ldp * sizeof(float);
            o3d_prefetch_l2(dpool + (size_t)g0 * ldp, bytes);
            o3d_prefetch_l2(sel + (size_t)g0 * ldp, bytes);
        }
    }
};

// BF16 operands (o3d_stack_t.precision 1, inference, and 2, training): the same loader, its transformed rows rounded to bf16
// (cvt.rn) where the 3xTF32 path splits them into hi / lo; the kernel then stores one bf16 image per stage and issues 2 wgmma
// k16 per 32-wide k-block.  A wrapper type rather than a flag, so that each precision is its own instantiation with no runtime
// branch in the hot loop.
template <class L> struct Bf16 : L {};
template <class L> struct is_bf16 { static constexpr bool value = false; };
template <class L> struct is_bf16<Bf16<L>> { static constexpr bool value = true; };
template <class L> struct is_lift { static constexpr bool value = std::is_same<L, TcLift>::value; };
template <class L> struct is_lift<Bf16<L>> { static constexpr bool value = is_lift<L>::value; };

// ---- epilogues: thread = one output channel `ch`, called once per 32-position column group ------------------
// LD: compile-time row stride of y (0 = use the runtime ldy)
template <int LD>
struct TcFwdEpi {
    float* y; int ldy; const float* bias; double* sum; double* sumsq;
    int S, log2S; float* ymax; float* ymin; int32_t* arg; int ldp;
    // per-thread running state (fp32 inside a 32-position group, fp64 across groups and tiles)
    float bv, mx, mn; int ax, an; double d1, d2;
    __device__ __forceinline__ void begin(int ch, int Nw) {
        d1 = d2 = 0.0;
        bv = (bias && ch < Nw) ? bias[ch] : 0.f;
        mx = -INFINITY; mn = INFINITY; ax = an = 0;
    }
    __device__ __forceinline__ void prefetch(int, int, int, int) {}
    __device__ __forceinline__ const int32_t* lift_gidx() const { return nullptr; }
    __device__ __forceinline__ const float* lift_s() const { return nullptr; }
    __device__ __forceinline__ void set_tile(const int32_t*, const float4*) {}
    // Fast path = a full group of 16 positions that lies inside one pooling group (S >= 16, the set-abstraction case):
    // no per-element range or group-boundary test, the max / min / first-arg scan is local to the 16 values and is merged
    // into the running (mx, ax, mn, an) of the pooling group with two compares.  Everything else takes the element-wise path.
    __device__ __forceinline__ void group(const uint32_t (&r)[16], int ch, int Nw, int pbase, int P) {
        if (ch >= Nw) return;
        float s1 = 0.f, s2 = 0.f;
        const int smask = S - 1;
        float* yp = y ? y + (size_t)pbase * ldy + ch : nullptr;
        if (pbase + 16 <= P && (S == 0 || S >= 16)) {
            float v[16];
#pragma unroll
            for (int j = 0; j < 16; ++j) v[j] = __uint_as_float(r[j]) + bv;
            if (yp) {
                const size_t st = LD ? (size_t)LD : (size_t)ldy;   // compile-time stride -> immediate store offsets
#pragma unroll
                for (int j = 0; j < 16; ++j) yp[j * st] = v[j];
            }
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                s1 += v[j];
                s2 = fmaf(v[j], v[j], s2);
            }
            if (S > 0) {
                float gm = v[0], gn = v[0];
                int ga = 0, gb = 0;
#pragma unroll
                for (int j = 1; j < 16; ++j) {
                    if (v[j] > gm) { gm = v[j]; ga = j; }
                    if (v[j] < gn) { gn = v[j]; gb = j; }
                }
                const int s0 = pbase & smask;
                if (s0 == 0) { mx = gm; ax = ga; mn = gn; an = gb; }
                else {
                    if (gm > mx) { mx = gm; ax = s0 + ga; }
                    if (gn < mn) { mn = gn; an = s0 + gb; }
                }
                if (s0 + 16 == S) {
                    const size_t o = (size_t)(pbase >> log2S) * ldp + ch;
                    ymax[o] = mx; ymin[o] = mn; arg[o] = ax | (an << 16);
                }
            }
        } else {
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                if (pbase + j >= P) break;
                const float v = __uint_as_float(r[j]) + bv;
                if (yp) yp[(size_t)j * ldy] = v;
                s1 += v;
                s2 = fmaf(v, v, s2);
                if (S > 0) {
                    const int s = (pbase + j) & smask;
                    if (s == 0) { mx = -INFINITY; mn = INFINITY; ax = an = 0; }
                    if (v > mx) { mx = v; ax = s; }
                    if (v < mn) { mn = v; an = s; }
                    if (s == smask) {
                        const size_t o = (size_t)((pbase + j) >> log2S) * ldp + ch;
                        ymax[o] = mx; ymin[o] = mn; arg[o] = ax | (an << 16);
                    }
                }
            }
        }
        d1 += (double)s1;
        d2 += (double)s2;
    }
    __device__ __forceinline__ void end(int ch, int Nw) {
        if (sum && ch < Nw) {
            atomicAdd(sum + ch, d1);
            atomicAdd(sumsq + ch, d2);
        }
    }
};

// LD: compile-time row stride shared by out and yprev (0 = use the runtime ldo / ldyp)
// LIFT: the previous layer is a lifted one (its raw output is re-evaluated from Z / s.u); a separate instantiation so that the
// ordinary dgrad kernels carry none of its state
template <int LD, bool LIFT = false>
struct TcDgradEpi {
    float* out; int ldo; const float* yprev; int ldyp; const float* scale; const float* shift; int relu;
    double* s1g; double* s2y;
    LiftView lv;             // lv.z / lv.s set: the previous layer's raw output is the lifted Y0 (re-evaluated, never stored)
    float sc, sh; double d1, d2;
    float yv[16];
    float u0, u1, u2, u3; const int32_t* gs; const float4* ss;   // lifted: this thread's u[j][ch]; the tile's gidx / s slices staged in shared memory
    __device__ __forceinline__ bool lifted() const { return LIFT; }
    __device__ __forceinline__ void begin(int ch, int Nw) {
        d1 = d2 = 0.0;
        sc = (scale && ch < Nw) ? scale[ch] : 1.f;
        sh = (shift && ch < Nw) ? shift[ch] : 0.f;
        if constexpr (LIFT) {
            const bool on = lv.u && ch < Nw;
            u0 = on ? lv.u[ch] : 0.f; u1 = on ? lv.u[lv.ldz + ch] : 0.f; u2 = on ? lv.u[2 * lv.ldz + ch] : 0.f; u3 = on ? lv.u[3 * lv.ldz + ch] : 0.f;
            gs = nullptr;
        }
    }
    __device__ __forceinline__ const int32_t* lift_gidx() const { return LIFT ? lv.gidx : nullptr; }
    __device__ __forceinline__ const float* lift_s() const { return LIFT ? lv.s : nullptr; }
    __device__ __forceinline__ void set_tile(const int32_t* g, const float4* s4) { if constexpr (LIFT) { gs = g; ss = s4; } }
    // lifted yprev: `col` = first column of the group inside the tile (index into the staged gidx slice)
    __device__ __forceinline__ void prefetch_lift(int ch, int pbase, int col, int P) {
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            const float z = lv.z ? __ldg(lv.z + (size_t)gs[col + j] * lv.ldz + ch) : 0.f;
            const float4 sv = lv.s ? ss[col + j] : make_float4(0.f, 0.f, 0.f, 0.f);
            yv[j] = lift_val(z, sv, u0, u1, u2, u3);
        }
    }
    // (an L2 prefetch of these rows one tile ahead was measured: 7-15 % slower, it competes with the loader's own window)
    // issue the previous layer's raw outputs for this column group before reading the staged accumulators (independent loads)
    __device__ __forceinline__ void prefetch(int ch, int Nw, int pbase, int P) {
        if (ch >= Nw) return;
        if constexpr (LIFT) { prefetch_lift(ch, pbase, pbase & (TC_N - 1), P); return; }
        if (!yprev) return;
        if (pbase + 16 <= P) {
            const float* yp = yprev + (size_t)pbase * ldyp + ch;
            const size_t st = LD ? (size_t)LD : (size_t)ldyp;
#pragma unroll
            for (int j = 0; j < 16; ++j) yv[j] = __ldg(yp + j * st);
        } else {
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const int pj = min(pbase + j, P - 1);      // clamped: the load is unconditional, group() masks by range
                yv[j] = __ldg(yprev + (size_t)pj * ldyp + ch);
            }
        }
    }
    __device__ __forceinline__ void group(const uint32_t (&r)[16], int ch, int Nw, int pbase, int P) {
        if (ch >= Nw) return;
        float s1 = 0.f, s2 = 0.f;
        float* op = out + (size_t)pbase * ldo + ch;
        if (pbase + 16 <= P) {          // full group: no per-element range test
            float v[16];
#pragma unroll
            for (int j = 0; j < 16; ++j) v[j] = __uint_as_float(r[j]);
            if (yprev || lifted()) {
                if (relu) {
#pragma unroll
                    for (int j = 0; j < 16; ++j) v[j] = fmaf(yv[j], sc, sh) > 0.f ? v[j] : 0.f;
                }
#pragma unroll
                for (int j = 0; j < 16; ++j) s2 = fmaf(v[j], yv[j], s2);
            }
            const size_t st = LD ? (size_t)LD : (size_t)ldo;       // compile-time stride -> immediate store offsets
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                s1 += v[j];
                op[j * st] = v[j];
            }
        } else {
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                if (pbase + j >= P) break;
                float v = __uint_as_float(r[j]);
                if (yprev || lifted()) {
                    if (relu && !(fmaf(yv[j], sc, sh) > 0.f)) v = 0.f;
                    s2 = fmaf(v, yv[j], s2);
                }
                s1 += v;
                op[(size_t)j * ldo] = v;
            }
        }
        d1 += (double)s1;
        d2 += (double)s2;
    }
    __device__ __forceinline__ void end(int ch, int Nw) {
        if (s1g && ch < Nw) {
            atomicAdd(s1g + ch, d1);
            atomicAdd(s2y + ch, d2);
        }
    }
};

// ------------------------------------------------------------------------------------------------------------
// pw_tc_kernel: one persistent CTA per SM and 128-channel tile; every role walks the same static sequence of 128-position
// tiles.  512 threads = 16 warps:
//   warps 0-3, 4-7  two consumer warpgroups.  Warpgroup h multiplies positions h*64 .. h*64+63 of the tile by the 128
//                   channels of the weight tile (wgmma m64n128k8, 3xTF32: 12 per k-block, accumulators in registers),
//                   stages the result in shared memory as [channel][position] and runs the epilogue on it: thread = one
//                   output channel walking 64 positions in groups of 16, so the batch statistics, the group max/min/arg and
//                   the ReLU-mask sums are plain per-thread loops and every global store of a warp is one coalesced line
//   warps 8-15      operand producers (256 threads, 4 neighbouring rows each): coalesced 16-byte loads issued one k-block
//                   ahead ("raw-first"), transform, hi/lo split, 128B-swizzled st.shared, fence.proxy.async, arrive.
//                   Producer thread 0 also streams the stage's pre-tiled, pre-swizzled weight image (hi|lo, 32 KB per k-block,
//                   written once per call by stack.cu's pack kernel) with cp.async.bulk onto the stage's "full" barrier, and
//                   asks for the next position tile's rows with cp.async.bulk.prefetch.L2.  (A 17th warp for that would
//                   cap every thread at 96 registers and make the consumers spill.)
// Shared memory: 2 stages x (Whi | Wlo | Xhi | Xlo, 64 KB) + 2 x 34 KB epilogue staging + barriers / lifted slices = 202 KB.
constexpr int TC_STAGES = 2;
constexpr int TC_STAGE_BYTES = 4 * TILE_BYTES;         // Whi | Wlo | Xhi | Xlo
constexpr int TC_EPI_LD = 68;                          // floats per staged channel row: 64 positions + 4 (no bank conflicts
                                                       // for the accumulator stores nor for the epilogue's float4 reads)
constexpr int TC_EPI_BYTES = TC_M * TC_EPI_LD * 4;     // one warpgroup's staging
constexpr int TC_THREADS = 512;
constexpr int TC_SMEM = TC_STAGES * TC_STAGE_BYTES + 2 * TC_EPI_BYTES + 1024 + 256 + 1024 + 4096;   // + alignment | barriers |
                                                                                                    //   gidx + s slices (lifted dgrad)

// accumulators of one warpgroup (m64 x N, rows = positions, columns = channels) -> stg[channel * TC_EPI_LD + position]
template <int R>
__device__ __forceinline__ void stage_acc(const float (&acc)[R], float* stg, int ld) {
    const int w = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
#pragma unroll
    for (int i = 0; i < R; ++i) {
        const int row = 16 * w + (lane >> 2) + 8 * ((i >> 1) & 1), col = 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
        stg[col * ld + row] = acc[i];
    }
}

template <class BLoad, class Epi>
__global__ void __launch_bounds__(TC_THREADS, 1)
    pw_tc_kernel(BLoad bl, const uint8_t* __restrict__ wtiles, int P, int K, int Nw, int nkb, Epi epi, int rev) {
    constexpr bool BF = is_bf16<BLoad>::value;
    constexpr int WBYTES = BF ? BF_TILE_BYTES : 2 * TILE_BYTES;   // weight image per (channel tile, k-block)
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint8_t* tail = smem + TC_STAGES * TC_STAGE_BYTES + 2 * TC_EPI_BYTES;
    uint64_t* full = reinterpret_cast<uint64_t*>(tail);      // [STAGES]  producers (+ weight copy) -> consumers
    uint64_t* empty = full + TC_STAGES;                       // [STAGES]  consumers (lane 0 of each of the 8 warps) -> producers

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int mt0 = blockIdx.y;                   // 128-channel tile of this CTA
    const int n_ptiles = (P + TC_N - 1) / TC_N;
    // `rev`: walk the position tiles from the last to the first.  Consecutive layers alternate the direction, so a layer
    // starts on the part of its input that the previous kernel touched last and that is still resident in the 50 MB L2.
    auto tile_of = [&](int t) { return rev ? n_ptiles - 1 - t : t; };

    if (threadIdx.x == 0) {
        for (int s = 0; s < TC_STAGES; ++s) {
            o3d_mbar_init(full + s, 256 + 1);
            o3d_mbar_init(empty + s, 8);
        }
        o3d_fence_mbar_init();
    }
    __syncthreads();

    if (warp < 8) {
        // ===================================================== consumers: wgmma + epilogue (2 warpgroups)
        const int h = warp >> 2;                      // warpgroup: positions h*64 .. h*64+63 of each tile
        const int tw = threadIdx.x & 127;
        const int ch = mt0 * TC_M + tw;
        float* stg = reinterpret_cast<float*>(smem + TC_STAGES * TC_STAGE_BYTES + h * TC_EPI_BYTES);
        int32_t* gsm = reinterpret_cast<int32_t*>(tail + 256);           // [2][TC_N] row indices
        float4* ssm = reinterpret_cast<float4*>(tail + 256 + 1024);      // [2][TC_N] per-position scalars
        epi.begin(ch, Nw);
        int stage = 0, phase = 0, buf = 0;
        for (int t = blockIdx.x; t < n_ptiles; t += gridDim.x) {
            const int pt0 = tile_of(t) * TC_N;
            {
                // lifted previous layer: stage the tile's 128 row indices (warpgroup 0) and per-position scalars (warpgroup 1)
                // once, both read them; the named barrier of tile t+1 orders the re-use of the slices by tile t+2
                const int32_t* gi = epi.lift_gidx();
                const float* si = epi.lift_s();
                if (gi || si) {
                    const int pp = min(pt0 + tw, P - 1);
                    if (gi && h == 0) gsm[buf * TC_N + tw] = __ldg(gi + pp);
                    if (si && h == 1) ssm[buf * TC_N + tw] = ld4g(si + (size_t)pp * 4);
                    asm volatile("bar.sync 1, 256;" ::: "memory");
                    epi.set_tile(gsm + buf * TC_N, ssm + buf * TC_N);
                }
            }
            const int pb = pt0 + h * 64;
            epi.prefetch(ch, Nw, pb, P);
            float acc[64];
#pragma unroll
            for (int i = 0; i < 64; ++i) acc[i] = 0.f;
            for (int kb = 0; kb < nkb; ++kb) {
                o3d_mbar_wait(full + stage, phase);
                const uint32_t sb = o3d_smem_u32(smem + stage * TC_STAGE_BYTES);
                wgmma_fence_acc(acc);
                wgmma_fence();
                if constexpr (BF) {
                    const uint32_t xb = sb + 2 * TILE_BYTES + h * (BF_TILE_BYTES / 2);
                    wgmma_bf16_kblock<128>(acc, make_desc_sw64(xb), make_desc_sw64(sb), kb == 0);
                } else {
                    const uint32_t xb = sb + 2 * TILE_BYTES + h * (TILE_BYTES / 2);    // rows h*64.. of the activation tile
                    wgmma_3xtf32_kblock<128>(acc, make_desc(xb), make_desc(xb + TILE_BYTES), make_desc(sb), make_desc(sb + TILE_BYTES),
                                             kb == 0);
                }
                wgmma_commit();
                wgmma_wait<0>();
                wgmma_fence_acc(acc);
                if (lane == 0) o3d_mbar_arrive(empty + stage);
                if (++stage == TC_STAGES) { stage = 0; phase ^= 1; }
            }
            asm volatile("bar.sync %0, 128;" ::"r"(2 + h) : "memory");     // the previous tile's epilogue is done with stg
            stage_acc(acc, stg, TC_EPI_LD);
            asm volatile("bar.sync %0, 128;" ::"r"(2 + h) : "memory");
            const float* row = stg + tw * TC_EPI_LD;
#pragma unroll 1
            for (int cg = 0; cg < 4; ++cg) {
                uint32_t r[16];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float4 v = *reinterpret_cast<const float4*>(row + cg * 16 + 4 * j);
                    r[4 * j] = __float_as_uint(v.x); r[4 * j + 1] = __float_as_uint(v.y);
                    r[4 * j + 2] = __float_as_uint(v.z); r[4 * j + 3] = __float_as_uint(v.w);
                }
                epi.group(r, ch, Nw, pb + cg * 16, P);
                if (cg + 1 < 4) epi.prefetch(ch, Nw, pb + (cg + 1) * 16, P);
            }
            buf ^= 1;
        }
        epi.end(ch, Nw);
    } else {
        // ===================================================== activation-operand producers (8 warps, 256 threads)
        // Per k-block: [raw rows of kb already in registers] -> wait for the stage -> transform, hi/lo split, swizzled
        // st.shared -> fence + arrive -> issue the raw loads of kb+1 (all back to back, nothing depends on them until
        // the next iteration, so they fly while the consumers work through the stages ahead).
        const int pt = (warp - 8) * 32 + lane;            // 0..255
        const int chunk = pt & 7;                         // 16-byte chunk (4 channels) inside the 128-byte row
        const int row0 = (pt >> 3) * 4;                   // 4 neighbouring rows row0 + i, i < 4 (one pooling group)
        int stage = 0, phase = 0;
        // The (tile, k-block) nest is walked as one flat sequence of items so that the raw loads of the item ahead — also
        // when it belongs to the next position tile — are in flight while the current one is being stored.
        struct Cur { int t, kb, p0; };
        auto advance = [&](Cur& c) {
            if (++c.kb == nkb) {
                c.kb = 0;
                c.t += gridDim.x;
                if (c.t < n_ptiles) c.p0 = tile_of(c.t) * TC_N;
            }
        };
        using Batch4 = typename BLoad::template Batch<4>;
        auto issue = [&](Batch4& r, typename BLoad::Coef& cf, const Cur& c) {
            if (c.t >= n_ptiles) return;
            const int k = c.kb * TC_K + chunk * 4;
            cf = bl.prep(k, K);
            bl.fetch(r, c.p0 + row0, 1, P, k, K);
        };
        Cur c0{(int)blockIdx.x, 0, 0};
        if (c0.t < n_ptiles) c0.p0 = tile_of(c0.t) * TC_N;
        Batch4 r0{};      // value-initialised: TcLift keeps a look-ahead tag in the batch
        typename BLoad::Coef f0 = bl.prep(chunk * 4, K);
        issue(r0, f0, c0);
        if (pt == 0 && c0.t < n_ptiles) bl.prefetch_rows(c0.p0, TC_N, P);
        while (c0.t < n_ptiles) {
            o3d_mbar_wait(empty + stage, phase ^ 1);
            if (pt == 0) {
                o3d_mbar_expect_tx(full + stage, WBYTES);
                o3d_bulk_g2s(smem + stage * TC_STAGE_BYTES, wtiles + ((size_t)mt0 * nkb + c0.kb) * WBYTES, WBYTES, full + stage);
                const int tn = c0.t + (int)gridDim.x;
                if (c0.kb == 0 && tn < n_ptiles) bl.prefetch_rows(tile_of(tn) * TC_N, TC_N, P);   // next tile of this CTA -> L2
            }
            uint8_t* xhi = smem + stage * TC_STAGE_BYTES + 2 * TILE_BYTES;
            uint8_t* xlo = xhi + TILE_BYTES;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float4 v = bl.finish(r0, f0, i, c0.p0 + row0 + i, P);
                if constexpr (BF) {
                    *reinterpret_cast<uint2*>(xhi + sw64(row0 + i, chunk >> 1) + (chunk & 1) * 8) = pack_bf16x4(v);
                } else {
                    const uint32_t off = sw128(row0 + i, chunk);
                    *reinterpret_cast<float4*>(xhi + off) = hi_part(v);
                    *reinterpret_cast<float4*>(xlo + off) = lo_part(v);
                }
            }
            o3d_fence_proxy_async();              // generic-proxy stores -> visible to the tensor core (async proxy)
            o3d_mbar_arrive(full + stage);
            if (++stage == TC_STAGES) { stage = 0; phase ^= 1; }
            advance(c0);
            issue(r0, f0, c0);
        }
    }
}

// ------------------------------------------------------------------------------------------------------------
// wgrad on the tensor core:  dW[m, n] += sum_p dY[p, m] * X[p, n]  over this CTA's slice of positions, one 128 x 128 tile
// of dW per CTA.  Both operands are position-major in global memory (channels contiguous) while wgmma takes tf32 operands
// K-major only, K being the position here.  Per 32-position k-block a stage holds
//   dY      as it comes, unsplit: rows = positions, 4 SWIZZLE_128B sub-images of 32 channels (WG_DY_SUB bytes each), written
//           with 16-byte stores.  The consumers read their A fragments (dY^T) from it with ld.shared, split them into hi / lo
//           in registers and issue register-fed MMAs (wgmma_tf32_rs_n128), so only B is read by the tensor core from shared
//           memory;
//   X^T     hi | lo, [128 channels x 32 positions] K-major SWIZZLE_128B tiles written by store_transposed (16-byte stores of
//           a 4 x 4 block transposed in registers).
//   warps 0-3, 4-7  consumers: warpgroup h accumulates rows m0 + h*64 .. of the tile (wgmma m64n128k8, 3xTF32), then writes
//                   its partial tile: plain stores into the split-K workspace part[split][m][n] (summed in a fixed order by
//                   wgrad_reduce_kernel: deterministic)
//   warps 8-15      producers: each thread owns 4 channels x 4 consecutive positions of each operand per k-block; producer
//                   thread 0 also keeps the L2 prefetch of the slice's rows WG_AHEAD k-blocks ahead of the stores (requesting
//                   the whole slice up front asks for more than the L2 holds across the grid, and the lines are evicted again
//                   before their k-block comes up)
// Shared memory: 4 stages x (dY 16 KB | X^T hi 16 KB | X^T lo 16 KB) (BF16: 3 stages x 64 KB) + alignment | barriers.
constexpr int WG_STAGES = 4;                           // 3xTF32
constexpr int WG_STAGE_BYTES = 3 * TILE_BYTES;
constexpr int WG_DY_SUB = TC_K * 128;                  // 4 KB: 32 positions x 32 channels of dY
constexpr int WG_BF_STAGES = 3;                        // BF16
constexpr int WG_BF_STAGE_BYTES = 4 * TILE_BYTES;
constexpr int WG_AHEAD = 4;
constexpr int WG_THREADS = 512;
constexpr int WG_SMEM = WG_STAGES * WG_STAGE_BYTES + 1024 + 256;
static_assert(WG_BF_STAGES * WG_BF_STAGE_BYTES == WG_STAGES * WG_STAGE_BYTES, "both precisions use one shared-memory size");
// 3xTF32: each role declares its register bound (setmaxnreg) where the roles part.  The bound is the launch's own 128 per
// thread, so nothing moves between the warpgroups, but ptxas then allocates the consumer and producer code separately:
// without it the lifted instantiation's producers spill (32 bytes) although each role fits in 128 registers on its own.
// A 120 / 136 split makes the consumers spill inside the MMA loop, and ptxas then serialises the wgmmas.
constexpr int WG_REGS = 128;

// X^T of one thread: positions p_first + 4 q .. p_first + 4 q + 3 (rows i of `raw`) x channels c_local .. c_local + 3 of a
// [channels x 32 positions] K-major SWIZZLE_128B tile (element (c, p) at sw128(c, p / 4) + 4 (p % 4); hi at `hi`, lo
// TILE_BYTES on).  The 4 x 4 block is transposed in registers, so each channel's 4 positions are one 16-byte chunk: 4
// st.shared.v4 per half.  Channel c's chunk lands in bank group q ^ (c & 7): the 8 lanes of a quarter-warp, same channels
// and q = 0 .. 7, hit 8 distinct groups.
template <class L>
__device__ __forceinline__ void store_transposed(const L& ld, const typename L::template Batch<4>& raw, const typename L::Coef& cf,
                                                 uint8_t* hi, int c_local, int p_first, int q, int pend) {
    float4 v[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) v[i] = ld.finish(raw, cf, i, p_first + 4 * q + i, pend);
    const float4 col[4] = {make_float4(v[0].x, v[1].x, v[2].x, v[3].x), make_float4(v[0].y, v[1].y, v[2].y, v[3].y),
                           make_float4(v[0].z, v[1].z, v[2].z, v[3].z), make_float4(v[0].w, v[1].w, v[2].w, v[3].w)};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const uint32_t off = sw128(c_local + j, q);
        *reinterpret_cast<float4*>(hi + off) = hi_part(col[j]);
        *reinterpret_cast<float4*>(hi + TILE_BYTES + off) = lo_part(col[j]);
    }
}

// BF16 (XB = Bf16<...>): no transpose.  The producers store both operands' rows position-major into the 64-byte-swizzle image
// of the forward path, dY at the stage's start and X WG_BF_X bytes on, each as four 32-channel sub-images of 32 positions
// (WG_BF_SUB bytes apart); the consumers read them MN-major (wgmma_bf16_tt_*, make_desc_sw64_mn): 2 k16 MMAs per k-block.
constexpr int WG_BF_SUB = TC_K * TC_BF_ROW;             // 2 KB: 32 positions x 32 channels
constexpr int WG_BF_X = 4 * WG_BF_SUB;

template <class L>
__device__ __forceinline__ void store_rows_bf16(const L& ld, const typename L::template Batch<4>& raw, const typename L::Coef& cf,
                                                uint8_t* img, int sub, int c_local, int p_first, int prow0, int pend) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int pl = prow0 + 8 * i;
        st_bf16_row4(img, sub, pl, c_local, ld.finish(raw, cf, i, p_first + pl, pend));
    }
}

template <class XB>
__global__ void __launch_bounds__(WG_THREADS, 1)
    pw_wgrad_tc_kernel(TcDy da, XB xb, int P, int M, int N, int chunk, float* __restrict__ part) {
    constexpr bool BF = is_bf16<XB>::value;
    constexpr int STAGES = BF ? WG_BF_STAGES : WG_STAGES;
    constexpr int STAGE_BYTES = BF ? WG_BF_STAGE_BYTES : WG_STAGE_BYTES;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
    uint64_t* empty = full + STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int m0 = blockIdx.z * TC_M, n0 = blockIdx.y * TC_N;
    // every split owns one contiguous slice of positions (DRAM-friendly)
    const int pbeg = blockIdx.x * chunk, pend = min(P, pbeg + chunk);
    const int nkb = pend > pbeg ? (pend - pbeg + TC_K - 1) / TC_K : 0;
    auto kpos = [&](int i) { return pbeg + i * TC_K; };

    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) {
            o3d_mbar_init(full + s, 256);
            o3d_mbar_init(empty + s, 8);
        }
        o3d_fence_mbar_init();
    }
    __syncthreads();

    if (warp < 8) {
        if constexpr (!BF) asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(WG_REGS));
        const int h = warp >> 2, w = warp & 3;
        float acc[64];
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[i] = 0.f;
        int stage = 0, phase = 0;
        for (int kb = 0; kb < nkb; ++kb) {
            o3d_mbar_wait(full + stage, phase);
            const uint32_t sb = o3d_smem_u32(smem + stage * STAGE_BYTES);
            if constexpr (BF) {
                wgmma_fence_acc(acc);
                wgmma_fence();
                const uint32_t ab = sb + h * 2 * WG_BF_SUB;                   // dY channels m0 + h*64 .. : sub-images 2h, 2h+1
#pragma unroll
                for (int ks = 0; ks < 2; ++ks)
                    wgmma_bf16_tt_n128(acc, make_desc_sw64_mn(ab + ks * 1024, WG_BF_SUB),
                                       make_desc_sw64_mn(sb + WG_BF_X + ks * 1024, WG_BF_SUB), (kb == 0 && ks == 0) ? 0u : 1u);
                wgmma_commit();
                wgmma_wait<0>();
                wgmma_fence_acc(acc);
            } else {
                // A = dY^T fragments of the 4 k-steps: rows (channels) h*64 + 16 w + lane / 4 (+ 8), i.e. sub-image 2 h + w / 2,
                // columns (positions) 8 ks + lane % 4 (+ 4); split into hi / lo here, as the producers split X^T
                const uint8_t* dyk = smem + stage * STAGE_BYTES + (2 * h + (w >> 1)) * WG_DY_SUB;
                const int mc = (16 * w + (lane >> 2)) & 31;
                uint32_t ahi[4][4], alo[4][4];
#pragma unroll
                for (int ks = 0; ks < TC_K / 8; ++ks) {
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const int p = ks * 8 + (lane & 3) + 4 * (i >> 1), m = mc + 8 * (i & 1);
                        const float x = *reinterpret_cast<const float*>(dyk + sw128(p, m >> 2) + 4 * (m & 3));
                        const float xh = hi1(x);
                        ahi[ks][i] = __float_as_uint(xh);
                        alo[ks][i] = __float_as_uint(x - xh);
                    }
                }
                const uint64_t bhi = make_desc(sb + TILE_BYTES), blo = make_desc(sb + 2 * TILE_BYTES);
                wgmma_fence_acc(acc);
                wgmma_fence();
#pragma unroll
                for (int ks = 0; ks < TC_K / 8; ++ks) {      // Alo.Bhi + Ahi.Blo + Ahi.Bhi, as wgmma_3xtf32_kblock
                    const uint64_t adv = (uint64_t)((ks * 32) >> 4);
                    wgmma_tf32_rs_n128(acc, alo[ks], bhi + adv, (kb == 0 && ks == 0) ? 0u : 1u);
                    wgmma_tf32_rs_n128(acc, ahi[ks], blo + adv, 1u);
                    wgmma_tf32_rs_n128(acc, ahi[ks], bhi + adv, 1u);
                }
                wgmma_commit();
                wgmma_wait<0>();
                wgmma_fence_acc(acc);
#pragma unroll
                for (int ks = 0; ks < TC_K / 8; ++ks) {
                    wgmma_fence_frag(ahi[ks]);
                    wgmma_fence_frag(alo[ks]);
                }
            }
            // after the wait: the stage's dY image (read into the fragments) and X^T (read by the MMAs) are free again
            if (lane == 0) o3d_mbar_arrive(empty + stage);
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
        const int Mt = TC_M * (int)gridDim.z, Nt = TC_N * (int)gridDim.y;
        float* __restrict__ out = part + (size_t)blockIdx.x * Mt * Nt;
#pragma unroll
        for (int i = 0; i < 64; i += 4) {
#pragma unroll
            for (int rr = 0; rr < 2; ++rr) {
                const int m = m0 + h * 64 + 16 * w + (lane >> 2) + 8 * rr, n = n0 + 8 * (i >> 2) + 2 * (lane & 3);
                // zeros when the slice is empty
                *reinterpret_cast<float2*>(out + (size_t)m * Nt + n) = make_float2(acc[i + 2 * rr], acc[i + 2 * rr + 1]);
            }
        }
    } else {
        if constexpr (!BF) asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(WG_REGS));
        // producers, thread = 4 channels x 4 positions of each operand per k-block
        //   3xTF32  dY: rows 4 pw .. 4 pw + 3 x channels 4 lane .. (16-byte row stores, a quarter-warp covers one 128-byte
        //           row of a sub-image); X: positions 4 (lane % 8) .. + 3 x channels 4 c4 .. (see store_transposed)
        //   BF16    both operands: channels 4 c4 .., positions prow0 + 8 i, i < 4
        const int pw = warp - 8;
        const int c4 = BF ? pw * 4 + (lane & 3) : pw * 4 + (lane >> 3), prow0 = lane >> 2;
        const int ca = BF ? c4 : lane, pa = BF ? prow0 : 4 * pw;              // dY channel quad, first row
        const int qx = lane & 7, px = BF ? prow0 : 4 * qx;                      // X first row
        constexpr int RS = BF ? 8 : 1;                                         // row stride of both operands
        const bool pt0 = pw == 0 && lane == 0;
        TcDy::Batch<4> ra = {};
        typename XB::template Batch<4> rb = {};
        auto fetch = [&](int kb) {
            da.fetch(ra, kpos(kb) + pa, RS, pend, m0 + ca * 4, M);
            xb.fetch(rb, kpos(kb) + px, RS, pend, n0 + c4 * 4, N);
        };
        auto prefetch = [&](int kb) {
            if (pt0 && kb < nkb) {
                da.prefetch_rows(kpos(kb), TC_K, pend);
                xb.prefetch_rows(kpos(kb), TC_K, pend);
            }
        };
        int stage = 0, phase = 0;
        for (int kb = 0; kb < WG_AHEAD; ++kb) prefetch(kb);
        if (nkb > 0) fetch(0);
        for (int kb = 0; kb < nkb; ++kb) {
            prefetch(kb + WG_AHEAD);
            o3d_mbar_wait(empty + stage, phase ^ 1);
            uint8_t* sbase = smem + stage * STAGE_BYTES;
            // the per-channel coefficients are re-read (L1-resident) per k-block: kept live across the loop they push the
            // lifted operand's producer past its register budget
            if constexpr (BF) {
                store_rows_bf16(da, ra, da.prep(m0 + c4 * 4, M), sbase, WG_BF_SUB, c4 * 4, kpos(kb), prow0, pend);
                store_rows_bf16(xb, rb, xb.prep(n0 + c4 * 4, N), sbase + WG_BF_X, WG_BF_SUB, c4 * 4, kpos(kb), prow0, pend);
            } else {
                const TcDy::Coef cf = da.prep(m0 + ca * 4, M);
                uint8_t* dy = sbase + (ca >> 3) * WG_DY_SUB;
#pragma unroll
                for (int i = 0; i < 4; ++i)
                    *reinterpret_cast<float4*>(dy + sw128(pa + i, ca & 7)) = da.finish(ra, cf, i, kpos(kb) + pa + i, pend);
                store_transposed(xb, rb, xb.prep(n0 + c4 * 4, N), sbase + TILE_BYTES, c4 * 4, kpos(kb), qx, pend);
            }
            o3d_fence_proxy_async();
            o3d_mbar_arrive(full + stage);
            if (kb + 1 < nkb) fetch(kb + 1);
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
    }
}

// dW[m, n] (+)= sum over splits of part[s][m][n]   (Mt x Nt partial tiles -> the M x N corner of dW)
// 8 lanes share one float4 of output (each sums every 8th split, then a 3-step shuffle tree): 8x more loads in flight.
__global__ void __launch_bounds__(256)
    wgrad_reduce_kernel(const float* __restrict__ part, int splits, int Mt, int Nt, int M, int N, float* __restrict__ dW,
                        int lddw) {
    const int sub = threadIdx.x & 7;
    const int n4 = (blockIdx.x * 32 + (threadIdx.x >> 3)) * 4, m = blockIdx.y;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (n4 < N && m < M) {
        const float* p = part + (size_t)m * Nt + n4;
        for (int s = sub; s < splits; s += 8) {
            const float4 v = __ldg(reinterpret_cast<const float4*>(p + (size_t)s * Mt * Nt));
            acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
        }
    }
#pragma unroll
    for (int o = 4; o >= 1; o >>= 1) {
        acc.x += __shfl_xor_sync(0xFFFFFFFFu, acc.x, o); acc.y += __shfl_xor_sync(0xFFFFFFFFu, acc.y, o);
        acc.z += __shfl_xor_sync(0xFFFFFFFFu, acc.z, o); acc.w += __shfl_xor_sync(0xFFFFFFFFu, acc.w, o);
    }
    if (sub == 0 && n4 < N && m < M) {
        float* o = dW + (size_t)m * lddw + n4;
        o[0] += acc.x;
        if (n4 + 1 < N) o[1] += acc.y;
        if (n4 + 2 < N) o[2] += acc.z;
        if (n4 + 3 < N) o[3] += acc.w;
    }
}

// ------------------------------------------------------------------------------------------------------------
// pw_bwd_tc_kernel: both gradients of one narrow layer (Cout = M and Cin = N in {64, 128}) in one persistent walk over
// 64-position tiles, so that every byte the two GEMMs share — dY's g / dpool / y rows and the layer input X — leaves HBM once:
//   dgrad  out[p, n] = sum_m dY[p, m] Wt[n, m]   (TcDgradEpi: ReLU mask, BN-backward sums, coalesced stores)
//   wgrad  dW[m, n] += sum_p dY[p, m] X[p, n]    (accumulated in registers over the CTA's tiles, written once to
//                                                 part[blockIdx.x] and summed in split order by wgrad_reduce_kernel)
// wgmma takes tf32 operands K-major only, and the two GEMMs contract dY along different axes.  dY is stored once, as dgrad's
// operand (rows = positions, m contiguous, hi | lo); wgrad's A operand dY^T is read from that image into registers in the
// wgmma fragment layout (wgmma_tf32_rs_*), and X^T is the producers' transposed store (store_transposed), as in
// pw_wgrad_tc_kernel.  Every value fed to an MMA is the loaders' finish() output split as the two-kernel path splits it.
//   warps 0-3, 4-7  consumer warpgroup h: dgrad of the tile's 64 positions x channels h*N/2 .. (m64 n{32,64}, weights from its
//                   own two-stage ring of pre-tiled images), then wgrad rows m = 64 h .. 64 h + 63 (when M = 128 or h = 0;
//                   m64 n{64,128}), then the dgrad epilogue from accumulators staged over the dead X^T image
//   warps 8-11      producers: dY k-blocks and X^T k-blocks of the tile, each operand's raw rows one item ahead; thread 0
//                   also asks for the CTA's next tile's rows with cp.async.bulk.prefetch.L2
// Shared memory: dY 4 x 16 KB | X^T 2 x 32 KB (epilogue staging 2 x 17 KB) | weight rings 2 x 2 x 16 KB | barriers, lifted slices.
constexpr int BW_TP = 64;                               // positions per tile
constexpr int BW_THREADS = 384;
constexpr int BW_DY = 0, BW_XT = 64 * 1024, BW_W = 128 * 1024, BW_TAIL = 192 * 1024;
constexpr int BW_SMEM = BW_TAIL + 256 + 1024 + 4096 + 1024;
// BF16 (XB = Bf16<...>): dY is stored once as a bf16 64-byte-swizzle image, rows = positions, one 4 KB image per 32-channel
// k-block.  dgrad reads it as its K-major A operand; wgrad reads the same image MN-major (transposed) as its A operand, in place
// of the register-fed dY^T fragments.  X is stored position-major the same way (one 4 KB image per 32 channels) as wgrad's
// MN-major B operand, with no transposed store, and the weight ring carries the bf16 dgrad images (one k16 pair per k-block).
constexpr int BW_BF_SUB = BW_TP * TC_BF_ROW;            // 4 KB: 64 positions x 32 channels

template <class XB, int N>
__global__ void __launch_bounds__(BW_THREADS, 1)
    pw_bwd_tc_kernel(TcDy da, XB xb, const uint8_t* __restrict__ wtiles, int P, int M, TcDgradEpi<N, is_lift<XB>::value> epi,
                     float* __restrict__ part) {
    constexpr bool BF = is_bf16<XB>::value;
    constexpr int NH = N / 2;                           // dgrad channels per consumer warpgroup
    constexpr int WSTAGE = BF ? NH * TC_BF_ROW : 2 * NH * 128;   // one ring stage: the bf16 rows, or hi | lo rows of NH channels
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint8_t* tail = smem + BW_TAIL;
    uint64_t* dy_full = reinterpret_cast<uint64_t*>(tail);
    uint64_t* dy_empty = dy_full + 1;
    uint64_t* xt_full = dy_full + 2;
    uint64_t* xt_empty = dy_full + 3;
    uint64_t* wfull = dy_full + 4;                      // [2 warpgroups][2 stages]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nkb = M / TC_K;                           // dY k-blocks (dgrad's K)
    const int n_ptiles = (P + BW_TP - 1) / BW_TP;
    const int my_tiles = blockIdx.x < n_ptiles ? (n_ptiles - 1 - blockIdx.x) / gridDim.x + 1 : 0;

    if (threadIdx.x == 0) {
        o3d_mbar_init(dy_full, 128);
        o3d_mbar_init(dy_empty, 8);
        o3d_mbar_init(xt_full, 128);
        o3d_mbar_init(xt_empty, 8);
        for (int s = 0; s < 4; ++s) o3d_mbar_init(wfull + s, 1);
        o3d_fence_mbar_init();
    }
    __syncthreads();

    if (warp < 8) {
        const int h = warp >> 2, w = warp & 3, tw = threadIdx.x & 127;
        uint8_t* wring = smem + BW_W + h * 2 * WSTAGE;
        const int n_witems = my_tiles * nkb;            // this warpgroup's weight images: (tile, k-block) in walk order
        auto load_w = [&](int item) {                   // rows h*NH .. of the image of k-block item % nkb, hi and lo
            const int s = item & 1;
            o3d_mbar_expect_tx(wfull + 2 * h + s, WSTAGE);
            if constexpr (BF) {
                const uint8_t* src = wtiles + (size_t)(item % nkb) * BF_TILE_BYTES + h * NH * TC_BF_ROW;
                o3d_bulk_g2s(wring + s * WSTAGE, src, WSTAGE, wfull + 2 * h + s);
            } else {
                const uint8_t* src = wtiles + (size_t)(item % nkb) * (2 * TILE_BYTES) + h * NH * 128;
                o3d_bulk_g2s(wring + s * WSTAGE, src, NH * 128, wfull + 2 * h + s);
                o3d_bulk_g2s(wring + s * WSTAGE + NH * 128, src + TILE_BYTES, NH * 128, wfull + 2 * h + s);
            }
        };
        if (tw == 0) {
            if (n_witems > 0) load_w(0);
            if (n_witems > 1) load_w(1);
        }
        const bool do_w = 64 * h < M;                   // wgrad rows of this warpgroup
        const int n_local = h * NH + (tw % NH);         // epilogue: thread = one output channel x NH / 2 positions
        const int q = tw / NH;
        constexpr int PPT = NH / 2;
        float* stg = reinterpret_cast<float*>(smem + BW_XT + h * (NH * TC_EPI_LD * 4));
        int32_t* gsm = reinterpret_cast<int32_t*>(tail + 256);           // [2][128] row indices (lifted X)
        float4* ssm = reinterpret_cast<float4*>(tail + 256 + 1024);      // [2][128] per-position scalars
        epi.begin(n_local, N);
        float wacc[N / 2];
#pragma unroll
        for (int i = 0; i < N / 2; ++i) wacc[i] = 0.f;
        int witem = 0, tphase = 0, buf = 0;
        for (int t = blockIdx.x; t < n_ptiles; t += gridDim.x) {
            const int pt0 = t * BW_TP;
            {
                const int32_t* gi = epi.lift_gidx();
                const float* si = epi.lift_s();
                if (gi || si) {
                    if (tw < BW_TP) {
                        const int pp = min(pt0 + tw, P - 1);
                        const int slot = buf * TC_N + ((pt0 + tw) & (TC_N - 1));
                        if (gi && h == 0) gsm[slot] = __ldg(gi + pp);
                        if (si && h == 1) ssm[slot] = ld4g(si + (size_t)pp * 4);
                    }
                    asm volatile("bar.sync 1, 256;" ::: "memory");
                    epi.set_tile(gsm + buf * TC_N, ssm + buf * TC_N);
                }
            }
            const int pb = pt0 + q * PPT;
            // ---- dgrad: D[64 positions, NH channels] over the nkb k-blocks of dY
            float dacc[NH / 2];
#pragma unroll
            for (int i = 0; i < NH / 2; ++i) dacc[i] = 0.f;
            o3d_mbar_wait(dy_full, tphase);
            for (int kb = 0; kb < nkb; ++kb, ++witem) {
                o3d_mbar_wait(wfull + 2 * h + (witem & 1), (witem >> 1) & 1);
                const uint32_t bb = o3d_smem_u32(wring + (witem & 1) * WSTAGE);
                wgmma_fence_acc(dacc);
                wgmma_fence();
                if constexpr (BF) {
                    wgmma_bf16_kblock<NH>(dacc, make_desc_sw64(o3d_smem_u32(smem + BW_DY + kb * BW_BF_SUB)), make_desc_sw64(bb), kb == 0);
                } else {
                    const uint32_t ab = o3d_smem_u32(smem + BW_DY + kb * TILE_BYTES);   // hi | lo, 8 KB each
                    wgmma_3xtf32_kblock<NH>(dacc, make_desc(ab), make_desc(ab + TILE_BYTES / 2), make_desc(bb), make_desc(bb + NH * 128),
                                            kb == 0);
                }
                wgmma_commit();
                wgmma_wait<0>();
                wgmma_fence_acc(dacc);
                asm volatile("bar.sync %0, 128;" ::"r"(2 + h) : "memory");   // the warpgroup is done with this ring stage
                if (tw == 0 && witem + 2 < n_witems) load_w(witem + 2);
            }
            // ---- wgrad: dW[64 h + 0..63, 0..N-1] += dY^T . X over the tile's 64 positions (8 k-steps)
            o3d_mbar_wait(xt_full, tphase);
            if constexpr (BF) {
                if (do_w) {   // rows m = 64 h .. : dY images 2h, 2h+1 read MN-major; X images read MN-major; 4 k16 steps
                    const uint32_t ab = o3d_smem_u32(smem + BW_DY + 2 * h * BW_BF_SUB), xb0 = o3d_smem_u32(smem + BW_XT);
                    wgmma_fence_acc(wacc);
                    wgmma_fence();
#pragma unroll
                    for (int ks = 0; ks < BW_TP / 16; ++ks) {
                        const uint64_t ad = make_desc_sw64_mn(ab + ks * 1024, BW_BF_SUB), bd = make_desc_sw64_mn(xb0 + ks * 1024, BW_BF_SUB);
                        if constexpr (N == 128) wgmma_bf16_tt_n128(wacc, ad, bd, 1u);
                        else wgmma_bf16_tt_n64(wacc, ad, bd, 1u);
                    }
                    wgmma_commit();
                    wgmma_wait<0>();
                    wgmma_fence_acc(wacc);
                }
            } else if (do_w) {
                const int mr = 16 * w + (lane >> 2);                 // fragment rows mr, mr + 8 of this warpgroup's 64
                const uint8_t* dyk = smem + BW_DY + (2 * h + (w >> 1)) * (TILE_BYTES);   // k-block of channels 64 h + mr
                const int mc = mr & 31;
                const uint32_t xt = o3d_smem_u32(smem + BW_XT);
#pragma unroll 1
                for (int ks = 0; ks < BW_TP / 8; ++ks) {
                    uint32_t ahi[4], alo[4];
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const int p = ks * 8 + (lane & 3) + 4 * (i >> 1), m = mc + 8 * (i & 1);
                        const uint32_t off = sw128(p, m >> 2) + 4 * (m & 3);
                        ahi[i] = *reinterpret_cast<const uint32_t*>(dyk + off);
                        alo[i] = *reinterpret_cast<const uint32_t*>(dyk + TILE_BYTES / 2 + off);
                    }
                    const uint32_t xb0 = xt + (ks >> 2) * (2 * TILE_BYTES) + (ks & 3) * 32;
                    const uint64_t bhi = make_desc(xb0), blo = make_desc(xb0 + TILE_BYTES);
                    wgmma_fence_acc(wacc);
                    wgmma_fence();
                    if constexpr (N == 128) {
                        wgmma_tf32_rs_n128(wacc, alo, bhi);
                        wgmma_tf32_rs_n128(wacc, ahi, blo);
                        wgmma_tf32_rs_n128(wacc, ahi, bhi);
                    } else {
                        wgmma_tf32_rs_n64(wacc, alo, bhi);
                        wgmma_tf32_rs_n64(wacc, ahi, blo);
                        wgmma_tf32_rs_n64(wacc, ahi, bhi);
                    }
                    wgmma_commit();
                    wgmma_wait<0>();                                  // the fragments' registers are re-used by the next step
                    wgmma_fence_acc(wacc);
                }
            }
            __syncwarp();
            if (lane == 0) o3d_mbar_arrive(dy_empty);
            // the first column group's input rows are requested only now: held across the MMAs they would push the lifted
            // instantiations past the register budget
            epi.prefetch(n_local, N, pb, P);
            asm volatile("bar.sync 4, 256;" ::: "memory");           // both warpgroups are done with X^T: staging goes over it
            stage_acc(dacc, stg, TC_EPI_LD);
            asm volatile("bar.sync %0, 128;" ::"r"(2 + h) : "memory");
            const float* row = stg + (tw % NH) * TC_EPI_LD + q * PPT;
#pragma unroll 1
            for (int cg = 0; cg < PPT / 16; ++cg) {
                uint32_t r[16];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float4 v = *reinterpret_cast<const float4*>(row + cg * 16 + 4 * j);
                    r[4 * j] = __float_as_uint(v.x); r[4 * j + 1] = __float_as_uint(v.y);
                    r[4 * j + 2] = __float_as_uint(v.z); r[4 * j + 3] = __float_as_uint(v.w);
                }
                epi.group(r, n_local, N, pb + cg * 16, P);
                if (cg + 1 < PPT / 16) epi.prefetch(n_local, N, pb + (cg + 1) * 16, P);
            }
            __syncwarp();
            if (lane == 0) o3d_mbar_arrive(xt_empty);
            tphase ^= 1;
            buf ^= 1;
        }
        epi.end(n_local, N);
        if (do_w) {
            float* __restrict__ out = part + (size_t)blockIdx.x * TC_M * TC_N;
#pragma unroll
            for (int i = 0; i < N / 2; i += 4) {
#pragma unroll
                for (int rr = 0; rr < 2; ++rr) {
                    const int m = 64 * h + 16 * w + (lane >> 2) + 8 * rr, n = 8 * (i >> 2) + 2 * (lane & 3);
                    *reinterpret_cast<float2*>(out + (size_t)m * TC_N + n) = make_float2(wacc[i + 2 * rr], wacc[i + 2 * rr + 1]);
                }
            }
        }
    } else {
        // ===================================================== producers (4 warps, 128 threads)
        const int pt = threadIdx.x - 256;
        const int chunk = pt & 7, row0 = (pt >> 3) * 4;               // dY: 4 neighbouring rows, 4 channels of a k-block
        // X: 4 channels 4 c4 .. x positions prow0 + 8 i (BF16), or 4 consecutive positions 4 (lane % 8) .. (3xTF32, see
        // store_transposed)
        const int pw = warp - 8, c4 = BF ? pw * 4 + (lane & 3) : pw * 4 + (lane >> 3), prow0 = lane >> 2;
        const int qx = lane & 7, px = BF ? prow0 : 4 * qx;
        constexpr int RS = BF ? 8 : 1;
        constexpr int NXH = N / 64;                                   // X^T pieces per 32-position k-block (64 channels each)
        const int n_items_x = 2 * NXH;
        // dY items (tile, kb) and X^T items (tile, j = 32-position half, channel half) are two flat sequences, each walked
        // with its raw rows one item ahead
        struct It { int t, i; };
        TcDy::Batch<4> ra{};
        typename XB::template Batch<4> rb{};
        It ca{(int)blockIdx.x, 0}, cb{(int)blockIdx.x, 0};
        auto fetch_a = [&](const It& c) {
            if (c.t < n_ptiles) da.fetch(ra, c.t * BW_TP + row0, 1, P, c.i * TC_K + chunk * 4, M);
        };
        auto fetch_b = [&](const It& c) {
            if (c.t < n_ptiles)
                xb.fetch(rb, c.t * BW_TP + (c.i >> (NXH - 1)) * TC_K + px, RS, P, (c.i & (NXH - 1)) * 64 + c4 * 4, N);
        };
        fetch_a(ca);
        fetch_b(cb);
        if (pt == 0 && ca.t < n_ptiles) { da.prefetch_rows(ca.t * BW_TP, BW_TP, P); xb.prefetch_rows(ca.t * BW_TP, BW_TP, P); }
        int tphase = 0;
        for (int t = blockIdx.x; t < n_ptiles; t += gridDim.x) {
            const int pt0 = t * BW_TP;
            if (pt == 0) {
                const int tn = t + (int)gridDim.x;
                if (tn < n_ptiles) { da.prefetch_rows(tn * BW_TP, BW_TP, P); xb.prefetch_rows(tn * BW_TP, BW_TP, P); }
            }
            o3d_mbar_wait(dy_empty, tphase ^ 1);
            for (int kb = 0; kb < nkb; ++kb) {
                const int k = kb * TC_K + chunk * 4;
                const TcDy::Coef cf = da.prep(k, M);
                if constexpr (BF) {
#pragma unroll
                    for (int i = 0; i < 4; ++i)
                        st_bf16_row4(smem + BW_DY + kb * BW_BF_SUB, 0, row0 + i, chunk * 4, da.finish(ra, cf, i, pt0 + row0 + i, P));
                } else {
                    uint8_t* hi = smem + BW_DY + kb * TILE_BYTES;
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const float4 v = da.finish(ra, cf, i, pt0 + row0 + i, P);
                        const uint32_t off = sw128(row0 + i, chunk);
                        *reinterpret_cast<float4*>(hi + off) = hi_part(v);
                        *reinterpret_cast<float4*>(hi + TILE_BYTES / 2 + off) = lo_part(v);
                    }
                }
                if (++ca.i == nkb) { ca.i = 0; ca.t += gridDim.x; }
                fetch_a(ca);
            }
            o3d_fence_proxy_async();
            o3d_mbar_arrive(dy_full);
            o3d_mbar_wait(xt_empty, tphase ^ 1);
            for (int it = 0; it < n_items_x; ++it) {
                const int j = it >> (NXH - 1), cl = (it & (NXH - 1)) * 64 + c4 * 4;
                if constexpr (BF)
                    store_rows_bf16(xb, rb, xb.prep(cl, N), smem + BW_XT + j * (TC_K * TC_BF_ROW), BW_BF_SUB, cl, pt0 + j * TC_K, prow0, P);
                else
                    store_transposed(xb, rb, xb.prep(cl, N), smem + BW_XT + j * (2 * TILE_BYTES), cl, pt0 + j * TC_K, qx, P);
                if (++cb.i == n_items_x) { cb.i = 0; cb.t += gridDim.x; }
                fetch_b(cb);
            }
            o3d_fence_proxy_async();
            o3d_mbar_arrive(xt_full);
            tphase ^= 1;
        }
    }
}

// Pre-tile a weight matrix W[rows, ld] (rows = output channels, k contiguous) into the per-(m_tile, k-block) shared-memory
// images the kernel bulk-copies: [hi 16 KB | lo 16 KB], K-major SWIZZLE_128B, zero padded.
__global__ void w_pretile_kernel(const float* __restrict__ W, int ld, int rows, int K, int nkb, uint8_t* __restrict__ out) {
    const int m_tile = blockIdx.y, kb = blockIdx.x;
    uint8_t* dst = out + ((size_t)m_tile * nkb + kb) * (2 * TILE_BYTES);
    for (int id = threadIdx.x; id < TC_M * 8; id += blockDim.x) {
        const int r = id >> 3, c = id & 7;
        const int row = m_tile * TC_M + r, k = kb * TC_K + c * 4;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (row < rows && k < K) v = *reinterpret_cast<const float4*>(W + (size_t)row * ld + k);
        const uint32_t off = sw128(r, c);
        *reinterpret_cast<float4*>(dst + off) = hi_part(v);
        *reinterpret_cast<float4*>(dst + TILE_BYTES + off) = lo_part(v);
    }
}

inline int ilog2_exact(int v) { int l = 0; while ((1 << l) < v) ++l; return l; }

// reverse: walk the position tiles from the last to the first (see pw_tc_kernel)
template <class BLoad, class Epi>
int launch_tc(BLoad bl, const uint8_t* wtiles, int P, int K, int Nw, Epi epi, bool reverse, cudaStream_t st, const char* name) {
    auto kern = pw_tc_kernel<BLoad, Epi>;
    O3D_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM), name);
    const int gy = (Nw + TC_M - 1) / TC_M;
    const int nkb = (K + TC_K - 1) / TC_K;
    const int n_ptiles = (P + TC_N - 1) / TC_N;
    int gx = o3d_num_sms() / gy;
    if (gx < 1) gx = 1;
    if (gx > n_ptiles) gx = n_ptiles;
    kern<<<dim3(gx, gy), TC_THREADS, TC_SMEM, st>>>(bl, wtiles, P, K, Nw, nkb, epi, reverse);
    O3D_CHECK_LAUNCH(name);
    return O3D_OK;
}

template <int LD, class BLoad>
int launch_fwd(const BLoad& bl, const void* wtiles, const float* bias, int P, int K, int Nw, float* y, int ldy, double* sum,
               double* sumsq, int S, float* ymax, float* ymin, int32_t* arg, int ldp, bool reverse, cudaStream_t st) {
    TcFwdEpi<LD> ep{};
    ep.y = y; ep.ldy = ldy; ep.bias = bias; ep.sum = sum; ep.sumsq = sumsq;
    ep.S = S; ep.ymax = ymax; ep.ymin = ymin; ep.arg = arg; ep.ldp = ldp;
    ep.log2S = 0;
    while ((1 << ep.log2S) < S) ++ep.log2S;
    return launch_tc(bl, (const uint8_t*)wtiles, P, K, Nw, ep, reverse, st, "o3d_pw_fwd_tc");
}

template <int LD, bool LIFT = false, class BL>
int launch_dgrad(const BL& bl, const void* wtiles_t, int P, int Cout, int Cin, float* out, int ldo, const float* yprev,
                 int ldyp, const float* pscale, const float* pshift, int prelu, double* s1, double* s2y, cudaStream_t st,
                 const LiftView* lv = nullptr) {
    if constexpr (!LIFT) {
        if (lv) return launch_dgrad<LD, true>(bl, wtiles_t, P, Cout, Cin, out, ldo, yprev, ldyp, pscale, pshift, prelu, s1, s2y, st, lv);
    }
    TcDgradEpi<LD, LIFT> ep{};
    if (lv) ep.lv = *lv;
    ep.out = out; ep.ldo = ldo; ep.yprev = yprev; ep.ldyp = ldyp; ep.scale = pscale; ep.shift = pshift; ep.relu = prelu;
    ep.s1g = s1; ep.s2y = s2y;
    // GEMM: D[pos, cin] = sum_cout dY[pos, cout] * Wt[cin, cout]  ->  "K" = Cout, "Nw" = Cin
    return launch_tc(bl, (const uint8_t*)wtiles_t, P, Cout, Cin, ep, false, st, "o3d_pw_dgrad_tc");
}

}  // namespace

extern "C" long long o3d_pw_tc_wtile_bytes(int rows, int K) {
    const long long mt = (rows + TC_M - 1) / TC_M, nkb = (K + TC_K - 1) / TC_K;
    return mt * nkb * 2 * TILE_BYTES;
}

extern "C" int o3d_pw_tc_pretile(const float* w, int ldw, int rows, int K, void* wtiles, void* stream) {
    O3D_REQUIRE(w && wtiles, O3D_ERR_ARG, "o3d_pw_tc_pretile: null pointer");
    O3D_REQUIRE((K & 3) == 0 && (ldw & 3) == 0, O3D_ERR_ARG, "o3d_pw_tc_pretile: K and ldw must be multiples of 4");
    O3D_REQUIRE(((uintptr_t)wtiles & 15) == 0 && ((uintptr_t)w & 15) == 0, O3D_ERR_ALIGN, "o3d_pw_tc_pretile: alignment");
    const int mt = (rows + TC_M - 1) / TC_M, nkb = (K + TC_K - 1) / TC_K;
    w_pretile_kernel<<<dim3(nkb, mt), 256, 0, (cudaStream_t)stream>>>(w, ldw, rows, K, nkb, (uint8_t*)wtiles);
    O3D_CHECK_LAUNCH("o3d_pw_tc_pretile");
    return O3D_OK;
}

int o3d_pw_fwd_tc_dir(const float* x, int ldx, const float* in_scale, const float* in_shift, int in_relu, const void* wtiles,
                      const float* bias, int P, int K, int N, float* y, int ldy, double* sum, double* sumsq, int S, float* ymax,
                      float* ymin, int32_t* arg, int ldp, void* stream, bool reverse, bool bf16) {
    O3D_REQUIRE(x && wtiles, O3D_ERR_ARG, "o3d_pw_fwd_tc: null pointer");
    O3D_REQUIRE(P >= 0 && K >= 4 && N >= 1 && (K & 3) == 0 && (ldx & 3) == 0, O3D_ERR_ARG, "o3d_pw_fwd_tc: bad sizes");
    O3D_REQUIRE(S == 0 || (P % S == 0 && 64 % S == 0 && ymax && ymin && arg), O3D_ERR_ARG,
                "o3d_pw_fwd_tc: pooling group size must divide 64 and P");
    if (P == 0) return O3D_OK;
    const int Nw = (N + 3) & ~3;
    TcAct bl{x, ldx, in_scale, in_shift, in_relu};
    // the usual activation widths get a compile-time row stride (immediate store offsets in the epilogue)
    cudaStream_t st = (cudaStream_t)stream;
    if (bf16) {
        Bf16<TcAct> bb{bl};
#define O3D_FWD_ARGS bb, wtiles, bias, P, K, Nw, y, ldy, sum, sumsq, S, ymax, ymin, arg, ldp, reverse, st
        if (ldy == 64) return launch_fwd<64>(O3D_FWD_ARGS);
        if (ldy == 128) return launch_fwd<128>(O3D_FWD_ARGS);
        if (ldy == 256) return launch_fwd<256>(O3D_FWD_ARGS);
        return launch_fwd<0>(O3D_FWD_ARGS);
#undef O3D_FWD_ARGS
    }
#define O3D_FWD_ARGS bl, wtiles, bias, P, K, Nw, y, ldy, sum, sumsq, S, ymax, ymin, arg, ldp, reverse, st
    if (ldy == 64) return launch_fwd<64>(O3D_FWD_ARGS);
    if (ldy == 128) return launch_fwd<128>(O3D_FWD_ARGS);
    if (ldy == 256) return launch_fwd<256>(O3D_FWD_ARGS);
    return launch_fwd<0>(O3D_FWD_ARGS);
#undef O3D_FWD_ARGS
}

extern "C" int o3d_pw_fwd_tc(const float* x, int ldx, const float* in_scale, const float* in_shift, int in_relu,
                             const void* wtiles, const float* bias, int P, int K, int N, float* y, int ldy, double* sum,
                             double* sumsq, int S, float* ymax, float* ymin, int32_t* arg, int ldp, void* stream) {
    return o3d_pw_fwd_tc_dir(x, ldx, in_scale, in_shift, in_relu, wtiles, bias, P, K, N, y, ldy, sum, sumsq, S, ymax, ymin, arg,
                             ldp, stream, false, false);
}

namespace {
int dgrad_tc_impl(const float* g, int ldg, const float* y, int ldy, const float* a, const float* b, const float* cc,
                  const float* dpool, const int32_t* sel, int S, int ldp, const void* wtiles_t, int P, int Cout, int Cin,
                  float* out, int ldo, const float* yprev, int ldyp, const float* pscale, const float* pshift, int prelu,
                  double* s1, double* s2y, void* stream, const LiftView* lv, bool bf16) {
    O3D_REQUIRE((g || dpool) && wtiles_t && out, O3D_ERR_ARG, "o3d_pw_dgrad_tc: null pointer");
    O3D_REQUIRE((Cout & 3) == 0 && (Cin & 3) == 0, O3D_ERR_ARG, "o3d_pw_dgrad_tc: channel counts must be multiples of 4");
    if (P == 0) return O3D_OK;
    TcDy bl{g, ldg, y, ldy, a, b, cc, dpool, sel, S > 0 ? S : 1, ldp, ilog2_exact(S > 0 ? S : 1)};
    cudaStream_t st = (cudaStream_t)stream;
    const int ld = (!yprev || ldyp == ldo) ? ldo : 0;   // one compile-time stride serves both out and yprev
    auto run = [&](const auto& ldr) {
#define O3D_DG_ARGS ldr, wtiles_t, P, Cout, Cin, out, ldo, yprev, ldyp, pscale, pshift, prelu, s1, s2y, st, lv
        if (ld == 64) return launch_dgrad<64>(O3D_DG_ARGS);
        if (ld == 128) return launch_dgrad<128>(O3D_DG_ARGS);
        if (ld == 256) return launch_dgrad<256>(O3D_DG_ARGS);
        return launch_dgrad<0>(O3D_DG_ARGS);
#undef O3D_DG_ARGS
    };
    return bf16 ? run(Bf16<TcDy>{bl}) : run(bl);   // bf16: wtiles_t holds bf16 images (o3d_stack_t.precision = 2)
}
}  // namespace

int o3d_pw_dgrad_tc_prec(const float* g, int ldg, const float* y, int ldy, const float* a, const float* b, const float* cc,
                         const float* dpool, const int32_t* sel, int S, int ldp, const void* wtiles_t, int P, int Cout, int Cin,
                         float* out, int ldo, const float* yprev, int ldyp, const float* pscale, const float* pshift, int prelu,
                         double* s1, double* s2y, void* stream, bool bf16) {
    return dgrad_tc_impl(g, ldg, y, ldy, a, b, cc, dpool, sel, S, ldp, wtiles_t, P, Cout, Cin, out, ldo, yprev, ldyp, pscale,
                         pshift, prelu, s1, s2y, stream, nullptr, bf16);
}

extern "C" int o3d_pw_dgrad_tc(const float* g, int ldg, const float* y, int ldy, const float* a, const float* b,
                               const float* cc, const float* dpool, const int32_t* sel, int S, int ldp,
                               const void* wtiles_t, int P, int Cout, int Cin, float* out, int ldo, const float* yprev,
                               int ldyp, const float* pscale, const float* pshift, int prelu, double* s1, double* s2y,
                               void* stream) {
    return dgrad_tc_impl(g, ldg, y, ldy, a, b, cc, dpool, sel, S, ldp, wtiles_t, P, Cout, Cin, out, ldo, yprev, ldyp, pscale,
                         pshift, prelu, s1, s2y, stream, nullptr, false);
}

// dgrad whose input side is a lifted first layer: the ReLU mask and the BatchNorm-backward sums use Y0 gathered from Z
int o3d_pw_dgrad_tc_lift_prec(const float* g, int ldg, const float* y, int ldy, const float* a, const float* b, const float* cc,
                              const float* dpool, const int32_t* sel, int S, int ldp, const void* wtiles_t, int P, int Cout,
                              int Cin, float* out, int ldo, const o3d_lift_t* lf, const int32_t* gidx, const float* pscale,
                              const float* pshift, int prelu, double* s1, double* s2y, void* stream, bool bf16) {
    O3D_REQUIRE(lf && (gidx || !lf->z) && (lf->z || lf->s) && lf->ldz == Cin, O3D_ERR_ARG, "o3d_pw_dgrad_tc_lift: lift descriptor");
    const LiftView lv{lf->z, lf->ldz, lf->z ? gidx : nullptr, lf->s, lf->u};
    return dgrad_tc_impl(g, ldg, y, ldy, a, b, cc, dpool, sel, S, ldp, wtiles_t, P, Cout, Cin, out, ldo, nullptr, 0, pscale,
                         pshift, prelu, s1, s2y, stream, &lv, bf16);
}

extern "C" int o3d_pw_dgrad_tc_lift(const float* g, int ldg, const float* y, int ldy, const float* a, const float* b,
                                    const float* cc, const float* dpool, const int32_t* sel, int S, int ldp,
                                    const void* wtiles_t, int P, int Cout, int Cin, float* out, int ldo,
                                    const o3d_lift_t* lf, const int32_t* gidx, const float* pscale, const float* pshift,
                                    int prelu, double* s1, double* s2y, void* stream) {
    return o3d_pw_dgrad_tc_lift_prec(g, ldg, y, ldy, a, b, cc, dpool, sel, S, ldp, wtiles_t, P, Cout, Cin, out, ldo, lf, gidx, pscale,
                                     pshift, prelu, s1, s2y, stream, false);
}

namespace {
// the splits write partial tiles into `part` (part_floats long) and wgrad_reduce_kernel adds their sum into dw in split order
// (deterministic)
template <class XB>
int launch_wgrad(const TcDy& da, const XB& xb, int P, int Cout, int Cin, float* dw, int lddw, float* part, long long part_floats,
                 cudaStream_t st) {
    auto kern = pw_wgrad_tc_kernel<XB>;
    O3D_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, WG_SMEM), "o3d_pw_wgrad_tc2");
    const int mt = (Cout + TC_M - 1) / TC_M, nt = (Cin + TC_N - 1) / TC_N;
    const int Mt = mt * TC_M, Nt = nt * TC_N;
    int splits = o3d_num_sms() / (mt * nt);
    if (splits < 1) splits = 1;
    const long long cap = part_floats / ((long long)Mt * Nt);
    if (splits > cap) splits = (int)cap;
    // small problems (the heads: a few thousand positions): every split writes and the reduction re-reads a whole
    // Mt x Nt partial tile, so at least 128 positions per split
    const int by_size = (P + 127) / 128;
    if (splits > by_size) splits = by_size;
    O3D_REQUIRE(splits >= 1, O3D_ERR_ARG, "o3d_pw_wgrad_tc2: workspace too small");
    int chunk = (P + splits - 1) / splits;
    chunk = ((chunk + TC_K - 1) / TC_K) * TC_K;
    splits = (P + chunk - 1) / chunk;
    kern<<<dim3(splits, nt, mt), WG_THREADS, WG_SMEM, st>>>(da, xb, P, Cout, Cin, chunk, part);
    O3D_CHECK_LAUNCH("o3d_pw_wgrad_tc2");
    dim3 rg((Cin / 4 + 31) / 32, Cout);
    wgrad_reduce_kernel<<<rg, 256, 0, st>>>(part, splits, Mt, Nt, Cout, Cin, dw, lddw);
    O3D_CHECK_LAUNCH("o3d_pw_wgrad_tc2: reduce");
    return O3D_OK;
}
inline TcLift make_tclift(const o3d_lift_t* lf, const int32_t* gidx, const float* scale, const float* shift, int relu) {
    return TcLift{LiftView{lf->z, lf->ldz, lf->z ? gidx : nullptr, lf->s, lf->u}, scale, shift, relu, 0};
}
}  // namespace

extern "C" long long o3d_pw_wgrad_tc2_workspace_floats(void) {
    return (long long)o3d_num_sms() * TC_M * TC_N;   // splits <= #SMs / tiles of dW, so splits * Mt * Nt <= #SMs * 128 * 128
}

int o3d_pw_wgrad_tc2_prec(const float* g, int ldg, const float* y, int ldy, const float* a, const float* b, const float* cc,
                          const float* dpool, const int32_t* sel, int S, int ldp, const float* x, int ldx, const float* in_scale,
                          const float* in_shift, int in_relu, int P, int Cout, int Cin, float* dw, int lddw, float* part,
                          long long part_floats, void* stream, bool bf16) {
    O3D_REQUIRE((g || dpool) && x && dw && part, O3D_ERR_ARG, "o3d_pw_wgrad_tc2: null pointer");
    O3D_REQUIRE((Cout & 3) == 0 && (Cin & 3) == 0 && (ldx & 3) == 0 && (lddw & 3) == 0, O3D_ERR_ARG,
                "o3d_pw_wgrad_tc2: channel counts / leading dimensions must be multiples of 4");
    if (P == 0) return O3D_OK;
    TcDy da{g, ldg, y, ldy, a, b, cc, dpool, sel, S > 0 ? S : 1, ldp, ilog2_exact(S > 0 ? S : 1)};
    TcAct xb{x, ldx, in_scale, in_shift, in_relu};
    if (bf16) return launch_wgrad(da, Bf16<TcAct>{xb}, P, Cout, Cin, dw, lddw, part, part_floats, (cudaStream_t)stream);
    return launch_wgrad(da, xb, P, Cout, Cin, dw, lddw, part, part_floats, (cudaStream_t)stream);
}

extern "C" int o3d_pw_wgrad_tc2(const float* g, int ldg, const float* y, int ldy, const float* a, const float* b,
                                const float* cc, const float* dpool, const int32_t* sel, int S, int ldp, const float* x,
                                int ldx, const float* in_scale, const float* in_shift, int in_relu, int P, int Cout,
                                int Cin, float* dw, int lddw, float* part, long long part_floats, void* stream) {
    return o3d_pw_wgrad_tc2_prec(g, ldg, y, ldy, a, b, cc, dpool, sel, S, ldp, x, ldx, in_scale, in_shift, in_relu, P, Cout, Cin,
                                 dw, lddw, part, part_floats, stream, false);
}

// ---- lifted first layer (o3d_lift_t): the next layer's GEMMs read Y0 through TcLift / the lifted dgrad epilogue ----------
int o3d_pw_wgrad_tc_lift_prec(const float* g, int ldg, const float* y, int ldy, const float* a, const float* b, const float* cc,
                              const float* dpool, const int32_t* sel, int S, int ldp, const o3d_lift_t* lf, const int32_t* gidx,
                              const float* in_scale, const float* in_shift, int in_relu, int P, int Cout, int Cin, float* dw,
                              int lddw, float* part, long long part_floats, void* stream, bool bf16) {
    O3D_REQUIRE((g || dpool) && lf && (gidx || !lf->z) && dw && part, O3D_ERR_ARG, "o3d_pw_wgrad_tc_lift: null pointer");
    O3D_REQUIRE((Cout & 3) == 0 && (Cin & 3) == 0 && lf->ldz == Cin && (lddw & 3) == 0, O3D_ERR_ARG,
                "o3d_pw_wgrad_tc_lift: channel counts / leading dimensions");
    if (P == 0) return O3D_OK;
    TcDy da{g, ldg, y, ldy, a, b, cc, dpool, sel, S > 0 ? S : 1, ldp, ilog2_exact(S > 0 ? S : 1)};
    TcLift xb = make_tclift(lf, gidx, in_scale, in_shift, in_relu);
    xb.la = TC_K;      // a producer thread's next fetch lies one k-block of positions further
    if (bf16) return launch_wgrad(da, Bf16<TcLift>{xb}, P, Cout, Cin, dw, lddw, part, part_floats, (cudaStream_t)stream);
    return launch_wgrad(da, xb, P, Cout, Cin, dw, lddw, part, part_floats, (cudaStream_t)stream);
}

extern "C" int o3d_pw_wgrad_tc_lift(const float* g, int ldg, const float* y, int ldy, const float* a, const float* b,
                                    const float* cc, const float* dpool, const int32_t* sel, int S, int ldp,
                                    const o3d_lift_t* lf, const int32_t* gidx, const float* in_scale, const float* in_shift,
                                    int in_relu, int P, int Cout, int Cin, float* dw, int lddw, float* part,
                                    long long part_floats, void* stream) {
    return o3d_pw_wgrad_tc_lift_prec(g, ldg, y, ldy, a, b, cc, dpool, sel, S, ldp, lf, gidx, in_scale, in_shift, in_relu, P, Cout,
                                     Cin, dw, lddw, part, part_floats, stream, false);
}

int o3d_pw_fwd_tc_lift_prec(const o3d_lift_t* lf, const int32_t* gidx, const float* in_scale, const float* in_shift, int in_relu,
                            const void* wtiles, const float* bias, int P, int K, int N, float* y, int ldy, double* sum,
                            double* sumsq, int S, float* ymax, float* ymin, int32_t* arg, int ldp, void* stream, bool bf16) {
    O3D_REQUIRE(lf && (gidx || !lf->z) && wtiles, O3D_ERR_ARG, "o3d_pw_fwd_tc_lift: null pointer");
    O3D_REQUIRE(P >= 0 && K >= 32 && N >= 1 && (K & 3) == 0 && lf->ldz == K, O3D_ERR_ARG, "o3d_pw_fwd_tc_lift: bad sizes");
    O3D_REQUIRE(S == 0 || (P % S == 0 && 64 % S == 0 && ymax && ymin && arg), O3D_ERR_ARG,
                "o3d_pw_fwd_tc_lift: pooling group size must divide 64 and P");
    if (P == 0) return O3D_OK;
    const int Nw = (N + 3) & ~3;
    const TcLift bl = make_tclift(lf, gidx, in_scale, in_shift, in_relu);
    cudaStream_t st = (cudaStream_t)stream;
    if (bf16) {
        const Bf16<TcLift> bb{bl};
#define O3D_FWD_ARGS bb, wtiles, bias, P, K, Nw, y, ldy, sum, sumsq, S, ymax, ymin, arg, ldp, false, st
        if (ldy == 64) return launch_fwd<64>(O3D_FWD_ARGS);
        if (ldy == 128) return launch_fwd<128>(O3D_FWD_ARGS);
        if (ldy == 256) return launch_fwd<256>(O3D_FWD_ARGS);
        return launch_fwd<0>(O3D_FWD_ARGS);
#undef O3D_FWD_ARGS
    }
#define O3D_FWD_ARGS bl, wtiles, bias, P, K, Nw, y, ldy, sum, sumsq, S, ymax, ymin, arg, ldp, false, st
    if (ldy == 64) return launch_fwd<64>(O3D_FWD_ARGS);
    if (ldy == 128) return launch_fwd<128>(O3D_FWD_ARGS);
    if (ldy == 256) return launch_fwd<256>(O3D_FWD_ARGS);
    return launch_fwd<0>(O3D_FWD_ARGS);
#undef O3D_FWD_ARGS
}

extern "C" int o3d_pw_fwd_tc_lift(const o3d_lift_t* lf, const int32_t* gidx, const float* in_scale, const float* in_shift,
                                  int in_relu, const void* wtiles, const float* bias, int P, int K, int N, float* y, int ldy,
                                  double* sum, double* sumsq, int S, float* ymax, float* ymin, int32_t* arg, int ldp,
                                  void* stream) {
    return o3d_pw_fwd_tc_lift_prec(lf, gidx, in_scale, in_shift, in_relu, wtiles, bias, P, K, N, y, ldy, sum, sumsq, S, ymax, ymin,
                                   arg, ldp, stream, false);
}

namespace {
template <class XB, int N>
int launch_bwd(const TcDy& da, const XB& xb, const void* wtiles_t, int P, int M, const TcDgradEpi<N, is_lift<XB>::value>& ep,
               float* dw, int lddw, float* part, long long part_floats, cudaStream_t st) {
    auto kern = pw_bwd_tc_kernel<XB, N>;
    O3D_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, BW_SMEM), "o3d_pw_bwd_tc");
    const int n_ptiles = (P + BW_TP - 1) / BW_TP;
    int gx = o3d_num_sms();
    if (gx > n_ptiles) gx = n_ptiles;
    O3D_REQUIRE(part_floats >= (long long)gx * TC_M * TC_N, O3D_ERR_ARG, "o3d_pw_bwd_tc: workspace too small");
    kern<<<gx, BW_THREADS, BW_SMEM, st>>>(da, xb, (const uint8_t*)wtiles_t, P, M, ep, part);
    O3D_CHECK_LAUNCH("o3d_pw_bwd_tc");
    dim3 rg((N / 4 + 31) / 32, M);
    wgrad_reduce_kernel<<<rg, 256, 0, st>>>(part, gx, TC_M, TC_N, M, N, dw, lddw);
    O3D_CHECK_LAUNCH("o3d_pw_bwd_tc: reduce");
    return O3D_OK;
}

template <class XB>
int bwd_tc_impl(const TcDy& da, const XB& xb, const void* wtiles_t, int P, int Cout, int Cin, float* out, const float* yprev,
                const LiftView* lv, const float* pscale, const float* pshift, int prelu, double* s1, double* s2y, float* dw,
                int lddw, float* part, long long part_floats, cudaStream_t st) {
    constexpr bool LIFT = is_lift<XB>::value;
    auto fill = [&](auto& ep) {
        if constexpr (LIFT) ep.lv = *lv;
        ep.out = out; ep.ldo = Cin; ep.yprev = yprev; ep.ldyp = Cin; ep.scale = pscale; ep.shift = pshift; ep.relu = prelu;
        ep.s1g = s1; ep.s2y = s2y;
    };
    if (Cin == 64) {
        TcDgradEpi<64, LIFT> ep{};
        fill(ep);
        return launch_bwd<XB, 64>(da, xb, wtiles_t, P, Cout, ep, dw, lddw, part, part_floats, st);
    }
    TcDgradEpi<128, LIFT> ep{};
    fill(ep);
    return launch_bwd<XB, 128>(da, xb, wtiles_t, P, Cout, ep, dw, lddw, part, part_floats, st);
}
}  // namespace

int o3d_pw_bwd_tc_prec(const float* g, int ldg, const float* y, int ldy, const float* a, const float* b, const float* cc,
                       const float* dpool, const int32_t* sel, int S, int ldp, const void* wtiles_t, const float* x,
                       const o3d_lift_t* lf, const int32_t* gidx, const float* in_scale, const float* in_shift, int in_relu, int P,
                       int Cout, int Cin, float* out, double* s1, double* s2y, float* dw, int lddw, float* part,
                       long long part_floats, void* stream, bool bf16) {
    O3D_REQUIRE((g || dpool) && wtiles_t && (x || lf) && out && dw && part, O3D_ERR_ARG, "o3d_pw_bwd_tc: null pointer");
    O3D_REQUIRE((Cout == 64 || Cout == 128) && (Cin == 64 || Cin == 128) && (lddw & 3) == 0, O3D_ERR_ARG,
                "o3d_pw_bwd_tc: channel counts must be 64 or 128");
    O3D_REQUIRE(!lf || ((gidx || !lf->z) && (lf->z || lf->s) && lf->ldz == Cin), O3D_ERR_ARG, "o3d_pw_bwd_tc: lift descriptor");
    if (P == 0) return O3D_OK;
    const TcDy da{g, ldg, y, ldy, a, b, cc, dpool, sel, S > 0 ? S : 1, ldp, ilog2_exact(S > 0 ? S : 1)};
    cudaStream_t st = (cudaStream_t)stream;
    if (lf) {
        TcLift xb = make_tclift(lf, gidx, in_scale, in_shift, in_relu);
        const LiftView lv = xb.lv;
        if (bf16)
            return bwd_tc_impl(da, Bf16<TcLift>{xb}, wtiles_t, P, Cout, Cin, out, nullptr, &lv, in_scale, in_shift, in_relu, s1, s2y,
                               dw, lddw, part, part_floats, st);
        return bwd_tc_impl(da, xb, wtiles_t, P, Cout, Cin, out, nullptr, &lv, in_scale, in_shift, in_relu, s1, s2y, dw, lddw, part,
                           part_floats, st);
    }
    // the ReLU mask / BN-backward sums read the layer input's raw rows when the previous layer has a BN or a ReLU
    const float* yprev = (in_scale || in_relu) ? x : nullptr;
    const TcAct xb{x, Cin, in_scale, in_shift, in_relu};
    if (bf16)
        return bwd_tc_impl(da, Bf16<TcAct>{xb}, wtiles_t, P, Cout, Cin, out, yprev, nullptr, in_scale, in_shift, in_relu, s1, s2y, dw,
                           lddw, part, part_floats, st);
    return bwd_tc_impl(da, xb, wtiles_t, P, Cout, Cin, out, yprev, nullptr, in_scale, in_shift, in_relu, s1, s2y, dw, lddw, part,
                       part_floats, st);
}

extern "C" int o3d_pw_bwd_tc(const float* g, int ldg, const float* y, int ldy, const float* a, const float* b, const float* cc,
                             const float* dpool, const int32_t* sel, int S, int ldp, const void* wtiles_t, const float* x,
                             const o3d_lift_t* lf, const int32_t* gidx, const float* in_scale, const float* in_shift, int in_relu,
                             int P, int Cout, int Cin, float* out, double* s1, double* s2y, float* dw, int lddw, float* part,
                             long long part_floats, void* stream) {
    return o3d_pw_bwd_tc_prec(g, ldg, y, ldy, a, b, cc, dpool, sel, S, ldp, wtiles_t, x, lf, gidx, in_scale, in_shift, in_relu, P,
                              Cout, Cin, out, s1, s2y, dw, lddw, part, part_floats, stream, false);
}
