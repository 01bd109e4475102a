/*
 * o3d_b200.h — C ABI of libo3d_b200.so (hand-written sm_90a kernels for the Open3DSOT hot path).
 *
 * Conventions (SURVEY.md §8b):
 *   - every pointer is a DEVICE pointer unless its name ends in `_host`; the caller owns all buffers,
 *     including scratch and pre-zeroed gradient outputs — nothing is allocated inside;
 *   - float = IEEE fp32, indices = int32, tensors dense row-major in the shape given in the comment;
 *   - `stream` is a cudaStream_t passed as void*; kernels are only enqueued (no synchronisation, no
 *     host-side state), so every entry point may be captured into a CUDA graph;
 *   - return value 0 = ok, <0 = argument / CUDA error; o3d_last_error() gives the text (thread-local);
 *   - no torch types anywhere.
 *
 * The first block mirrors, one to one, the nine pybind entry points of `pointnet2_ops._ext` that the
 * reference binds at pointnet2/utils/pointnet2_utils.py:17 and calls at :56,:92,:98,:125,:162,:184,:217,
 * :237,:268 (tensor layouts and result conventions identical).  The second block holds the fused
 * supersets used by the native modules (channels-last activations).
 */
#ifndef O3D_B200_H
#define O3D_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define O3D_B200_VERSION 100

int o3d_version(void);
const char* o3d_last_error(void);
int o3d_opt_threads(int work);  /* upstream cuda_utils.h opt_n_threads(): defines the FPS tie order */
int o3d_device_sms(void);

/* ------------------------------------------------------------------------------------------------
 * Block 1 — drop-in for pointnet2_ops._ext
 * ---------------------------------------------------------------------------------------------- */

/* _ext.furthest_point_sampling(xyz, npoint)            pointnet2_utils.py:56
 * xyz (B,N,3) f32 -> idx (B,npoint) i32. Starts at index 0, skips points with |p|^2 <= 1e-3,
 * ties resolved exactly as the upstream block reduction does.  N <= 16384.                      */
int o3d_fps(const float* xyz, int B, int N, int npoint, int32_t* idx, void* stream);

/* _ext.gather_points(features, idx)                    pointnet2_utils.py:92
 * features (B,C,N), idx (B,M) -> out (B,C,M)                                                    */
int o3d_gather(const float* features, const int32_t* idx, int B, int C, int N, int M, float* out, void* stream);

/* _ext.gather_points_grad(grad_out, idx, N)            pointnet2_utils.py:98
 * grad_out (B,C,M), idx (B,M) -> grad_features (B,C,N), MUST be zero-filled by the caller       */
int o3d_gather_grad(const float* grad_out, const int32_t* idx, int B, int C, int N, int M, float* grad_features,
                    void* stream);

/* _ext.ball_query(new_xyz, xyz, radius, nsample)       pointnet2_utils.py:268
 * new_xyz (B,M,3), xyz (B,N,3) -> idx (B,M,nsample): first nsample indices in ascending order with
 * d^2 < radius^2 (strict, fp32), remaining slots = first hit, no hit = 0.                        */
int o3d_ball_query(const float* new_xyz, const float* xyz, int B, int N, int M, float radius, int nsample,
                   int32_t* idx, void* stream);

/* _ext.group_points(features, idx)                     pointnet2_utils.py:217
 * features (B,C,N), idx (B,M,S) -> out (B,C,M,S)                                                */
int o3d_group(const float* features, const int32_t* idx, int B, int C, int N, int M, int S, float* out, void* stream);

/* _ext.group_points_grad(grad_out, idx, N)             pointnet2_utils.py:237
 * grad_out (B,C,M,S), idx (B,M,S) -> grad_features (B,C,N), zero-filled by the caller           */
int o3d_group_grad(const float* grad_out, const int32_t* idx, int B, int C, int N, int M, int S, float* grad_features,
                   void* stream);

/* _ext.three_nn(unknown, known)                        pointnet2_utils.py:125
 * unknown (B,n,3), known (B,m,3) -> dist2 (B,n,3) SQUARED distances, idx (B,n,3); ties -> lower index;
 * m < 3 leaves +inf / 0 in the unused slots (upstream 1e40 cast to float).                      */
int o3d_three_nn(const float* unknown, const float* known, int B, int n, int m, float* dist2, int32_t* idx,
                 void* stream);

/* _ext.three_interpolate(features, idx, weight)        pointnet2_utils.py:162
 * features (B,c,m), idx (B,n,3), weight (B,n,3) -> out (B,c,n)                                   */
int o3d_three_interpolate(const float* features, const int32_t* idx, const float* weight, int B, int c, int m, int n,
                          float* out, void* stream);

/* _ext.three_interpolate_grad(grad_out, idx, weight, m) pointnet2_utils.py:184
 * grad_out (B,c,n) -> grad_features (B,c,m), zero-filled by the caller                          */
int o3d_three_interpolate_grad(const float* grad_out, const int32_t* idx, const float* weight, int B, int c, int n,
                               int m, float* grad_features, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Block 2 — fused supersets (channels-last activations: a feature tensor is (B, N, C), so one
 * point's channel vector is one contiguous, 16-byte-aligned row; C % 4 == 0)
 * ---------------------------------------------------------------------------------------------- */

/* QueryAndGroup.forward in one kernel (pointnet2_utils.py:299-339): ball query + xyz grouping +
 * centre subtraction (+ /radius) + feature grouping + concat.
 *   xyz (B,N,3), new_xyz (B,M,3), feat_cl (B,N,C) or NULL (C=0)
 *   -> idx (B,M,S) (may be NULL), grouped_cl (B,M,S,C+4): [features(C) | dx dy dz | 0]
 * (the reference's channel order [xyz, features] is restored by the weight packing of the MLP).  */
int o3d_ballquery_group(const float* xyz, const float* new_xyz, const float* feat_cl, int B, int N, int M, int C,
                        float radius, int nsample, int normalize_xyz, int32_t* idx, float* grouped_cl, void* stream);

/* Backward of the grouping above w.r.t. features and (optionally) coordinates.
 *   grad_grouped_cl (B,M,S,C+4), idx (B,M,S)
 *   -> grad_feat_cl (B,N,C) += ..., grad_xyz (B,N,3) += ..., grad_new_xyz (B,M,3) -= sum_s ...
 * all three accumulated with fp32 reductions (pre-zeroed by caller; any may be NULL).            */
int o3d_ballquery_group_grad(const float* grad_grouped_cl, const int32_t* idx, int B, int N, int M, int C, int S,
                             float radius, int normalize_xyz, float* grad_feat_cl, float* grad_xyz,
                             float* grad_new_xyz, void* stream);

/* PointnetFPModule's three_nn + inverse-distance weights + three_interpolate in one kernel
 * (pointnet2_modules.py:187-195): unknown (B,n,3), known (B,m,3), known_feat_cl (B,m,c)
 *   -> out_cl (B,n,c), idx (B,n,3), weight (B,n,3)  (idx/weight kept for the backward)            */
int o3d_three_nn_interpolate(const float* unknown, const float* known, const float* known_feat_cl, int B, int n, int m,
                             int c, float* out_cl, int32_t* idx, float* weight, void* stream);
int o3d_three_nn_interpolate_grad(const float* grad_out_cl, const int32_t* idx, const float* weight, int B, int n, int m,
                                  int c, float* grad_known_feat_cl, void* stream);

/* BoxAwareXCorr grouping by an explicit (top-k) index list (models/head/xcorr.py:87-90), channels-last:
 * feat_cl (B,N,C), idx (B,L) -> out_cl (B,L,C); the gradient is accumulated into a pre-zeroed (B,N,C).   */
int o3d_group_rows(const float* feat_cl, const int32_t* idx, int B, int N, int L, int C, float* out_cl, void* stream);
int o3d_group_rows_grad(const float* grad_out_cl, const int32_t* idx, int B, int N, int L, int C, float* grad_feat_cl,
                        void* stream);

/* Cross-correlation front ends (models/head/xcorr.py).  The MLP + max-pool behind either of them is a lifted stack
 * (o3d_lift_t below), which also provides the gradient of the BoxAware grouping (indices carry no gradient).
 *
 * o3d_xcorr_boxaware_fwd — BoxAwareXCorr (xcorr.py:81-88: cdist + argsort + [:k]): template_bc (B,M,D), search_bc (B,N,D),
 *   D <= 16, k <= 8 -> idx (B,N,k): the k template points with the nearest box cloud per search point, nearest first,
 *   equal distances in ascending template order; squared distances by direct differences (see csrc/xcorr.cu).
 * o3d_xcorr_p2b_fwd — P2B_XCorr's cosine map (xcorr.py:37-38): tfeat_cl (B,n1,C), sfeat_cl (B,n2,C) channels-last
 *   -> sim (B,n2,n1) = <t_i / max(|t_i|, eps), s_j / max(|s_j|, eps)>; tnorm (B,n1) / snorm (B,n2) (nullable) keep the
 *   norms for the backward.
 * o3d_xcorr_p2b_bwd — dsim (B,n2,n1) -> d_tfeat_cl (B,n1,C), d_sfeat_cl (B,n2,C) (either may be NULL; plain stores).   */
int o3d_xcorr_boxaware_fwd(const float* template_bc, const float* search_bc, int B, int M, int N, int D, int k, int32_t* idx,
                           void* stream);
int o3d_xcorr_p2b_fwd(const float* tfeat_cl, const float* sfeat_cl, int B, int n1, int n2, int C, float eps, float* sim,
                      float* tnorm, float* snorm, void* stream);
int o3d_xcorr_p2b_bwd(const float* dsim, const float* sim, const float* tfeat_cl, const float* sfeat_cl, const float* tnorm,
                      const float* snorm, int B, int n1, int n2, int C, float eps, float* d_tfeat_cl, float* d_sfeat_cl,
                      void* stream);

/* ------------------------------------------------------------------------------------------------
 * Block 3 — point-wise MLP layers (SharedMLP / Seq of the reference: 1x1 conv + BatchNorm + ReLU
 * [+ max-pool over nsample / k / template points]; pointnet2/utils/pytorch_utils.py:12-37,68-121,
 * pointnet2_modules.py:64-73, models/head/xcorr.py:47-51,98-101).
 * Activations are channels-last matrices X[P, ld] (ld % 4 == 0, 16-byte aligned rows); weights are
 * zero-padded to multiples of 4 in both dimensions.  All statistics buffers are fp64, pre-zeroed.
 * ---------------------------------------------------------------------------------------------- */

/* Y[p,n] = sum_k A(X)[p,k] * wt[k,n] (+ bias[n]),  A(v) = relu?(v*in_scale[k] + in_shift[k]) (scale/shift nullable).
 * wt is the TRANSPOSED weight [K, ldw].  Optional outputs: y (raw pre-BN, nullable), sum / sumsq (per-channel
 * batch statistics), and for S > 0 the per-group (S consecutive positions; S | 128, S | P) ymax / ymin / arg
 * (argmax | argmin << 16), each [P/S, ldp].                                                        */
int o3d_pw_fwd(const float* x, int ldx, const float* in_scale, const float* in_shift, int in_relu, const float* wt,
               int ldw, const float* bias, int P, int K, int N, float* y, int ldy, double* sum, double* sumsq, int S,
               float* ymax, float* ymin, int32_t* arg, int ldp, void* stream);

/* The layer's output gradient is given implicitly as  dY = a*g + b + cc*y  (batch-norm backward; a == NULL -> dY = g)
 * with g either dense [P, ldg] or pooled: g[p,c] = (p % S == sel[p/S,c]) ? dpool[p/S,c] : 0.
 * dgrad: out[p,n] = sum_c dY[p,c] * w[c,n]; if yprev != NULL the previous layer's ReLU mask
 *        [yprev*pscale+pshift > 0] is applied and s1 += out, s2y += out*yprev are accumulated.      */
int o3d_pw_dgrad(const float* g, int ldg, const float* y, int ldy, const float* a, const float* b, const float* cc,
                 const float* dpool, const int32_t* sel, int S, int ldp, const float* w, int ldw, int P, int Cout,
                 int Cin, float* out, int ldo, const float* yprev, int ldyp, const float* pscale, const float* pshift,
                 int prelu, double* s1, double* s2y, void* stream);

/* wgrad: dw[m,n] += sum_p dY[p,m] * A(X)[p,n]   (dw pre-zeroed, [Cout, lddw], fp32 reductions)       */
int o3d_pw_wgrad(const float* g, int ldg, const float* y, int ldy, const float* a, const float* b, const float* cc,
                 const float* dpool, const int32_t* sel, int S, int ldp, const float* x, int ldx, const float* in_scale,
                 const float* in_shift, int in_relu, int P, int Cout, int Cin, float* dw, int lddw, void* stream);

/* BatchNorm bookkeeping (torch semantics: biased variance to normalise, unbiased for running_var, momentum
 * update, num_batches_tracked += 1): scale = gamma*invstd, shift = beta - mean*scale.               */
int o3d_bn_fwd_finalize(const double* sum, const double* sumsq, double count, const float* gamma, const float* beta,
                        float* running_mean, float* running_var, long long* num_batches_tracked, float momentum,
                        float eps, int training, int C, float* scale, float* shift, float* mean, float* invstd,
                        void* stream);
/* `training`: bit 0 = batch statistics were used; bit 1 = ACCUMULATE into dgamma / dbeta instead of overwriting them. */
int o3d_bn_bwd_finalize(const double* s1, const double* s2y, double count, const float* gamma, const float* mean,
                        const float* invstd, int training, int C, float* a, float* b, float* cc, float* dgamma,
                        float* dbeta, void* stream);

/* Pooled activation: out[g,c] = relu?(scale*ysel + shift), ysel = scale >= 0 ? ymax : ymin, sel = its position. */
int o3d_pool_finalize(const float* ymax, const float* ymin, const int32_t* arg, const float* scale, const float* shift,
                      int relu, int G, int C, int ldp, float* out, int ldo, int32_t* sel, float* ysel, void* stream);
int o3d_pool_bwd_prep(const float* dout, int ldd, const float* out, int ldo, const float* ysel, int relu, int G, int C,
                      int ldp, float* dpool, double* s1, double* s2y, void* stream);
/* Dense activation and its backward preparation (g = dout * [out > 0], s1 = sum g, s2y = sum g*y).   */
int o3d_act_apply(const float* y, int ldy, const float* scale, const float* shift, int relu, int P, int C, float* out,
                  int ldo, void* stream);
int o3d_dense_bwd_prep(const float* dout, int ldd, const float* out, int ldo, const float* y, int ldy, int relu, int P,
                       int C, float* g, int ldg, double* s1, double* s2y, void* stream);

/* Tensor-core (Hopper wgmma, 3xTF32) variants of o3d_pw_fwd / o3d_pw_dgrad for >= 128 output channels and
 * K >= 32.  The weight operand is passed pre-tiled: o3d_pw_tc_pretile() rewrites a row-major matrix
 * w[rows, ldw] (rows = the GEMM's output channels, K contiguous) into per-(128-row tile, 32-wide k-block)
 * shared-memory images [hi | lo], K-major SWIZZLE_128B, that the kernel streams with cp.async.bulk.
 * forward:  rows = Cout, K = Cin   (w = the padded conv weight)
 * dgrad  :  rows = Cin,  K = Cout  (w = its transpose)                                                */
long long o3d_pw_tc_wtile_bytes(int rows, int K);
int o3d_pw_tc_pretile(const float* w, int ldw, int rows, int K, void* wtiles, void* stream);
int o3d_pw_fwd_tc(const float* x, int ldx, const float* in_scale, const float* in_shift, int in_relu, const void* wtiles,
                  const float* bias, int P, int K, int N, float* y, int ldy, double* sum, double* sumsq, int S,
                  float* ymax, float* ymin, int32_t* arg, int ldp, void* stream);
int o3d_pw_dgrad_tc(const float* g, int ldg, const float* y, int ldy, const float* a, const float* b, const float* cc,
                    const float* dpool, const int32_t* sel, int S, int ldp, const void* wtiles_t, int P, int Cout,
                    int Cin, float* out, int ldo, const float* yprev, int ldyp, const float* pscale,
                    const float* pshift, int prelu, double* s1, double* s2y, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Block 4 — a whole MLP stack (SharedMLP / Seq) per call.  The descriptor carries the raw parameter
 * pointers of the reference modules in their checkpoint layout (weight [cout, cin] row-major, BN
 * gamma/beta/running stats); packing, per-layer GEMMs, BN bookkeeping, pooling and — backward —
 * BN-backward, wgrad, dgrad and un-packing of the gradients are all enqueued by one call.
 * ---------------------------------------------------------------------------------------------- */
#define O3D_MAX_LAYERS 8

/* Row counts P at which a stack's kernel plan changes, so that a layer's arithmetic depends on which side of them P lies:
 *   O3D_TC_MIN_P_INFER / O3D_TC_MIN_P_TRAIN: below it (eval / training mode) no layer runs the tensor-core forward, every
 *     layer runs the exact-fp32 CUDA-core GEMM;
 *   O3D_TC_BWD_MIN_P: the tensor-core data gradient, which a lifted stack also needs to keep its first layer's output virtual;
 *   O3D_FWD_SKINNY_MIN_P: a CUDA-core forward layer with at most 8 input columns and no pooling streams through the skinny
 *     kernel from here on.
 * o3d_stack_plan_thresholds(d, out) (declared after o3d_stack_t below) writes to out[0 .. 3] the ones that can change the eval-mode plan of the stack `d`
 * (whatever its P) and returns how many.  A caller that needs one result at several row counts (the live tracker's occupancy
 * buckets) keeps every stack on one side of each of them.                                                           */
#define O3D_TC_MIN_P_TRAIN 128
#define O3D_TC_MIN_P_INFER 16
#define O3D_TC_BWD_MIN_P 128
#define O3D_FWD_SKINNY_MIN_P 4096

/* "Lifted" first layer.  When the first 1x1 convolution of a stack acts on GROUPED rows — QueryAndGroup
 * (pointnet2_utils.py:317-329: [xyz(idx) - centre, features(idx)]), BoxAwareXCorr's top-k grouping (xcorr.py:87-90) or
 * P2B_XCorr's [similarity, template xyz, template feature] fusion tensor (xcorr.py:39-46) — its linearity lets the
 * feature part of the convolution run ONCE per source point instead of once per (centre, neighbour) position:
 *     Y0[p, c] = Z[row(p), c] + s[p][0] * u[0][c] + s[p][1] * u[1][c] + s[p][2] * u[2][c] + s[p][3] * u[3][c]
 *       Z = W0_f . source features  (zrows x C0, computed by an ordinary one-layer stack over the source points; optional)
 *       s = up to four per-position scalars with their weight columns u: the relative coordinates (dx, dy, dz) of a set
 *           abstraction layer — applied directly, in the reference's difference-then-multiply form — or P2B's cosine
 *           similarity (optional)
 * Neither the grouped tensor nor Y0 is written to memory: Y0 exists only inside the operand loaders / epilogues of
 * the next layer's GEMMs (tensor-core path), its batch statistics come from one gather pass, and the backward is a
 * scatter of dY0 into dZ / ds / du.  Layer 0 of the descriptor then carries only BatchNorm / ReLU (weight NULL).
 * row(p) = cloud(p) * rows_per_cloud + (ridx ? ridx[p] : p % ridx_mod),  cloud(p) = p / pos_per_cloud.             */
typedef struct o3d_lift_t {
    const float* z;        /* [zrows, ldz], ldz == round4(C0), or NULL (no gathered part)             */
    int ldz;
    const int32_t* ridx;   /* [P] source row of each position, local to its cloud, or NULL            */
    int ridx_mod;          /* used when ridx == NULL                                                  */
    int rows_per_cloud;    /* Z rows per cloud                                                        */
    int pos_per_cloud;     /* positions per cloud                                                     */
    int grp;               /* work unit of the gather / scatter passes: consecutive positions per thread (power of two
                              dividing P; the ball-query group size, so that first-hit padding merges)               */
    const float* s;        /* [P, 4] (unused columns zero) or NULL                                    */
    const float* u;        /* [4, ldz] (unused rows zero) or NULL                                     */
    /* backward outputs (NULL = not wanted), all zero-filled by the caller                           */
    float* d_z;            /* [zrows, ldz]   += scatter of dY0                                        */
    float* d_s;            /* [P, 4]         += dY0 . u[j]                                            */
    float* d_u;            /* [4, ldz]       += sum_p s[p][j] * dY0[p]                                */
} o3d_lift_t;

typedef struct o3d_stack_t {
    int n_layers;   /* 1..O3D_MAX_LAYERS */
    int P;          /* positions (rows of the channels-last input)                               */
    int K0;         /* input row length (multiple of 4, zero padded)                             */
    int S;          /* pooling group size over consecutive positions (0 = dense output)          */
    int training;   /* BatchNorm uses batch statistics and updates the running ones              */
    int use_tc;     /* allow the wgmma 3xTF32 kernels where the shape qualifies: bit 0 = forward + dgrad, bit 1 = wgrad */
    int xyz_first;  /* layer-0 weight columns are [xyz(3) | features(c0)], input rows [features | dx dy dz 0] */
    int c0;         /* real feature channels of layer 0 when xyz_first                           */
    int dx_cols;    /* backward: only the first dx_cols input columns need a gradient (0 = all K0) */
    int cin[O3D_MAX_LAYERS], cout[O3D_MAX_LAYERS], relu[O3D_MAX_LAYERS], has_bn[O3D_MAX_LAYERS];
    float momentum[O3D_MAX_LAYERS], eps[O3D_MAX_LAYERS];
    const float* weight[O3D_MAX_LAYERS];
    const float* bias[O3D_MAX_LAYERS];
    const float* gamma[O3D_MAX_LAYERS];
    const float* beta[O3D_MAX_LAYERS];
    float* running_mean[O3D_MAX_LAYERS];
    float* running_var[O3D_MAX_LAYERS];
    long long* num_batches_tracked[O3D_MAX_LAYERS];
    /* backward outputs, same layouts as the parameters (NULL = not wanted) */
    float* d_weight[O3D_MAX_LAYERS];
    float* d_bias[O3D_MAX_LAYERS];
    float* d_gamma[O3D_MAX_LAYERS];
    float* d_beta[O3D_MAX_LAYERS];
    const o3d_lift_t* lift;   /* non-NULL: layer 0 is lifted (weight[0] == NULL, cout[0] = C0, K0 = round4(C0), x unused) */
    int accumulate;           /* backward: d_weight / d_bias / d_gamma / d_beta are ADDED to (the caller's persistent .grad buffers —
                                 saves one elementwise add per parameter and call); 0 = overwritten                            */
    const void* prepared;     /* non-NULL (inference only): parameter block filled by o3d_stack_prepare(); the forward then
                                 neither packs weights nor finalises BatchNorm                                            */
    int precision;            /* operands of the tensor-core forward GEMMs: 0 = 3xTF32 (default, fp32-grade), 1 = BF16 operands with
                                 FP32 accumulation.  1 is for inference on a prepared block only: o3d_stack_forward returns
                                 O3D_ERR_ARG with training, keep_for_backward or no `prepared`, and the prepare / size calls
                                 refuse a training descriptor.  The block then holds one bf16 image per weight tile (2 bytes per
                                 weight instead of 8) and the forward takes the bf16 pw_tc / sa_fused kernels.  Layers that the
                                 plan sends to the exact-fp32 CUDA-core kernels (K < 32, P < 16, ...) stay fp32 either way;
                                 accumulation, BatchNorm, ReLU, pooling and the first SA layer's coordinate term are fp32 too.
                                 2 = BF16 training: BF16 operands with FP32 accumulation for the tensor-core forward, dgrad and
                                 wgrad GEMMs.  Valid with training = 1 only (with or without keep_for_backward, and in
                                 o3d_stack_backward); the size and prepare calls refuse it for an eval-mode descriptor.  The
                                 weights are rounded to bf16 once per call when they are packed (the forward and the dgrad
                                 images, 8 KB per tile instead of 32 KB), and each GEMM input row where 3xTF32 would split it.
                                 The stored pre-BN outputs, batch statistics, BN-backward sums, ReLU masks, pooling, the split-K
                                 partial tiles and their fixed-order reduction, the lifted layer's gather / scatter passes and
                                 every CUDA-core layer stay fp32.                                                          */
} o3d_stack_t;

int o3d_stack_plan_thresholds(const o3d_stack_t* d, int* out);   /* see O3D_TC_MIN_P_INFER above */

long long o3d_stack_workspace_bytes(const o3d_stack_t* d, int backward);
/* Static-weight inference (the B=1 tracking loop): pack the weights / fold the running BN statistics once. */
long long o3d_stack_prepared_bytes(const o3d_stack_t* d);
int o3d_stack_prepare(const o3d_stack_t* d, void* block, void* stream);
/* out: [P or P/S, round4(cout_last)]; ws_fwd must stay alive (untouched) until the backward call. */
int o3d_stack_forward(const o3d_stack_t* d, const float* x, void* ws_fwd, float* out, int keep_for_backward,
                      void* stream);
/* dout: contiguous [rows, round4(cout_last)]; dx: [P, K0] or NULL (columns >= dx_cols are left undefined when
 * dx_cols > 0). */
int o3d_stack_backward(const o3d_stack_t* d, const float* x, const void* ws_fwd, void* ws_bwd, const float* out,
                       const float* dout, float* dx, void* stream);

/* A whole set-abstraction layer in ONE kernel, inference only (running BatchNorm statistics, no saved tensors): replaces the
 * body of _PointnetSAModuleBase.forward — QueryAndGroup (pointnet2/utils/pointnet2_utils.py:299-339), the SharedMLP and the
 * max-pool over nsample (pointnet2/utils/pointnet2_modules.py:58-76) — for one (grouper, mlp) scale.
 * d describes the SharedMLP in the reference's layout: xyz_first = 1, c0 = feature channels C, cin[0] = 3 + C, every cout <= 256,
 * C <= 288; P / K0 / S / lift are ignored, and training too unless precision = 1, which it refuses.  o3d_sa_fused_prepare() packs the
 * weights (pre-tiled TF32 hi | lo images, or with precision = 1 one bf16 image per tile for the BF16 kernel) and
 * folds BatchNorm + bias into per-channel scale / shift once; `block` (o3d_sa_fused_prepared_bytes() bytes) then serves every call.
 * xyz [B, N, 3], new_xyz [B, M, 3], feat_cl [B, N, ldf] channels-last (NULL iff c0 == 0), out [B * M, ldo] channels-last,
 * idx (nullable) [B, M, nsample] receives the ball-query result.  nsample must divide 64 and M be a multiple of 64 / nsample. */
long long o3d_sa_fused_prepared_bytes(const o3d_stack_t* d);
int o3d_sa_fused_prepare(const o3d_stack_t* d, void* block, void* stream);
int o3d_sa_fused_forward(const o3d_stack_t* d, const void* block, const float* xyz, const float* new_xyz, const float* feat_cl,
                         int ldf, int B, int N, int M, float radius, int nsample, int normalize, float* out, int ldo, int32_t* idx,
                         void* stream);

/* Lifted first layer (o3d_lift_t), helpers used by o3d_stack_forward/backward.
 * o3d_lift_stats : gidx[p] = global Z row of position p; sum / sumsq (nullable) += per-channel batch statistics of Y0;
 *                  y0 (nullable) receives Y0 itself [P, C0] (the CUDA-core fallback reads it as an ordinary activation).
 * o3d_lift_scatter: dY0 = a*g + b + cc*Y0 (a == NULL: dY0 = g) scattered into lf->d_z / d_cc / d_s / d_u (see o3d_lift_t);
 *                  y0 NULL = re-gather Y0 from Z.
 * o3d_pw_*_tc_lift: the tensor-core GEMMs of the layer AFTER the lifted one, reading Y0 through gidx (never stored).
 *                  wgrad: split-K into the workspace `part`, as o3d_pw_wgrad_tc2.                                       */
int o3d_lift_stats(const o3d_lift_t* lf, int P, int C0, int32_t* gidx, float* y0, double* sum, double* sumsq, void* stream);
int o3d_lift_scatter(const o3d_lift_t* lf, int P, int C0, const int32_t* gidx, const float* y0, const float* g, int ldg,
                     const float* a, const float* b, const float* cc, void* stream);
int o3d_pw_fwd_tc_lift(const o3d_lift_t* lf, const int32_t* gidx, const float* in_scale, const float* in_shift, int in_relu,
                       const void* wtiles, const float* bias, int P, int K, int N, float* y, int ldy, double* sum,
                       double* sumsq, int S, float* ymax, float* ymin, int32_t* arg, int ldp, void* stream);
int o3d_pw_dgrad_tc_lift(const float* g, int ldg, const float* y, int ldy, const float* a, const float* b, const float* cc,
                         const float* dpool, const int32_t* sel, int S, int ldp, const void* wtiles_t, int P, int Cout,
                         int Cin, float* out, int ldo, const o3d_lift_t* lf, const int32_t* gidx, const float* pscale,
                         const float* pshift, int prelu, double* s1, double* s2y, void* stream);
int o3d_pw_wgrad_tc_lift(const float* g, int ldg, const float* y, int ldy, const float* a, const float* b, const float* cc,
                         const float* dpool, const int32_t* sel, int S, int ldp, const o3d_lift_t* lf, const int32_t* gidx,
                         const float* in_scale, const float* in_shift, int in_relu, int P, int Cout, int Cin, float* dw,
                         int lddw, float* part, long long part_floats, void* stream);

/* Both gradients of one layer with Cout, Cin in {64, 128} in one kernel: the dgrad of o3d_pw_dgrad_tc(_lift) into out
 * [P, Cin] (its ReLU mask and BN-backward sums read x's raw rows when in_scale or in_relu is set, or Y0 when lf is given)
 * and the weight gradient of o3d_pw_wgrad_tc2 / o3d_pw_wgrad_tc_lift added into dw.  X is x [P, Cin] or, with lf, the lifted
 * first layer.  part: o3d_pw_wgrad_tc2_workspace_floats() floats; the partials are summed in a fixed order (deterministic). */
int o3d_pw_bwd_tc(const float* g, int ldg, const float* y, int ldy, const float* a, const float* b, const float* cc,
                  const float* dpool, const int32_t* sel, int S, int ldp, const void* wtiles_t, const float* x,
                  const o3d_lift_t* lf, const int32_t* gidx, const float* in_scale, const float* in_shift, int in_relu, int P,
                  int Cout, int Cin, float* out, double* s1, double* s2y, float* dw, int lddw, float* part,
                  long long part_floats, void* stream);

/* wgrad on the tensor core (operands transposed to K-major SWIZZLE_128B tiles), 128 x 128 tiles of dW per CTA, split over
 * positions; the per-split partial tiles go to `part` (o3d_pw_wgrad_tc2_workspace_floats() floats) and a second kernel adds
 * their sum into dw in a fixed order (deterministic).                                                               */
long long o3d_pw_wgrad_tc2_workspace_floats(void);
int o3d_pw_wgrad_tc2(const float* g, int ldg, const float* y, int ldy, const float* a, const float* b, const float* cc,
                     const float* dpool, const int32_t* sel, int S, int ldp, const float* x, int ldx,
                     const float* in_scale, const float* in_shift, int in_relu, int P, int Cout, int Cin, float* dw,
                     int lddw, float* part, long long part_floats, void* stream);

/* Adam over a flat fp32 parameter bucket (torch.optim.Adam semantics; the reference uses betas (0.5, 0.999),
 * eps 1e-6: models/base_model.py:28-36).  state = device float[2] {step count (incremented by the call), lr}.  */
int o3d_adam_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, long long n, float* state,
                  float beta1, float beta2, float eps, float weight_decay, void* stream);

/* Block 5 — box-frame crop of LiDAR scans (tracking frame loop and training-pair construction; replaces the host numpy of
 * datasets/points_utils.py generate_subwindow :223-254, cropAndCenterPC :102-124, crop_pc_axis_aligned :147-173).
 *   local[b,i,:] = R[b]^T (scans[frame[b],i,:] - center[b]);  keep[b,i] = i < count[frame[b]] && |local| < half[b] per axis
 * scans [F,N,3]; count [F] int64 or NULL (all N valid); frame [B] int64 or NULL (frame b = b); rot [B,9] row-major with
 * the box axes in its columns; half [B,3] = (l, w, h) * scale / 2 + offset.                                        */
int o3d_crop_box_frame(const float* scans, const long long* count, const long long* frame, const float* center,
                       const float* rot, const float* half, int B, int N, float* local, unsigned char* keep, void* stream);

/* The crop of o3d_crop_box_frame appended to a per-slot history (the template of shape_aggregation 'all'): for every slot b
 * with frame[b] >= 0, the points i < count[frame[b]] of scan frame[b] strictly inside half[b] in the frame of box b (the same
 * local coordinates as o3d_crop_box_frame, bit for bit) are written in scan order to hist[b, hist_count[b] + j] with
 * hist_keep set there, for positions < H only; hist_count[b] then grows by the number kept, including those that did not fit.
 * frame[b] < 0 leaves slot b untouched.  hist [B,H,3], hist_keep [B,H] bytes, hist_count [B] int64; count nullable. */
int o3d_crop_append(const float* scans, const long long* count, const long long* frame, const float* center, const float* rot,
                    const float* half, int B, int N, int H, float* hist, unsigned char* hist_keep, long long* hist_count,
                    void* stream);

/* Fixed-shape resampling of a masked candidate set (datasets/points_utils.py:24-40 regularize_pc, device form): per cloud,
 * n = #keep;  n >= size: the `size` kept candidates with the smallest keys u_perm, in ascending key order (a uniform draw
 * without replacement);  2 < n < size: draw i = the floor(u_pick[i] * n)-th kept candidate;  n <= 2: zeros.
 * points [B, N, 3], keep [B, N] (bytes, non-zero = kept), u_perm [B, N] and u_pick [B, size] uniform in [0, 1),
 * scratch [B, N] int32, out [B, size, 3], src [B, size] int64 (source index of every output point), n_out (nullable) [B] int64.
 * size <= 2048. */
int o3d_resample(const float* points, const unsigned char* keep, const float* u_perm, const float* u_pick, int B, int N, int size,
                 int32_t* scratch, float* out, long long* src, long long* n_out, void* stream);

/* Crop + resample of a shared scan for K targets in one kernel (one CTA per target; the live multi-target tracker's crops).
 * Target k's candidates are [prefix[k, 0 .. Np-1], crop of scans[frame[k]]]: element e < Np is prefix point e (already in the
 * box frame) when prefix_keep[k, e] != 0; element Np + i is point i of the scan in the frame of box k, kept when
 * i < count[frame[k]] and |local| < half[k] per axis (o3d_crop_box_frame's test and coordinates, bit for bit).  The result is
 * o3d_resample of those candidates with the keyed draws of o3d_keyed_uniform: u_perm = stream perm_stream over Np + N elements,
 * u_pick = stream pick_stream over size elements, both for (seed, key[k], key_frame[k]) — bitwise the same output and survivor
 * count as crop_box_frame -> keyed_uniform -> resample on the concatenation, without its (K, Np + N) intermediates.
 * scans [S, N, 3], count [S] int64 or NULL, frame [K] int64, center [K, 3], rot [K, 9], half [K, 3] (all may be NULL when N = 0:
 * prefix only); prefix [K, Np, 3], prefix_keep [K, Np] bytes (NULL when Np = 0); key / key_frame [K] int64;
 * scratch [K, 2, Np + N] int32 (written for survivors only); out [K, size, 3]; n_out (nullable) [K] int64.
 * K <= 65535, 1 <= size <= 2048. */
int o3d_crop_resample(const float* scans, const long long* count, const long long* frame, const float* center, const float* rot,
                      const float* half, int N, const float* prefix, const unsigned char* prefix_keep, int Np, unsigned int seed,
                      const long long* key, const long long* key_frame, int perm_stream, int pick_stream, int K, int size,
                      int32_t* scratch, float* out, long long* n_out, void* stream);

/* Scan ingest for the live tracker's feeds (one sensor or recorded scene each): every feed that gets a new scan this step hands
 * its raw point rows, as stored, and the reader's affine transforms; one launch writes them all as float32 xyz.
 * Descriptor i: rows [rows, stride] of float32 (is_f64 = 0) or float64 (is_f64 = 1) at byte `offset` of the slab, x y z first;
 * each row is moved through xf[0], then xf[1] (the first n_xf of them; row-major 3x4 [R | t]: p <- R p + t) in float64 and written
 * to scans[feed, half, 0 .. rows-1] as float32; count[feed, half] = rows.
 * desc_host: the descriptors in host memory, checked before the launch; desc: the same n_desc descriptors in device memory (the
 * kernel reads these).  scans [feeds, 2, max_points, 3] fp32, count [feeds, 2] int64.  Checks: feed in [0, feeds), half 0 / 1,
 * stride in [3, 16], n_xf in [0, 2], rows in [0, max_points], the rows inside [0, slab_bytes) at an element-aligned offset, no two
 * descriptors with the same (feed, half), n_desc <= 2 * feeds.  n_desc = 0: nothing is launched. */
typedef struct {
    long long offset;  /* byte offset of the first row in the slab */
    int rows;          /* number of rows (points) */
    int stride;        /* values per row */
    int is_f64;        /* 0: float32 rows, 1: float64 rows */
    int feed;          /* destination feed */
    int half;          /* destination half of the feed's ping-pong pair */
    int n_xf;          /* transforms applied, in order */
    double xf[2][12];  /* row-major 3x4 [R | t] */
} o3d_scan_desc_t;
int o3d_scan_ingest(const o3d_scan_desc_t* desc_host, const o3d_scan_desc_t* desc, int n_desc, const void* slab, long long slab_bytes,
                    int feeds, int max_points, float* scans, long long* count, void* stream);

/* In-box point counts of the live tracker's evidence (nuscenes points_in_box as the inclusive test in the box frame):
 *   n_in[k] = #{ i < count[frame[k]] : |R[k]^T (scans[frame[k], i, :] - center[k])| <= half[k] per axis }
 * with the box-frame coordinates in fp32, (dx R[0][j] + dy R[1][j]) + dz R[2][j], every operation rounded on its own (no FMA
 * contraction): tracking/boxes.py box_point_counts bit for bit, so the counts equal it exactly.  n_in is zeroed inside the call
 * (an async memset, then one launch); the per-block counts are summed with integer atomics, so the result does not depend on
 * the order blocks run in.  No host sync; capturable.  scans [S, N, 3], count [S] int64 or NULL (all N valid), frame [K]
 * int64, center [K, 3], rot [K, 9] row-major with the box axes in its columns, half [K, 3], n_in [K] int32.  K <= 65535. */
int o3d_box_points(const float* scans, const long long* count, const long long* frame, const float* center, const float* rot,
                   const float* half, int N, int K, int* n_in, void* stream);

/* The live tracker's per-row write-back (tracking/multi_tracker.py track_update, the tensor formulation it equals bit for bit):
 * row i < b reads its slot's state at src[i] and writes it at dst[i] (slots are distinct; padding rows read an idle row and write
 * one nothing reads).  With adv[i] = 0 the state is copied unchanged.  With adv[i] = 1 (P = the network's box: center / rot,
 * n = points[i], t' = t[src] + 1):
 *   points, score <- n, score[i];  first_flag <- 0;  t <- t';  box <- P
 *   rule:  hit = n >= min_points;  misses <- hit ? 0 : misses + 1;  lost <- lost | misses >= patience (every row)
 *   coast (needs rule), gap = (float)(t' - hit_t):
 *     hit:  v = (P.c - hit_c) / gap;  vel <- hit_t == 0 ? v : alpha v + beta vel;  hit_c <- P.c;  hit_t <- t'
 *     miss: box centre <- hit_c + vel gap, rotation the previous one (vel, hit_c, hit_t hold)
 *     coasting <- !hit && !lost
 * Detection matches (optional; all four fields null = none, the behaviour above): match [b] int32, the row's detection from
 * o3d_box_associate (-1: none), match_box [b, 12] its centre and row-major rotation.  An advanced row takes detection <- match[i]
 * and reacquired <- (match[i] >= 0 and a miss under the rule); a re-acquired row is handled as a hit whose box is the detection's
 * centre and rotation (the slot keeps its wlh): misses <- 0, and with coast the velocity sample, hit_c / hit_t and coasting
 * follow the hit rules with P.c = the detection's centre.  A matched hit writes P as without matches.
 * Every fp32 operation is rounded on its own (no FMA contraction).  One thread per row, no atomics, no host sync, capturable.
 * Slot state: box_c [., 3], box_r [., 9] row-major, t / hit_t int64, first_flag / score fp32, points / misses / detection int32,
 * lost / coasting / reacquired bool (one byte), vel / hit_c [., 3].  Refused: a null descriptor or pointer (the match fields:
 * some but not all null), b outside 0 .. 65535, rule / coast not 0 / 1, coast without rule, min_points < 0 or patience < 1 with
 * the rule, alpha outside (0, 1] with coast.  b = 0 launches nothing. */
typedef struct o3d_track_update_t {
    int b;
    const long long* src;
    const long long* dst;
    const unsigned char* adv;
    const float* center;       /* [b, 3] the network's box */
    const float* rot;          /* [b, 9] */
    const int* points;         /* [b] its in-box count */
    const float* score;        /* [b] */
    float* box_c;              /* slot state */
    float* box_r;
    long long* t;
    float* first_flag;
    int* slot_points;
    float* slot_score;
    int* misses;
    unsigned char* lost;
    float* vel;
    float* hit_c;
    long long* hit_t;
    unsigned char* coasting;
    int rule;
    int min_points;
    int patience;
    int coast;
    float alpha;
    float beta;
    const int* match;          /* [b] o3d_box_associate's match, or NULL (no detections) */
    const float* match_box;    /* [b, 12] */
    int* slot_detection;       /* slot state: the last advance's detection index, -1 for none */
    unsigned char* slot_reacquired;
} o3d_track_update_t;
int o3d_track_update(const o3d_track_update_t* p, void* stream);

/* Detection matching of the live tracker (tracking/multi_tracker.py associate_tensors, which it equals exactly), one CTA per
 * feed, run before o3d_track_update in the same step.  Row i < b of the step belongs to feed[i] and takes part when adv[i]; it
 * is matched against the centre it would write without detections, pred (o3d_track_update's arithmetic, csrc/track_predict.cuh):
 * P = center[i] on a hit or without the rule (hit = points[i] >= min_points), and with coast on a miss hit_c + vel * gap with
 * gap = (float)(t[src[i]] + 1 - hit_t[src[i]]) from the slot state at src[i].  Feed f's detections this advance are
 * det[f, d, :] for d < count[f] when fed[f] != 0 (none otherwise); a row is 16 floats: centre (3), wlh (3), row-major rotation
 * with the box axes in its columns (9), score.  Distance: d2 = dx*dx + dy*dy over the plane axes axis0 / axis1, each operation
 * rounded on its own; a pair is a candidate when d2 <= gate2.  Per feed, the candidates are taken greedily in ascending
 * (d2, row, detection) order, a pair accepted when its row and its detection are both still free; score plays no part.
 * Writes, for every row: pred [b, 3] (NaN for a row that does not take part), match [b] int32 (the detection, -1 for none),
 * match_box [b, 12] (the matched detection's centre and rotation; zeros without a match).  For every fed feed and d < count[f]:
 * rec_det[f, d] <- det[f, d], rec_slot[f, d] <- src of the row detection d matched, or -1; rec_count[f] <- count[f].  Rows
 * d >= count[f] and the records of a feed that is not fed are left as they are.  count is read on the device: the caller checks 0 <= count[f] <= D before it
 * uploads it.  No atomics, no host sync, capturable.  Refused: a null descriptor or pointer, b outside 0 .. 65535, F < 1, D
 * outside 1 .. 1024, gate2 not finite or <= 0, axis0 / axis1 not distinct values in {0, 1, 2}, rule / coast not 0 / 1, coast
 * without rule, min_points < 0 with the rule.  b = 0 launches nothing. */
typedef struct o3d_box_associate_t {
    int b;                     /* rows of the step */
    int F;                     /* feeds */
    int D;                     /* detections per feed, at most (the row stride of det / rec_det / rec_slot) */
    int axis0, axis1;          /* the plane the distance is measured in */
    float gate2;               /* squared gate, float32 */
    int rule, min_points, coast;
    const long long* src;      /* [b] slot of each row */
    const long long* feed;     /* [b] feed of each row */
    const unsigned char* adv;  /* [b] */
    const float* center;       /* [b, 3] the network's box */
    const int* points;         /* [b] its in-box count */
    const long long* t;        /* slot state (read at src[i]): frame counter before this advance */
    const long long* hit_t;
    const float* hit_c;        /* [., 3] */
    const float* vel;          /* [., 3] */
    const long long* fed;      /* [F] the feed got a scan this advance */
    const int* count;          /* [F] detections of the feed this advance */
    const float* det;          /* [F, D, 16] */
    float* pred;               /* [b, 3] out */
    int* match;                /* [b] out */
    float* match_box;          /* [b, 12] out */
    float* rec_det;            /* [F, D, 16] per-feed records */
    int* rec_count;            /* [F] */
    int* rec_slot;             /* [F, D] */
} o3d_box_associate_t;
int o3d_box_associate(const o3d_box_associate_t* p, void* stream);

/* Target births of the live tracker (tracking/multi_tracker.py birth_tensors, which it equals exactly), one CTA for every feed,
 * run after o3d_box_associate and o3d_track_update in the same step.  The birth list holds R entries (birth_slot[e],
 * birth_feed[e]): the slots the host reserved for this advance, grouped by ascending feed, padded with birth_feed = -1.  Feed
 * f's entries are its r_f reserved slots in order.  For every feed with r_f > 0, fed[f] != 0 and count[f] > 0, detection
 * d < count[f] of det[f] is a candidate when rec_slot[f, d] < 0 (o3d_box_associate left it unmatched), its score det[f, d, 15]
 * >= min_score, and d2 > gate2 to the pred centre of every row i < b with feed[i] == f and adv[i] (d2 = dx*dx + dy*dy over the
 * plane axes, dx = pred - det, each operation rounded on its own).  The candidates are ranked by descending score (-0 as +0),
 * then ascending d, and walked in rank order: a candidate whose d2 (candidate minus born) to a candidate already born from
 * this feed is <= gate2 is passed over; otherwise it is born into the feed's next reserved slot; the walk ends when the slots
 * run out.  The n-th birth of the call (feeds ascending, then rank) gets id = id_base + next + n, and next grows by the births.
 * A birth at entry e, slot k, detection d writes the slot state add(id, box, feed=f) writes (box from the row: centre, wlh,
 * row-major rotation; first_flag 1, active 1, key id, t 0, slot_feed f, points -1, score NaN, misses 0, lost 0, vel 0,
 * hit_c = centre, hit_t 0, coasting 0, detection -1, reacquired 0), rec_slot[f, d] <- k and log[e] = (k, id, f, d); every
 * other log entry is (-1, -1, -1, -1).  The first-frame crop is the caller's.  No atomics, no host sync, capturable.
 * Refused: a null descriptor or pointer (feed / adv / pred may be null when b = 0), b outside 0 .. 65535, F < 1, D outside
 * 1 .. 1024, R outside 1 .. 65535, gate2 not finite or <= 0, min_score not finite, axis0 / axis1 not distinct values in
 * {0, 1, 2}, id_base < 0. */
typedef struct o3d_track_birth_t {
    int b;                     /* rows of the step (0: a step that advances no row) */
    int F;                     /* feeds */
    int D;                     /* detections per feed, at most (the row stride of det / rec_slot) */
    int R;                     /* birth list entries */
    int axis0, axis1;          /* the plane the distance is measured in */
    float gate2;               /* squared gate, float32 */
    float min_score;
    long long id_base;         /* the first born id */
    const long long* feed;     /* [b] feed of each row */
    const unsigned char* adv;  /* [b] */
    const float* pred;         /* [b, 3] o3d_box_associate's pred */
    const long long* fed;      /* [F] */
    const int* count;          /* [F] */
    const float* det;          /* [F, D, 16] */
    int* rec_slot;             /* [F, D] the matching's records, updated for the born detections */
    const long long* birth_slot;   /* [R] */
    const long long* birth_feed;   /* [R] */
    long long* next;           /* [1] births so far */
    long long* log;            /* [R, 4] out */
    float* box_c;              /* slot state, as o3d_track_update's */
    float* box_s;
    float* box_r;
    float* first_flag;
    unsigned char* active;
    long long* key;
    long long* t;
    long long* slot_feed;
    int* points;
    float* score;
    int* misses;
    unsigned char* lost;
    float* vel;
    float* hit_c;
    long long* hit_t;
    unsigned char* coasting;
    int* detection;
    unsigned char* reacquired;
} o3d_track_birth_t;
int o3d_track_birth(const o3d_track_birth_t* p, void* stream);

/* Block 6 — split evaluation with K tracklets in flight (tracking/batched_tracker.py).
 *
 * o3d_keyed_uniform: out [K, n] uniform [0, 1) draws of one stream.  Slot k's element e is a pure function of
 *   (seed, tracklet[k], frame[k], stream, e): Philox4x32-10 (cuRAND's constants) with key = (seed, (uint32) tracklet[k]) and
 *   counter = (e / 4, (uint32) frame[k], stream, 0); word e % 4 of the block -> (w >> 8) * 2^-24.  tracklet / frame [K] int64.
 *   K <= 65535.
 * o3d_track_metrics: utils/metrics.py estimateOverlap(gt, result, dim, up_axis) and estimateAccuracy(...) in fp64, one slot per
 *   thread.  The result box is the slot's fp32 state: center [K, 3], rot [K, 9] (row-major), wlh [K, 3]; the ground truth is fp64,
 *   indexed by the slot's pool frame: gt_center [F, 3], gt_rot [F, 9], gt_wlh [F, 3], frame [K] int64 (< 0 = idle slot: writes
 *   nothing).  dim = 2 (bird's-eye IoU, distance over the up axis components) or 3.  up_mask: bit i set <=> up_axis[i] != 0.
 *   Writes overlap[frame[k]] and distance[frame[k]] ([F] fp64).                                                               */
int o3d_keyed_uniform(const long long* tracklet, const long long* frame, int K, unsigned int seed, int stream, int n, float* out,
                      void* cuda_stream);
int o3d_track_metrics(const float* center, const float* rot, const float* wlh, const double* gt_center, const double* gt_rot,
                      const double* gt_wlh, const long long* frame, int K, int dim, int up_mask, double* overlap, double* distance,
                      void* stream);

#ifdef __cplusplus
}
#endif
#endif /* O3D_B200_H */
