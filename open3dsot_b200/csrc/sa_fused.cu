// A whole PointNet++ set-abstraction layer in ONE kernel — inference (static weights, running BatchNorm statistics).
//
// Replaces, for eval-mode forward passes, the body of _PointnetSAModuleBase.forward (pointnet2/utils/pointnet2_modules.py:58-76):
//   QueryAndGroup (ball_query + 2x group_points + centre subtraction [+ /radius] + cat, pointnet2_utils.py:299-339),
//   the SharedMLP (conv1x1 + BatchNorm(running stats) + ReLU, pt_utils.py) and the max-pool over nsample (F.max_pool2d).
// The training path (stack.cu: lifted first layer, batch statistics, saved tensors for the backward) keeps its multi-kernel
// form; this kernel is what the B = 1 tracking loop and model.eval() forward passes run.
//
// One CTA owns 64 positions = 64 / nsample neighbouring centres of one cloud and carries them through every layer:
//   A. the cloud's coordinates are staged into shared memory, one warp per centre runs the ball query (same code and order
//      as ball_query.cu) and keeps idx[64] and (dx, dy, dz)[64] in shared memory;
//   B. the 64 neighbour feature rows are gathered (coalesced 128-byte segments), split into TF32 hi / lo parts and stored as
//      the K-major SWIZZLE_128B activation operand (k-blocks of 32 channels: hi [64 x 128 B] | lo [64 x 128 B]);
//   C. per layer, the two warpgroups issue 3xTF32 wgmma (M = the 64 positions, K = 8; warpgroup h takes output channels
//      h*64 .. h*64+63 of a one-tile layer, or the whole 128-channel tile h of a two-tile layer) over all k-blocks, weights
//      arriving as pre-tiled hi | lo images (o3d_sa_fused_prepare) through a bulk-copy ring that runs ahead across layers;
//      accumulators live in registers.  The epilogue adds the coordinate term of the first layer W0[:, 0:3] . (dx, dy, dz)
//      with plain FMAs (exact fp32 — the same split as the training path's lifted first layer), applies the folded
//      BatchNorm + ReLU and writes the result, hi / lo split, over the activation operand IN PLACE once every MMA of the
//      layer has retired: the layer's output never leaves the SM;
//   D. the last layer's result is staged [position][channel] over the (then dead) operand and weight ring, and one thread
//      per channel max-pools each centre's nsample positions and stores one channels-last row per centre.
// HBM / L2 traffic per CTA: the cloud's coordinates, 64 feature rows, the weight images, 64 / nsample output rows.
//
//   warps 0-7: query / gather / MMA / epilogue (two warpgroups) | 8: weight streamer
#include "common.cuh"
#include "ball_query.cuh"
#include "tc_ptx.cuh"
#include "../../include/o3d_b200.h"

namespace {

constexpr int SF_POS = 64;                  // positions per CTA
constexpr int SF_THREADS = 288;
constexpr int SF_ACT_KB = 2 * SF_POS * 128; // bytes per activation k-block: hi | lo
constexpr int SF_WTILE = 2 * TILE_BYTES;    // one weight tile (128 channels x 32 k): hi | lo
// BF16 variant: one bf16 image per k-block / tile instead of hi | lo, rows of 64 bytes (SWIZZLE_64B)
template <bool BF> constexpr int SF_ACT_KB_OF = BF ? SF_POS * TC_BF_ROW : SF_ACT_KB;
template <bool BF> constexpr int SF_WTILE_OF = BF ? BF_TILE_BYTES : SF_WTILE;
constexpr int SF_MAX_SLOTS = 6;
constexpr int SF_MISC = 128 + SF_POS * 4 + SF_POS * 16;   // barriers | idx | rel

struct SfLayer {
    int cout, n_mt, nkb, relu, mma;
    uint32_t vec_off;      // floats from the block start: scale[n_mt * 128] | shift[n_mt * 128]
};
struct SfParams {
    int n, Cp, ldf, N, M, S, BM;
    float radius, radius2;
    int normalize;
    int act_bytes, nslot;
    uint32_t wx_off;       // floats: W0's coordinate columns, [3][n_mt0 * 128]
    uint32_t tiles_off;    // bytes: weight tiles in consumption order (layer, channel tile, k-block)
    SfLayer l[O3D_MAX_LAYERS];
};

__device__ __forceinline__ float2 ld2g(const float* p) { return __ldg(reinterpret_cast<const float2*>(p)); }
__device__ __forceinline__ void sts_v4(uint32_t a, const float4& v) {
    asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(a), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ void sts_v2(uint32_t a, const uint2& v) {
    asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(a), "r"(v.x), "r"(v.y) : "memory");
}

// One layer on the two warpgroups.  NT = output channels per warpgroup: 64 (a one-tile layer, split) or 128 (tile h).
// Every warpgroup walks every weight tile of the layer (waits for it, releases it) so that the ring's phases stay in step.
// BF: bf16 operands (one wgmma k16 pair per k-block), the layer's output rounded to bf16 where the 3xTF32 path splits it.
template <int NT, bool BF>
__device__ __forceinline__ void sf_layer(const SfParams& prm, int l, uint8_t* act, uint8_t* ring, uint64_t* full, uint64_t* empty,
                                         int& slot, int& phase, const uint8_t* __restrict__ block, const float4* s_rel, int g0,
                                         float* __restrict__ out, int ldo) {
    const SfLayer& L = prm.l[l];
    constexpr int ACT_KB = SF_ACT_KB_OF<BF>, WTILE = SF_WTILE_OF<BF>;
    const int h = threadIdx.x >> 7, w = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
    float acc[NT / 2];
#pragma unroll
    for (int i = 0; i < NT / 2; ++i) acc[i] = 0.f;
    if (L.mma) {
        for (int mt = 0; mt < L.n_mt; ++mt) {
            for (int kb = 0; kb < L.nkb; ++kb) {
                o3d_mbar_wait(full + slot, phase);
                if (NT == 64 || mt == h) {
                    const uint32_t wb = o3d_smem_u32(ring + slot * WTILE) + (NT == 64 ? h * (WTILE / (BF ? 2 : 4)) : 0);
                    const uint32_t ab = o3d_smem_u32(act + kb * ACT_KB);
                    wgmma_fence_acc(acc);
                    wgmma_fence();
                    if constexpr (BF)
                        wgmma_bf16_kblock<NT>(acc, make_desc_sw64(ab), make_desc_sw64(wb), kb == 0);
                    else
                        wgmma_3xtf32_kblock<NT>(acc, make_desc(ab), make_desc(ab + SF_ACT_KB / 2), make_desc(wb),
                                                make_desc(wb + TILE_BYTES), kb == 0);
                    wgmma_commit();
                    wgmma_wait<0>();
                    wgmma_fence_acc(acc);
                }
                __syncwarp();
                if (lane == 0) o3d_mbar_arrive(empty + slot);
                if (++slot == prm.nslot) { slot = 0; phase ^= 1; }
            }
        }
    }
    asm volatile("bar.sync 1, 256;" ::: "memory");   // every MMA reading the operand has retired: it may be overwritten
    const bool first = l == 0, last = l == prm.n - 1;
    const int next_nkb = last ? 0 : prm.l[l + 1].nkb;
    const int ldv = L.n_mt * 128;                     // scale | shift (and W0's coordinate columns) per channel
    const int lds = ldv + 8;                          // last layer: staged [position][channel] row stride
    const float* vecs = reinterpret_cast<const float*>(block);
    float* stg = reinterpret_cast<float*>(act);
    const float floor_v = L.relu ? 0.f : -INFINITY;
    float4 rel[2] = {};
    if (first) {
        rel[0] = s_rel[16 * w + (lane >> 2)];
        rel[1] = s_rel[16 * w + (lane >> 2) + 8];
    }
#pragma unroll
    for (int j = 0; j < NT / 8; ++j) {
        const int ch = h * NT + 8 * j + 2 * (lane & 3);   // this thread's channels ch, ch + 1
        if (!last && (ch >> 5) >= next_nkb) continue;     // padding no later layer reads (uniform over the warp)
        const float2 sc = ld2g(vecs + L.vec_off + ch), sh = ld2g(vecs + L.vec_off + ldv + ch);
        float2 wx0 = make_float2(0.f, 0.f), wx1 = wx0, wx2 = wx0;
        if (first) {
            wx0 = ld2g(vecs + prm.wx_off + ch);
            wx1 = ld2g(vecs + prm.wx_off + ldv + ch);
            wx2 = ld2g(vecs + prm.wx_off + 2 * ldv + ch);
        }
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const int pos = 16 * w + (lane >> 2) + 8 * r;
            float a0 = acc[4 * j + 2 * r], a1 = acc[4 * j + 2 * r + 1];
            if (first) {
                a0 = fmaf(wx2.x, rel[r].z, fmaf(wx1.x, rel[r].y, fmaf(wx0.x, rel[r].x, a0)));
                a1 = fmaf(wx2.y, rel[r].z, fmaf(wx1.y, rel[r].y, fmaf(wx0.y, rel[r].x, a1)));
            }
            const float v0 = fmaxf(fmaf(a0, sc.x, sh.x), floor_v), v1 = fmaxf(fmaf(a1, sc.y, sh.y), floor_v);
            if (!last && BF) {
                *reinterpret_cast<uint32_t*>(act + (ch >> 5) * ACT_KB + sw64(pos, (ch & 31) >> 3) + (ch & 7) * 2) = pack_bf16x2(v0, v1);
            } else if (!last) {
                uint8_t* dst = act + (ch >> 5) * SF_ACT_KB + sw128(pos, (ch & 31) >> 2) + (ch & 3) * 4;
                const float h0 = hi1(v0), h1 = hi1(v1);
                *reinterpret_cast<float2*>(dst) = make_float2(h0, h1);
                *reinterpret_cast<float2*>(dst + SF_ACT_KB / 2) = make_float2(v0 - h0, v1 - h1);
            } else {
                *reinterpret_cast<float2*>(stg + pos * lds + ch) = make_float2(v0, v1);
            }
        }
    }
    if (!last) {
        o3d_fence_proxy_async();                      // generic-proxy stores -> visible to the next layer's wgmma
        asm volatile("bar.sync 1, 256;" ::: "memory");
        return;
    }
    asm volatile("bar.sync 1, 256;" ::: "memory");
    // ---- D. max-pool over each centre's nsample positions: thread = channel
    const int ch = threadIdx.x;
    const int S = prm.S;
    if (ch >= ((L.cout + 31) & ~31) || ch >= ldo) return;
    const bool real = ch < L.cout;
    for (int g = 0; g < SF_POS / S; ++g) {
        float mx = -INFINITY;
        for (int p = g * S; p < (g + 1) * S; ++p) mx = fmaxf(mx, stg[p * lds + ch]);
        const int gg = g0 + g;
        if (gg < prm.BM) out[(size_t)gg * ldo + ch] = real ? mx : 0.f;
    }
}

template <bool BF>
__global__ void __launch_bounds__(SF_THREADS, 1)
    sa_fused_kernel(const SfParams prm, const uint8_t* __restrict__ block, const float* __restrict__ xyz,
                    const float* __restrict__ new_xyz, const float* __restrict__ feat, float* __restrict__ out, int ldo,
                    int32_t* __restrict__ idx_out) {
    constexpr int ACT_KB = SF_ACT_KB_OF<BF>, WTILE = SF_WTILE_OF<BF>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint8_t* act = smem;
    uint8_t* ring = smem + prm.act_bytes;
    uint8_t* misc = ring + prm.nslot * WTILE;
    uint64_t* full = reinterpret_cast<uint64_t*>(misc);       // [SF_MAX_SLOTS] weight tile landed
    uint64_t* empty = full + SF_MAX_SLOTS;                    // [SF_MAX_SLOTS] both warpgroups are done with the slot
    int32_t* s_idx = reinterpret_cast<int32_t*>(misc + 128);
    float4* s_rel = reinterpret_cast<float4*>(misc + 128 + SF_POS * 4);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nslot = prm.nslot;
    const bool mma0 = prm.l[0].mma != 0;

    if (threadIdx.x == 0) {
        for (int s = 0; s < SF_MAX_SLOTS; ++s) {
            o3d_mbar_init(full + s, 1);
            o3d_mbar_init(empty + s, 8);
        }
        o3d_fence_mbar_init();
    }
    __syncthreads();

    if (warp == 8) {
        // ===================================================== weight streamer: runs ahead of the MMAs, across layers
        if (lane == 0) {
            const uint8_t* src = block + prm.tiles_off;
            int slot = 0, phase = 0;
            for (int l = 0; l < prm.n; ++l) {
                const SfLayer& L = prm.l[l];
                if (!L.mma) continue;
                for (int t = 0; t < L.n_mt * L.nkb; ++t) {
                    o3d_mbar_wait(empty + slot, phase ^ 1);
                    o3d_mbar_expect_tx(full + slot, WTILE);
                    o3d_bulk_g2s(ring + slot * WTILE, src, WTILE, full + slot);
                    src += WTILE;
                    if (++slot == nslot) { slot = 0; phase ^= 1; }
                }
            }
        }
    } else {
        // ===================================================== query / gather / MMA / epilogue (256 threads)
        const int tid = threadIdx.x;
        const int S = prm.S, N = prm.N, M = prm.M;
        const int cpc = SF_POS / S;                     // centres of this CTA
        const int g0 = blockIdx.x * cpc;                // first centre, global over B * M (M % cpc == 0: one cloud per CTA)
        const int b = g0 / M;
        // ---- A. ball query
        float* s_xyz = reinterpret_cast<float*>(act);
        const float* cloud = xyz + (size_t)b * N * 3;
        for (int i = tid; i < 3 * N; i += 256) s_xyz[i] = __ldg(cloud + i);
        asm volatile("bar.sync 1, 256;" ::: "memory");
        for (int ci = warp; ci < cpc; ci += 8) {
            const int g = g0 + ci;
            int32_t* o = s_idx + ci * S;
            if (g < prm.BM) {
                const float* c = new_xyz + (size_t)g * 3;
                const float cx = __ldg(c), cy = __ldg(c + 1), cz = __ldg(c + 2);
                warp_ball_query(s_xyz, N, cx, cy, cz, prm.radius2, S, o, lane);
                __syncwarp();
                for (int i = lane; i < S; i += 32) {
                    const int k = o[i];
                    float dx = __fsub_rn(s_xyz[k * 3 + 0], cx), dy = __fsub_rn(s_xyz[k * 3 + 1], cy),
                          dz = __fsub_rn(s_xyz[k * 3 + 2], cz);
                    if (prm.normalize) {
                        dx = __fdiv_rn(dx, prm.radius);
                        dy = __fdiv_rn(dy, prm.radius);
                        dz = __fdiv_rn(dz, prm.radius);
                    }
                    s_rel[ci * S + i] = make_float4(dx, dy, dz, 0.f);
                    if (idx_out) idx_out[(size_t)g * S + i] = k;
                }
            } else {
                for (int i = lane; i < S; i += 32) {
                    o[i] = 0;
                    s_rel[ci * S + i] = make_float4(0.f, 0.f, 0.f, 0.f);
                }
            }
            __syncwarp();
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");   // idx / rel complete; the staged coordinates are dead from here on
        // ---- B. gather the feature rows into the activation operand
        if (mma0) {
            const int chunk = tid & 7, r0 = tid >> 3;    // rows r0 and r0 + 32, 16-byte chunk `chunk` of every k-block
            const float* f0 = feat + ((size_t)b * N + s_idx[r0]) * prm.ldf + chunk * 4;
            const float* f1 = feat + ((size_t)b * N + s_idx[r0 + 32]) * prm.ldf + chunk * 4;
            const uint32_t o0 = BF ? sw64(r0, chunk >> 1) + (chunk & 1) * 8 : sw128(r0, chunk);
            const uint32_t o1 = BF ? sw64(r0 + 32, chunk >> 1) + (chunk & 1) * 8 : sw128(r0 + 32, chunk);
            const int nkb = prm.l[0].nkb;
            for (int kb0 = 0; kb0 < nkb; kb0 += 4) {
                float4 v0[4], v1[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int k = (kb0 + j) * 32 + chunk * 4;
                    const bool on = kb0 + j < nkb && k < prm.Cp;
                    v0[j] = on ? ld4g(f0 + (kb0 + j) * 32) : make_float4(0.f, 0.f, 0.f, 0.f);
                    v1[j] = on ? ld4g(f1 + (kb0 + j) * 32) : make_float4(0.f, 0.f, 0.f, 0.f);
                }
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    if (kb0 + j >= nkb) break;
                    const uint32_t hi = o3d_smem_u32(act) + (uint32_t)((kb0 + j) * ACT_KB);
                    if constexpr (BF) {
                        sts_v2(hi + o0, pack_bf16x4(v0[j]));
                        sts_v2(hi + o1, pack_bf16x4(v1[j]));
                    } else {
                        const uint32_t lo = hi + SF_ACT_KB / 2;
                        sts_v4(hi + o0, hi_part(v0[j]));
                        sts_v4(lo + o0, lo_part(v0[j]));
                        sts_v4(hi + o1, hi_part(v1[j]));
                        sts_v4(lo + o1, lo_part(v1[j]));
                    }
                }
            }
        }
        o3d_fence_proxy_async();
        asm volatile("bar.sync 1, 256;" ::: "memory");   // the first layer's operand is complete
        // ---- C / D. per layer: MMAs -> (+ coordinate term) -> BatchNorm + ReLU -> next operand | max-pool
        int slot = 0, phase = 0;
        for (int l = 0; l < prm.n; ++l) {
            if (prm.l[l].n_mt == 2) sf_layer<128, BF>(prm, l, act, ring, full, empty, slot, phase, block, s_rel, g0, out, ldo);
            else sf_layer<64, BF>(prm, l, act, ring, full, empty, slot, phase, block, s_rel, g0, out, ldo);
        }
    }
}

// ---- parameter block ------------------------------------------------------------------------------------------------
struct SfPackLayer {
    const float *w, *bias, *gamma, *beta, *mean, *var;
    float eps;
    int cout, cin, col0 /* first source column of the tiled part */, kreal /* tiled source columns */, nkb, n_mt, has_bn, mma;
    uint32_t vec_off;
    size_t tile_off;
};
struct SfPackArgs { SfPackLayer l[O3D_MAX_LAYERS]; uint32_t wx_off; int bf16; };

// blockIdx.y = layer; a thread owns 4 consecutive k of one (padded) output channel
__global__ void sa_fused_pack_kernel(const SfPackArgs args, uint8_t* __restrict__ block) {
    const SfPackLayer& L = args.l[blockIdx.y];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int rows = L.n_mt * 128;
    float* vec = reinterpret_cast<float*>(block) + L.vec_off;
    if (i < rows) {
        float sc = 0.f, sh = 0.f;
        if (i < L.cout) {
            sc = 1.f;
            if (L.has_bn) {
                const float istd = 1.0f / sqrtf(L.var[i] + L.eps);
                sc = (L.gamma ? L.gamma[i] : 1.f) * istd;
                sh = (L.beta ? L.beta[i] : 0.f) - L.mean[i] * sc;
            }
            if (L.bias) sh = fmaf(sc, L.bias[i], sh);
        }
        vec[i] = sc;
        vec[rows + i] = sh;
        if (blockIdx.y == 0) {
            float* wx = reinterpret_cast<float*>(block) + args.wx_off;
#pragma unroll
            for (int j = 0; j < 3; ++j) wx[j * rows + i] = i < L.cout ? L.w[(size_t)i * L.cin + j] : 0.f;
        }
    }
    if (!L.mma) return;
    const int k4n = L.nkb * 8;
    if (i >= rows * k4n) return;
    const int n = i / k4n, k = (i % k4n) * 4;
    float v[4] = {0.f, 0.f, 0.f, 0.f};
    if (n < L.cout) {
#pragma unroll
        for (int j = 0; j < 4; ++j)
            if (k + j < L.kreal) v[j] = L.w[(size_t)n * L.cin + L.col0 + k + j];
    }
    if (args.bf16) {   // one bf16 image per tile, rounded to nearest even
        uint8_t* dst = block + L.tile_off + ((size_t)(n >> 7) * L.nkb + (k >> 5)) * BF_TILE_BYTES + sw64(n & 127, (k & 31) >> 3) +
                       ((k >> 2) & 1) * 8;
        *reinterpret_cast<uint2*>(dst) = pack_bf16x4(make_float4(v[0], v[1], v[2], v[3]));
        return;
    }
    uint8_t* dst = block + L.tile_off + ((size_t)(n >> 7) * L.nkb + (k >> 5)) * SF_WTILE + sw128(n & 127, (k & 31) >> 2);
    *reinterpret_cast<float4*>(dst) = make_float4(hi1(v[0]), hi1(v[1]), hi1(v[2]), hi1(v[3]));
    *reinterpret_cast<float4*>(dst + TILE_BYTES) = make_float4(v[0] - hi1(v[0]), v[1] - hi1(v[1]), v[2] - hi1(v[2]), v[3] - hi1(v[3]));
}

struct SfPlan {
    SfParams prm;
    size_t tile_off[O3D_MAX_LAYERS];
    size_t bytes;
    int max_kb;
    bool bf16;     // d->precision == 1: bf16 weight tiles and the BF16 kernel
};

// d: the SA layer's SharedMLP as a stack description — xyz_first = 1, c0 = feature channels, K0 = round4(c0) + 4 (unused here)
bool sf_plan(const o3d_stack_t* d, SfPlan& p) {
    if (!d || d->n_layers < 1 || d->n_layers > O3D_MAX_LAYERS || !d->xyz_first || d->c0 < 0) return false;
    if (d->precision != 0 && (d->precision != 1 || d->training)) return false;   // bf16 is for inference only
    p.bf16 = d->precision == 1;
    SfParams& q = p.prm;
    q.n = d->n_layers;
    const int C = d->c0;
    if (d->cin[0] != C + 3 || C > 288) return false;     // 9 k-blocks of input features: 144 KB operand + a two-slot weight ring
    q.Cp = (C + 3) & ~3;
    size_t off = 0;   // floats
    p.max_kb = 0;
    for (int l = 0; l < q.n; ++l) {
        SfLayer& L = q.l[l];
        L.cout = d->cout[l];
        if (L.cout < 1 || L.cout > 256) return false;
        if (l > 0 && d->cin[l] != d->cout[l - 1]) return false;
        if (d->has_bn[l] && (!d->running_mean[l] || !d->running_var[l])) return false;
        L.n_mt = (L.cout + 127) / 128;
        L.relu = d->relu[l];
        const int kreal = l == 0 ? C : d->cout[l - 1];
        L.nkb = (kreal + 31) / 32;
        L.mma = L.nkb > 0;
        L.vec_off = (uint32_t)off;
        off += 2 * (size_t)L.n_mt * 128;
        if (L.nkb > p.max_kb) p.max_kb = L.nkb;        // the operand buffer holds the k-blocks a layer reads
    }
    q.wx_off = (uint32_t)off;
    off += 3 * (size_t)q.l[0].n_mt * 128;
    size_t bytes = (off * sizeof(float) + 1023) & ~(size_t)1023;
    q.tiles_off = (uint32_t)bytes;
    for (int l = 0; l < q.n; ++l) {
        p.tile_off[l] = bytes;
        if (q.l[l].mma) bytes += (size_t)q.l[l].n_mt * q.l[l].nkb * (p.bf16 ? BF_TILE_BYTES : SF_WTILE);
    }
    p.bytes = bytes;
    return true;
}

}  // namespace

extern "C" long long o3d_sa_fused_prepared_bytes(const o3d_stack_t* d) {
    SfPlan p;
    if (!sf_plan(d, p)) return -1;
    return (long long)p.bytes;
}

extern "C" int o3d_sa_fused_prepare(const o3d_stack_t* d, void* block, void* stream) {
    O3D_REQUIRE(d && block, O3D_ERR_ARG, "o3d_sa_fused_prepare: null pointer");
    SfPlan p;
    O3D_REQUIRE(sf_plan(d, p), O3D_ERR_ARG, "o3d_sa_fused_prepare: this SharedMLP does not fit the fused layer (see o3d_sa_fused_forward)");
    SfPackArgs a{};
    a.wx_off = p.prm.wx_off;
    a.bf16 = p.bf16;
    int work_max = 0;
    for (int l = 0; l < p.prm.n; ++l) {
        const SfLayer& L = p.prm.l[l];
        SfPackLayer& q = a.l[l];
        O3D_REQUIRE(d->weight[l], O3D_ERR_ARG, "o3d_sa_fused_prepare: layer %d has no weight", l);
        q.w = d->weight[l]; q.bias = d->bias[l]; q.gamma = d->gamma[l]; q.beta = d->beta[l];
        q.mean = d->running_mean[l]; q.var = d->running_var[l]; q.eps = d->eps[l];
        q.cout = L.cout; q.cin = d->cin[l];
        q.col0 = l == 0 ? 3 : 0;
        q.kreal = l == 0 ? d->c0 : d->cout[l - 1];
        q.nkb = L.nkb; q.n_mt = L.n_mt; q.has_bn = d->has_bn[l]; q.mma = L.mma;
        q.vec_off = L.vec_off; q.tile_off = p.tile_off[l];
        int work = L.n_mt * 128 * (L.nkb > 0 ? L.nkb * 8 : 1);
        if (work > work_max) work_max = work;
    }
    sa_fused_pack_kernel<<<dim3((work_max + 255) / 256, p.prm.n), 256, 0, (cudaStream_t)stream>>>(a, (uint8_t*)block);
    O3D_CHECK_LAUNCH("o3d_sa_fused_prepare");
    return O3D_OK;
}

extern "C" int o3d_sa_fused_forward(const o3d_stack_t* d, const void* block, const float* xyz, const float* new_xyz,
                                    const float* feat_cl, int ldf, int B, int N, int M, float radius, int nsample, int normalize,
                                    float* out, int ldo, int32_t* idx, void* stream) {
    O3D_REQUIRE(d && block && xyz && new_xyz && out, O3D_ERR_ARG, "o3d_sa_fused_forward: null pointer");
    SfPlan p;
    O3D_REQUIRE(sf_plan(d, p), O3D_ERR_ARG, "o3d_sa_fused_forward: SharedMLP outside the fused layer's range (<= 256 channels per layer)");
    O3D_REQUIRE(B >= 0 && N >= 1 && M >= 0, O3D_ERR_ARG, "o3d_sa_fused_forward: bad sizes B=%d N=%d M=%d", B, N, M);
    O3D_REQUIRE(nsample >= 1 && SF_POS % nsample == 0 && M % (SF_POS / nsample) == 0, O3D_ERR_ARG,
                "o3d_sa_fused_forward: nsample=%d must divide %d and npoint=%d be a multiple of %d", nsample, SF_POS, M,
                SF_POS / (nsample > 0 && SF_POS % nsample == 0 ? nsample : 1));
    O3D_REQUIRE((d->c0 == 0) == (feat_cl == nullptr), O3D_ERR_ARG, "o3d_sa_fused_forward: features / c0 mismatch");
    O3D_REQUIRE(!feat_cl || (ldf >= p.prm.Cp && (ldf & 3) == 0 && (reinterpret_cast<uintptr_t>(feat_cl) & 15) == 0), O3D_ERR_ARG,
                "o3d_sa_fused_forward: feature rows must be 16-byte aligned with ldf >= round4(c0)");
    const int last = p.prm.n - 1;
    O3D_REQUIRE(ldo >= p.prm.l[last].cout, O3D_ERR_ARG, "o3d_sa_fused_forward: ldo=%d < %d output channels", ldo, p.prm.l[last].cout);
    if (B == 0 || M == 0) return O3D_OK;
    SfParams prm = p.prm;
    prm.ldf = ldf; prm.N = N; prm.M = M; prm.S = nsample; prm.BM = B * M;
    prm.radius = radius; prm.radius2 = radius * radius; prm.normalize = normalize;
    const int act_kb = p.bf16 ? SF_ACT_KB_OF<true> : SF_ACT_KB, wtile = p.bf16 ? SF_WTILE_OF<true> : SF_WTILE;
    int act = p.max_kb * act_kb;
    const int cloud = ((N * 12 + 1023) / 1024) * 1024;
    if (act < cloud) act = cloud;
    if (act < SF_ACT_KB) act = SF_ACT_KB;
    const int budget = 227 * 1024 - 1024 - SF_MISC - act;
    int nslot = budget / wtile;
    if (nslot > SF_MAX_SLOTS) nslot = SF_MAX_SLOTS;
    int tiles = 0;
    for (int l = 0; l < prm.n; ++l) tiles += prm.l[l].mma ? prm.l[l].n_mt * prm.l[l].nkb : 0;
    if (nslot > tiles && tiles >= 2) nslot = tiles;       // a short stack needs no deeper ring
    O3D_REQUIRE(nslot >= 2, O3D_ERR_ARG, "o3d_sa_fused_forward: N=%d points per cloud do not fit the shared-memory staging", N);
    if (p.bf16) {   // the last layer's [position][channel] fp32 staging spans the operand and the ring, which bf16 makes smaller
        const int staging = SF_POS * (p.prm.l[last].n_mt * 128 + 8) * 4;
        if (act + nslot * wtile < staging) act = ((staging - nslot * wtile + 1023) / 1024) * 1024;
    }
    prm.act_bytes = act;
    const int cpc = SF_POS / nsample;
    const int grid = (B * M) / cpc;
    prm.nslot = nslot;
    const int smem = 1024 + act + nslot * wtile + SF_MISC;
    auto kern = p.bf16 ? sa_fused_kernel<true> : sa_fused_kernel<false>;
    O3D_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem), "o3d_sa_fused_forward: smem attribute");
    kern<<<grid, SF_THREADS, smem, (cudaStream_t)stream>>>(prm, (const uint8_t*)block, xyz, new_xyz, feat_cl, out, ldo, idx);
    O3D_CHECK_LAUNCH("o3d_sa_fused_forward");
    return O3D_OK;
}
