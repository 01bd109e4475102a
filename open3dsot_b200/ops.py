"""Tensor-level entry points: torch tensors in, C-ABI calls on the current CUDA stream, torch tensors out.

torch is used for device memory and the stream only.  Argument checks follow upstream `pointnet2_ops`
(CHECK_CONTIGUOUS / CHECK_IS_FLOAT / CHECK_IS_INT / CHECK_CUDA -> RuntimeError; "CPU not supported").
"""
import ctypes

import numpy as np
import torch

from . import _lib


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _chk_f(t, name):
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor (CPU not supported)")
    if t.dtype != torch.float32:
        raise RuntimeError(f"{name} must be a float tensor")
    if not t.is_contiguous():
        raise RuntimeError(f"{name} must be a contiguous tensor")


def _chk_i(t, name):
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor (CPU not supported)")
    if t.dtype != torch.int32:
        raise RuntimeError(f"{name} must be an int tensor")
    if not t.is_contiguous():
        raise RuntimeError(f"{name} must be a contiguous tensor")


LAUNCHES = 0  # kernels enqueued through the C ABI (bench.py reports it as gpu_launches)


def _call(name, *args):
    global LAUNCHES
    LAUNCHES += 1
    _lib.check(getattr(_lib.lib(), name)(*args), name)


# ------------------------------------------------------------------ the nine `_ext` entry points
def furthest_point_sampling(xyz, npoint):
    _chk_f(xyz, "xyz")
    B, N, _ = xyz.shape
    out = torch.empty(B, npoint, dtype=torch.int32, device=xyz.device)
    _call("o3d_fps", xyz.data_ptr(), B, N, int(npoint), out.data_ptr(), _stream())
    return out


def gather_points(features, idx):
    _chk_f(features, "features"); _chk_i(idx, "idx")
    B, C, N = features.shape
    M = idx.shape[1]
    out = torch.empty(B, C, M, dtype=torch.float32, device=features.device)
    _call("o3d_gather", features.data_ptr(), idx.data_ptr(), B, C, N, M, out.data_ptr(), _stream())
    return out


def gather_points_grad(grad_out, idx, N):
    _chk_f(grad_out, "grad_out"); _chk_i(idx, "idx")
    B, C, M = grad_out.shape
    out = torch.zeros(B, C, N, dtype=torch.float32, device=grad_out.device)
    _call("o3d_gather_grad", grad_out.data_ptr(), idx.data_ptr(), B, C, int(N), M, out.data_ptr(), _stream())
    return out


def ball_query(new_xyz, xyz, radius, nsample):
    _chk_f(new_xyz, "new_xyz"); _chk_f(xyz, "xyz")
    B, N, _ = xyz.shape
    M = new_xyz.shape[1]
    out = torch.empty(B, M, nsample, dtype=torch.int32, device=xyz.device)
    _call("o3d_ball_query", new_xyz.data_ptr(), xyz.data_ptr(), B, N, M, float(radius), int(nsample), out.data_ptr(),
          _stream())
    return out


def group_points(features, idx):
    _chk_f(features, "features"); _chk_i(idx, "idx")
    B, C, N = features.shape
    _, M, S = idx.shape
    out = torch.empty(B, C, M, S, dtype=torch.float32, device=features.device)
    _call("o3d_group", features.data_ptr(), idx.data_ptr(), B, C, N, M, S, out.data_ptr(), _stream())
    return out


def group_points_grad(grad_out, idx, N):
    _chk_f(grad_out, "grad_out"); _chk_i(idx, "idx")
    B, C, M, S = grad_out.shape
    out = torch.zeros(B, C, N, dtype=torch.float32, device=grad_out.device)
    _call("o3d_group_grad", grad_out.data_ptr(), idx.data_ptr(), B, C, int(N), M, S, out.data_ptr(), _stream())
    return out


def three_nn(unknown, known):
    _chk_f(unknown, "unknown"); _chk_f(known, "known")
    B, n, _ = unknown.shape
    m = known.shape[1]
    dist2 = torch.empty(B, n, 3, dtype=torch.float32, device=unknown.device)
    idx = torch.empty(B, n, 3, dtype=torch.int32, device=unknown.device)
    _call("o3d_three_nn", unknown.data_ptr(), known.data_ptr(), B, n, m, dist2.data_ptr(), idx.data_ptr(), _stream())
    return dist2, idx


def three_interpolate(features, idx, weight):
    _chk_f(features, "features"); _chk_i(idx, "idx"); _chk_f(weight, "weight")
    B, c, m = features.shape
    n = idx.shape[1]
    out = torch.empty(B, c, n, dtype=torch.float32, device=features.device)
    _call("o3d_three_interpolate", features.data_ptr(), idx.data_ptr(), weight.data_ptr(), B, c, m, n, out.data_ptr(),
          _stream())
    return out


def three_interpolate_grad(grad_out, idx, weight, m):
    _chk_f(grad_out, "grad_out"); _chk_i(idx, "idx"); _chk_f(weight, "weight")
    B, c, n = grad_out.shape
    out = torch.zeros(B, c, int(m), dtype=torch.float32, device=grad_out.device)
    _call("o3d_three_interpolate_grad", grad_out.data_ptr(), idx.data_ptr(), weight.data_ptr(), B, c, n, int(m),
          out.data_ptr(), _stream())
    return out


# ------------------------------------------------------------------ fused supersets (channels-last)
def ballquery_group(xyz, new_xyz, feat_cl, radius, nsample, normalize_xyz=False, return_idx=True):
    """xyz (B,N,3), new_xyz (B,M,3), feat_cl (B,N,C)|None -> grouped (B,M,S,C+4) [feat | dx dy dz 0], idx (B,M,S)."""
    _chk_f(xyz, "xyz"); _chk_f(new_xyz, "new_xyz")
    B, N, _ = xyz.shape
    M = new_xyz.shape[1]
    C = 0
    if feat_cl is not None:
        _chk_f(feat_cl, "feat_cl")
        C = feat_cl.shape[2]
    grouped = torch.empty(B, M, nsample, C + 4, dtype=torch.float32, device=xyz.device)
    idx = torch.empty(B, M, nsample, dtype=torch.int32, device=xyz.device) if return_idx else None
    _call("o3d_ballquery_group", xyz.data_ptr(), new_xyz.data_ptr(), feat_cl.data_ptr() if C else None, B, N, M, C,
          float(radius), int(nsample), int(bool(normalize_xyz)), idx.data_ptr() if return_idx else None,
          grouped.data_ptr(), _stream())
    return grouped, idx


def ballquery_group_grad(grad_grouped, idx, N, radius, normalize_xyz, need_feat=True, need_xyz=False,
                         need_new_xyz=False):
    _chk_f(grad_grouped, "grad_grouped"); _chk_i(idx, "idx")
    B, M, S, row = grad_grouped.shape
    C = row - 4
    dev = grad_grouped.device
    gf = torch.zeros(B, N, C, dtype=torch.float32, device=dev) if (need_feat and C) else None
    gx = torch.zeros(B, N, 3, dtype=torch.float32, device=dev) if need_xyz else None
    gn = torch.zeros(B, M, 3, dtype=torch.float32, device=dev) if need_new_xyz else None
    _call("o3d_ballquery_group_grad", grad_grouped.data_ptr(), idx.data_ptr(), B, int(N), M, C, S, float(radius),
          int(bool(normalize_xyz)), gf.data_ptr() if gf is not None else None,
          gx.data_ptr() if gx is not None else None, gn.data_ptr() if gn is not None else None, _stream())
    return gf, gx, gn


def three_nn_interpolate(unknown, known, known_feat_cl):
    """unknown (B,n,3), known (B,m,3), known_feat_cl (B,m,c) -> out_cl (B,n,c), idx (B,n,3), weight (B,n,3)."""
    _chk_f(unknown, "unknown"); _chk_f(known, "known"); _chk_f(known_feat_cl, "known_feat_cl")
    B, n, _ = unknown.shape
    m, c = known_feat_cl.shape[1], known_feat_cl.shape[2]
    out = torch.empty(B, n, c, dtype=torch.float32, device=unknown.device)
    idx = torch.empty(B, n, 3, dtype=torch.int32, device=unknown.device)
    w = torch.empty(B, n, 3, dtype=torch.float32, device=unknown.device)
    _call("o3d_three_nn_interpolate", unknown.data_ptr(), known.data_ptr(), known_feat_cl.data_ptr(), B, n, m, c,
          out.data_ptr(), idx.data_ptr(), w.data_ptr(), _stream())
    return out, idx, w


def three_nn_interpolate_grad(grad_out_cl, idx, weight, m):
    _chk_f(grad_out_cl, "grad_out_cl"); _chk_i(idx, "idx"); _chk_f(weight, "weight")
    B, n, c = grad_out_cl.shape
    g = torch.zeros(B, int(m), c, dtype=torch.float32, device=grad_out_cl.device)
    _call("o3d_three_nn_interpolate_grad", grad_out_cl.data_ptr(), idx.data_ptr(), weight.data_ptr(), B, n, int(m), c,
          g.data_ptr(), _stream())
    return g


# ------------------------------------------------------------------ cross-correlation front ends (models/head/xcorr.py)
def boxaware_topk(template_bc, search_bc, k):
    """template_bc (B,M,D), search_bc (B,N,D) -> idx (B,N,k) int32: nearest template box clouds per search point."""
    _chk_f(template_bc, "template_bc"); _chk_f(search_bc, "search_bc")
    B, M, D = template_bc.shape
    N = search_bc.shape[1]
    idx = torch.empty(B, N, int(k), dtype=torch.int32, device=search_bc.device)
    _call("o3d_xcorr_boxaware_fwd", template_bc.data_ptr(), search_bc.data_ptr(), B, M, N, D, int(k), idx.data_ptr(), _stream())
    return idx


def p2b_cosine(tfeat_cl, sfeat_cl, eps=1e-8):
    """tfeat_cl (B,n1,C), sfeat_cl (B,n2,C) -> sim (B,n2,n1), tnorm (B,n1), snorm (B,n2)."""
    _chk_f(tfeat_cl, "tfeat_cl"); _chk_f(sfeat_cl, "sfeat_cl")
    B, n1, C = tfeat_cl.shape
    n2 = sfeat_cl.shape[1]
    dev = tfeat_cl.device
    sim = torch.empty(B, n2, n1, dtype=torch.float32, device=dev)
    tn = torch.empty(B, n1, dtype=torch.float32, device=dev)
    sn = torch.empty(B, n2, dtype=torch.float32, device=dev)
    _call("o3d_xcorr_p2b_fwd", tfeat_cl.data_ptr(), sfeat_cl.data_ptr(), B, n1, n2, C, float(eps), sim.data_ptr(), tn.data_ptr(),
          sn.data_ptr(), _stream())
    return sim, tn, sn


def p2b_cosine_grad(dsim, sim, tfeat_cl, sfeat_cl, tn, sn, eps=1e-8, need_t=True, need_s=True):
    _chk_f(dsim, "dsim")
    B, n1, C = tfeat_cl.shape
    n2 = sfeat_cl.shape[1]
    dt = torch.empty_like(tfeat_cl) if need_t else None
    dsf = torch.empty_like(sfeat_cl) if need_s else None
    _call("o3d_xcorr_p2b_bwd", dsim.data_ptr(), sim.data_ptr(), tfeat_cl.data_ptr(), sfeat_cl.data_ptr(), tn.data_ptr(),
          sn.data_ptr(), B, n1, n2, C, float(eps), dt.data_ptr() if need_t else None, dsf.data_ptr() if need_s else None, _stream())
    return dt, dsf


# ------------------------------------------------------------------ box-frame crop (tracking loop / training sampler)
RESAMPLE_MAX_SIZE = 2048


def resample(points, keep, size, u_perm, u_pick):
    """Fixed-shape resampling in one kernel (csrc/resample.cu; semantics of tracking/sampling.py): points (B, N, 3) fp32 CUDA,
    keep (B, N) bool, u_perm (B, N) / u_pick (B, size) uniform [0, 1) -> out (B, size, 3), src (B, size) int64, n (B,) int64."""
    _chk_f(points, "points")
    B, N, _ = points.shape
    keep = keep.contiguous()
    u_perm, u_pick = u_perm.contiguous(), u_pick.contiguous()
    assert keep.dtype == torch.bool and keep.shape == (B, N) and u_perm.shape == (B, N) and u_pick.shape == (B, size)
    assert u_perm.dtype == torch.float32 and u_pick.dtype == torch.float32
    dev = points.device
    scratch = torch.empty(B, N, dtype=torch.int32, device=dev)
    out = torch.empty(B, size, 3, device=dev)
    src = torch.empty(B, size, dtype=torch.int64, device=dev)
    n = torch.empty(B, dtype=torch.int64, device=dev)
    _call("o3d_resample", points.data_ptr(), keep.data_ptr(), u_perm.data_ptr(), u_pick.data_ptr(), B, N, int(size),
          scratch.data_ptr(), out.data_ptr(), src.data_ptr(), n.data_ptr(), _stream())
    return out, src, n


def crop_box_frame(scans, center, rot, half, frame=None, count=None):
    """scans (F, N, 3) fp32 CUDA; center (B, 3), rot (B, 3, 3), half (B, 3); frame (B,) int64 picks a scan per sample
    (None: sample b reads scan b), count (F,) int64 = valid points per scan.  Returns local (B, N, 3), keep (B, N) bool."""
    _chk_f(scans, "scans")
    F, N, _ = scans.shape
    B = center.shape[0]
    center, rot, half = (t.contiguous().float() for t in (center, rot, half))
    local = torch.empty(B, N, 3, device=scans.device)
    keep = torch.empty(B, N, dtype=torch.bool, device=scans.device)
    _call("o3d_crop_box_frame", scans.data_ptr(), None if count is None else count.data_ptr(),
          None if frame is None else frame.data_ptr(), center.data_ptr(), rot.data_ptr(), half.data_ptr(), B, N,
          local.data_ptr(), keep.data_ptr(), _stream())
    return local, keep


def crop_append(scans, center, rot, half, frame, count, hist, hist_keep, hist_count):
    """o3d_crop_box_frame's crop appended in place to per-slot histories (csrc/geometry.cu): scans (F, N, 3) fp32 CUDA; center
    (B, 3), rot (B, 3, 3), half (B, 3); frame (B,) int64, < 0 = slot untouched; count (F,) int64 or None; hist (B, H, 3) fp32,
    hist_keep (B, H) bool, hist_count (B,) int64.  Kept points go, in scan order, to positions hist_count[b] + j < H, and
    hist_count[b] grows by the full number kept."""
    _chk_f(scans, "scans"); _chk_f(hist, "hist")
    F, N, _ = scans.shape
    B, H, _ = hist.shape
    for t, name in ((frame, "frame"), (hist_count, "hist_count")) + (() if count is None else ((count, "count"),)):
        if not t.is_cuda or t.dtype != torch.int64 or not t.is_contiguous():
            raise RuntimeError(f"{name} must be a contiguous int64 CUDA tensor")
    assert frame.shape == (B,) and hist_count.shape == (B,) and hist_keep.shape == (B, H)
    assert hist_keep.dtype == torch.bool and hist_keep.is_contiguous()
    center, rot, half = (t.contiguous().float() for t in (center, rot, half))
    _call("o3d_crop_append", scans.data_ptr(), None if count is None else count.data_ptr(), frame.data_ptr(), center.data_ptr(),
          rot.data_ptr(), half.data_ptr(), B, N, H, hist.data_ptr(), hist_keep.data_ptr(), hist_count.data_ptr(), _stream())


def _chk_i64(t, name):
    if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != torch.int64 or not t.is_contiguous():
        raise RuntimeError(f"{name} must be a contiguous int64 CUDA tensor")


def crop_resample(scans, count, frame, center, rot, half, size, seed, key, key_frame, perm_stream, pick_stream, prefix=None,
                  prefix_keep=None):
    """Crop of a shared scan per target, resampled to `size` points, in one kernel (csrc/crop_resample.cu): scans (S, N, 3) fp32
    CUDA, count (S,) int64 or None, frame (K,) int64 picks each target's scan; center (K, 3), rot (K, 3, 3), half (K, 3) as
    `crop_box_frame` takes them; prefix (K, Np, 3) fp32 / prefix_keep (K, Np) bool: candidates already in the box frame that come
    before the crop; key / key_frame (K,) int64 and the perm / pick stream ids key the draws as `keyed_uniform` does.
    Returns out (K, size, 3) and the survivor counts (K,) int64, bitwise equal to `crop_box_frame` -> `keyed_uniform` ->
    `resample` on the concatenation [prefix, crop]."""
    _chk_f(scans, "scans")
    _, N, _ = scans.shape
    K = key.shape[0]
    for t, name in ((key, "key"), (key_frame, "key_frame")) + ((frame, "frame"),) + (() if count is None else ((count, "count"),)):
        _chk_i64(t, name)
    assert key_frame.shape == (K,) and frame.shape == (K,)
    center, rot, half = (t.contiguous().float() for t in (center, rot, half))
    assert center.shape == (K, 3) and rot.shape == (K, 3, 3) and half.shape == (K, 3)
    Np = 0
    if prefix is not None:
        _chk_f(prefix, "prefix")
        Np = prefix.shape[1]
        assert prefix.shape == (K, Np, 3) and prefix_keep.shape == (K, Np) and prefix_keep.dtype == torch.bool
        assert prefix_keep.is_contiguous()
    dev = scans.device
    scratch = torch.empty(K, 2, Np + N, dtype=torch.int32, device=dev)
    out = torch.empty(K, int(size), 3, device=dev)
    n = torch.empty(K, dtype=torch.int64, device=dev)
    _call("o3d_crop_resample", scans.data_ptr(), None if count is None else count.data_ptr(), frame.data_ptr(), center.data_ptr(),
          rot.data_ptr(), half.data_ptr(), N, None if prefix is None else prefix.data_ptr(),
          None if prefix is None else prefix_keep.data_ptr(), Np, int(seed) & 0xFFFFFFFF, key.data_ptr(), key_frame.data_ptr(),
          int(perm_stream), int(pick_stream), K, int(size), scratch.data_ptr(), out.data_ptr(), n.data_ptr(), _stream())
    return out, n


def box_points(scans, count, frame, center, rot, half, out=None):
    """In-box point counts (csrc/box_points.cu): scans (S, N, 3) fp32 CUDA, count (S,) int64 or None, frame (K,) int64 picks
    each row's scan; center (K, 3), rot (K, 3, 3), half (K, 3).  Returns (K,) int32 (or writes `out`): the points i <
    count[frame[k]] with |R^T (p - c)| <= half in every component, exactly `tracking.boxes.box_point_counts`."""
    _chk_f(scans, "scans")
    _, N, _ = scans.shape
    _chk_i64(frame, "frame")
    if count is not None:
        _chk_i64(count, "count")
    K = frame.shape[0]
    center, rot, half = (t.contiguous().float() for t in (center, rot, half))
    assert center.shape == (K, 3) and rot.shape == (K, 3, 3) and half.shape == (K, 3)
    if out is None:
        out = torch.empty(K, dtype=torch.int32, device=scans.device)
    _chk_i(out, "out")
    assert out.shape == (K,)
    _call("o3d_box_points", scans.data_ptr(), None if count is None else count.data_ptr(), frame.data_ptr(), center.data_ptr(),
          rot.data_ptr(), half.data_ptr(), N, K, out.data_ptr(), _stream())
    return out


# slot state of the live tracker's write-back: (attribute, dtype, values per row)
TRACK_SLOTS = (("box_c", torch.float32, 3), ("box_r", torch.float32, 9), ("t", torch.int64, 1), ("first_flag", torch.float32, 1),
               ("points", torch.int32, 1), ("score", torch.float32, 1), ("misses", torch.int32, 1), ("lost", torch.bool, 1),
               ("vel", torch.float32, 3), ("hit_c", torch.float32, 3), ("hit_t", torch.int64, 1), ("coasting", torch.bool, 1))


def track_update(slots, src, dst, adv, center, rot, points, score, rule=None, coast=None, match=None):
    """The live tracker's per-row write-back in one kernel (csrc/track_update.cu), in place on `slots` (an object with the
    TRACK_SLOTS attributes, contiguous CUDA tensors of the same number of rows): row i reads slot src[i] and writes slot dst[i].
    adv (b,) bool; center (b, 3), rot (b, 3, 3), points (b,) int32, score (b,) float32: the network's box and its evidence.
    `rule`: None or (min_points, patience); `coast`: None or (alpha, beta), float32 values.  `match`: None or (match (b,) int32,
    match_box (b, 12) float32 from `box_associate`, detection and reacquired: the slot state of MATCH_SLOTS, with the rows of
    `slots`).  Exactly `tracking.multi_tracker.track_update_tensors`."""
    b = adv.shape[0]
    rows = slots.box_c.shape[0]
    for name, dtype, n in TRACK_SLOTS:
        t = getattr(slots, name)
        if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != dtype or not t.is_contiguous() \
                or t.shape[0] != rows or t.numel() != rows * n:
            raise RuntimeError(f"track_update: slot state {name} must be a contiguous {dtype} CUDA tensor of {rows} x {n}")
    _chk_i64(src, "src")
    _chk_i64(dst, "dst")
    _chk_f(center, "center")
    _chk_f(rot, "rot")
    _chk_f(score, "score")
    _chk_i(points, "points")
    if not adv.is_cuda or adv.dtype != torch.bool or not adv.is_contiguous():
        raise RuntimeError("adv must be a contiguous bool CUDA tensor")
    assert src.shape == dst.shape == points.shape == score.shape == (b,) and center.shape == (b, 3) and rot.shape == (b, 3, 3)
    ptrs = [None] * 4
    if match is not None:
        m, m_box, detection, reacquired = match
        _chk_i(m, "match")
        _chk_f(m_box, "match_box")
        assert m.shape == (b,) and m_box.shape == (b, 12)
        for t, (name, dtype) in zip((detection, reacquired), MATCH_SLOTS):
            if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != dtype or not t.is_contiguous() or t.shape != (rows,):
                raise RuntimeError(f"track_update: slot state {name} must be a contiguous {dtype} CUDA tensor of {rows}")
        ptrs = [t.data_ptr() for t in (m, m_box, detection, reacquired)]
    d = _lib.TrackUpdateDesc(b, src.data_ptr(), dst.data_ptr(), adv.data_ptr(), center.data_ptr(), rot.data_ptr(),
                             points.data_ptr(), score.data_ptr(), *(getattr(slots, name).data_ptr() for name, _, _ in TRACK_SLOTS),
                             rule is not None, *(rule or (0, 1)), coast is not None, *(coast or (1.0, 0.0)), *ptrs)
    _call("o3d_track_update", ctypes.byref(d), _stream())


# the write-back's detection state per slot: (attribute, dtype)
MATCH_SLOTS = (("detection", torch.int32), ("reacquired", torch.bool))
# values of one detection row: centre (3), wlh (3), row-major rotation with the box axes in its columns (9), score
DETECTION_VALUES = 16
MAX_DETECTIONS = 1024


def box_associate(src, feed, adv, center, points, slots, fed, count, det, records, gate2, axes, rule=None, coast=False):
    """Match each feed's detections to the step's advancing rows (csrc/associate.cu, one CTA per feed): greedy in ascending
    (d2, row, detection) order over the pairs with d2 <= gate2, d2 the squared distance over the plane `axes` between the
    detection's centre and the centre the row writes without detections (`coast`: whether a miss coasts).  src / feed (b,) int64,
    adv (b,) bool, center (b, 3) / points (b,) int32: the network's box and its in-box count; `slots`: the slot state (t, hit_t,
    hit_c, vel attributes); fed (F,) int64, count (F,) int32 (checked on the host before its upload: 0 .. D), det (F, D, 16)
    float32; `records`: (rec_det (F, D, 16), rec_count (F,) int32, rec_slot (F, D) int32), updated for the fed feeds.  `gate2`: a
    float32 value; `rule`: None or (min_points, patience).  Returns (pred (b, 3), match (b,) int32, match_box (b, 12)), exactly
    `tracking.multi_tracker.associate_tensors`."""
    b = adv.shape[0]
    _chk_i64(src, "src")
    _chk_i64(feed, "feed")
    _chk_i64(fed, "fed")
    _chk_f(center, "center")
    _chk_i(points, "points")
    _chk_i(count, "count")
    _chk_f(det, "det")
    if not adv.is_cuda or adv.dtype != torch.bool or not adv.is_contiguous():
        raise RuntimeError("adv must be a contiguous bool CUDA tensor")
    F, D, n = det.shape
    assert n == DETECTION_VALUES and src.shape == feed.shape == points.shape == (b,) and center.shape == (b, 3)
    assert fed.shape == count.shape == (F,)
    rec_det, rec_count, rec_slot = records
    _chk_f(rec_det, "rec_det")
    _chk_i(rec_count, "rec_count")
    _chk_i(rec_slot, "rec_slot")
    assert rec_det.shape == (F, D, n) and rec_count.shape == (F,) and rec_slot.shape == (F, D)
    for name, chk in (("t", _chk_i64), ("hit_t", _chk_i64), ("hit_c", _chk_f), ("vel", _chk_f)):
        chk(getattr(slots, name), name)
    dev = adv.device
    pred = torch.empty(b, 3, device=dev)
    match = torch.empty(b, dtype=torch.int32, device=dev)
    match_box = torch.empty(b, 12, device=dev)
    d = _lib.AssociateDesc(b, F, D, int(axes[0]), int(axes[1]), float(gate2), rule is not None, (rule or (0, 1))[0], bool(coast),
                           *(t.data_ptr() for t in (src, feed, adv, center, points, slots.t, slots.hit_t, slots.hit_c, slots.vel,
                                                    fed, count, det, pred, match, match_box, rec_det, rec_count, rec_slot)))
    _call("o3d_box_associate", ctypes.byref(d), _stream())
    return pred, match, match_box


# slot state a birth writes, in o3d_track_birth_t's order: (attribute, dtype, values per row)
BIRTH_SLOTS = (("box_c", torch.float32, 3), ("box_s", torch.float32, 3), ("box_r", torch.float32, 9),
               ("first_flag", torch.float32, 1), ("active", torch.bool, 1), ("key", torch.int64, 1), ("t", torch.int64, 1),
               ("slot_feed", torch.int64, 1), ("points", torch.int32, 1), ("score", torch.float32, 1), ("misses", torch.int32, 1),
               ("lost", torch.bool, 1), ("vel", torch.float32, 3), ("hit_c", torch.float32, 3), ("hit_t", torch.int64, 1),
               ("coasting", torch.bool, 1), ("detection", torch.int32, 1), ("reacquired", torch.bool, 1))


def track_birth(feed, adv, pred, fed, count, det, rec_slot, birth_list, next_id, log, slots, gate2, axes, min_score, id_base):
    """Start targets from each feed's unmatched detections in one kernel (csrc/track_birth.cu, one CTA): feed (b,) int64, adv
    (b,) bool, pred (b, 3) float32 from `box_associate`; fed (F,) int64, count (F,) int32, det (F, D, 16) float32, rec_slot (F,
    D) int32 (updated for the born detections); birth_list (2, R) int64: reserved slots and their feeds (-1: padding); next_id
    (1,) int64, the births so far (advanced); log (R, 4) int64 out; `slots`: an object with the BIRTH_SLOTS attributes,
    contiguous CUDA tensors of the same number of rows.  `gate2` / `min_score`: float32 values.  Exactly
    `tracking.multi_tracker.birth_tensors`."""
    b = adv.shape[0]
    rows = slots.box_c.shape[0]
    for name, dtype, n in BIRTH_SLOTS:
        t = getattr(slots, name)
        if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != dtype or not t.is_contiguous() \
                or t.shape[0] != rows or t.numel() != rows * n:
            raise RuntimeError(f"track_birth: slot state {name} must be a contiguous {dtype} CUDA tensor of {rows} x {n}")
    for t, name in ((feed, "feed"), (fed, "fed"), (birth_list, "birth_list"), (next_id, "next_id"), (log, "log")):
        _chk_i64(t, name)
    _chk_f(pred, "pred")
    _chk_f(det, "det")
    _chk_i(count, "count")
    _chk_i(rec_slot, "rec_slot")
    if not adv.is_cuda or adv.dtype != torch.bool or not adv.is_contiguous():
        raise RuntimeError("adv must be a contiguous bool CUDA tensor")
    F, D, n = det.shape
    R = birth_list.shape[1]
    assert n == DETECTION_VALUES and feed.shape == (b,) and pred.shape == (b, 3) and fed.shape == count.shape == (F,)
    assert rec_slot.shape == (F, D) and birth_list.shape == (2, R) and next_id.shape == (1,) and log.shape == (R, 4)
    d = _lib.BirthDesc(b, F, D, R, int(axes[0]), int(axes[1]), float(gate2), float(min_score), int(id_base),
                       *(t.data_ptr() for t in (feed, adv, pred, fed, count, det, rec_slot, birth_list[0], birth_list[1], next_id,
                                                log)),
                       *(getattr(slots, name).data_ptr() for name, _, _ in BIRTH_SLOTS))
    _call("o3d_track_birth", ctypes.byref(d), _stream())


# ------------------------------------------------------------------ scan ingest for the live tracker's feeds (csrc/scan_ingest.cu)
# o3d_scan_desc_t, field for field
SCAN_DESC = np.dtype([("offset", "<i8"), ("rows", "<i4"), ("stride", "<i4"), ("is_f64", "<i4"), ("feed", "<i4"), ("half", "<i4"),
                      ("n_xf", "<i4"), ("xf", "<f8", (2, 12))])
assert SCAN_DESC.itemsize == 224


def pack_scans(items, head=0):
    """Pack raw scans for one `scan_ingest` call into one pinned host buffer: [head bytes | descriptors | rows].  `items`: (feed,
    half, rows, transforms) with rows an (n, stride) float32 / float64 array as stored and transforms a list of at most two 3x4 (or
    4x4) affine matrices applied in order.  Returns (buffer (uint8 torch tensor, pinned when CUDA is available), descriptors
    (a SCAN_DESC numpy view into the buffer), byte offset of the descriptors, byte offset of the rows)."""
    items = list(items)
    rows = []
    for feed, _, r, _ in items:
        r = np.asarray(r)
        if r.ndim != 2:
            raise ValueError(f"scan_ingest: the rows of feed {feed} have shape {r.shape}; expected (points, values per row)")
        rows.append(np.ascontiguousarray(r if r.dtype in (np.float32, np.float64) else r.astype(np.float64)))
    d0 = -(-int(head) // 16) * 16
    s0 = d0 + len(items) * SCAN_DESC.itemsize
    offs, at = [], 0
    for r in rows:
        offs.append(at)
        at += -(-r.nbytes // 16) * 16
    buf = torch.empty(s0 + at, dtype=torch.uint8, pin_memory=torch.cuda.is_available())
    host = buf.numpy()
    desc = host[d0:s0].view(SCAN_DESC)
    desc["xf"] = 0.0
    for i, ((feed, half, _, xfs), r, o) in enumerate(zip(items, rows, offs)):
        xfs = list(xfs)
        if len(xfs) > 2:
            raise ValueError(f"scan_ingest: {len(xfs)} transforms for feed {feed}; at most two")
        for name, v in (("offset", o), ("rows", r.shape[0]), ("stride", r.shape[1]), ("is_f64", int(r.dtype == np.float64)),
                        ("feed", int(feed)), ("half", int(half)), ("n_xf", len(xfs))):
            desc[name][i] = v
        for k, m in enumerate(xfs):
            desc["xf"][i, k] = np.asarray(m, np.float64)[:3, :4].reshape(12)
        host[s0 + o:s0 + o + r.nbytes] = r.reshape(-1).view(np.uint8)
    return buf, desc, d0, s0


def scan_ingest(scans, count, desc, dev_buf, desc_at, slab_at):
    """Write raw scans into the feeds' halves of scans (F, 2, N, 3) fp32 CUDA and set count (F, 2) int64, in one launch
    (csrc/scan_ingest.cu).  `desc`: the SCAN_DESC host descriptors (checked before the launch); `dev_buf`: the device copy of the
    `pack_scans` buffer, with the descriptors at byte `desc_at` and the rows from byte `slab_at`."""
    _chk_f(scans, "scans")
    _chk_i64(count, "count")
    F, two, N, _ = scans.shape
    assert two == 2 and count.shape == (F, 2) and desc.dtype == SCAN_DESC and desc.flags.c_contiguous
    if not dev_buf.is_cuda or dev_buf.dtype != torch.uint8 or not dev_buf.is_contiguous():
        raise RuntimeError("dev_buf must be a contiguous uint8 CUDA tensor")
    base = dev_buf.data_ptr()
    _call("o3d_scan_ingest", desc.ctypes.data, base + desc_at, len(desc), base + slab_at, dev_buf.numel() - slab_at, F, N,
          scans.data_ptr(), count.data_ptr(), _stream())


# ------------------------------------------------------------------ split evaluation, K tracklets in flight (tracking/batched_tracker.py)
def keyed_uniform(tracklet, frame, seed, stream, n, out=None):
    """Counter-based uniform [0, 1) draws (csrc/track_eval.cu): tracklet (K,) / frame (K,) int64 CUDA -> out (K, n) fp32, row k a pure
    function of (seed, tracklet[k], frame[k], stream, element): Philox4x32-10, key (seed, tracklet), counter (e // 4, frame, stream, 0)."""
    for t, name in ((tracklet, "tracklet"), (frame, "frame")):
        if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != torch.int64 or not t.is_contiguous():
            raise RuntimeError(f"{name} must be a contiguous int64 CUDA tensor")
    K = tracklet.shape[0]
    assert frame.shape == (K,)
    if out is None:
        out = torch.empty(K, int(n), device=tracklet.device)
    _chk_f(out, "out")
    assert out.shape == (K, int(n))
    _call("o3d_keyed_uniform", tracklet.data_ptr(), frame.data_ptr(), K, int(seed) & 0xFFFFFFFF, int(stream), int(n), out.data_ptr(),
          _stream())
    return out


def up_mask(up_axis):
    """Bit i set <=> up_axis[i] != 0 (the axes utils/metrics.py selects with `np.array(up_axis) != 0`)."""
    return sum(1 << i for i, a in enumerate(up_axis) if a != 0)


def track_metrics(center, rot, wlh, gt_center, gt_rot, gt_wlh, frame, dim, up_axis, overlap, distance):
    """estimateOverlap(gt, result, dim, up_axis) / estimateAccuracy in fp64 per slot (csrc/track_eval.cu): result box center (K, 3),
    rot (K, 3, 3), wlh (K, 3) fp32; ground truth gt_* (F, 3) / (F, 3, 3) / (F, 3) fp64; frame (K,) int64 pool frame of each slot
    (< 0 = idle).  Writes overlap[frame[k]] / distance[frame[k]] of the fp64 (F,) records in place."""
    for t, name in ((center, "center"), (rot, "rot"), (wlh, "wlh")):
        _chk_f(t, name)
    for t, name in ((gt_center, "gt_center"), (gt_rot, "gt_rot"), (gt_wlh, "gt_wlh"), (overlap, "overlap"), (distance, "distance")):
        if not t.is_cuda or t.dtype != torch.float64 or not t.is_contiguous():
            raise RuntimeError(f"{name} must be a contiguous float64 CUDA tensor")
    if not frame.is_cuda or frame.dtype != torch.int64 or not frame.is_contiguous():
        raise RuntimeError("frame must be a contiguous int64 CUDA tensor")
    K = center.shape[0]
    assert rot.shape == (K, 3, 3) and wlh.shape == (K, 3) and frame.shape == (K,)
    _call("o3d_track_metrics", center.data_ptr(), rot.data_ptr(), wlh.data_ptr(), gt_center.data_ptr(), gt_rot.data_ptr(),
          gt_wlh.data_ptr(), frame.data_ptr(), K, int(dim), up_mask(up_axis), overlap.data_ptr(), distance.data_ptr(), _stream())
