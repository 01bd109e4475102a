"""Box geometry of the tracking frame loop as batched tensor math (CPU or CUDA tensors, no host round trips).

A box is `Box(center (...,3), wlh (...,3), rot (...,3,3))`; the reference carries the orientation as a pyquaternion
Quaternion (datasets/data_classes.py:128-257) but only ever composes, inverts and applies it, so the rotation matrix is
the natural device-side form: q1*q2 -> R1 @ R2, q.inverse -> R^T, Quaternion(axis=z, degrees=a) -> rotz(a).
Point clouds are (N, 3) row-major tensors (the reference keeps (3, N) numpy arrays).

Functions cite the reference lines whose behaviour they reproduce (datasets/points_utils.py unless noted)."""
from typing import NamedTuple

import torch


class Box(NamedTuple):
    center: torch.Tensor   # (..., 3)
    wlh: torch.Tensor      # (..., 3)  width (y extent), length (x extent), height (z extent)
    rot: torch.Tensor      # (..., 3, 3)

    def to(self, *a, **k):
        return Box(self.center.to(*a, **k), self.wlh.to(*a, **k), self.rot.to(*a, **k))


def make_box(center, wlh, rot=None, yaw_degrees=None, device=None, dtype=torch.float32):
    c = torch.as_tensor(center, dtype=dtype, device=device)
    s = torch.as_tensor(wlh, dtype=dtype, device=device)
    if rot is None:
        rot = rotz(torch.as_tensor(0.0 if yaw_degrees is None else yaw_degrees, dtype=dtype, device=device), degrees=True)
    return Box(c, s, torch.as_tensor(rot, dtype=dtype, device=device))


def rotz(angle, degrees=True):
    """Rotation about +z by `angle` (tensor, any batch shape) -> (..., 3, 3)."""
    a = torch.deg2rad(angle) if degrees else angle
    c, s = torch.cos(a), torch.sin(a)
    z, o = torch.zeros_like(a), torch.ones_like(a)
    return torch.stack([torch.stack([c, -s, z], -1), torch.stack([s, c, z], -1), torch.stack([z, z, o], -1)], -2)


_SIGNS = ((1, 1, 1, 1, -1, -1, -1, -1), (1, -1, -1, 1, 1, -1, -1, 1), (1, 1, -1, -1, 1, 1, -1, -1))
_SIGN_CACHE = {}


def _signs(like):
    """(3, 8) corner signs on `like`'s device; cached so that no host->device copy happens inside a graph capture."""
    key = (like.device, like.dtype)
    if key not in _SIGN_CACHE:
        _SIGN_CACHE[key] = torch.tensor(_SIGNS, dtype=like.dtype, device=like.device)
    return _SIGN_CACHE[key]


def corners(box: Box, wlh_factor=1.0):
    """(..., 8, 3) corners in the reference's order (data_classes.py:229-252): x forward = length, y left = width."""
    w, l, h = (box.wlh * wlh_factor).unbind(-1)
    sx, sy, sz = _signs(box.wlh)
    local = torch.stack([l[..., None] / 2 * sx, w[..., None] / 2 * sy, h[..., None] / 2 * sz], -1)   # (..., 8, 3)
    return local @ box.rot.transpose(-1, -2) + box.center[..., None, :]


def to_box_frame(points, box: Box):
    """Points expressed in the frame of `box`: R^T (p - c)  (translate(-c) then rotate(R^T), e.g. :223-242)."""
    return (points - box.center[..., None, :]) @ box.rot


def from_box_frame(points, box: Box):
    return points @ box.rot.transpose(-1, -2) + box.center[..., None, :]


def axis_aligned_mask(points, box: Box, offset=0.0, scale=1.0):
    """crop_pc_axis_aligned (:147-173): strictly inside the axis-aligned hull of the scaled box, padded by `offset`."""
    c = corners(Box(box.center, box.wlh * scale, box.rot))
    maxi, mini = c.max(-2).values + offset, c.min(-2).values - offset
    return ((points > mini[..., None, :]) & (points < maxi[..., None, :])).all(-1)


def subwindow(points, box: Box, scale, offset=2.0):
    """generate_subwindow, oriented (:223-254): returns (points in the frame of `box`, keep mask)."""
    local = to_box_frame(points, box)
    canon = Box(torch.zeros_like(box.center), box.wlh, torch.eye(3, dtype=box.rot.dtype, device=box.rot.device).expand_as(box.rot))
    return local, axis_aligned_mask(local, canon, offset=offset, scale=scale)


def crop_and_center(points, box: Box, offset=0.0, scale=1.0):
    """cropAndCenterPC (:102-124): coarse world-frame crop (4x scale, 2x offset), then the exact crop in the box frame.
    Returns (points in the box frame, keep mask, canonical box)."""
    coarse = axis_aligned_mask(points, box, offset=2 * offset, scale=4 * scale)
    local = to_box_frame(points, box)
    canon = Box(torch.zeros_like(box.center), box.wlh, torch.eye(3, dtype=box.rot.dtype, device=box.rot.device).expand_as(box.rot))
    return local, coarse & axis_aligned_mask(local, canon, offset=offset, scale=scale), canon


def crop_in_box_frame(scans, box: Box, scale, offset, frame=None, count=None):
    """The common core of generate_subwindow (:223-254) and cropAndCenterPC (:102-124) over a batch: scans (F, N, 3), one box
    per sample (B leading dim), `frame` (B,) picks each sample's scan, `count` (F,) the valid points per scan.
    Returns (local (B, N, 3) = points in the box frame, keep (B, N) = strictly inside the scaled box padded by `offset`).
    cropAndCenterPC's coarse world-frame pre-crop (4x scale, 2x offset) contains the exact box and is skipped.
    CUDA fp32 inputs go through one fused kernel (csrc/geometry.cu); other tensors through the tensor formulation."""
    half = torch.stack([box.wlh[..., 1], box.wlh[..., 0], box.wlh[..., 2]], -1) * (scale / 2) + offset      # l, w, h on x, y, z
    if scans.is_cuda and scans.dtype == torch.float32:
        from .. import ops
        return ops.crop_box_frame(scans.contiguous(), box.center, box.rot, half, frame, count)
    pts = scans if frame is None else scans[frame]
    local = to_box_frame(pts, box)
    keep = (local.abs() < half[..., None, :]).all(-1)
    if count is not None:
        n = count if frame is None else count[frame]
        keep = keep & (torch.arange(pts.shape[-2], device=pts.device)[None, :] < n[:, None])
    return local, keep


def crop_append(scans, box: Box, scale, offset, frame, count, hist, hist_keep, hist_count):
    """`crop_in_box_frame`'s kept points appended in place to per-slot histories, in scan order — getModel's concatenation
    (:88-100) one frame at a time.  scans (F, N, 3), one box per slot, frame (B,) (< 0: the slot is untouched), count (F,) or
    None; hist (B, H, 3), hist_keep (B, H) bool, hist_count (B,) int64.  Slot b's kept points go to positions
    hist_count[b] + j, those at H or beyond are dropped, and hist_count[b] grows by the full number kept, so an overflow shows
    as hist_count > H.  CUDA fp32 inputs go through one kernel (csrc/geometry.cu); other tensors through the tensor formulation."""
    half = torch.stack([box.wlh[..., 1], box.wlh[..., 0], box.wlh[..., 2]], -1) * (scale / 2) + offset
    if scans.is_cuda and scans.dtype == torch.float32:
        from .. import ops
        ops.crop_append(scans.contiguous(), box.center, box.rot, half, frame, count, hist, hist_keep, hist_count)
        return
    H = hist_keep.shape[1]
    local, keep = crop_in_box_frame(scans, box, scale, offset, frame.clamp(min=0), count)
    keep = keep & (frame >= 0)[:, None]
    pos = hist_count[:, None] + torch.cumsum(keep, 1) - 1
    b, i = torch.nonzero(keep & (pos < H), as_tuple=True)
    hist[b, pos[b, i]] = local[b, i].to(hist.dtype)
    hist_keep[b, pos[b, i]] = True
    hist_count += keep.sum(1)


def inclusive_half(wlh, wlh_factor=1.0):
    """Half extents (l, w, h on x, y, z) of nuscenes points_in_box's box scaled by `wlh_factor` (its inclusive test)."""
    return torch.stack([wlh[..., 1], wlh[..., 0], wlh[..., 2]], -1) * (wlh_factor / 2)


def box_point_counts(scans, count, frame, center, rot, half, rows=16):
    """The tensor formulation of `ops.box_points` (csrc/box_points.cu): for every row k, the points i < count[frame[k]] of
    scans[frame[k]] with |R^T (p - c)| <= half[k] in every component, as (K,) int32.  scans (S, N, 3) fp32, count (S,) or None,
    frame (K,), center (K, 3), rot (K, 3, 3), half (K, 3).  The box-frame coordinates are `to_box_frame`'s sum over the rows of R
    in order, (d_x R[0] + d_y R[1]) + d_z R[2], one rounded fp32 operation at a time, which is what the kernel computes.  Runs
    `rows` rows at a time, so that (rows, N, 3) is the largest intermediate."""
    N = scans.shape[1]
    n_valid = torch.full((scans.shape[0],), N, dtype=torch.int64, device=scans.device) if count is None else count.clamp(0, N)
    idx = torch.arange(N, device=scans.device)
    out = []
    for k0 in range(0, frame.shape[0], rows):
        f = frame[k0:k0 + rows]
        R = rot[k0:k0 + rows, None]                                          # (r, 1, 3, 3)
        d = scans[f] - center[k0:k0 + rows, None, :]
        local = d[..., 0:1] * R[..., 0, :] + d[..., 1:2] * R[..., 1, :]
        local = local + d[..., 2:3] * R[..., 2, :]
        inside = (local.abs() <= half[k0:k0 + rows, None, :]).all(-1) & (idx[None, :] < n_valid[f][:, None])
        out.append(inside.sum(1))
    return torch.cat(out).to(torch.int32) if out else torch.zeros(0, dtype=torch.int32, device=scans.device)


def point_to_box_distance(points, box: Box, wlh_factor=1.0):
    """get_point_to_box_distance (:127-144): (..., N, 9) distances to the centre and the eight corners."""
    ref = torch.cat([box.center[..., None, :], corners(box, wlh_factor)], -2)                  # (..., 9, 3)
    return (points[..., :, None, :] - ref[..., None, :, :]).square().sum(-1).sqrt()


def offset_box(box: Box, offset, degrees=True, use_z=False, limit_box=True, rand=None):
    """getOffsetBB (:43-85).  `offset` = (..., 4): dx, dy, dz, angle in the box frame (a 3-vector dx, dy, angle is the
    use_z=False form).  Net effect: centre += R @ (dx, dy, dz*use_z), R <- R @ rotz(angle).  `rand` (..., 2) supplies the
    uniform(-1, 1) replacements limit_box draws for out-of-range dx / dy (torch.rand-based when None)."""
    if offset.shape[-1] == 3:
        offset = torch.stack([offset[..., 0], offset[..., 1], torch.zeros_like(offset[..., 0]), offset[..., 2]], -1)
        use_z = False
    dx, dy, dz, ang = offset.unbind(-1)
    if limit_box:
        if rand is None:
            rand = torch.rand(offset.shape[:-1] + (2,), dtype=offset.dtype, device=offset.device) * 2 - 1
        dx = torch.where(dx > box.wlh[..., 0], rand[..., 0], dx)
        dy = torch.where(dy > torch.clamp(box.wlh[..., 1], max=2.0), rand[..., 1], dy)
        if use_z:
            dz = torch.where(dz > box.wlh[..., 2], torch.zeros_like(dz), dz)
    t = torch.stack([dx, dy, dz if use_z else torch.zeros_like(dz)], -1)
    center = box.center + (box.rot @ t[..., None])[..., 0]
    return Box(center, box.wlh, box.rot @ rotz(ang, degrees))
