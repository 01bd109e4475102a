"""On-device construction of siamese training batches (SURVEY.md §8f rank 3).

The reference builds every template-search pair on the host (datasets/sampler.py:16-79 `siamese_processing`, driven by
`PointTrackingSampler.__getitem__` :213-243, ten DataLoader workers per GPU): numpy crops, pyquaternion box algebra, a
Python call per pair.  At the rate the fused training step consumes pairs (thousands per second per GPU) that pipeline is
the bottleneck, so here the tracklets live on the device as padded tensors and one call produces a whole batch with
batched tensor math: frame selection, the two random box offsets, template = first-frame crop + offset previous-frame crop
(getModel), search area = sub-window around the offset current box, segmentation labels, box regression target, fixed-shape
resampling and the two BoxClouds.  Output keys, shapes and dtypes are those of the reference's collated batch.

Samples the reference rejects (<= 20 template or search points: it catches the AssertionError and draws another index)
are drawn here as an oversampled pool; the first `batch_size` valid ones are returned."""
import torch

from ..tracking import boxes as bx
from ..tracking.sampling import resample_batched


class DeviceTracklets:
    """Tracklets as padded device tensors: scans (F, Nmax, 3) + valid counts (F,), one box per frame, and for every frame
    the index of its tracklet's first frame and of its predecessor (clamped at the start: sampler.py:229-231)."""

    def __init__(self, tracklets, device, max_points=None):
        frames = [f for t in tracklets for f in t]
        nmax = max_points or max(f["pc"].points.shape[1] for f in frames)
        F = len(frames)
        self.scans = torch.zeros(F, nmax, 3, device=device)
        self.count = torch.zeros(F, dtype=torch.long, device=device)
        c, s, r, first, prev = [], [], [], [], []
        k = 0
        for t in tracklets:
            for j, f in enumerate(t):
                if f["pc"].points.shape[1] > nmax:
                    raise ValueError(f"DeviceTracklets: a scan has {f['pc'].points.shape[1]} points > max_points={nmax}; "
                                     "raise max_points (scans are never truncated silently)")
                pts = torch.as_tensor(f["pc"].points, dtype=torch.float32).t()
                self.scans[k + j, : pts.shape[0]] = pts.to(device)
                self.count[k + j] = pts.shape[0]
                b = f["3d_bbox"]
                c.append(torch.as_tensor(b.center, dtype=torch.float32))
                s.append(torch.as_tensor(b.wlh, dtype=torch.float32))
                r.append(torch.as_tensor(b.rotation_matrix, dtype=torch.float32))
                first.append(k)
                prev.append(k + max(j - 1, 0))
            k += len(t)
        self.center, self.wlh, self.rot = (torch.stack(x).to(device) for x in (c, s, r))
        self.first = torch.tensor(first, device=device)
        self.prev = torch.tensor(prev, device=device)
        self.num_frames = F

    def box(self, idx):
        return bx.Box(self.center[idx], self.wlh[idx], self.rot[idx])

    def valid(self, idx):
        n = self.scans.shape[1]
        return torch.arange(n, device=self.scans.device)[None, :] < self.count[idx][:, None]


def transform_box(box: bx.Box, ref: bx.Box):
    """points_utils.transform_box (:257-262): `box` expressed in the frame of `ref`."""
    center = ((box.center - ref.center)[..., None, :] @ ref.rot)[..., 0, :]
    return bx.Box(center, box.wlh, ref.rot.transpose(-1, -2) @ box.rot)


def in_box_mask(points, box: bx.Box):
    """points_utils.get_in_box_mask (:273-300): strictly inside the oriented box."""
    local = bx.to_box_frame(points, box)
    half = torch.stack([box.wlh[..., 1], box.wlh[..., 0], box.wlh[..., 2]], -1)[..., None, :] / 2     # l, w, h along x, y, z
    return (local.abs() < half).all(-1)


def _augment(data, cfg, idx, box, draws, key, generator):
    """The reference's optional `apply_augmentation` transform on the frames `idx` (sampler.py:31-35 / :102-105):
    returns (scans (B, N, 3) or None when augmentation is off, per-sample valid counts, box)."""
    if not cfg.get("use_augmentation", False):
        return None, None, box
    dev = data.scans.device
    B = idx.shape[0]
    d = (draws or {}).get(key)
    if d is None:
        u = torch.rand(B, 6, device=dev, generator=generator)
        d = {"trans": u[:, :3] * 0.6 - 0.3, "rot": u[:, 3] * 20 - 10, "flip_x": u[:, 4] < 0.5, "flip_y": u[:, 5] < 0.5}
    pts, box = apply_augmentation(data.scans[idx], box, d["trans"], d["rot"], d["flip_x"], d["flip_y"], data.valid(idx))
    return pts, data.count[idx], box


def siamese_batch(data: DeviceTracklets, cfg, frame_ids, candidate_ids, draws=None, generator=None):
    """siamese_processing for the frames `frame_ids` (B,) with candidate indices `candidate_ids` (B,).
    `draws` may carry explicit random numbers (tests): 'template_offset' (B, 3) uniform(-0.3, 0.3) draws, 'search_offset'
    (B, 3) standard-normal draws, 'u_t', 'u_pick_t', 'u_s', 'u_pick_s' for the two resamplings.
    Returns (batch dict, valid (B,) bool)."""
    dev = data.scans.device
    B = frame_ids.shape[0]
    draws = draws or {}
    deg = 5.0 if cfg.degrees else 0.08726646259971647                 # 5 degrees, in the unit the boxes are offset in
    ang_scale = torch.cat([torch.ones(2, device=dev), torch.full((1,), deg, device=dev)])   # fills only: graph-capturable
    cand0 = candidate_ids == 0
    # ---- template: offset the previous frame's box, merge with the first frame's crop (sampler.py:37-46)
    off_t = draws.get("template_offset")
    if off_t is None:
        off_t = torch.rand(B, 3, device=dev, generator=generator) * 0.6 - 0.3
    off_t = torch.where(cand0[:, None], torch.zeros_like(off_t), off_t * ang_scale)
    i_first, i_prev = data.first[frame_ids], data.prev[frame_ids]
    def limit_rand(key):
        r = draws.get(key)
        if r is None and cfg.data_limit_box:
            r = torch.rand(B, 2, device=dev, generator=generator) * 2 - 1
        return r
    t_box = bx.offset_box(data.box(i_prev), off_t, degrees=cfg.degrees, limit_box=cfg.data_limit_box,
                          rand=limit_rand("limit_rand_t"))
    f_local, f_keep = bx.crop_in_box_frame(data.scans, data.box(i_first), cfg.model_bb_scale, cfg.model_bb_offset, i_first, data.count)
    p_local, p_keep = bx.crop_in_box_frame(data.scans, t_box, cfg.model_bb_scale, cfg.model_bb_offset, i_prev, data.count)
    canon = bx.Box(torch.zeros_like(t_box.center), t_box.wlh, torch.eye(3, device=dev).expand_as(t_box.rot))
    cand = torch.cat([f_local, p_local], 1)
    keep = torch.cat([f_keep, p_keep], 1)
    template, _, n_t = resample_batched(cand, keep, cfg.template_size, draws.get("u_t"), draws.get("u_pick_t"), generator)
    # ---- search area around the offset current box (sampler.py:50-63)
    off_s = draws.get("search_offset")
    if off_s is None:
        off_s = torch.randn(B, 3, device=dev, generator=generator)
    off_s = off_s * ang_scale.sqrt()            # N(0, diag(1, 1, 5 deg)): KalmanFiltering.reset
    if cfg.get("num_candidates", 1) > 1:
        off_s = torch.where(cand0[:, None], torch.zeros_like(off_s), off_s)
    aug_pts, aug_count, gt = _augment(data, cfg, frame_ids, data.box(frame_ids), draws, "aug_search", generator)
    sample_bb = bx.offset_box(gt, off_s, degrees=cfg.degrees, limit_box=cfg.data_limit_box, rand=limit_rand("limit_rand_s"))
    if aug_pts is None:
        s_local, s_keep = bx.crop_in_box_frame(data.scans, sample_bb, cfg.search_bb_scale, cfg.search_bb_offset, frame_ids, data.count)
    else:
        s_local, s_keep = bx.crop_in_box_frame(aug_pts, sample_bb, cfg.search_bb_scale, cfg.search_bb_offset, None, aug_count)
    s_box = transform_box(gt, sample_bb)
    search, src, n_s = resample_batched(s_local, s_keep, cfg.search_size, draws.get("u_s"), draws.get("u_pick_s"), generator)
    seg = in_box_mask(search, s_box).float()
    box_label = torch.cat([s_box.center, -off_s[:, 2:3]], 1)
    batch = {"template_points": template, "search_points": search, "box_label": box_label, "bbox_size": s_box.wlh,
             "seg_label": seg}
    if cfg.get("box_aware", False):
        batch["points2cc_dist_t"] = bx.point_to_box_distance(template, canon)
        batch["points2cc_dist_s"] = bx.point_to_box_distance(search, s_box)
    batch["_n_template"], batch["_n_search"] = n_t, n_s          # survivor counts (diagnostics; dropped by next_batch)
    return batch, (n_t > 20) & (n_s > 20)


def apply_augmentation(points, box: bx.Box, trans, rot_deg, flip_x, flip_y, valid=None, wlh_factor=1.25):
    """points_utils.apply_augmentation / apply_transform (:303-362), batched: the points inside the 1.25x box move rigidly
    with it — mirror in the box frame (x: the box also turns by 180 degrees so that +x stays the heading; y), rotate by
    `rot_deg` about the box's z, shift by `trans` (box frame) — everything else stays.  points (B, N, 3), trans (B, 3),
    rot_deg (B,), flip_x / flip_y (B,) bool.  Returns (points, box)."""
    inside = in_box_inclusive(points, box, wlh_factor)
    if valid is not None:
        inside = inside & valid
    local = bx.to_box_frame(points, box)
    sx = torch.where(flip_x, -1.0, 1.0).to(points.dtype)
    sy = torch.where(flip_y, -1.0, 1.0).to(points.dtype)
    local = local * torch.stack([sx, sy, torch.ones_like(sx)], -1)[:, None, :]
    rz = bx.rotz(rot_deg.to(points.dtype), degrees=True)
    local = local @ rz.transpose(-1, -2) + trans[:, None, :]
    moved = bx.from_box_frame(local, box)
    turn = bx.rotz(torch.where(flip_x, 180.0, 0.0).to(points.dtype), degrees=True)
    new_box = bx.Box(box.center + (box.rot @ trans[..., None])[..., 0], box.wlh, box.rot @ rz @ turn)
    return torch.where(inside[..., None], moved, points), new_box


def in_box_inclusive(points, box: bx.Box, wlh_factor=1.0):
    """nuscenes geometry_utils.points_in_box (used at sampler.py:130-132): its three projection tests 0 <= v.e <= e.e are the
    inclusive form of |local| <= half * wlh_factor in the box frame."""
    local = bx.to_box_frame(points, box)
    half = torch.stack([box.wlh[..., 1], box.wlh[..., 0], box.wlh[..., 2]], -1)[..., None, :] * (wlh_factor / 2)
    return (local.abs() <= half).all(-1)


def yaw_of(rot, degrees):
    """Signed rotation angle about +z of a (..., 3, 3) yaw rotation — pyquaternion's `degrees * axis[-1]` (sampler.py:149-156)."""
    a = torch.atan2(rot[..., 1, 0], rot[..., 0, 0])
    return torch.rad2deg(a) if degrees else a


def motion_batch(data: DeviceTracklets, cfg, frame_ids, candidate_ids, draws=None, generator=None):
    """motion_processing (sampler.py:82-181) for the frames `frame_ids` (B,): previous + current sub-windows in the frame of
    the (randomly offset) previous box, stacked with timestamp / prior-targetness channels, segmentation labels, box /
    previous-box / motion regression targets, motion-state label and the three BoxClouds.  Returns (batch, valid (B,))."""
    dev = data.scans.device
    B = frame_ids.shape[0]
    draws = draws or {}
    n = cfg.point_sample_size
    deg = 5.0 if cfg.degrees else 0.08726646259971647
    ang_scale = torch.cat([torch.ones(2, device=dev), torch.full((1,), deg, device=dev)])
    cand0 = candidate_ids == 0
    i_prev = data.prev[frame_ids]
    prev_aug, prev_cnt, prev_box = _augment(data, cfg, i_prev, data.box(i_prev), draws, "aug_prev", generator)
    this_aug, this_cnt, this_box = _augment(data, cfg, frame_ids, data.box(frame_ids), draws, "aug_this", generator)
    off = draws.get("offset")
    if off is None:
        off = torch.rand(B, 3, device=dev, generator=generator) * 0.6 - 0.3
    off = torch.where(cand0[:, None], torch.zeros_like(off), off * ang_scale)
    rand = draws.get("limit_rand")
    if rand is None and cfg.data_limit_box:
        rand = torch.rand(B, 2, device=dev, generator=generator) * 2 - 1
    ref = bx.offset_box(prev_box, off, degrees=cfg.degrees, limit_box=cfg.data_limit_box, rand=rand)
    # enough target points in the previous GT box (sampler.py:99-100)
    def crop(aug, cnt, idx, box, scale, offset):
        if aug is None:
            return bx.crop_in_box_frame(data.scans, box, scale, offset, idx, data.count)
        return bx.crop_in_box_frame(aug, box, scale, offset, None, cnt)
    # the reference counts the target points BEFORE the augmentation (sampler.py:99-100, on the original frame)
    p_gt_local, p_gt_keep = bx.crop_in_box_frame(data.scans, data.box(i_prev), 1.0, 0.0, i_prev, data.count)
    half_gt = torch.stack([prev_box.wlh[:, 1], prev_box.wlh[:, 0], prev_box.wlh[:, 2]], -1)[:, None, :] / 2
    n_target = ((p_gt_local.abs() <= half_gt).all(-1) & data.valid(i_prev)).sum(1)
    p_local, p_keep = crop(prev_aug, prev_cnt, i_prev, ref, cfg.bb_scale, cfg.bb_offset)
    t_local, t_keep = crop(this_aug, this_cnt, frame_ids, ref, cfg.bb_scale, cfg.bb_offset)
    this_b, prev_b = transform_box(this_box, ref), transform_box(prev_box, ref)
    canon = bx.Box(torch.zeros_like(ref.center), ref.wlh, torch.eye(3, device=dev).expand_as(ref.rot))
    motion_b = transform_box(this_b, prev_b)
    prev_pts, _, n_p = resample_batched(p_local, p_keep, n, draws.get("u_p"), draws.get("u_pick_p"), generator)
    this_pts, _, n_t = resample_batched(t_local, t_keep, n, draws.get("u_t"), draws.get("u_pick_t"), generator)
    seg_this = in_box_inclusive(this_pts, this_b, 1.25)
    seg_prev = in_box_inclusive(prev_pts, prev_b, 1.25)
    mask_prev = in_box_inclusive(prev_pts, canon, 1.25).float()
    mask_prev = torch.where(cand0[:, None], mask_prev, mask_prev * 0.6 + 0.2)             # 0.2 / 0.8: the prior box is not GT
    col = lambda pts, t, m: torch.cat([pts, torch.full_like(pts[..., :1], t), m[..., None]], -1)
    points = torch.cat([col(prev_pts, 0.0, mask_prev), col(this_pts, 0.1, torch.full_like(mask_prev, 0.5))], 1)
    lab = lambda b: torch.cat([b.center, yaw_of(b.rot, cfg.degrees)[:, None]], 1)
    batch = {"points": points, "box_label": lab(this_b), "box_label_prev": lab(prev_b), "motion_label": lab(motion_b),
             "motion_state_label": ((this_b.center - prev_b.center).norm(dim=1) > cfg.motion_threshold).long(),
             "bbox_size": this_b.wlh, "seg_label": torch.cat([seg_prev, seg_this], 1).long()}
    if cfg.get("box_aware", False):
        cand_bc = bx.point_to_box_distance(prev_pts, canon)
        batch.update({"prev_bc": bx.point_to_box_distance(prev_pts, prev_b), "this_bc": bx.point_to_box_distance(this_pts, this_b),
                      "candidate_bc": torch.cat([cand_bc, torch.zeros_like(cand_bc)], 1)})
    batch["_n_prev"], batch["_n_this"], batch["_n_target"] = n_p, n_t, n_target
    return batch, (n_target > 10) & (n_t > 20)


class DeviceSiameseSampler:
    """(`DeviceMotionSampler` below is the same class bound to `motion_batch`.)
    Drop-in source of training batches: `next_batch()` returns `(batch, valid)`: the reference's batch dict on the device
    and a (B,) bool mask that is all-True unless every sample of the oversampled pool was rejected.
    On CUDA the construction (≈ 340 small launches, host-bound when issued eagerly) is captured once in a CUDA graph;
    every replay draws new frames and offsets (graph-safe philox offsets of the default CUDA generator) into the same
    static output tensors — consume or copy a batch before asking for the next one."""

    def __init__(self, tracklets, cfg, device, oversample=1.5, seed=0, max_points=None, use_graph=True, processing=None):
        self.processing = processing or siamese_batch           # `motion_batch` for the motion-centric models
        self.data = tracklets if isinstance(tracklets, DeviceTracklets) else DeviceTracklets(tracklets, device, max_points)
        self.cfg = cfg
        dev = self.data.scans.device
        self.use_graph = bool(use_graph) and dev.type == "cuda"
        # a captured graph can only advance the default CUDA generator; the eager path keeps its own seeded generator
        self.gen = None if self.use_graph else torch.Generator(device=dev).manual_seed(seed)
        if self.use_graph:
            torch.cuda.manual_seed(seed)
        self.oversample = oversample
        self.num_candidates = cfg.get("num_candidates", 1)
        self._graphs = {}

    def __len__(self):
        """Samples per epoch, as the reference's PointTrackingSampler counts them: every frame once per candidate."""
        return self.data.num_frames * self.num_candidates

    def _build(self, B, indices=None):
        pool = int(B * self.oversample) + 1
        dev = self.data.scans.device
        if indices is None:
            index = torch.randint(0, len(self), (pool,), device=dev, generator=self.gen)
        else:       # the epoch's samples first; the random rest of the pool stands in for the ones that are rejected
            index = torch.cat([indices, torch.randint(0, len(self), (pool - B,), device=dev, generator=self.gen)])
        batch, valid = self.processing(self.data, self.cfg, index // self.num_candidates, index % self.num_candidates,
                                       generator=self.gen)
        order = torch.argsort((~valid).to(torch.int8), stable=True)           # valid samples first, original order kept
        # the reference redraws until a sample is valid (sampler.py:230-242); here the pool is oversampled and, should it
        # still hold fewer than B valid samples, the valid ones are re-used cyclically (fixed shapes, graph-safe) — a
        # rejected sample is never handed to the training step unless the whole pool was rejected
        nvalid = valid.sum().clamp(min=1)
        order = order[torch.arange(B, device=dev) % nvalid]
        return {k: v[order] for k, v in batch.items() if not k.startswith("_")}, valid[order]

    def next_batch(self, batch_size=None, indices=None):
        """`indices`: optional (B,) int64 device tensor of sample indices in [0, len(self)) (frame * num_candidates +
        candidate), the reference's epoch order; by default every sample is drawn at random.  Sample i of the batch is
        indices[i] unless the reference would reject it; then valid samples move up and random valid draws fill the end."""
        B = batch_size or self.cfg.batch_size
        if indices is not None and tuple(indices.shape) != (B,):
            raise ValueError(f"next_batch: indices of shape {tuple(indices.shape)} for a batch of {B}")
        if not self.use_graph:
            return self._build(B, indices)
        key = (B, indices is not None)
        if key not in self._graphs:
            static = None if indices is None else torch.zeros(B, dtype=torch.int64, device=self.data.scans.device)
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                self._build(B, static)                           # warm-up: allocator, lazy initialisations
            torch.cuda.current_stream().wait_stream(s)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                out = self._build(B, static)
            self._graphs[key] = (g, out, static)
        g, out, static = self._graphs[key]
        if static is not None:
            static.copy_(indices, non_blocking=True)
        g.replay()
        return out


class DeviceMotionSampler(DeviceSiameseSampler):
    """MotionTrackingSampler + motion_processing (sampler.py:82-181, :262-288) on the device."""

    def __init__(self, tracklets, cfg, device, **kw):
        super().__init__(tracklets, cfg, device, processing=motion_batch, **kw)
