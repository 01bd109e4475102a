"""Synthetic KITTI-shaped training batches (replaces datasets/* of the reference, which is CPU
data preparation and out of scope — SURVEY.md §2.1 rows 12-15, §8d).

`synthetic_siamese_batch` emits exactly the dict `siamese_processing` builds
(datasets/sampler.py:67-78): template_points (B,M,3), search_points (B,N,3), box_label (B,4),
bbox_size (B,3), seg_label (B,N), and for box-aware models points2cc_dist_t (B,M,9),
points2cc_dist_s (B,N,9) — distances to the box centre and its 8 corners
(datasets/points_utils.py:127-143).  Clouds are resampled to the fixed size *with replacement*
whenever the crop holds fewer points (datasets/points_utils.py:24-40), so exact duplicate
points — and therefore exact distance ties in FPS / ball query — are the norm, as on KITTI.

All randomness comes from a numpy Generator seeded by the caller: the same seed gives the same
batch on every box.
"""
import numpy as np
import torch

CAR_WLH = (1.6, 3.9, 1.56)
PED_WLH = (0.7, 0.9, 1.8)


def _box_points(center, wlh, yaw):
    """centre + 8 corners of a yawed box, (9,3). x forward / y left / z up."""
    w, l, h = wlh
    xs = np.array([1, 1, 1, 1, -1, -1, -1, -1]) * (l / 2)
    ys = np.array([1, -1, -1, 1, 1, -1, -1, 1]) * (w / 2)
    zs = np.array([1, 1, -1, -1, 1, 1, -1, -1]) * (h / 2)
    c, s = np.cos(yaw), np.sin(yaw)
    cx = c * xs - s * ys
    cy = s * xs + c * ys
    corners = np.stack([cx, cy, zs], 1) + center[None]
    return np.concatenate([center[None], corners], 0)


def _surface_points(rng, n, wlh, noise=0.02):
    """n points on the surface of an axis-aligned box centred at 0 (LiDAR sees ~2 sides + roof)."""
    w, l, h = wlh
    face = rng.choice(3, size=n, p=[0.45, 0.35, 0.20])
    u = rng.uniform(-0.5, 0.5, size=(n, 3)) * np.array([l, w, h])
    pts = u.copy()
    pts[face == 0, 1] = -w / 2          # near side
    pts[face == 1, 0] = -l / 2          # rear
    pts[face == 2, 2] = h / 2           # roof
    return pts + rng.normal(0, noise, size=(n, 3))


def _resample(rng, pts, size, extra=None):
    """regularize_pc semantics: choice without replacement if enough points, else with replacement."""
    n = pts.shape[0]
    if n == size:
        sel = np.arange(n)
    else:
        sel = rng.choice(n, size=size, replace=size > n)
    return pts[sel], sel


def _in_box(pts, center, wlh, yaw):
    w, l, h = wlh
    d = pts - center[None]
    c, s = np.cos(-yaw), np.sin(-yaw)
    x = c * d[:, 0] - s * d[:, 1]
    y = s * d[:, 0] + c * d[:, 1]
    return (np.abs(x) <= l / 2) & (np.abs(y) <= w / 2) & (np.abs(d[:, 2]) <= h / 2)


def _cdist(a, b):
    return np.sqrt(((a[:, None, :] - b[None, :, :]) ** 2).sum(-1))


def synthetic_siamese_batch(batch_size, template_size=512, search_size=1024, seed=20260924, box_aware=True,
                            wlh=CAR_WLH, uniform=False, device="cpu", pin_memory=False):
    """One training batch for BAT / P2B.  `uniform=True` is the sparse-ball stress distribution
    (points uniform in the crop → heavy first-hit padding in ball query)."""
    rng = np.random.default_rng(seed)
    w, l, h = wlh
    out = {k: [] for k in ("template_points", "search_points", "box_label", "bbox_size", "seg_label",
                           "points2cc_dist_t", "points2cc_dist_s")}
    t_half = np.array([l, w, h]) * 1.25 / 2                      # model_bb_scale 1.25, offset 0
    s_half = np.array([l, w, h]) * 1.25 / 2 + 2.0                 # search_bb_scale 1.25, offset 2
    for _ in range(batch_size):
        # ---------------- template: object-centred crop
        if uniform:
            ut = int(rng.integers(template_size // 2, template_size + 1))
            tp = rng.uniform(-1, 1, size=(ut, 3)) * t_half
        else:
            ut = int(rng.integers(48, template_size + 1))
            tp = _surface_points(rng, ut, wlh)
            tp = np.clip(tp, -t_half, t_half)
        tp, _ = _resample(rng, tp, template_size)
        t_bc = _cdist(tp, _box_points(np.zeros(3), wlh, 0.0))
        # ---------------- search: crop around a perturbed box (Kalman offset, sampler.py:53-57)
        off = np.array([rng.normal(0, 1) * 0.5, rng.normal(0, 1) * 0.5, 0.0])
        off[:2] = np.clip(off[:2], -1.5, 1.5)
        dyaw = np.deg2rad(rng.normal(0, 5.0))
        center = np.array([-off[0], -off[1], 0.0])               # gt box seen from the perturbed crop frame
        us = int(rng.integers(64, search_size + 1))
        if uniform:
            sp = rng.uniform(-1, 1, size=(us, 3)) * s_half
        else:
            n_car = max(8, int(0.30 * us)); n_gnd = int(0.50 * us); n_cl = max(0, us - n_car - n_gnd)
            car = _surface_points(rng, n_car, wlh)
            c, s = np.cos(-dyaw), np.sin(-dyaw)
            car = np.stack([c * car[:, 0] - s * car[:, 1], s * car[:, 0] + c * car[:, 1], car[:, 2]], 1) + center
            gnd = np.stack([rng.uniform(-s_half[0], s_half[0], n_gnd), rng.uniform(-s_half[1], s_half[1], n_gnd),
                            -h / 2 + rng.normal(0, 0.03, n_gnd)], 1)
            cl = rng.uniform(-1, 1, size=(n_cl, 3)) * s_half
            sp = np.concatenate([car, gnd, cl], 0)
            sp = np.clip(sp, -s_half, s_half)
            sp = sp[rng.permutation(sp.shape[0])]
        sp, _ = _resample(rng, sp, search_size)
        seg = _in_box(sp, center, wlh, -dyaw).astype(np.float32)
        s_bc = _cdist(sp, _box_points(center, wlh, -dyaw))
        out["template_points"].append(tp); out["search_points"].append(sp)
        out["box_label"].append(np.array([center[0], center[1], center[2], np.rad2deg(dyaw)]))
        out["bbox_size"].append(np.array(wlh)); out["seg_label"].append(seg)
        out["points2cc_dist_t"].append(t_bc); out["points2cc_dist_s"].append(s_bc)
    batch = {k: torch.from_numpy(np.stack(v).astype(np.float32)) for k, v in out.items()}
    if not box_aware:
        batch.pop("points2cc_dist_t"); batch.pop("points2cc_dist_s")
    if pin_memory and torch.cuda.is_available():
        batch = {k: v.pin_memory() for k, v in batch.items()}
    if device != "cpu":
        batch = {k: v.to(device, non_blocking=True) for k, v in batch.items()}
    return batch


def synthetic_motion_batch(batch_size, point_sample_size=1024, seed=20260924, wlh=CAR_WLH, device="cpu"):
    """One M2-Track training batch with the schema of `motion_processing` (datasets/sampler.py:140-179):
    points (B,2P,5)=[xyz, timestamp∈{0,0.1}, prior-mask], candidate_bc (B,2P,9), seg_label (B,2P),
    box_label / box_label_prev / motion_label (B,4), motion_state_label (B,), prev_bc / this_bc (B,P,9)."""
    rng = np.random.default_rng(seed)
    P = point_sample_size
    w, l, h = wlh
    half = np.array([l, w, h]) * 1.25 / 2 + 2.0
    keys = ("points", "candidate_bc", "seg_label", "box_label", "box_label_prev", "motion_label",
            "motion_state_label", "prev_bc", "this_bc", "bbox_size")
    out = {k: [] for k in keys}
    for _ in range(batch_size):
        frames, bcs, segs, centers, yaws = [], [], [], [], []
        motion = np.array([rng.normal(0, 0.4), rng.normal(0, 0.2), 0.0, np.deg2rad(rng.normal(0, 3))])
        prev_c = np.array([rng.normal(0, 0.3), rng.normal(0, 0.3), 0.0]); prev_yaw = np.deg2rad(rng.normal(0, 3))
        for t, (c0, y0) in enumerate([(prev_c, prev_yaw), (prev_c + motion[:3], prev_yaw + motion[3])]):
            u = int(rng.integers(64, P + 1))
            n_car = max(8, int(0.3 * u)); n_gnd = int(0.5 * u); n_cl = max(0, u - n_car - n_gnd)
            car = _surface_points(rng, n_car, wlh)
            c, s = np.cos(y0), np.sin(y0)
            car = np.stack([c * car[:, 0] - s * car[:, 1], s * car[:, 0] + c * car[:, 1], car[:, 2]], 1) + c0
            gnd = np.stack([rng.uniform(-half[0], half[0], n_gnd), rng.uniform(-half[1], half[1], n_gnd),
                            -h / 2 + rng.normal(0, 0.03, n_gnd)], 1)
            cl = rng.uniform(-1, 1, size=(n_cl, 3)) * half
            pts = np.concatenate([car, gnd, cl], 0)
            pts = pts[rng.permutation(pts.shape[0])]
            pts, _ = _resample(rng, pts, P)
            frames.append(pts); centers.append(c0); yaws.append(y0)
            segs.append(_in_box(pts, c0, wlh, y0).astype(np.float32))
            bcs.append(_cdist(pts, _box_points(c0, wlh, y0)))
        ts = np.concatenate([np.zeros((P, 1)), np.full((P, 1), 0.1)], 0)
        prior = np.concatenate([np.where(segs[0] > 0, rng.choice([0.8, 1.0], P), rng.choice([0.0, 0.2], P)),
                                np.full(P, 0.5)])[:, None]
        out["points"].append(np.concatenate([np.concatenate(frames, 0), ts, prior], 1))
        cand = _cdist(np.concatenate(frames, 0), _box_points(prev_c, wlh, prev_yaw))
        out["candidate_bc"].append(cand)
        out["seg_label"].append(np.concatenate(segs))
        out["box_label"].append(np.array([*centers[1], yaws[1]]))
        out["box_label_prev"].append(np.array([*centers[0], yaws[0]]))
        out["motion_label"].append(motion)
        out["motion_state_label"].append(float(np.linalg.norm(motion[:3]) > 0.15))
        out["prev_bc"].append(bcs[0]); out["this_bc"].append(bcs[1]); out["bbox_size"].append(np.array(wlh))
    batch = {k: torch.from_numpy(np.stack(v).astype(np.float32)) for k, v in out.items()}
    batch["seg_label"] = batch["seg_label"].long()
    batch["motion_state_label"] = batch["motion_state_label"].long()
    if device != "cpu":
        batch = {k: v.to(device, non_blocking=True) for k, v in batch.items()}
    return batch


def synthetic_sequence(n_frames=8, n_points=20000, seed=20260924, wlh=CAR_WLH, speed=0.6, yaw_rate=2.0, n_object=600):
    """A synthetic tracklet with the schema of the reference's test datasets (datasets/kitti.py:150-205:
    a list of {"pc": PointCloud (3, N), "3d_bbox": Box}): one car-sized box driving along a gently curved path through
    ground + clutter returns.  Frame i: centre advances `speed` m along its heading, heading turns `yaw_rate` degrees."""
    from .data_classes import Box, PointCloud
    rng = np.random.default_rng(seed)
    center, yaw = np.array([8.0, 2.0, -0.8 + wlh[2] / 2]), np.deg2rad(15.0)
    ground = np.stack([rng.uniform(-10, 40, n_points), rng.uniform(-20, 20, n_points), np.full(n_points, -0.8)], 1)
    clutter = rng.uniform([-10, -20, -0.8], [40, 20, 2.0], size=(n_points // 10, 3))
    frames = []
    for _ in range(n_frames):
        c, s = np.cos(yaw), np.sin(yaw)
        rot = np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])
        obj = _surface_points(rng, n_object, wlh) @ rot.T + center[None]
        bg = np.concatenate([ground + rng.normal(0, 0.01, ground.shape), clutter])
        bg = bg[~_in_box(bg, center, np.asarray(wlh) * 1.05, yaw)]
        pts = np.concatenate([obj, bg[: n_points - n_object]]).astype(np.float32)
        frames.append({"pc": PointCloud(pts.T.copy()), "3d_bbox": Box(center.copy(), wlh, rot.copy())})
        center = center + speed * np.array([c, s, 0.0])
        yaw = yaw + np.deg2rad(yaw_rate)
    return frames


def synthetic_scene(n_frames=8, n_points=60000, n_objects=8, seed=20260924, wlh=CAR_WLH, n_object=300, extent=60.0):
    """A scan stream with several moving boxes: {"scans": [(n_points, 3) float32 per frame], "boxes": [[Box per frame] per
    object]}.  Objects start on a grid over [-extent, extent]^2, each with its own heading, speed and turn rate; every scan has
    `n_object` surface points per object over ground + clutter returns (points inside any box removed), `n_points` in all."""
    from .data_classes import Box
    rng = np.random.default_rng(seed)
    side = int(np.ceil(np.sqrt(n_objects)))
    cells = np.linspace(-extent * 0.8, extent * 0.8, side) if side > 1 else np.zeros(1)
    z0 = -0.8 + wlh[2] / 2
    state = [(np.array([cells[i % side] + rng.uniform(-2, 2), cells[i // side] + rng.uniform(-2, 2), z0]),
              rng.uniform(-np.pi, np.pi), rng.uniform(0.2, 0.8), np.deg2rad(rng.uniform(-3, 3))) for i in range(n_objects)]
    n_bg = max(n_points - n_objects * n_object, 0)
    ground = np.stack([rng.uniform(-extent, extent, n_bg), rng.uniform(-extent, extent, n_bg), np.full(n_bg, -0.8)], 1)
    clutter = rng.uniform([-extent, -extent, -0.8], [extent, extent, 2.0], size=(n_bg // 10, 3))
    scans, boxes = [], [[] for _ in range(n_objects)]
    for _ in range(n_frames):
        objs, bg = [], np.concatenate([ground + rng.normal(0, 0.01, ground.shape), clutter])
        for i, (center, yaw, speed, turn) in enumerate(state):
            c, s = np.cos(yaw), np.sin(yaw)
            rot = np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])
            objs.append(_surface_points(rng, n_object, wlh) @ rot.T + center[None])
            bg = bg[~_in_box(bg, center, np.asarray(wlh) * 1.05, yaw)]
            boxes[i].append(Box(center.copy(), wlh, rot.copy()))
            state[i] = (center + speed * np.array([c, s, 0.0]), yaw + turn, speed, turn)
        pts = np.concatenate(objs + [bg])[:n_points]
        if pts.shape[0] < n_points:
            pts = np.concatenate([pts, bg[rng.integers(0, len(bg), n_points - pts.shape[0])]])
        scans.append(pts.astype(np.float32))
    return {"scans": scans, "boxes": boxes}
