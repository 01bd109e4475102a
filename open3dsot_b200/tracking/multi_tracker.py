"""Live tracking of many targets through one scan stream: K slots advanced together by one captured step per scan.

`DeviceTracker` follows one target and `BatchedDeviceTracker` replays pre-loaded tracklets with ground truth for every frame;
this tracker takes the scans as they arrive and targets as they appear and disappear:
  * `step(points)` copies the scan into a static (2, N, 3) ping-pong buffer (the one copy of the scan) and replays one captured
    step that advances every active slot to it: search crop of the new scan around the slot's result box, template = the
    first-frame crop (kept per slot) + the previous scan's crop in the result box ('firstandprevious', or either one alone for
    'first' / 'previous'), or for motion models (M2-Track) the previous and current scans' crops, then BoxCloud, the network in
    eval mode, the best proposal and the box update, exactly as `BatchedDeviceTracker._step`.  Which buffer holds the current /
    previous scan is a device index flipped inside the graph, so one capture serves every step;
  * every crop is one `o3d_crop_resample` launch for all slots (csrc/crop_resample.cu): crop and resampling in one kernel with
    the keyed draws computed in place, never a (K, N) array;
  * `add(id, box)` starts a target on the most recent scan (`DeviceTracker.reset`'s computation) and `drop(id)` frees its slot,
    both between steps and without a host synchronisation;
  * a slot's draws are keyed by (seed, target id, frame within the target's track), so a target's result does not depend on its
    slot, on the other targets or on `max_targets`.
Idle slots run on a fixed dummy box and report nothing: the cost of a step follows `max_targets`, not the number of active
targets.  Ground-truth reference boxes (reference_BB 'previous_gt' / 'current_gt') have no meaning on a live stream, and
shape_aggregation 'all' is not supported here; both are refused."""
import numpy as np
import torch

from .. import ops, runtime
from . import boxes as bx
from .batched_tracker import (STREAM_LIMIT_BOX, STREAM_SEARCH_PERM, STREAM_SEARCH_PICK, STREAM_TEMPLATE_PERM, STREAM_TEMPLATE_PICK,
                              best_proposal, canonical, motion_data)
from .device_tracker import is_motion, tracking_modes


def _half(box, scale, offset):
    """crop_in_box_frame's half extents (l, w, h on x, y, z), the same expression so that the crop test is the same."""
    return torch.stack([box.wlh[..., 1], box.wlh[..., 0], box.wlh[..., 2]], -1) * (scale / 2) + offset


def _box_values(box):
    """(center, wlh, 3x3 rotation) as float64 numpy arrays from a data_classes.Box or a tracking.boxes.Box."""
    if isinstance(box, bx.Box):
        return tuple(np.asarray(t.detach().cpu(), dtype=np.float64) for t in box)
    return np.asarray(box.center, np.float64), np.asarray(box.wlh, np.float64), np.asarray(box.rotation_matrix, np.float64)


class MultiTargetTracker:
    """`max_targets` slots over scans of at most `max_points` points.  `seed` keys the random draws; `use_graph`: capture the
    step in a CUDA graph on the first `step()` (eager otherwise).  Call `step(scan)` for every scan of the stream, `add(id, box)`
    to start a target on the scan just given, `drop(id)` to end it."""

    def __init__(self, model, max_points, max_targets, seed=0, use_graph=True):
        self.model = model.eval()
        self.cfg = cfg = model.config
        self.dev = dev = next(model.parameters()).device
        self.use_graph = bool(use_graph) and dev.type == "cuda"
        self.seed = int(seed)
        self.needs_bc = hasattr(model, "mlp_bc")
        self.motion = is_motion(model)
        self.mode, ref_mode = tracking_modes(model)
        if ref_mode != "previous_result":
            raise ValueError(f"reference_BB '{ref_mode}': a live stream has no ground truth; use 'previous_result'")
        if self.mode == "all":
            raise ValueError("shape_aggregation 'all' is not supported by the live multi-target tracker")
        self.N = N = int(max_points)
        self.K = K = int(max_targets)
        if N < 1 or K < 1 or K > 65535:
            raise ValueError(f"max_points={N} and max_targets={K} must be >= 1 (max_targets <= 65535)")
        f = dict(device=dev, dtype=torch.float32)
        i64 = dict(device=dev, dtype=torch.int64)
        self.scans = torch.zeros(2, N, 3, **f)
        self.count = torch.zeros(2, **i64)
        self.cur = torch.ones(K, **i64)                  # per slot: the buffer holding the most recent scan (all equal) ...
        self.prev = torch.zeros(K, **i64)                # ... and the one holding the scan before it
        self._cur = 1                                     # host mirror of cur
        self.arange = torch.arange(N, device=dev)
        # slot state; idle slots hold the dummy box
        self.box_c = torch.zeros(K, 3, **f)
        self.box_s = torch.ones(K, 3, **f)
        self.box_r = torch.eye(3, **f).repeat(K, 1, 1)
        self.first_flag = torch.zeros(K, **f)
        self.active = torch.zeros(K, dtype=torch.bool, device=dev)
        self.key = torch.zeros(K, **i64)                  # target id of the slot (the key of its draws)
        self.t = torch.zeros(K, **i64)                    # frame within the target's track
        self.u_lim = torch.zeros(K, 2, **f)
        if self.mode in ("firstandprevious", "first"):
            self.first_local = torch.zeros(K, N, 3, **f)
            self.first_keep = torch.zeros(K, N, dtype=torch.bool, device=dev)
        self.slot_of = {}                                 # target id -> slot
        self.scans_seen = 0
        self.graph = None

    # ------------------------------------------------------------------ one step for all slots, fixed shapes
    def _crop(self, which, box, half, perm, pick, size, prefix=False):
        scans = self.scans if which is not None else self.scans[:, :0]
        frame = which if which is not None else self.cur
        pre = (self.first_local, self.first_keep) if prefix else (None, None)
        out, _ = ops.crop_resample(scans, self.count, frame, box.center, box.rot, half, size, self.seed, self.key, self.t, perm,
                                   pick, *pre)
        return out

    def _inputs(self, box):
        cfg = self.cfg
        if self.motion:
            h = _half(box, cfg.bb_scale, cfg.bb_offset)
            n = cfg.point_sample_size
            prev_pts = self._crop(self.prev, box, h, STREAM_TEMPLATE_PERM, STREAM_TEMPLATE_PICK, n)
            this_pts = self._crop(self.cur, box, h, STREAM_SEARCH_PERM, STREAM_SEARCH_PICK, n)
            return motion_data(cfg, box, prev_pts, this_pts, self.first_flag)
        search = self._crop(self.cur, box, _half(box, cfg.search_bb_scale, cfg.search_bb_offset), STREAM_SEARCH_PERM,
                            STREAM_SEARCH_PICK, cfg.search_size)
        h = _half(box, cfg.model_bb_scale, cfg.model_bb_offset)
        if self.mode == "first":                          # the first-frame crop alone: no scan in the candidate set
            template = self._crop(None, box, h, STREAM_TEMPLATE_PERM, STREAM_TEMPLATE_PICK, cfg.template_size, prefix=True)
        else:
            template = self._crop(self.prev, box, h, STREAM_TEMPLATE_PERM, STREAM_TEMPLATE_PICK, cfg.template_size,
                                  prefix=self.mode == "firstandprevious")
        data = {"template_points": template, "search_points": search}
        if self.needs_bc:
            data["points2cc_dist_t"] = bx.point_to_box_distance(template, canonical(box))
        return data

    def _step(self):
        cfg = self.cfg
        with torch.no_grad(), runtime.static_weights_scope():
            self.prev.copy_(self.cur)
            self.cur.neg_().add_(1)
            self.t.add_(self.active.long())
            ops.keyed_uniform(self.key, self.t, self.seed, STREAM_LIMIT_BOX, 2, out=self.u_lim)
            box = bx.Box(self.box_c, self.box_s, self.box_r)
            est = best_proposal(self.model(self._inputs(box))["estimation_boxes"])
            new = bx.offset_box(box, est, degrees=cfg.degrees, use_z=cfg.use_z, limit_box=cfg.limit_box, rand=self.u_lim * 2 - 1)
            a = self.active[:, None]
            self.box_c.copy_(torch.where(a, new.center, self.box_c))            # idle slots keep the dummy box
            self.box_r.copy_(torch.where(a[..., None], new.rot, self.box_r))
            self.first_flag.zero_()

    def _capture(self):
        # the warm-up runs a real step; the state it advances is restored before the captured graph's first replay
        state = (self.cur, self.prev, self.t, self.box_c, self.box_r, self.first_flag, self.u_lim)
        snap = [t.clone() for t in state]
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            self._step()                                                       # warm-up (allocations, weight packing)
        torch.cuda.current_stream().wait_stream(s)
        for t, v in zip(state, snap):
            t.copy_(v)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self._step()
        for t, v in zip(state, snap):
            t.copy_(v)

    # ------------------------------------------------------------------ public interface
    def step(self, points, n_valid=None):
        """Load the next scan (`points` (n, 3), the first `n_valid` valid; a CUDA tensor, or a host tensor copied without a
        sync) and advance every active target to it.  Returns `boxes()`: device views of the slots' state, no host sync."""
        n = points.shape[0]
        if n > self.N:
            raise ValueError(f"max_points: the scan has {n} points, the tracker was built for {self.N}")
        n_valid = n if n_valid is None else int(n_valid)
        nxt = 1 - self._cur
        self.scans[nxt, :n].copy_(points, non_blocking=True)
        self.count[nxt].fill_(min(n_valid, n))
        if not self.use_graph:
            self._step()
        else:
            if self.graph is None:
                self._capture()
            self.graph.replay()
        self._cur = nxt
        self.scans_seen += 1
        return self.boxes()

    def add(self, target_id, box):
        """Start target `target_id` on the most recent scan with `box` (a data_classes.Box or a tracking.boxes.Box): the box is
        its result on that scan, and the template's first-frame crop is taken from it.  No host sync."""
        tid = int(target_id)
        if tid in self.slot_of:
            raise ValueError(f"target_id {tid} is already active")
        if len(self.slot_of) >= self.K:
            raise ValueError(f"max_targets: all {self.K} slots are taken; drop a target first")
        if self.scans_seen == 0:
            raise RuntimeError("add() starts a target on the most recent scan: call step() with a scan first")
        k = min(set(range(self.K)) - set(self.slot_of.values()))
        c, s, r = _box_values(box)
        vals = torch.tensor(np.concatenate([c, s, r.reshape(-1)]), dtype=torch.float32)
        if self.dev.type == "cuda":
            vals = vals.pin_memory().to(self.dev, non_blocking=True)                # no host sync
        self.box_c[k].copy_(vals[0:3])
        self.box_s[k].copy_(vals[3:6])
        self.box_r[k].copy_(vals[6:15].view(3, 3))
        if self.mode in ("firstandprevious", "first"):
            cfg, cur = self.cfg, self._cur
            b = bx.Box(self.box_c[k], self.box_s[k], self.box_r[k])
            local, keep, _ = bx.crop_and_center(self.scans[cur], b, offset=cfg.model_bb_offset, scale=cfg.model_bb_scale)
            self.first_local[k].copy_(local)
            self.first_keep[k].copy_(keep & (self.arange < self.count[cur]))
        # fill_ on a view, not `x[k] = value`: indexed assignment of a Python scalar copies it from the host and synchronises
        self.first_flag[k].fill_(1.0)
        self.active[k].fill_(True)
        self.key[k].fill_(tid)
        self.t[k].zero_()
        self.slot_of[tid] = k

    def drop(self, target_id):
        """End target `target_id` and free its slot (it returns to the dummy box).  No host sync."""
        tid = int(target_id)
        if tid not in self.slot_of:
            raise ValueError(f"target_id {tid} is not active")
        k = self.slot_of.pop(tid)
        self.active[k].fill_(False)
        self.box_c[k].zero_()
        self.box_s[k].fill_(1.0)
        self.box_r[k].copy_(torch.eye(3, device=self.dev))
        self.key[k].zero_()
        self.t[k].zero_()
        if self.mode in ("firstandprevious", "first"):
            self.first_keep[k].zero_()

    def boxes(self):
        """Device state of the slots: ids (K,) int64 (-1 for an idle slot), center (K, 3), wlh (K, 3), rot (K, 3, 3), active (K,)."""
        return {"ids": torch.where(self.active, self.key, torch.full_like(self.key, -1)), "center": self.box_c, "wlh": self.box_s,
                "rot": self.box_r, "active": self.active}

    def snapshot(self):
        """A device copy of the slots' boxes, (K, 15) = centre, wlh, row-major rotation; `results()` without the read-back."""
        return torch.cat([self.box_c, self.box_s, self.box_r.reshape(self.K, 9)], 1)

    def targets(self):
        """{target id: slot} of the active targets (host state)."""
        return dict(self.slot_of)

    def results(self):
        """{target id: data_classes.Box} of the active targets, read back from the device once."""
        from ..datasets.data_classes import Box
        host = self.snapshot().cpu().double().numpy()
        return {tid: Box(host[k, 0:3], host[k, 3:6], host[k, 6:15].reshape(3, 3)) for tid, k in self.slot_of.items()}


def track_stream(model, scans, starts, ends, max_targets, seed=0, max_points=None, use_graph=True):
    """Track targets through a stream of scans.  `scans`: iterable of (n, 3) tensors; `starts`: {frame: [(id, Box), ...]} — each
    target starts on that scan with that box; `ends`: {id: last frame} (a target without an entry runs to the end of the
    stream).  `max_points`: the scan buffer's size (default: the largest scan, which needs the whole stream up front).
    Returns {id: {frame: data_classes.Box}}, from the frame a target starts on to its last frame; the device is read back once."""
    from ..datasets.data_classes import Box
    if max_points is None:
        scans = list(scans)
        max_points = max((s.shape[0] for s in scans), default=1)
    trk = MultiTargetTracker(model, max_points, max_targets, seed=seed, use_graph=use_graph)
    dev = trk.dev
    records = []                                                              # (frame, {id: slot}, device snapshot)
    for t, pts in enumerate(scans):
        pts = torch.as_tensor(pts)
        if pts.device != dev:
            pts = pts.to(dev, dtype=torch.float32, non_blocking=True)
        trk.step(pts.float())
        for tid, box in starts.get(t, ()):
            trk.add(tid, box)
        live = trk.targets()
        if live:
            records.append((t, live, trk.snapshot()))
        for tid in live:
            if ends.get(tid, -1) == t:
                trk.drop(tid)
    out = {}
    if records:
        host = torch.stack([r[2] for r in records]).cpu().double().numpy()
        for (t, live, _), h in zip(records, host):
            for tid, k in live.items():
                out.setdefault(tid, {})[t] = Box(h[k, 0:3], h[k, 3:6], h[k, 6:15].reshape(3, 3))
    return out
