"""Split evaluation with K tracklets in flight: the graph-captured frame of `DeviceTracker` with a slot dimension.

`DeviceTracker` runs one B=1 frame per replay, which leaves most of the GPU idle (FPS and resampling run one CTA per
cloud).  Here a chunk of tracklets sits on the device as a `DeviceTracklets` pool (padded scans, per-frame first /
previous indices, fp32 boxes) plus fp64 copies of the ground-truth boxes, and K slots each track one tracklet of it:
  * one fixed-shape step advances every slot by one frame — search crop of the current frame in the reference box's frame
    (the slot's result box, or the pool's ground truth of the previous / current frame for reference_BB 'previous_gt' /
    'current_gt'), template crop of the previous frame in the result box's frame, template = first-frame crop + previous crop
    (or, for shape_aggregation 'all', the slot's history: the crops of every past frame, appended once per step by
    csrc/geometry.cu's o3d_crop_append), resampling, BoxCloud, the network in eval mode, best proposal, box update of the
    reference box, and the overlap / centre distance of the new box against the ground truth (csrc/track_eval.cu) written
    into a record indexed by the pool frame — and is captured once in a CUDA graph;
  * the random draws of a slot (resampling, limit_box) are keyed by (seed, tracklet id, frame within the tracklet), so a
    tracklet's result does not depend on the slot it runs in or on K;
  * between replays, a slot whose tracklet has ended is re-filled with the next one (`DeviceTracker.reset`'s computation for
    that tracklet, issued without a host sync); the host plans that schedule from the tracklet lengths, longest first;
  * the host synchronises once per chunk, to copy the records back (and, in 'all' mode, the slots' peak history counts: a
    chunk whose history overflowed its capacity runs again with the capacity raised, so nothing is truncated).
Idle slots run on a valid dummy frame and record nothing."""
import heapq

import numpy as np
import torch

from .. import ops, runtime
from ..datasets.device_sampler import DeviceTracklets
from . import boxes as bx
from .device_tracker import HISTORY_POINTS, is_motion, tracking_modes
from .sampling import resample_batched

# keyed-draw streams of one frame, in DeviceTracker's buffer layout: u_s (perm, pick), u_t (perm, pick), limit_box's two draws
STREAM_SEARCH_PERM, STREAM_SEARCH_PICK, STREAM_TEMPLATE_PERM, STREAM_TEMPLATE_PICK, STREAM_LIMIT_BOX = range(5)


def canonical(box):
    """The slots' boxes moved to the origin, axis-aligned (the frame the template / previous points are expressed in)."""
    return bx.Box(torch.zeros_like(box.center), box.wlh, torch.eye(3, device=box.center.device).expand_as(box.rot))


def motion_data(cfg, box, prev_pts, this_pts, first_flag):
    """DeviceTracker._inputs_motion's input dict with a slot dimension, from the resampled previous / current crops (K, n, 3):
    the previous points masked 1 / 0 by the box on the first frame (first_flag (K,) = 1), 0.8 / 0.2 afterwards."""
    half = torch.stack([box.wlh[:, 1], box.wlh[:, 0], box.wlh[:, 2]], -1) * (1.25 / 2)
    inside = (prev_pts.abs() <= half[:, None, :]).all(-1).float()
    first = first_flag[:, None]
    mask_prev = inside * (0.6 + 0.4 * first) + 0.2 * (1 - first)             # 1 / 0 on the first frame, 0.8 / 0.2 afterwards
    col = lambda pts, t, m: torch.cat([pts, torch.full_like(pts[..., :1], t), m[..., None]], -1)
    data = {"points": torch.cat([col(prev_pts, 0.0, mask_prev), col(this_pts, 0.1, torch.full_like(mask_prev, 0.5))], 1)}
    if getattr(cfg, "box_aware", False):
        bc = bx.point_to_box_distance(prev_pts, canonical(box))
        data["candidate_bc"] = torch.cat([bc, torch.zeros_like(bc)], 1)
    return data


def best_proposal(est):
    """(K, num_proposal, 5) proposals -> (K, 4) offsets of the highest-scoring one per slot; (K, 4) passes through."""
    if est.dim() == 3:
        best = est[:, :, 4].argmax(1)
        est = est.gather(1, best[:, None, None].expand(-1, 1, est.shape[-1]))[:, 0, :4]
    return est


def best_proposal_score(est):
    """(K, num_proposal, 5) proposals -> (`best_proposal`'s (K, 4) offsets, (K,) the score, column 4, of that proposal)."""
    best = est[:, :, 4].argmax(1)
    row = est.gather(1, best[:, None, None].expand(-1, 1, est.shape[-1]))[:, 0]
    return row[:, :4], row[:, 4]


def plan_schedule(lengths, slots):
    """Slot schedule of one chunk.  `lengths`: frames per tracklet, in pool order.  Tracklets are admitted longest first
    (ties in input order), each into the slot that frees first (lowest slot on ties); a tracklet of n frames holds its slot
    for n - 1 steps, and tracklets of fewer than two frames never take one.
    Returns {"offsets": pool frame index of every tracklet's frame 0, "admissions": per step, the (slot, tracklet) pairs to
    admit before it, "steps": number of steps, "slots": slots used}."""
    lengths = [int(n) for n in lengths]
    offsets = np.concatenate([[0], np.cumsum(lengths)[:-1]]).astype(np.int64) if lengths else np.zeros(0, np.int64)
    order = sorted((j for j, n in enumerate(lengths) if n > 1), key=lambda j: -lengths[j])
    k_used = min(int(slots), len(order))
    free = [(0, k) for k in range(k_used)]                    # (step at which the slot is free, slot)
    admissions, steps = [], 0
    for j in order:
        t, k = heapq.heappop(free)
        end = t + lengths[j] - 1
        steps = max(steps, end)
        admissions.extend([] for _ in range(t + 1 - len(admissions)))
        admissions[t].append((k, j))
        heapq.heappush(free, (end, k))
    admissions.extend([] for _ in range(steps - len(admissions)))
    return {"offsets": offsets, "admissions": admissions, "steps": steps, "slots": k_used}


def pool_frame_bytes(max_points):
    """Device bytes one frame of a chunk occupies: the padded scan, the pool's indices and fp32 box, the fp64 ground truth,
    the next-frame bound and the records (result box, overlap, distance), rounded up."""
    return 12 * int(max_points) + 512


def history_bytes(slots, capacity):
    """Device bytes of the 'all' template history of `slots` slots: points (12 B) and keep mask (1 B) per position, plus the
    template's permutation draw (4 B) and the resampling's compaction scratch (4 B) over the same positions."""
    return int(slots) * int(capacity) * (12 + 1 + 4 + 4)


def plan_chunks(lengths, frame_bytes, max_resident_bytes, fixed_bytes=0):
    """Consecutive groups of tracklets (input order) whose frames fit `max_resident_bytes` beside `fixed_bytes` of per-chunk
    state (the 'all' history); a tracklet is never split."""
    budget = max_resident_bytes - fixed_bytes
    chunks, cur, used = [], [], 0
    for j, n in enumerate(lengths):
        need = int(n) * frame_bytes
        if need > budget:
            raise ValueError(f"tracklet {j} needs {need} bytes on the device beside {fixed_bytes} bytes of slot state, more than "
                             f"max_resident_bytes={max_resident_bytes}")
        if cur and used + need > budget:
            chunks.append(cur)
            cur, used = [], 0
        cur.append(j)
        used += need
    if cur:
        chunks.append(cur)
    return chunks


class BatchedDeviceTracker:
    """K slots tracking the tracklets of one chunk.  `tracklets`: lists of {"pc", "3d_bbox"}; `ids`: their tracklet ids
    (the key of their random draws; default 0..n-1); `max_points`: padded scan size (default: the largest scan);
    `history`: starting capacity (points per slot) of the 'all' template history, raised by `run()` when a slot needs more."""

    def __init__(self, model, tracklets, slots, seed=0, ids=None, max_points=None, use_graph=True, history=HISTORY_POINTS,
                 precision="fp32"):
        self.precision = runtime.check_precision(precision)
        self.model = model.eval()
        self.cfg = cfg = model.config
        self.dev = dev = next(model.parameters()).device
        self.use_graph = bool(use_graph) and dev.type == "cuda"
        self.seed = int(seed)
        self.needs_bc = hasattr(model, "mlp_bc")
        self.motion = is_motion(model)
        self.mode, self.ref_mode = tracking_modes(model)
        lengths = [len(t) for t in tracklets]
        self.ids = list(range(len(tracklets))) if ids is None else [int(i) for i in ids]
        self.plan = plan_schedule(lengths, slots)
        self.pool = P = DeviceTracklets(tracklets, dev, max_points)
        F, N = P.num_frames, P.scans.shape[1]
        self.F, self.N = F, N
        frames = [f["3d_bbox"] for t in tracklets for f in t]
        f64 = dict(device=dev, dtype=torch.float64)
        self.gt_c = torch.tensor(np.stack([b.center for b in frames]), **f64)
        self.gt_r = torch.tensor(np.stack([b.rotation_matrix for b in frames]), **f64)
        self.gt_s = torch.tensor(np.stack([b.wlh for b in frames]), **f64)
        self.stop = torch.tensor(np.repeat(self.plan["offsets"] + np.asarray(lengths, np.int64), lengths), device=dev)
        self.arange = torch.arange(N, device=dev)
        K = self.K = max(self.plan["slots"], 1)
        f = dict(device=dev, dtype=torch.float32)
        # slot state
        self.box_c = torch.zeros(K, 3, **f)
        self.box_s = torch.ones(K, 3, **f)
        self.box_r = torch.eye(3, **f).repeat(K, 1, 1)
        if self.mode != "all":
            self.first_local = torch.zeros(K, N, 3, **f)
            self.first_keep = torch.zeros(K, N, dtype=torch.bool, device=dev)
        self.first_flag = torch.zeros(K, **f)
        self.frame = torch.full((K,), -1, dtype=torch.int64, device=dev)       # pool frame being tracked, -1 = idle
        self.tracklet = torch.zeros(K, dtype=torch.int64, device=dev)
        # keyed draws, refreshed inside the step
        size_s = cfg.point_sample_size if self.motion else cfg.search_size
        size_t = cfg.point_sample_size if self.motion else cfg.template_size
        self.u_s = (torch.zeros(K, N, **f), torch.zeros(K, size_s, **f))
        self.u_t = (torch.zeros(K, 2 * N, **f), torch.zeros(K, size_t, **f))
        self.u_lim = torch.zeros(K, 2, **f)
        # records, indexed by pool frame; row F takes the idle slots' writes
        self.rec_c = torch.zeros(F + 1, 3, **f)
        self.rec_r = torch.zeros(F + 1, 3, 3, **f)
        self.overlap = torch.zeros(F, **f64)
        self.distance = torch.zeros(F, **f64)
        if self.mode == "all":
            self.hist_count = torch.zeros(K, dtype=torch.int64, device=dev)
            self.hist_peak = torch.zeros(K, dtype=torch.int64, device=dev)  # largest count of each slot over the chunk
            self._alloc_history(int(history))
        self.graph = None

    def _alloc_history(self, H):
        """History buffers for H points per slot (contents undefined until admission); drops the captured graph."""
        K = self.K
        self.hist = torch.zeros(K, H, 3, device=self.dev)
        self.hist_keep = torch.zeros(K, H, dtype=torch.bool, device=self.dev)
        self.u_t = (torch.zeros(K, H, device=self.dev), self.u_t[1])          # the template draw is over the history
        self.H = H
        self.graph = None

    # ------------------------------------------------------------------ one step for all slots, fixed shapes
    def _draw(self, local):
        for stream, buf in zip(range(5), (*self.u_s, *self.u_t, self.u_lim)):
            ops.keyed_uniform(self.tracklet, local, self.seed, stream, buf.shape[1], out=buf)

    def _inputs_motion(self, f, box):
        """DeviceTracker._inputs_motion with a slot dimension."""
        cfg, P, N = self.cfg, self.pool, self.N
        n = cfg.point_sample_size
        p_local, p_keep = bx.crop_in_box_frame(P.scans, box, cfg.bb_scale, cfg.bb_offset, P.prev[f], P.count)
        t_local, t_keep = bx.crop_in_box_frame(P.scans, box, cfg.bb_scale, cfg.bb_offset, f, P.count)
        prev_pts, _, _ = resample_batched(p_local, p_keep, n, self.u_t[0][:, :N], self.u_t[1])
        this_pts, _, _ = resample_batched(t_local, t_keep, n, self.u_s[0], self.u_s[1])
        return motion_data(cfg, box, prev_pts, this_pts, self.first_flag)

    def _canon(self, box):
        return canonical(box)

    def _inputs(self, f, box, ref, active):
        """DeviceTracker._inputs with a slot dimension: `box` the slots' result boxes, `ref` their reference boxes."""
        if self.motion:
            return self._inputs_motion(f, box)
        cfg, P, mode = self.cfg, self.pool, self.mode
        s_local, s_keep = bx.crop_in_box_frame(P.scans, ref, cfg.search_bb_scale, cfg.search_bb_offset, f, P.count)
        search, _, _ = resample_batched(s_local, s_keep, cfg.search_size, *self.u_s)
        if mode == "all":
            # append the previous frame's crop in the current result box; the history then holds frames 0 .. t-1
            prev = torch.where(active, P.prev[f], torch.full_like(f, -1))
            bx.crop_append(P.scans, box, cfg.model_bb_scale, cfg.model_bb_offset, prev, P.count, self.hist, self.hist_keep,
                           self.hist_count)
            torch.maximum(self.hist_peak, self.hist_count, out=self.hist_peak)
            cand, keep = self.hist, self.hist_keep
        elif mode == "first":
            cand, keep = self.first_local, self.first_keep
        else:
            p_local, p_keep = bx.crop_in_box_frame(P.scans, box, cfg.model_bb_scale, cfg.model_bb_offset, P.prev[f], P.count)
            if mode == "firstandprevious":
                cand, keep = torch.cat([self.first_local, p_local], 1), torch.cat([self.first_keep, p_keep], 1)
            else:
                cand, keep = p_local, p_keep
        template, _, _ = resample_batched(cand, keep, cfg.template_size, self.u_t[0][:, : cand.shape[1]], self.u_t[1])
        data = {"template_points": template, "search_points": search}
        if self.needs_bc:
            data["points2cc_dist_t"] = bx.point_to_box_distance(template, self._canon(box))
        return data

    def _step(self):
        cfg, P = self.cfg, self.pool
        with torch.no_grad(), runtime.static_weights_scope(), runtime.inference_precision_scope(self.precision):
            active = self.frame >= 0
            f = self.frame.clamp(min=0)                                        # idle slots track pool frame 0, unrecorded
            self._draw(f - P.first[f])
            box = bx.Box(self.box_c, self.box_s, self.box_r)
            if self.ref_mode == "previous_result":
                ref = box
            else:
                ref = P.box(P.prev[f] if self.ref_mode == "previous_gt" else f)
            est = best_proposal(self.model(self._inputs(f, box, ref, active))["estimation_boxes"])
            new = bx.offset_box(ref, est, degrees=cfg.degrees, use_z=cfg.use_z, limit_box=cfg.limit_box, rand=self.u_lim * 2 - 1)
            self.box_c.copy_(new.center)
            self.box_r.copy_(new.rot)
            if ref is not box:
                self.box_s.copy_(new.wlh)                                      # the result takes the reference box's size
            row = f.masked_fill(~active, self.F)
            self.rec_c.index_copy_(0, row, self.box_c)
            self.rec_r.index_copy_(0, row, self.box_r)
            ops.track_metrics(self.box_c, self.box_r, self.box_s, self.gt_c, self.gt_r, self.gt_s, self.frame, cfg.IoU_space,
                              cfg.up_axis, self.overlap, self.distance)
            self.first_flag.zero_()
            nxt = f + 1
            self.frame.copy_(torch.where(active & (nxt < self.stop[f]), nxt, torch.full_like(nxt, -1)))

    def _capture(self):
        # every slot is idle here, so the warm-up step changes no state that a replay reads before admission rewrites it
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            self._step()                                                       # warm-up (allocations, weight packing)
        torch.cuda.current_stream().wait_stream(s)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self._step()

    # ------------------------------------------------------------------ admission, between replays
    def admit(self, k, j):
        """Slot k starts tracklet j of the chunk: DeviceTracker.reset on its first frame, without a host sync."""
        cfg, P = self.cfg, self.pool
        f0 = int(self.plan["offsets"][j])
        self.box_c[k].copy_(P.center[f0])
        self.box_s[k].copy_(P.wlh[f0])
        self.box_r[k].copy_(P.rot[f0])
        if self.mode == "all":
            self.hist_count[k] = 0
            self.hist_keep[k].zero_()
        elif not self.motion:
            box = bx.Box(P.center[f0], P.wlh[f0], P.rot[f0])
            local, keep, _ = bx.crop_and_center(P.scans[f0], box, offset=cfg.model_bb_offset, scale=cfg.model_bb_scale)
            self.first_local[k].copy_(local)
            self.first_keep[k].copy_(keep & (self.arange < P.count[f0]))
        self.first_flag[k] = 1.0
        self.frame[k] = f0 + 1
        self.tracklet[k] = self.ids[j]

    def step(self):
        if not self.use_graph:
            self._step()
            return
        if self.graph is None:
            self._capture()
        self.graph.replay()

    def track(self):
        """Enqueue the whole schedule of the chunk: admissions and steps, no host synchronisation."""
        if self.plan["steps"] and self.use_graph and self.graph is None:
            self._capture()
        for t in range(self.plan["steps"]):
            for k, j in self.plan["admissions"][t]:
                self.admit(k, j)
            self.step()

    def run(self):
        """Track every tracklet of the chunk; returns host copies of the records after the chunk's one synchronisation:
        (overlap (F,), distance (F,), result centre (F, 3), result rotation (F, 3, 3)); frame-0 entries are left at 0.
        In 'all' mode, a chunk in which some slot's history outgrew its capacity runs again with the capacity raised to
        cover it, so the result is that of an unbounded history."""
        self.track()
        while self.mode == "all":
            peak = int(self.hist_peak.max())
            if peak <= self.H:
                break
            self._alloc_history(-(-peak * 5 // 4 // 4096) * 4096)               # headroom: the rerun's trajectory may differ
            self.hist_peak.zero_()
            self.hist_count.zero_()
            self.track()
        F = self.F
        return (self.overlap.cpu().numpy(), self.distance.cpu().numpy(), self.rec_c[:F].cpu().double().numpy(),
                self.rec_r[:F].cpu().double().numpy())
