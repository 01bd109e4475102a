"""B=1 tracking inference with the whole frame on the device (SURVEY.md §8f rank 2).

The reference's frame loop (models/base_model.py:44-117, :166-247) crops and resamples on the host with numpy /
pyquaternion, uploads two small clouds, runs the network, downloads the proposals (`.cpu().numpy()`, :48) and updates the
box on the host.  Here a frame is: scan already on the device -> search-area crop in the previous box's frame
(generate_search_area :197-218; reference_BB 'previous_gt' / 'current_gt': the ground-truth box the caller passes) ->
template = first-frame crop + previous-frame crop (generate_template :166-195, shape_aggregation 'firstandprevious' /
'first' / 'previous'), or for 'all' the crops of every past frame, each in its own result box, appended to a history buffer
-> fixed-shape resampling (sampling.py) -> BoxCloud of the template (bat.py:41-55) -> network in eval mode on the fused
kernels -> best proposal -> box update (getOffsetBB) of the reference box.
Every tensor has a static shape, nothing is read back, so the frame is captured once in a CUDA graph and replayed."""
import torch

from . import boxes as bx
from .sampling import resample

HISTORY_POINTS = 1 << 18        # starting capacity of the 'all' template history, points per tracklet (it grows on demand)


def template_mode(cfg):
    """shape_aggregation the way generate_template reads it (substring tests, in its order): 'firstandprevious', 'first',
    'previous' or 'all'; anything else is a ValueError."""
    raw = cfg.get("shape_aggregation", "firstandprevious")
    for mode in ("FIRSTANDPREVIOUS", "FIRST", "PREVIOUS", "ALL"):
        if mode in str(raw).upper():
            return mode.lower()
    raise ValueError(f"unknown shape_aggregation '{raw}'")


def reference_mode(cfg):
    """reference_BB the way generate_search_area reads it: 'previous_result', 'previous_gt' or 'current_gt'."""
    raw = cfg.get("reference_BB", "previous_result")
    for mode in ("PREVIOUS_RESULT", "PREVIOUS_GT", "CURRENT_GT"):
        if mode in str(raw).upper():
            return mode.lower()
    raise ValueError(f"unknown reference_BB '{raw}'")


def is_motion(model):
    """Motion-centric models (M2-Track): a two-frame input instead of template + search area."""
    return "point_sample_size" in model.config and not hasattr(model, "backbone")


def tracking_modes(model):
    """(template mode, reference mode) of a model's config; motion models ignore both settings, as the reference's
    MotionBaseModel.build_input_dict does: (None, 'previous_result')."""
    if is_motion(model):
        return None, "previous_result"
    return template_mode(model.config), reference_mode(model.config)


class DeviceTracker:
    """`reset(points, box)` on a tracklet's first frame, then `step(points, n_valid, ref_box)` per frame.  `seed` keys the
    random draws; `history`: starting capacity (points) of the 'all' template history.  Motion models (M2-Track) ignore
    shape_aggregation and reference_BB, as the reference's MotionBaseModel does.  `precision`: "fp32" (3xTF32 GEMMs, default) or
    "bf16" (BF16 operands, FP32 accumulation: runtime.inference_precision_scope) for the network's tensor-core layers."""

    def __init__(self, model, max_points, use_graph=True, seed=1, history=HISTORY_POINTS, precision="fp32"):
        from .. import runtime
        self.precision = runtime.check_precision(precision)
        self.model = model.eval()
        self.cfg = model.config
        self.dev = next(model.parameters()).device
        self.max_points = int(max_points)
        self.use_graph = bool(use_graph) and self.dev.type == "cuda"
        self.seed = int(seed)
        self.gen = torch.Generator(device=self.dev).manual_seed(seed)
        self.needs_bc = hasattr(model, "mlp_bc")            # BAT consumes the template BoxCloud
        self.motion = is_motion(model)                      # M2-Track style two-frame input
        self.mode, self.ref_mode = tracking_modes(model)
        f = dict(device=self.dev, dtype=torch.float32)
        n = self.max_points
        # static buffers (graph inputs / state)
        self.scan = torch.zeros(n, 3, **f)
        self.scan_valid = torch.zeros(n, dtype=torch.bool, device=self.dev)
        self.first_local = torch.zeros(n, 3, **f)           # first-frame object crop, canonical frame
        self.first_keep = torch.zeros(n, dtype=torch.bool, device=self.dev)
        self.prev_scan = torch.zeros(n, 3, **f)
        self.prev_valid = torch.zeros(n, dtype=torch.bool, device=self.dev)
        self.box_c = torch.zeros(3, **f)
        self.box_s = torch.ones(3, **f)
        self.box_r = torch.eye(3, **f)
        # uniform draws of the two resamplings: refreshed per frame OUTSIDE the captured graph (seeded, reproducible)
        size_s = self.cfg.point_sample_size if self.motion else self.cfg.search_size
        size_t = self.cfg.point_sample_size if self.motion else self.cfg.template_size
        self.u_s = (torch.zeros(n, **f), torch.zeros(size_s, **f))
        self.u_t = (torch.zeros(2 * n, **f), torch.zeros(size_t, **f))
        self.first_flag = torch.ones((), **f)               # 1 on the first tracked frame (prior box = ground truth), then 0
        # reference box of the search area and of the box update in the ground-truth modes (step's ref_box)
        self.ref_c, self.ref_s, self.ref_r = torch.zeros(3, **f), torch.ones(3, **f), torch.eye(3, **f)
        if self.mode == "all":
            # history of the 'all' template: the crops of frames 0 .. t-1, each in its result box, in frame and scan order
            i64 = dict(device=self.dev, dtype=torch.int64)
            self.scan_count, self.prev_count = torch.zeros(1, **i64), torch.zeros(1, **i64)
            self.slot0 = torch.zeros(1, **i64)              # the one slot's scan index and tracklet id
            self.frame_id = torch.zeros(1, **i64)
            self.hist_count = torch.zeros(1, **i64)
            self.hist_bound = 0                             # host upper bound of hist_count
            self.prev_n = 0                                 # valid points of the previous scan: what the next append can add
            self._alloc_history(int(history))
        self.graph = None
        self.frames = 0

    def _alloc_history(self, H, keep_count=0):
        """(Re)allocate the history for H points, keeping its first `keep_count` entries; the captured graph is dropped."""
        f = dict(device=self.dev, dtype=torch.float32)
        hist, keep = torch.zeros(1, H, 3, **f), torch.zeros(1, H, dtype=torch.bool, device=self.dev)
        if keep_count:
            hist[:, :keep_count].copy_(self.hist[:, :keep_count])
            keep[:, :keep_count].copy_(self.hist_keep[:, :keep_count])
        self.hist, self.hist_keep, self.H = hist, keep, H
        self.u_t = (torch.zeros(H, **f), self.u_t[1])      # the template draw is over the history
        self.graph = None

    # ------------------------------------------------------------------ state helpers
    def _box(self):
        return bx.Box(self.box_c, self.box_s, self.box_r)

    def _ref_box(self):
        """The box the search area is cropped in and the offset is applied to (generate_search_area's ref_bb)."""
        return self._box() if self.ref_mode == "previous_result" else bx.Box(self.ref_c, self.ref_s, self.ref_r)

    def _set_ref(self, ref_box):
        if self.ref_mode == "previous_result":
            return
        if ref_box is None:
            raise ValueError(f"reference_BB '{self.ref_mode}' needs the ground-truth reference box: step(..., ref_box=...)")
        rb = ref_box.to(self.dev)
        self.ref_c.copy_(rb.center); self.ref_s.copy_(rb.wlh); self.ref_r.copy_(rb.rot)

    def _load_scan(self, points, n_valid=None):
        n = points.shape[0]
        if n > self.max_points:
            raise ValueError(f"scan has {n} points, tracker was built for {self.max_points}")
        self.scan.zero_()
        self.scan[:n].copy_(points)
        n_valid = n if n_valid is None else int(n_valid)
        self.scan_valid.zero_()
        self.scan_valid[:n_valid] = True
        if self.mode == "all":
            self.scan_count.fill_(n_valid)
        return n_valid

    def reset(self, points, box: bx.Box):
        """First frame: remember the object crop (cropAndCenterPC of the first box) and the box itself; in 'all' mode empty
        the history (the first step appends this frame's crop)."""
        n = self._load_scan(points)
        box = box.to(self.dev)
        self.box_c.copy_(box.center); self.box_s.copy_(box.wlh); self.box_r.copy_(box.rot)
        if self.mode == "all":
            self.hist_count.zero_()
            self.hist_keep.zero_()
            self.prev_count.copy_(self.scan_count)
            self.hist_bound, self.prev_n = 0, n
        elif not self.motion:
            local, keep, _ = bx.crop_and_center(self.scan, box, offset=self.cfg.model_bb_offset, scale=self.cfg.model_bb_scale)
            self.first_local.copy_(local)
            self.first_keep.copy_(keep & self.scan_valid)
        self.first_flag.fill_(1.0)
        self.prev_scan.copy_(self.scan)
        self.prev_valid.copy_(self.scan_valid)
        self.frames = 1
        return self._box()

    # ------------------------------------------------------------------ one frame, fixed shapes
    def _inputs_motion(self):
        """MotionBaseModel.build_input_dict (models/base_model.py:255-303) on static buffers."""
        cfg, box = self.cfg, self._box()
        b1 = bx.Box(box.center[None], box.wlh[None], box.rot[None])
        n = cfg.point_sample_size
        p_local, p_keep = bx.crop_in_box_frame(self.prev_scan[None], b1, cfg.bb_scale, cfg.bb_offset)
        t_local, t_keep = bx.crop_in_box_frame(self.scan[None], b1, cfg.bb_scale, cfg.bb_offset)
        prev_pts, _ = resample(p_local[0], p_keep[0] & self.prev_valid, n, u_perm=self.u_t[0][: self.max_points], u_pick=self.u_t[1])
        this_pts, _ = resample(t_local[0], t_keep[0] & self.scan_valid, n, u_perm=self.u_s[0], u_pick=self.u_s[1])
        half = torch.stack([box.wlh[1], box.wlh[0], box.wlh[2]]) * (1.25 / 2)
        inside = (prev_pts.abs() <= half).all(-1).float()
        f = self.first_flag
        mask_prev = inside * (0.6 + 0.4 * f) + 0.2 * (1 - f)               # 1 / 0 on the first frame, 0.8 / 0.2 afterwards
        col = lambda pts, t, m: torch.cat([pts, torch.full_like(pts[:, :1], t), m[:, None]], -1)
        data = {"points": torch.cat([col(prev_pts, 0.0, mask_prev), col(this_pts, 0.1, torch.full_like(mask_prev, 0.5))], 0)[None]}
        if getattr(cfg, "box_aware", False):
            canon = bx.Box(torch.zeros_like(box.center), box.wlh, torch.eye(3, device=self.dev))
            bc = bx.point_to_box_distance(prev_pts, canon)
            data["candidate_bc"] = torch.cat([bc, torch.zeros_like(bc)], 0)[None]
        return data

    def _inputs(self):
        if self.motion:
            return self._inputs_motion()
        cfg, box, ref = self.cfg, self._box(), self._ref_box()
        b1 = bx.Box(box.center[None], box.wlh[None], box.rot[None])
        r1 = bx.Box(ref.center[None], ref.wlh[None], ref.rot[None])

        def build_template():
            # template: first-frame crop (+ previous-frame crop around the previous result), or every past frame's crop
            mode = self.mode
            if mode == "all":
                bx.crop_append(self.prev_scan[None], b1, cfg.model_bb_scale, cfg.model_bb_offset, self.slot0, self.prev_count,
                               self.hist, self.hist_keep, self.hist_count)
                cand, keep = self.hist[0], self.hist_keep[0]
            elif mode == "first":
                cand, keep = self.first_local, self.first_keep
            else:
                p_local, p_keep = bx.crop_in_box_frame(self.prev_scan[None], b1, cfg.model_bb_scale, cfg.model_bb_offset)
                p_local, p_keep = p_local[0], p_keep[0] & self.prev_valid
                if mode == "firstandprevious":
                    cand, keep = torch.cat([self.first_local, p_local]), torch.cat([self.first_keep, p_keep])
                else:
                    cand, keep = p_local, p_keep
            template, _ = resample(cand, keep, cfg.template_size, u_perm=self.u_t[0][: cand.shape[0]], u_pick=self.u_t[1])
            bc = None
            if self.needs_bc:
                canon = bx.Box(torch.zeros_like(box.center), box.wlh, torch.eye(3, device=self.dev))
                bc = bx.point_to_box_distance(template, canon)[None]
            return template[None], bc

        from .. import fused
        # the two crops + draws are independent: the template's run on the side stream (a parallel branch of the frame's graph)
        overlap = fused.branch_overlap(self.scan)
        join = fused.run_ahead(build_template) if overlap else None
        # search area: current scan in the frame of the reference box (previous result, or the caller's ground truth)
        s_local, s_keep = bx.crop_in_box_frame(self.scan[None], r1, cfg.search_bb_scale, cfg.search_bb_offset)
        s_local, s_keep = s_local[0], s_keep[0]
        search, _ = resample(s_local, s_keep & self.scan_valid, cfg.search_size, u_perm=self.u_s[0], u_pick=self.u_s[1])
        template, bc = join() if overlap else build_template()
        data = {"template_points": template, "search_points": search[None]}
        if bc is not None:
            data["points2cc_dist_t"] = bc
        return data

    def _frame(self):
        cfg = self.cfg
        from .. import runtime
        # the tracker never changes the weights: eval-mode stacks pack them / fold their BatchNorm once, not per frame
        with torch.no_grad(), runtime.static_weights_scope(), runtime.inference_precision_scope(self.precision):
            out = self.model(self._inputs())
            est = out["estimation_boxes"][0]                                   # (num_proposal, 5) or (4,)
            if est.dim() == 2:
                est = est.index_select(0, est[:, 4].argmax().reshape(1))[0, :4]    # (indexing by a 0-d tensor would sync)
            new = bx.offset_box(self._ref_box(), est, degrees=cfg.degrees, use_z=cfg.use_z, limit_box=cfg.limit_box)
            self.box_c.copy_(new.center); self.box_r.copy_(new.rot)
            if self.ref_mode != "previous_result":
                self.box_s.copy_(new.wlh)                                       # the result takes the reference box's size
            self.prev_scan.copy_(self.scan); self.prev_valid.copy_(self.scan_valid)
            if self.mode == "all":
                self.prev_count.copy_(self.scan_count)
            self.first_flag.zero_()

    def _reserve_history(self):
        """Make room for this step's append, which adds at most the previous scan's valid points.  The host bound on the count
        is exact only after a read-back, so the count is read (one synchronisation) only when the bound could pass H, and
        the history grows (copied, graph captured again) only when the exact count could."""
        need = self.hist_bound + self.prev_n
        if need > self.H:
            self.hist_bound = int(self.hist_count[0])
            need = self.hist_bound + self.prev_n
            if need > self.H:
                self._alloc_history(max(need, 2 * self.H), keep_count=min(self.hist_bound, self.H))
        self.hist_bound = need

    def _draw(self):
        """Per-frame uniform draws, outside the graph.  The 'all' history's permutation draw is keyed by (seed, tracklet 0,
        frame) on the device, so it does not depend on the history's capacity; the others come from the tracker's generator."""
        if self.mode != "all":
            for u in self.u_s + self.u_t:
                u.uniform_(generator=self.gen)
            return
        for u in self.u_s + self.u_t[1:]:
            u.uniform_(generator=self.gen)
        if self.dev.type == "cuda":
            from .. import ops
            from .batched_tracker import STREAM_TEMPLATE_PERM
            self.frame_id.fill_(self.frames)
            ops.keyed_uniform(self.slot0, self.frame_id, self.seed, STREAM_TEMPLATE_PERM, self.H, out=self.u_t[0].view(1, -1))
        else:
            self.u_t[0].uniform_(generator=self.gen)

    def step(self, points, n_valid=None, ref_box=None):
        """Next frame: `points` (n, 3) device tensor, the first `n_valid` valid.  `ref_box`: this frame's reference box,
        required in the reference_BB modes 'previous_gt' (the previous frame's ground truth) and 'current_gt' (this frame's).
        Returns the tracked box (views of the tracker's state buffers)."""
        if self.frames == 0:
            raise RuntimeError("call reset() with the first frame and its box before step()")
        self._set_ref(ref_box)
        if self.mode == "all":
            self._reserve_history()
        n = self._load_scan(points, n_valid)
        self._draw()
        if not self.use_graph:
            self._frame()
        elif self.graph is None:
            state = (self.box_c, self.box_s, self.box_r, self.prev_scan, self.prev_valid, self.first_flag)
            if self.mode == "all":
                state += (self.hist_keep, self.hist_count, self.prev_count)
            snap = [t.clone() for t in state]
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                self._frame()                                                   # warm-up (allocations, autotuning)
            torch.cuda.current_stream().wait_stream(s)
            for t, v in zip(state, snap):
                t.copy_(v)
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph):
                self._frame()
            for t, v in zip(state, snap):
                t.copy_(v)
            self.graph.replay()
        else:
            self.graph.replay()
        self.frames += 1
        if self.mode == "all":
            self.prev_n = n
        return self._box()
