"""Live tracking of many targets through one scan stream: K slots advanced together by one captured step per scan.

`DeviceTracker` follows one target and `BatchedDeviceTracker` replays pre-loaded tracklets with ground truth for every frame;
this tracker takes the scans as they arrive and targets as they appear and disappear:
  * `step(points)` copies the scan into a static (2, N, 3) ping-pong buffer (the one copy of the scan) and replays a captured
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
Occupancy buckets.  A step runs over the targets it advances only: the host forms the work list (the active slots whose feed got
a scan, in slot order) and runs the step at the smallest bucket that holds it, out of the powers of two below `max_targets` and
`max_targets` itself.  Each bucket has its own captured graph, all captured on the first advance and sharing one memory pool; the
graph gathers its rows' state (box, key, frame, first-frame flag and prefix, feed) through the work list, uploaded without a
sync, and scatters the box, frame counter and first-frame flag back into their slots; padding rows read an idle row and write
nowhere that is read.  Slots never move, so `boxes()` / `snapshot()` keep the slot layout.  Rows of a step are independent, and
the smallest bucket is one at which every MLP stack keeps the kernel plan it has over all slots (o3d_stack_plan_thresholds), so a
target's boxes are bitwise the same at every bucket.  A step therefore costs what its bucket costs, not what `max_targets` does;
an advance with no target to advance runs the ingest alone.

Feeds.  A feed is one sequence of scans: one sensor, or one recorded scene.  With `feeds=F` the scan buffer is (F, 2, N, 3), every
slot follows one feed, and each feed has its own ping-pong parity.  `put(feed, points)` (xyz) or `put_raw(feed, rows, transforms)`
(a scan's point rows as stored, with the reader's affine transforms) stages the next scan of a feed; `advance()` brings every
staged scan in (host scans: one packed host->device copy and one `o3d_scan_ingest` launch for all feeds, csrc/scan_ingest.cu) and
replays the one captured step.  A feed that got no scan since the last `advance()` holds still: its slots keep their box, frame
counter, first-frame flag and parity.  Since draws are keyed by target id and frame within the track, a target's boxes depend
neither on its feed, nor on the other feeds, nor on F.  `step(points)` is `put(0, points)` + `advance()` for one feed.
Evidence and lost targets.  After the box update, every advanced row also records the number of points of the scan it advanced
on inside its new box scaled by 1.25 (`o3d_box_points`, csrc/box_points.cu) and the model's score (BAT / P2B: the best
proposal's column 4; M2-Track: the share of the current frame's sampled points segmented as target).  With
`lost=(min_points, patience)` the step also counts consecutive advances below `min_points` and declares the target lost at
`patience` of them; a lost target is held from then on (its box, frame counter, first-frame flag and evidence stay those of
that advance) until the host drops it (`lost_targets()` / `drop_lost()`).  All of it runs inside the captured step, per row, so
it neither synchronises nor depends on the bucket, K or the other targets.
Device memory: feeds * 2 * max_points * 12 bytes of scans, plus per slot the crop scratch and, for the first-frame template
modes, max_points * 13 bytes of first-frame crop.  Ground-truth reference boxes (reference_BB 'previous_gt' / 'current_gt') have no meaning on a live stream, and
shape_aggregation 'all' is not supported here; both are refused."""
import weakref

import numpy as np
import torch

from .. import ops, runtime
from . import boxes as bx
from .batched_tracker import (STREAM_LIMIT_BOX, STREAM_SEARCH_PERM, STREAM_SEARCH_PICK, STREAM_TEMPLATE_PERM, STREAM_TEMPLATE_PICK,
                              best_proposal, best_proposal_score, canonical, motion_data)
from .device_tracker import is_motion, tracking_modes


def _half(box, scale, offset):
    """crop_in_box_frame's half extents (l, w, h on x, y, z), the same expression so that the crop test is the same."""
    return torch.stack([box.wlh[..., 1], box.wlh[..., 0], box.wlh[..., 2]], -1) * (scale / 2) + offset


# nuscenes points_in_box's wlh_factor for the evidence's in-box count: the factor the reference's M2-Track segmentation labels use
EVIDENCE_WLH_FACTOR = 1.25


def check_lost_rule(lost):
    """`lost=`: None (no target is ever declared lost) or (min_points, patience), ints with min_points >= 0, patience >= 1."""
    if lost is None:
        return None
    try:
        min_points, patience = lost
    except (TypeError, ValueError):
        raise ValueError(f"lost={lost!r}: expected None or (min_points, patience)") from None
    if isinstance(min_points, bool) or isinstance(patience, bool) or int(min_points) != min_points or int(patience) != patience:
        raise ValueError(f"lost={lost!r}: min_points and patience are integers")
    if min_points < 0:
        raise ValueError(f"lost: min_points={min_points} must be >= 0")
    if patience < 1:
        raise ValueError(f"lost: patience={patience} must be >= 1")
    return int(min_points), int(patience)


def _box_values(box):
    """(center, wlh, 3x3 rotation) as float64 numpy arrays from a data_classes.Box or a tracking.boxes.Box."""
    if isinstance(box, bx.Box):
        return tuple(np.asarray(t.detach().cpu(), dtype=np.float64) for t in box)
    return np.asarray(box.center, np.float64), np.asarray(box.wlh, np.float64), np.asarray(box.rotation_matrix, np.float64)


class ScanFeeds:
    """The scan feeds of one or more live trackers: `feeds` ping-pong buffers (F, 2, max_points, 3) with their point counts, the
    per-feed parity (host mirrors and the device copy the captured steps read) and the scans staged for the next advance.
    `put` / `put_raw` stage a feed's next scan; `ingest()` brings every staged scan in with one packed host->device copy and one
    `o3d_scan_ingest` launch and flips the parity of the feeds that got one.  Trackers built over the same store
    (`MultiTargetTracker(..., feeds=store)`) read the same scans: one copy and one ingest serve them all.  Since an ingest moves
    every feed's parity for all of them, only the store's `owner` advances: the first tracker built over it, or the
    MultiClassTracker that holds the trackers sharing it."""

    def __init__(self, max_points, feeds=1, device="cuda"):
        self.N = N = int(max_points)
        self.F = F = int(feeds)
        dev = torch.device(device)
        if dev.type == "cuda" and dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        self.dev = dev
        if N < 1 or F < 1:
            raise ValueError(f"max_points={N} and feeds={F} must be >= 1")
        i64 = dict(device=dev, dtype=torch.int64)
        self.scans = torch.zeros(F, 2, N, 3, device=dev, dtype=torch.float32)
        self.count = torch.zeros(F, 2, **i64)
        # per feed: fed by this advance (0 / 1), the half holding its most recent scan, the half holding the scan before it;
        # written from the host mirrors below before every step
        self.fstate = torch.tensor([[0] * F, [1] * F, [0] * F], **i64)
        self.fcur, self.fprev = [1] * F, [0] * F
        self.feed_seen = [0] * F                          # scans advanced per feed
        self.scans_seen = 0                               # scans advanced over all feeds
        self.staged = {}                                  # feed -> None (already in its buffer) or (rows, transforms)
        self._owner = None                                # weak reference to the one tracker whose advance() ingests

    @property
    def owner(self):
        return None if self._owner is None else self._owner()

    @owner.setter
    def owner(self, tracker):
        self._owner = None if tracker is None else weakref.ref(tracker)

    def claim(self, tracker):
        """Make `tracker` the store's owner, the one whose advance() ingests; a store has one owner."""
        if self.owner is not None and self.owner is not tracker:
            raise ValueError("these scan feeds already belong to another tracker, which advances them; build the trackers that "
                             "share them through a MultiClassTracker")
        self.owner = tracker

    def feed(self, feed):
        f = int(feed)
        if not 0 <= f < self.F:
            raise ValueError(f"feed {f} out of range: the tracker has feeds 0 .. {self.F - 1}")
        return f

    def _stage(self, feed, n):
        f = self.feed(feed)
        if f in self.staged:
            raise ValueError(f"feed {f} already has a scan staged: advance() before the next put")
        if n > self.N:
            raise ValueError(f"max_points: the scan has {n} points, the tracker was built for {self.N}")
        return f

    def put(self, feed, points, n_valid=None):
        """Stage the next scan of `feed`: `points` (n, 3), the first `n_valid` valid.  A CUDA tensor is copied into the feed's next
        buffer at once; a host tensor or array goes through the packed copy and the ingest kernel of the next `ingest()`.  No
        host sync."""
        n = points.shape[0]
        f = self._stage(feed, n)
        n_valid = n if n_valid is None else min(int(n_valid), n)
        if isinstance(points, torch.Tensor) and (points.device == self.dev or self.dev.type != "cuda"):
            nxt = 1 - self.fcur[f]
            self.scans[f, nxt, :n].copy_(points, non_blocking=True)
            self.count[f, nxt].fill_(n_valid)
            self.staged[f] = None
        else:
            rows = points.numpy() if isinstance(points, torch.Tensor) else np.asarray(points)
            self.staged[f] = (rows[:n_valid], ())

    def put_raw(self, feed, rows, transforms=()):
        """Stage the next scan of `feed` as a reader stores it: `rows` (n, stride) float32 / float64 (x, y, z first, 3 <= stride
        <= 16) and up to two affine transforms (3x4 or 4x4, applied in order in float64, as the readers apply them on the host).
        The next `ingest()` moves every staged raw scan to the device in one copy and one `o3d_scan_ingest` launch."""
        rows = np.asarray(rows)
        if self.dev.type != "cuda":
            raise RuntimeError("put_raw: scan ingest runs on the GPU; this tracker is not on a CUDA device")
        if rows.ndim != 2 or not 3 <= rows.shape[1] <= 16:
            raise ValueError(f"put_raw: rows of shape {rows.shape}; expected (points, 3 .. 16 values per row)")
        transforms = [np.asarray(m, np.float64) for m in transforms]
        if len(transforms) > 2 or any(m.shape not in ((3, 4), (4, 4)) for m in transforms):
            raise ValueError("put_raw: at most two transforms, each 3x4 or 4x4")
        f = self._stage(feed, rows.shape[0])
        self.staged[f] = (rows, transforms)

    def ingest(self):
        """Bring in every staged scan, on the current stream: the feeds that got one flip their parity and are marked fed in
        `fstate`, the others hold.  No host sync."""
        F, staged = self.F, self.staged
        raw = [(f, 1 - self.fcur[f], v[0], v[1]) for f, v in sorted(staged.items()) if v is not None]
        for f in staged:
            self.fprev[f], self.fcur[f] = self.fcur[f], 1 - self.fcur[f]
            self.feed_seen[f] += 1
        state = np.array([[int(f in staged) for f in range(F)], self.fcur, self.fprev], dtype=np.int64)
        if self.dev.type == "cuda":
            # one host->device copy per step: the feeds' state, the ingest descriptors and every raw scan's rows
            buf, desc, d0, s0 = ops.pack_scans(raw, head=state.nbytes)
            buf.numpy()[:state.nbytes] = state.reshape(-1).view(np.uint8)
            dev = buf.to(self.dev, non_blocking=True)
            self.fstate.copy_(dev[:state.nbytes].view(torch.int64).view(3, F))
            if raw:
                ops.scan_ingest(self.scans, self.count, desc, dev, d0, s0)
        else:
            self.fstate.copy_(torch.from_numpy(state))
        self.scans_seen += len(staged)
        staged.clear()


def capture_step(step, state, pool=None):
    """Capture `step()` in a CUDA graph (in the memory pool `pool`, or a private one).  The warm-up runs a real step
    (allocations, weight packing) on a side stream; `state`, the tensors a step advances, is put back after it and after the
    capture, so the graph's first replay is the first step."""
    snap = [t.clone() for t in state]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    for t, v in zip(state, snap):
        t.copy_(v)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, pool=pool):
        step()
    for t, v in zip(state, snap):
        t.copy_(v)
    return graph


# ------------------------------------------------------------------ occupancy buckets
def occupancy_buckets(K, smallest=1):
    """The row counts a K-slot tracker's step runs at: the powers of two from `smallest` up to below K, then K itself."""
    out, b = [], 1
    while b < K:
        if b >= smallest:
            out.append(b)
        b *= 2
    return tuple(out) + (K,)


def smallest_bucket(K, rows):
    """The fewest step rows at which every MLP stack of a K-row step keeps its kernel plan.  `rows`: (P, T) pairs from
    runtime.stack_rows_scope() over that step, a stack's row count P (proportional to the step's rows) with each row count T at
    which its plan changes (o3d_stack_plan_thresholds).  A stack below T at K is below it at every smaller size; one at or
    above it must stay there, which takes ceil(T * K / P) rows."""
    return max([-(-t * K // p) for p, t in rows if p >= t], default=1)


def bucket_for(n, buckets):
    """The smallest bucket that holds n rows."""
    return next(b for b in buckets if b >= n)


def work_slots(slot_feed, fed):
    """The work list of one advance: the slots of `slot_feed` ({slot: feed} of the active targets) whose feed is in `fed`, in
    slot order."""
    return sorted(k for k, f in slot_feed.items() if f in fed)


def work_rows(slots, K):
    """(2, K) int64: the rows a bucket step gathers its state from (the work list, then K, the idle row) and the rows it
    scatters its results to (the work list, then K + 1, a row nothing reads)."""
    n = len(slots)
    return np.array([list(slots) + [K] * (K - n), list(slots) + [K + 1] * (K - n)], dtype=np.int64)


class MultiTargetTracker:
    """`max_targets` slots over `feeds` scan feeds of at most `max_points` points per scan.  `seed` keys the random draws;
    `use_graph`: capture the step of every occupancy bucket in a CUDA graph on the first advance (eager otherwise).  With one feed, call `step(scan)` for
    every scan of the stream; with several, `put` / `put_raw` the feeds' next scans and `advance()`.  `add(id, box, feed=)` starts
    a target on its feed's most recent scan, `drop(id)` ends it.  `feeds` is a number of feeds, or a `ScanFeeds` store the
    tracker shares with others (MultiClassTracker): only the store's owner advances (its ingest serves every tracker on the
    store), and `_run()` advances this one tracker's slots.  `lost`: None (no target is ever declared lost) or
    (min_points, patience), the end-of-track rule the step applies on the device; `boxes()` / `evidence()` report every slot's
    evidence either way."""

    def __init__(self, model, max_points, max_targets, seed=0, use_graph=True, feeds=1, precision="fp32", lost=None):
        self.precision = runtime.check_precision(precision)
        self.lost_rule = check_lost_rule(lost)
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
        shared = isinstance(feeds, ScanFeeds)
        self.F = F = feeds.F if shared else int(feeds)
        if N < 1 or K < 1 or K > 65535 or F < 1:
            raise ValueError(f"max_points={N}, max_targets={K} and feeds={F} must be >= 1 (max_targets <= 65535)")
        if shared:
            if feeds.dev != dev or feeds.N != N:
                raise ValueError(f"the scan feeds hold {feeds.N} points per scan on {feeds.dev}; the tracker was asked for "
                                 f"max_points={N} on {dev}")
            self.scan_feeds = feeds
        else:
            self.scan_feeds = ScanFeeds(N, F, dev)
        if self.scan_feeds.owner is None:
            self.scan_feeds.claim(self)
        f = dict(device=dev, dtype=torch.float32)
        i64 = dict(device=dev, dtype=torch.int64)
        self.arange = torch.arange(N, device=dev)
        # Slot state, K + 2 rows: the K slots (the public attributes are views of them), row K the idle state the padding rows of
        # a bucket step read, row K + 1 where they write.  Idle slots and row K hold the dummy box.
        self._slot_feed = torch.zeros(K + 2, **i64)
        self._box_c = torch.zeros(K + 2, 3, **f)
        self._box_s = torch.ones(K + 2, 3, **f)
        self._box_r = torch.eye(3, **f).repeat(K + 2, 1, 1)
        self._first_flag = torch.zeros(K + 2, **f)
        self._active = torch.zeros(K + 2, dtype=torch.bool, device=dev)
        self._key = torch.zeros(K + 2, **i64)             # target id of the slot (the key of its draws)
        self._t = torch.zeros(K + 2, **i64)               # frame within the target's track
        # Evidence of the last advance: points of its scan in the box scaled by EVIDENCE_WLH_FACTOR (-1 before the first), the
        # model's score (NaN before the first), consecutive advances below the rule's min_points, and whether the rule fired
        self._points = torch.full((K + 2,), -1, device=dev, dtype=torch.int32)
        self._score = torch.full((K + 2,), float("nan"), **f)
        self._misses = torch.zeros(K + 2, device=dev, dtype=torch.int32)
        self._lost = torch.zeros(K + 2, dtype=torch.bool, device=dev)
        self.slot_feed, self.box_c, self.box_s, self.box_r = (x[:K] for x in (self._slot_feed, self._box_c, self._box_s, self._box_r))
        self.first_flag, self.active, self.key, self.t = (x[:K] for x in (self._first_flag, self._active, self._key, self._t))
        self.points, self.score, self.misses, self.lost = (x[:K] for x in (self._points, self._score, self._misses, self._lost))
        if self.mode in ("firstandprevious", "first"):
            self._first_local = torch.zeros(K + 2, N, 3, **f)
            self._first_keep = torch.zeros(K + 2, N, dtype=torch.bool, device=dev)
            self.first_local, self.first_keep = self._first_local[:K], self._first_keep[:K]
        self.slot_of = {}                                 # target id -> slot
        self._feed_of = {}                                # slot -> feed of the active targets (host mirror of slot_feed)
        # The work list of the next bucket step, (2, K) as work_rows() lays it out; one host->device copy per advance.
        self._work = torch.zeros(2, K, **i64)
        self._buckets = None                              # the step sizes (occupancy_buckets), fixed on the first advance
        self.graphs = {}                                  # bucket -> captured step

    # the feed state lives in the (possibly shared) ScanFeeds store
    scans = property(lambda self: self.scan_feeds.scans)
    count = property(lambda self: self.scan_feeds.count)
    fstate = property(lambda self: self.scan_feeds.fstate)
    feed_seen = property(lambda self: self.scan_feeds.feed_seen)
    _fcur = property(lambda self: self.scan_feeds.fcur)
    _fprev = property(lambda self: self.scan_feeds.fprev)
    _staged = property(lambda self: self.scan_feeds.staged)

    @property
    def scans_seen(self):
        return self.scan_feeds.scans_seen

    @scans_seen.setter
    def scans_seen(self, n):
        self.scan_feeds.scans_seen = n

    # ------------------------------------------------------------------ one step over a bucket of rows, fixed shapes
    def _crop(self, r, which, box, half, perm, pick, size, prefix=False):
        scans = self.scans.view(2 * self.F, self.N, 3)
        scans = scans if which is not None else scans[:, :0]
        frame = which if which is not None else r["cur"]
        pre = r["first"] if prefix else (None, None)
        out, _ = ops.crop_resample(scans, self.count.view(2 * self.F), frame, box.center, box.rot, half, size, self.seed, r["key"],
                                   r["t"], perm, pick, *pre)
        return out

    def _inputs(self, r, box):
        cfg = self.cfg
        if self.motion:
            h = _half(box, cfg.bb_scale, cfg.bb_offset)
            n = cfg.point_sample_size
            prev_pts = self._crop(r, r["prev"], box, h, STREAM_TEMPLATE_PERM, STREAM_TEMPLATE_PICK, n)
            this_pts = self._crop(r, r["cur"], box, h, STREAM_SEARCH_PERM, STREAM_SEARCH_PICK, n)
            return motion_data(cfg, box, prev_pts, this_pts, r["first_flag"])
        search = self._crop(r, r["cur"], box, _half(box, cfg.search_bb_scale, cfg.search_bb_offset), STREAM_SEARCH_PERM,
                            STREAM_SEARCH_PICK, cfg.search_size)
        h = _half(box, cfg.model_bb_scale, cfg.model_bb_offset)
        if self.mode == "first":                          # the first-frame crop alone: no scan in the candidate set
            template = self._crop(r, None, box, h, STREAM_TEMPLATE_PERM, STREAM_TEMPLATE_PICK, cfg.template_size, prefix=True)
        else:
            template = self._crop(r, r["prev"], box, h, STREAM_TEMPLATE_PERM, STREAM_TEMPLATE_PICK, cfg.template_size,
                                  prefix=self.mode == "firstandprevious")
        data = {"template_points": template, "search_points": search}
        if self.needs_bc:
            data["points2cc_dist_t"] = bx.point_to_box_distance(template, canonical(box))
        return data

    def _step(self, b):
        """Advance the first `b` rows of the work list `_work`: gather their slots' state, run the network on b rows and scatter
        the box, frame counter and first-frame flag back.  Padding rows read the idle row K, which is never active, and write
        row K + 1.  Every intermediate is dropped when the step ends; the results live in the slot state, allocated outside any
        capture, which is what lets the bucket graphs share one memory pool."""
        cfg = self.cfg
        with torch.no_grad(), runtime.static_weights_scope(), runtime.inference_precision_scope(self.precision):
            r, box, dst = self._gather(b)
            u_lim = ops.keyed_uniform(r["key"], r["t"], self.seed, STREAM_LIMIT_BOX, 2)
            out = self.model(self._inputs(r, box))
            if self.motion:
                est = best_proposal(out["estimation_boxes"])
                # the share of the current frame's sampled points segmented as target (argmax: ties go to background)
                seg = out["seg_logits"][:, :, cfg.point_sample_size:]
                score = (seg[:, 1] > seg[:, 0]).sum(1).float() / cfg.point_sample_size
            else:
                est, score = best_proposal_score(out["estimation_boxes"])
            new = bx.offset_box(box, est, degrees=cfg.degrees, use_z=cfg.use_z, limit_box=cfg.limit_box, rand=u_lim * 2 - 1)
            scans = self.scans.view(2 * self.F, self.N, 3)
            points = ops.box_points(scans, self.count.view(2 * self.F), r["cur"], new.center, new.rot,
                                    bx.inclusive_half(new.wlh, EVIDENCE_WLH_FACTOR))
            self._scatter(r, box, new, dst, points, score)

    def _gather(self, b):
        """The state of the first `b` rows of the work list: (rows {cur, prev, key, t, first_flag, adv[, first]}, box, the rows
        to scatter to)."""
        src, dst = self._work[0, :b], self._work[1, :b]
        fed, fcur, fprev = self.fstate
        feed = self._slot_feed.index_select(0, src)
        # a lost target holds from the advance it was declared lost on
        adv = self._active.index_select(0, src) & (fed[feed] != 0) & ~self._lost.index_select(0, src)
        r = {"cur": feed * 2 + fcur[feed], "prev": feed * 2 + fprev[feed], "key": self._key.index_select(0, src),
             "t": self._t.index_select(0, src) + adv.long(), "first_flag": self._first_flag.index_select(0, src), "adv": adv}
        if self.mode in ("firstandprevious", "first"):
            r["first"] = (self._first_local.index_select(0, src), self._first_keep.index_select(0, src))
        box = bx.Box(self._box_c.index_select(0, src), self._box_s.index_select(0, src), self._box_r.index_select(0, src))
        return r, box, dst

    def _scatter(self, r, box, new, dst, points, score):
        """Write the advanced rows' box, frame counter, first-frame flag and evidence back to their slots, and apply the end-of-track
        rule to them (rows that hold keep theirs)."""
        adv = r["adv"]
        a = adv[:, None]
        src = self._work[0, :adv.shape[0]]
        self._box_c.index_copy_(0, dst, torch.where(a, new.center, box.center))
        self._box_r.index_copy_(0, dst, torch.where(a[..., None], new.rot, box.rot))
        self._t.index_copy_(0, dst, r["t"])
        self._first_flag.index_copy_(0, dst, r["first_flag"].masked_fill(adv, 0.0))
        self._points.index_copy_(0, dst, torch.where(adv, points, self._points.index_select(0, src)))
        self._score.index_copy_(0, dst, torch.where(adv, score.float(), self._score.index_select(0, src)))
        if self.lost_rule is not None:
            min_points, patience = self.lost_rule
            misses = self._misses.index_select(0, src)
            misses = torch.where(adv, torch.where(points < min_points, misses + 1, torch.zeros_like(misses)), misses)
            self._misses.index_copy_(0, dst, misses)
            self._lost.index_copy_(0, dst, self._lost.index_select(0, src) | (misses >= patience))

    def _state(self):
        """The slot state a step writes (what the warm-up before a capture must put back)."""
        return (self._t, self._box_c, self._box_r, self._first_flag, self._points, self._score, self._misses, self._lost)

    def _plan(self):
        """First advance: the bucket sizes, from the row counts of the network's stacks in one step over all K slots (its
        writes are put back), then, with graphs, one captured step per bucket, largest first, all in one memory pool: only one
        of them replays at a time and none reads memory another wrote.  Eager, one step per bucket instead.  Either way only this
        advance synchronises."""
        K = self.K
        if self._buckets is None:
            snap = [t.clone() for t in self._state()]
            with runtime.stack_rows_scope() as rows:
                self._step(K)
            for t, v in zip(self._state(), snap):
                t.copy_(v)
            self._buckets = occupancy_buckets(K, smallest_bucket(K, rows))
        if self.use_graph:
            pool = torch.cuda.graph_pool_handle()
            for b in sorted(self._buckets, reverse=True):
                self.graphs[b] = capture_step(lambda b=b: self._step(b), self._state(), pool)
        else:
            # one step at every bucket size (its writes put back), so that the prepared weight blocks of every row count are
            # built, and synchronise, here rather than on the first advance that reaches that size
            snap = [t.clone() for t in self._state()]
            for b in self._buckets:
                self._step(b)
                for t, v in zip(self._state(), snap):
                    t.copy_(v)

    def _run(self, fed):
        """Advance the active targets of the feeds in `fed` to the scans the feed store has just brought in: upload the work list
        and replay the captured step of its bucket (or run the eager step at that size).  The first call fixes the buckets and
        captures every bucket's step, so that later calls never synchronise."""
        slots = work_slots(self._feed_of, fed)
        first = self._buckets is None or (self.use_graph and not self.graphs)
        if not slots and not first:
            return
        w = torch.from_numpy(work_rows(slots, self.K))
        # a fresh pinned buffer for every advance: it is not rewritten before its copy runs
        self._work.copy_(w.pin_memory() if self.dev.type == "cuda" else w, non_blocking=True)
        if first:
            self._plan()
        if not slots:
            return
        b = bucket_for(len(slots), self._buckets)
        if self.use_graph:
            self.graphs[b].replay()
        else:
            self._step(b)

    # ------------------------------------------------------------------ public interface
    def _feed(self, feed):
        return self.scan_feeds.feed(feed)

    def put(self, feed, points, n_valid=None):
        """Stage the next scan of `feed` (ScanFeeds.put): a CUDA tensor is copied into the feed's next buffer at once, a host
        tensor or array goes through the packed copy and the ingest kernel of the next `advance()`.  No host sync."""
        self.scan_feeds.put(feed, points, n_valid)

    def put_raw(self, feed, rows, transforms=()):
        """Stage the next scan of `feed` as a reader stores it (ScanFeeds.put_raw): the next `advance()` ingests it on the
        device."""
        self.scan_feeds.put_raw(feed, rows, transforms)

    def advance(self):
        """Bring in every staged scan and advance the active targets of those feeds to it, in one replay of the captured step;
        the other feeds hold.  Returns `boxes()`: device views of the slots' state, no host sync."""
        if self.scan_feeds.owner is not self:
            raise RuntimeError("advance(): this tracker shares scan feeds that another tracker owns; an ingest here would move "
                               "every sharing tracker's scans without advancing them, so advance the owner")
        fed = set(self.scan_feeds.staged)
        self.scan_feeds.ingest()
        self._run(fed)
        return self.boxes()

    def step(self, points, n_valid=None):
        """One-feed form: load the next scan (`points` (n, 3), the first `n_valid` valid; a CUDA tensor, or a host tensor moved
        without a sync) and advance every active target to it: `put(0, points)` + `advance()`."""
        if self.F != 1:
            raise ValueError(f"step() drives a one-feed tracker; with feeds={self.F} use put() / put_raw() and advance()")
        self.put(0, points, n_valid)
        return self.advance()

    def add(self, target_id, box, feed=0):
        """Start target `target_id` on the most recent scan of `feed` with `box` (a data_classes.Box or a tracking.boxes.Box): the
        box is its result on that scan, and the template's first-frame crop is taken from it.  No host sync."""
        tid = int(target_id)
        f = self._feed(feed)
        if tid in self.slot_of:
            raise ValueError(f"target_id {tid} is already active")
        if len(self.slot_of) >= self.K:
            raise ValueError(f"max_targets: all {self.K} slots are taken; drop a target first")
        if (self.scans_seen if self.F == 1 else self.feed_seen[f]) == 0:
            raise RuntimeError(f"add() starts a target on the most recent scan of its feed: call step() / advance() with a scan "
                               f"of feed {f} first")
        k = min(set(range(self.K)) - set(self.slot_of.values()))
        c, s, r = _box_values(box)
        vals = torch.tensor(np.concatenate([c, s, r.reshape(-1)]), dtype=torch.float32)
        if self.dev.type == "cuda":
            vals = vals.pin_memory().to(self.dev, non_blocking=True)                # no host sync
        self.box_c[k].copy_(vals[0:3])
        self.box_s[k].copy_(vals[3:6])
        self.box_r[k].copy_(vals[6:15].view(3, 3))
        if self.mode in ("firstandprevious", "first"):
            cfg, cur = self.cfg, self._fcur[f]
            b = bx.Box(self.box_c[k], self.box_s[k], self.box_r[k])
            local, keep, _ = bx.crop_and_center(self.scans[f, cur], b, offset=cfg.model_bb_offset, scale=cfg.model_bb_scale)
            self.first_local[k].copy_(local)
            self.first_keep[k].copy_(keep & (self.arange < self.count[f, cur]))
        self.slot_feed[k].fill_(f)
        # fill_ on a view, not `x[k] = value`: indexed assignment of a Python scalar copies it from the host and synchronises
        self.first_flag[k].fill_(1.0)
        self.active[k].fill_(True)
        self.key[k].fill_(tid)
        self.t[k].zero_()
        self._reset_evidence(k)
        self.slot_of[tid] = k
        self._feed_of[k] = f

    def drop(self, target_id):
        """End target `target_id` and free its slot (it returns to the dummy box).  No host sync."""
        tid = int(target_id)
        if tid not in self.slot_of:
            raise ValueError(f"target_id {tid} is not active")
        k = self.slot_of.pop(tid)
        del self._feed_of[k]
        self.active[k].fill_(False)
        self.box_c[k].zero_()
        self.box_s[k].fill_(1.0)
        self.box_r[k].copy_(torch.eye(3, device=self.dev))
        self.key[k].zero_()
        self.t[k].zero_()
        self.slot_feed[k].zero_()
        self._reset_evidence(k)
        if self.mode in ("firstandprevious", "first"):
            self.first_keep[k].zero_()

    def _reset_evidence(self, k):
        self.points[k].fill_(-1)
        self.score[k].fill_(float("nan"))
        self.misses[k].zero_()
        self.lost[k].fill_(False)

    def boxes(self):
        """Device state of the slots: ids (K,) int64 (-1 for an idle slot), center (K, 3), wlh (K, 3), rot (K, 3, 3), active (K,),
        and the evidence of each slot's last advance: points (K,) int32, score (K,) float32 (-1 / NaN before the first advance)
        and lost (K,) bool."""
        return {"ids": torch.where(self.active, self.key, torch.full_like(self.key, -1)), "center": self.box_c, "wlh": self.box_s,
                "rot": self.box_r, "active": self.active, "points": self.points, "score": self.score, "lost": self.lost}

    def evidence(self):
        """A device copy of the slots' evidence, (K, 4) float32 = points in the box, score, consecutive misses, lost (0 / 1)."""
        return torch.stack([self.points.float(), self.score, self.misses.float(), self.lost.float()], 1)

    def _record(self):
        """`snapshot()` and `evidence()` side by side, (K, 19), in one copy."""
        return torch.cat([self.box_c, self.box_s, self.box_r.reshape(self.K, 9), self.points.float()[:, None], self.score[:, None],
                          self.misses.float()[:, None], self.lost.float()[:, None]], 1)

    def lost_targets(self):
        """Ids of the active targets the end-of-track rule has declared lost, read back from the device (one sync)."""
        lost = self.lost.cpu().numpy()
        return sorted(tid for tid, k in self.slot_of.items() if lost[k])

    def drop_lost(self):
        """`drop` every target of `lost_targets()`; returns their ids."""
        ids = self.lost_targets()
        for tid in ids:
            self.drop(tid)
        return ids

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


def track_stream(model, scans, starts, ends, max_targets, seed=0, max_points=None, use_graph=True, precision="fp32"):
    """Track targets through a stream of scans.  `scans`: iterable of (n, 3) tensors; `starts`: {frame: [(id, Box), ...]} — each
    target starts on that scan with that box; `ends`: {id: last frame} (a target without an entry runs to the end of the
    stream).  `max_points`: the scan buffer's size (default: the largest scan, which needs the whole stream up front).
    Returns {id: {frame: data_classes.Box}}, from the frame a target starts on to its last frame; the device is read back once."""
    from ..datasets.data_classes import Box
    runtime.check_precision(precision)
    if max_points is None:
        scans = list(scans)
        max_points = max((s.shape[0] for s in scans), default=1)
    trk = MultiTargetTracker(model, max_points, max_targets, seed=seed, use_graph=use_graph, precision=precision)
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


def scene_peak(n_frames, starts, ends):
    """The largest number of a scene's targets active at once (a target is active from its start frame through its end frame,
    both included; without an end it runs to the scene's last frame)."""
    delta = [0] * (n_frames + 1)
    for t, group in starts.items():
        for tid, _ in group:
            delta[t] += 1
            delta[min(ends.get(tid, n_frames - 1), n_frames - 1) + 1] -= 1
    peak = live = 0
    for d in delta:
        live += d
        peak = max(peak, live)
    return peak


def class_peaks(n_frames, starts, ends):
    """`scene_peak` per class, for targets keyed (class, id): {class: the most targets of that class active at once}."""
    classes = dict.fromkeys(tid[0] for group in starts.values() for tid, _ in group)
    return {c: scene_peak(n_frames, {t: [(tid, b) for tid, b in group if tid[0] == c] for t, group in starts.items()}, ends)
            for c in classes}


def feed_schedule(lengths, peaks, feeds, max_targets):
    """When and on which feed every scene runs.  Scenes are admitted longest first (ties in scene order); the next scene waits
    for a free feed and for `peaks[i]` free slots, the most targets it has active at once, which stay reserved until it ends.  A
    feed is reused from the step after its scene's last frame.  Returns [(scene, feed, first step)] in admission order; scene i
    runs its frame t at step first + t.  Per class: `max_targets` {class: slots} and `peaks[i]` {class: peak} (class_peaks);
    a scene then waits until every class has its peak free."""
    n = len(lengths)
    per_class = isinstance(max_targets, dict)
    cap = {c: int(k) for c, k in max_targets.items()} if per_class else {None: int(max_targets)}
    need = [{c: q for c, q in p.items() if q > 0} for p in peaks] if per_class else [{None: p} for p in peaks]
    for i in range(n):
        if lengths[i] < 1:
            raise ValueError(f"scene {i} has no frames")
        for c, p in need[i].items():
            if not per_class:
                if p > cap[c]:
                    raise ValueError(f"max_targets={cap[c]}: scene {i} has {p} targets active at once and can never fit")
            elif p > cap.get(c, 0):
                raise ValueError(f"max_targets[{c!r}]={cap.get(c, 0)}: scene {i} has {p} targets of class {c!r} active at once "
                                 f"and can never fit")
    order = sorted(range(n), key=lambda i: -lengths[i])
    free_feeds, free_slots, running, out = list(range(int(feeds))), dict(cap), [], []
    step, q = 0, 0
    while q < n:
        for e, i, f in [r for r in running if r[0] < step]:
            running.remove((e, i, f))
            free_feeds.append(f)
            for c, p in need[i].items():
                free_slots[c] += p
        free_feeds.sort()
        while q < n and free_feeds and all(p <= free_slots[c] for c, p in need[order[q]].items()):
            i = order[q]
            f = free_feeds.pop(0)
            for c, p in need[i].items():
                free_slots[c] -= p
            running.append((step + lengths[i] - 1, i, f))
            out.append((i, f, step))
            q += 1
        if q < n:
            step = min(e for e, _, _ in running) + 1
    return out


def _scene_targets(scenes):
    """{target: scene} (ids must be unique over all scenes) and, per scene, {frame: targets dropped after it}."""
    scene_of, last = {}, []
    for i, sc in enumerate(scenes):
        T = int(sc["frames"])
        for group in sc["starts"].values():
            for tid, _ in group:
                if tid in scene_of:
                    raise ValueError(f"target id {tid} appears in scenes {scene_of[tid]} and {i}; ids must be unique")
                scene_of[tid] = i
        drops = {}
        for group in sc["starts"].values():
            for tid, _ in group:
                drops.setdefault(min(sc["ends"].get(tid, T - 1), T - 1), []).append(tid)
        last.append(drops)
    return scene_of, last


def run_scenes(trk, add, drop, scenes, sched, chunk=256, evidence=False):
    """Drive `trk` (a MultiTargetTracker or a MultiClassTracker) through `scenes` on the feeds and steps of `sched`
    (feed_schedule); `add(tid, box, feed)` / `drop(tid)` start and end a target, `trk.targets()` maps the live targets to rows of
    `trk.snapshot()`.  A host thread reads the next step's scans while the current step runs; the boxes and the evidence are read
    back from the device together every `chunk` steps.  A target the tracker's end-of-track rule declares lost has its results
    end at the frame it was declared lost on; its slot is still freed at its planned end, so the schedule stays what
    `feed_schedule` planned.  Returns, per scene, {id: {t: data_classes.Box}}, and with `evidence`, per scene
    {id: {t: (points in the box, score)}} as well."""
    from concurrent.futures import ThreadPoolExecutor

    from ..datasets.data_classes import Box
    scene_of, last = _scene_targets(scenes)
    lengths = [int(sc["frames"]) for sc in scenes]
    n_steps = max((s0 + lengths[i] for i, _, s0 in sched), default=0)
    work = [[] for _ in range(n_steps)]                                        # per step: (feed, scene, frame)
    first = {}
    for i, f, s0 in sched:
        first[i] = s0
        for t in range(lengths[i]):
            work[s0 + t].append((f, i, t))
    out = [{} for _ in scenes]
    ev = [{} for _ in scenes]
    ended = set()                                                             # targets declared lost, in a decoded step
    pending, inflight = [], []

    def load(step):
        return [(f, i, t, scenes[i]["scan"](t)) for f, i, t in work[step]]

    def read_back():                                                          # start a chunk's device -> host copy
        snaps = torch.stack([r[2] for r in pending])
        host = torch.empty(snaps.shape, dtype=snaps.dtype, pin_memory=snaps.is_cuda)
        host.copy_(snaps, non_blocking=True)
        done = torch.cuda.Event() if snaps.is_cuda else None
        if done is not None:
            done.record()
        inflight.append(([(s, live) for s, live, _ in pending], host, done))
        pending.clear()

    def decode():                                                             # finish the oldest chunk
        recs, host, done = inflight.pop(0)
        if done is not None:
            done.synchronize()
        h = host.double().numpy()
        for (s, live), hs in zip(recs, h):
            for tid, k in live.items():
                if tid in ended:
                    continue
                i = scene_of[tid]
                out[i].setdefault(tid, {})[s - first[i]] = Box(hs[k, 0:3], hs[k, 3:6], hs[k, 6:15].reshape(3, 3))
                ev[i].setdefault(tid, {})[s - first[i]] = (int(hs[k, 15]), float(hs[k, 16]))
                if hs[k, 18] != 0:
                    ended.add(tid)

    with ThreadPoolExecutor(max_workers=1) as pool:
        nxt = pool.submit(load, 0) if n_steps else None
        for s in range(n_steps):
            items = nxt.result()
            if s + 1 < n_steps:
                nxt = pool.submit(load, s + 1)                               # read ahead while this step runs
            for f, i, t, scan in items:
                if isinstance(scan, tuple):
                    trk.put_raw(f, *scan)
                else:
                    trk.put(f, torch.as_tensor(scan))
            trk.advance()
            for f, i, t, _ in items:
                for tid, box in scenes[i]["starts"].get(t, ()):
                    add(tid, box, f)
            live = trk.targets()
            if live:
                pending.append((s, live, trk._record()))
            for f, i, t, _ in items:
                for tid in last[i].get(t, ()):
                    if tid in live:
                        drop(tid)
            if len(pending) >= chunk:
                read_back()
                if len(inflight) > 1:
                    decode()
    if pending:
        read_back()
    while inflight:
        decode()
    return (out, ev) if evidence else out


def track_feeds(model, scenes, feeds, max_targets, seed=0, max_points=None, use_graph=True, chunk=256, precision="fp32", lost=None,
                evidence=False):
    """Track many scenes through one tracker with `feeds` scan feeds (`feed_schedule` decides which scene runs when and where).
    `scenes`: [{"frames": number of scans, "scan": t -> the scene's scan t, either (rows, transforms) for `put_raw` or an (n, 3)
    tensor / array for `put`, "starts": {t: [(id, Box), ...]}, "ends": {id: last t}}]; a target without an end runs to its scene's
    last frame, and target ids are unique over all scenes.  `max_points`: the scan buffer's size (required).
    A host thread reads the next step's scans while the current step runs; the boxes are read back from the device every
    `chunk` steps.  Returns, per scene, {id: {t: data_classes.Box}} from the frame a target starts on to its last frame.
    `lost`: the tracker's end-of-track rule (MultiTargetTracker); a lost target's results end at the frame it was declared lost
    on.  With `evidence`, also returns, per scene, {id: {t: (points in the box, score)}} over the same frames."""
    runtime.check_precision(precision)
    lost = check_lost_rule(lost)
    if max_points is None:
        raise ValueError("track_feeds: give max_points, the largest scan of the scenes")
    _scene_targets(scenes)
    lengths = [int(sc["frames"]) for sc in scenes]
    peaks = [scene_peak(lengths[i], sc["starts"], sc["ends"]) for i, sc in enumerate(scenes)]
    sched = feed_schedule(lengths, peaks, feeds, max_targets)
    trk = MultiTargetTracker(model, max_points, max_targets, seed=seed, use_graph=use_graph, feeds=feeds, precision=precision,
                             lost=lost)
    return run_scenes(trk, lambda tid, box, f: trk.add(tid, box, feed=f), trk.drop, scenes, sched, chunk, evidence)
