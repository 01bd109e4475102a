"""Multi-object tracking scores of tracking runs: CLEAR MOT (MOTA, MOTP, switches, fragmentations, mostly tracked / lost) and
the identity scores (IDF1), computed on the device (`o3d_mot_clear`, csrc/mot_eval.cu) with motmetrics' event rules.

A run is a list of sequences, a sequence a list of frames, a frame a pair (ground truth, hypotheses), each a list of (id, Box).
Ids are unique within a frame and never cross sequences.  A pair (object, hypothesis) of a frame is valid when, in fp64,
  metric "iou":      iou = utils.metrics.estimateOverlap(gt, hyp, dim, up_axis) >= threshold (threshold in (0, 1]), cost 1 - iou;
  metric "distance": d = estimateAccuracy(gt, hyp, dim, up_axis) <= threshold (finite, > 0), cost d.
Each frame, as motmetrics' MOTAccumulator.update with its defaults (no switch time limit):
  1. carry-over: the objects in the frame's order; object o whose last matched hypothesis m[o] is in the frame, still
     unmatched and valid with o is matched to it (a MATCH);
  2. assignment: among the remaining objects and hypotheses, a matching of maximum cardinality over the valid pairs and of
     least total cost among those (motmetrics' construction: the invalid pairs at 2 r c + 1, r the smaller side, c one more
     than the largest |cost| of a valid pair, through scipy's linear_sum_assignment, assignments to invalid pairs dropped).  A
     new pair (o, h) is a SWITCH when m[o] exists and differs from h, else a MATCH; then m[o] = h;
  3. unmatched objects are MISSes, unmatched hypotheses FALSE POSITIVEs.
Per sequence: the counts (num_objects = ground-truth boxes, num_predictions = hypothesis boxes, num_matches, num_switches,
num_misses, num_false_positives), total_cost (the matched and switched pairs' costs, in frame order then object order),
num_fragmentations (per object, tracked -> missed transitions between its first and last tracked frames), mostly_tracked /
partially_tracked / mostly_lost (tracked share of an object's frames >= 0.8 / otherwise / < 0.2), and the identity scores:
c[o, h] = the frames in which (o, h) is a valid pair, idtp = the largest sum of c over one-to-one object / hypothesis
assignments, idfn = num_objects - idtp, idfp = num_predictions - idtp.  Derived: mota = 1 - (misses + switches + false
positives) / objects, motp = total_cost / (matches + switches) (for IoU, 1 - mean_iou, also reported), idf1 = 2 idtp /
(objects + predictions), idp = idtp / predictions, idr = idtp / objects; a ratio with a zero denominator is NaN.  The total
over sequences sums the counts, total_cost, the MT / PT / ML counts and idtp, and recomputes the ratios.

`mot_metrics` runs the device kernel; `mot_reference` is the plain-loop numpy / scipy statement of the same rules that the
tests hold the kernel to."""
from typing import NamedTuple

import numpy as np
from scipy.optimize import linear_sum_assignment

MAX_BOXES = 256           # ground-truth boxes, and hypothesis boxes, of one frame (O3D_MOT_MAX_BOXES)
METRICS = ("iou", "distance")
COUNTERS = ("num_objects", "num_predictions", "num_matches", "num_switches", "num_misses", "num_false_positives",
            "num_fragmentations")
BOX_VALUES = 15           # centre (3), wlh (3), row-major rotation (9)


class MotRun(NamedTuple):
    """A run packed into arrays: sequence s has frames seq_frame[s] .. seq_frame[s+1] - 1; frame f has the ground-truth boxes
    frame_gt[f] .. frame_gt[f+1] - 1 and the hypothesis boxes frame_hyp[f] .. frame_hyp[f+1] - 1, in the frame's order."""
    seq_frame: np.ndarray     # (S + 1,) int64
    frame_gt: np.ndarray      # (F + 1,) int64
    frame_hyp: np.ndarray     # (F + 1,) int64
    gt_id: np.ndarray         # (NG,) int64
    hyp_id: np.ndarray        # (NH,) int64
    gt_box: np.ndarray        # (NG, 15) float64
    hyp_box: np.ndarray       # (NH, 15) float64


def box_values(box):
    """A Box as its 15 packed values: centre, wlh, row-major rotation."""
    return np.concatenate([np.asarray(box.center, np.float64).reshape(3), np.asarray(box.wlh, np.float64).reshape(3),
                           np.asarray(box.rotation_matrix, np.float64).reshape(9)])


def values_box(v):
    from ..datasets.data_classes import Box
    return Box(v[0:3], v[3:6], v[6:15].reshape(3, 3))


def pack_run(sequences):
    """A run given as sequences of frames (gt, hyp), each a list of (id, Box), as a MotRun."""
    seq_frame, frame_gt, frame_hyp = [0], [0], [0]
    ids, boxes = ([], []), ([], [])
    for s, seq in enumerate(sequences):
        for f, frame in enumerate(seq):
            try:
                gt, hyp = frame
            except (TypeError, ValueError):
                raise ValueError(f"mot: sequence {s} frame {f}: expected a pair (ground truth, hypotheses)") from None
            for side, items in enumerate((gt, hyp)):
                for item in items:
                    try:
                        i, box = item
                        ids[side].append(int(i))
                        boxes[side].append(box_values(box))
                    except (TypeError, ValueError, AttributeError):
                        raise ValueError(f"mot: sequence {s} frame {f}: expected (id, Box) items, got {item!r}") from None
            frame_gt.append(len(ids[0]))
            frame_hyp.append(len(ids[1]))
        seq_frame.append(len(frame_gt) - 1)
    arr = lambda v: np.asarray(v, np.int64)
    box = lambda b: np.asarray(b, np.float64).reshape(-1, BOX_VALUES)
    return MotRun(arr(seq_frame), arr(frame_gt), arr(frame_hyp), arr(ids[0]), arr(ids[1]), box(boxes[0]), box(boxes[1]))


def check_scoring(metric, threshold, dim=2, up_axis=(0, -1, 0)):
    """(metric, threshold, dim, up_axis) checked: ValueError for an unknown metric, a threshold outside (0, 1] (IoU) or not finite
    and > 0 (distance), dim not 2 / 3, an up_axis that names no axis."""
    if metric not in METRICS:
        raise ValueError(f"mot: metric must be one of {METRICS}, got {metric!r}")
    try:
        threshold = float(threshold)
    except (TypeError, ValueError):
        raise ValueError(f"mot: threshold must be a number, got {threshold!r}") from None
    if metric == "iou" and not 0.0 < threshold <= 1.0:
        raise ValueError(f"mot: an IoU threshold must be in (0, 1], got {threshold}")
    if metric == "distance" and not (np.isfinite(threshold) and threshold > 0.0):
        raise ValueError(f"mot: a distance threshold must be finite and > 0, got {threshold}")
    if dim not in (2, 3):
        raise ValueError(f"mot: dim must be 2 or 3, got {dim!r}")
    up_axis = tuple(up_axis)
    if len(up_axis) != 3 or not any(a != 0 for a in up_axis):
        raise ValueError(f"mot: up_axis must be three values naming an axis, got {up_axis}")
    return metric, threshold, dim, up_axis


class _Dense(NamedTuple):
    gt_obj: np.ndarray        # (NG,) int32: dense object index within the sequence
    hyp_idx: np.ndarray       # (NH,) int32
    obj_off: np.ndarray       # (S + 1,) int64
    hyp_off: np.ndarray
    cooc_off: np.ndarray
    max_gt: int
    max_hyp: int


def _offsets(name, off, first_end):
    off = np.asarray(off)
    if off.ndim != 1 or off.dtype.kind not in "iu" or len(off) < 1 or off[0] != 0 or (np.diff(off) < 0).any() \
            or off[-1] != first_end:
        raise ValueError(f"mot: {name} must be non-decreasing int offsets from 0 to {first_end}")
    return off.astype(np.int64)


def check_run(run):
    """Refuse (ValueError) a malformed MotRun: offsets, shapes, more than 256 boxes per frame and side, a non-finite box value
    or an id twice in one frame.  Returns the run with the sequences' dense object / hypothesis indices (_Dense)."""
    if not isinstance(run, MotRun):
        run = pack_run(run)
    gt_id, hyp_id = np.asarray(run.gt_id), np.asarray(run.hyp_id)
    gt_box, hyp_box = np.asarray(run.gt_box, np.float64), np.asarray(run.hyp_box, np.float64)
    if gt_id.ndim != 1 or hyp_id.ndim != 1 or gt_id.dtype.kind not in "iu" or hyp_id.dtype.kind not in "iu":
        raise ValueError("mot: gt_id / hyp_id must be 1-D int arrays")
    if gt_box.shape != (len(gt_id), BOX_VALUES) or hyp_box.shape != (len(hyp_id), BOX_VALUES):
        raise ValueError(f"mot: gt_box / hyp_box must be (boxes, {BOX_VALUES}) arrays beside their ids")
    if not (np.isfinite(gt_box).all() and np.isfinite(hyp_box).all()):
        raise ValueError("mot: every box value must be finite")
    frame_gt = _offsets("frame_gt", run.frame_gt, len(gt_id))
    frame_hyp = _offsets("frame_hyp", run.frame_hyp, len(hyp_id))
    if len(frame_gt) != len(frame_hyp):
        raise ValueError("mot: frame_gt and frame_hyp must have one entry per frame, plus one")
    seq_frame = _offsets("seq_frame", run.seq_frame, len(frame_gt) - 1)
    n_gt, n_hyp = np.diff(frame_gt), np.diff(frame_hyp)
    big = np.nonzero((n_gt > MAX_BOXES) | (n_hyp > MAX_BOXES))[0]
    if len(big):
        f = int(big[0])
        raise ValueError(f"mot: frame {f} has {n_gt[f]} ground-truth and {n_hyp[f]} hypothesis boxes; at most {MAX_BOXES} each")
    S = len(seq_frame) - 1
    gt_obj, hyp_idx = np.empty(len(gt_id), np.int32), np.empty(len(hyp_id), np.int32)
    off = {"gt": [0], "hyp": [0]}
    for side, ids, fr, out in (("gt", gt_id, frame_gt, gt_obj), ("hyp", hyp_id, frame_hyp, hyp_idx)):
        frame_of = np.repeat(np.arange(len(fr) - 1), np.diff(fr))
        if len(np.unique(np.stack([frame_of, ids]), axis=1).T) != len(ids):
            raise ValueError(f"mot: an id appears twice in one frame ({'ground truth' if side == 'gt' else 'hypotheses'})")
        for s in range(S):
            a, b = fr[seq_frame[s]], fr[seq_frame[s + 1]]
            uniq, inv = np.unique(ids[a:b], return_inverse=True)
            out[a:b] = inv
            off[side].append(off[side][-1] + len(uniq))
    obj_off, hyp_off = np.asarray(off["gt"], np.int64), np.asarray(off["hyp"], np.int64)
    cooc_off = np.concatenate([[0], np.cumsum(np.diff(obj_off) * np.diff(hyp_off))]).astype(np.int64)
    run = MotRun(seq_frame, frame_gt, frame_hyp, gt_id, hyp_id, gt_box, hyp_box)
    return run, _Dense(gt_obj, hyp_idx, obj_off, hyp_off, cooc_off, int(n_gt.max(initial=0)), int(n_hyp.max(initial=0)))


def _ratios(d, metric):
    div = lambda a, b: a / b if b else float("nan")
    d["idfn"] = d["num_objects"] - d["idtp"]
    d["idfp"] = d["num_predictions"] - d["idtp"]
    d["mota"] = 1.0 - div(d["num_misses"] + d["num_switches"] + d["num_false_positives"], d["num_objects"])
    d["motp"] = div(d["total_cost"], d["num_matches"] + d["num_switches"])
    if metric == "iou":
        d["mean_iou"] = 1.0 - d["motp"]
    d["idf1"] = div(2 * d["idtp"], d["num_objects"] + d["num_predictions"])
    d["idp"] = div(d["idtp"], d["num_predictions"])
    d["idr"] = div(d["idtp"], d["num_objects"])
    return d


def sequence_scores(counts, total_cost, present, tracked, cooc, metric):
    """One sequence's scores from its counts (COUNTERS order), cost sum, per-object frames present / tracked and co-occurrence
    matrix c (objects x hypotheses)."""
    d = {k: int(v) for k, v in zip(COUNTERS, counts)}
    d["total_cost"] = float(total_cost)
    ratio = np.asarray(tracked, np.float64) / np.maximum(np.asarray(present, np.float64), 1)
    d["mostly_tracked"] = int((ratio >= 0.8).sum())
    d["mostly_lost"] = int((ratio < 0.2).sum())
    d["partially_tracked"] = len(ratio) - d["mostly_tracked"] - d["mostly_lost"]
    d["idtp"] = 0
    if cooc.size:
        r, c = linear_sum_assignment(cooc, maximize=True)
        d["idtp"] = int(cooc[r, c].sum())
    return _ratios(d, metric)


def total_scores(sequences, metric):
    """The total over sequences' scores: counts, total_cost, MT / PT / ML and idtp summed, the ratios recomputed."""
    keys = COUNTERS + ("mostly_tracked", "partially_tracked", "mostly_lost", "idtp")
    d = {k: sum(s[k] for s in sequences) for k in keys}
    d["total_cost"] = float(sum(s["total_cost"] for s in sequences))
    return _ratios(d, metric)


class SequenceCounts(NamedTuple):
    """One sequence's events: counts in COUNTERS order, the cost sum, per-object frames present / tracked, and the
    co-occurrence matrix c (objects x hypotheses, dense per-sequence indices)."""
    counts: np.ndarray
    total_cost: float
    present: np.ndarray
    tracked: np.ndarray
    cooc: np.ndarray


def _scores(raw, metric):
    seqs = [sequence_scores(r.counts, r.total_cost, r.present, r.tracked, r.cooc, metric) for r in raw]
    return {"total": total_scores(seqs, metric), "sequences": seqs}


def upload_run(run, dense, device="cuda"):
    """The kernel's inputs of a checked run (`check_run`) as CUDA tensors, in `ops.mot_clear`'s order (an empty side padded to
    one row, which no frame reads)."""
    import torch
    up = lambda a, dtype: torch.as_tensor(np.ascontiguousarray(a, dtype=dtype)).to(device)
    pad = lambda a: a if len(a) else np.zeros((1,) + a.shape[1:], a.dtype)
    return (up(run.seq_frame, np.int64), up(run.frame_gt, np.int64), up(run.frame_hyp, np.int64), up(dense.obj_off, np.int64),
            up(dense.hyp_off, np.int64), up(dense.cooc_off, np.int64), up(pad(dense.gt_obj), np.int32),
            up(pad(dense.hyp_idx), np.int32), up(pad(run.gt_box), np.float64), up(pad(run.hyp_box), np.float64))


def work_rows(S):
    """Scratch rows (CTAs) of one launch: one per sequence, at most two per SM."""
    from .. import _lib
    return max(1, min(S, 2 * _lib.lib().o3d_device_sms()))


def device_counts(run, metric, threshold, dim=2, up_axis=(0, -1, 0), device="cuda"):
    """Each sequence's SequenceCounts from one `o3d_mot_clear` launch on the current stream and one read-back."""
    import torch

    from .. import ops
    metric, threshold, dim, up_axis = check_scoring(metric, threshold, dim, up_axis)
    run, dense = check_run(run)
    S = len(run.seq_frame) - 1
    outs = ops.mot_clear(*upload_run(run, dense, device), metric, threshold, dim, up_axis, dense.max_gt, dense.max_hyp,
                         work_rows(S))
    host = [t.to("cpu", non_blocking=True) for t in outs]
    torch.cuda.current_stream().synchronize()
    counts, cost_sum, obj, cooc = (t.numpy() for t in host)
    raw = []
    for s in range(S):
        o0, o1 = dense.obj_off[s], dense.obj_off[s + 1]
        c = cooc[dense.cooc_off[s]:dense.cooc_off[s + 1]].reshape(int(o1 - o0), int(dense.hyp_off[s + 1] - dense.hyp_off[s]))
        raw.append(SequenceCounts(counts[s], float(cost_sum[s]), obj[o0:o1, 0], obj[o0:o1, 1], c))
    return raw


def mot_metrics(run, metric, threshold, dim=2, up_axis=(0, -1, 0), device="cuda"):
    """Score a run on the device: {"total": {...}, "sequences": [{...}, ...]} with the keys of the module docstring.  `run`:
    sequences of frames (gt, hyp), each a list of (id, Box), or a MotRun.  One `o3d_mot_clear` launch on the current stream, one
    read-back, then each sequence's IDF1 assignment on the host.  Refuses (ValueError) what `check_scoring` / `check_run` do."""
    return _scores(device_counts(run, metric, threshold, dim, up_axis, device), metric)


# ------------------------------------------------------------------ the reference: the rules above as the plain loop
def expensive_edges(costs):
    """motmetrics.lap.add_expensive_edges: the invalid (NaN) entries at 2 r c + 1 (r the smaller side, c = 1 + the largest |cost|
    of a valid entry); unchanged when every entry is valid, zeros when none is."""
    valid = np.isfinite(costs)
    if valid.all():
        return costs.copy()
    if not valid.any():
        return np.zeros_like(costs)
    r = min(costs.shape)
    c = np.abs(costs[valid]).max() + 1
    return np.where(valid, costs, 2 * r * c + 1)


def reference_counts(run, metric, threshold, dim=2, up_axis=(0, -1, 0)):
    """`device_counts` on the host, frame by frame: per pair utils.metrics.estimateOverlap (each box's footprint computed once)
    or estimateAccuracy, motmetrics' event rules, scipy's linear_sum_assignment on the remainder."""
    from ..utils.metrics import _footprint, estimateAccuracy, estimateOverlap
    metric, threshold, dim, up_axis = check_scoring(metric, threshold, dim, up_axis)
    run, dense = check_run(run)
    raw = []
    for s in range(len(run.seq_frame) - 1):
        n_obj = int(dense.obj_off[s + 1] - dense.obj_off[s])
        n_hyp = int(dense.hyp_off[s + 1] - dense.hyp_off[s])
        cooc = np.zeros((n_obj, n_hyp), np.int64)
        present, tracked = np.zeros(n_obj, np.int64), np.zeros(n_obj, np.int64)
        history = [[] for _ in range(n_obj)]           # per object and frame present: tracked or not
        last = {}                                      # object -> its last matched hypothesis
        n = dict.fromkeys(COUNTERS, 0)
        total_cost = 0.0
        for f in range(run.seq_frame[s], run.seq_frame[s + 1]):
            ga, gb, ha, hb = run.frame_gt[f], run.frame_gt[f + 1], run.frame_hyp[f], run.frame_hyp[f + 1]
            objs, hyps = dense.gt_obj[ga:gb], dense.hyp_idx[ha:hb]
            gboxes = [values_box(v) for v in run.gt_box[ga:gb]]
            hboxes = [values_box(v) for v in run.hyp_box[ha:hb]]
            G, H = len(objs), len(hyps)
            cost = np.full((G, H), np.nan)
            if metric == "iou":
                gfp = [_footprint(b, up_axis) for b in gboxes]
                hfp = [_footprint(b, up_axis) for b in hboxes]
            for a in range(G):
                for b in range(H):
                    if metric == "iou":
                        iou = estimateOverlap(gboxes[a], hboxes[b], dim, up_axis, footprints=(gfp[a], hfp[b]))
                        if iou >= threshold:
                            cost[a, b] = 1.0 - iou
                    else:
                        d = estimateAccuracy(gboxes[a], hboxes[b], dim, up_axis)
                        if d <= threshold:
                            cost[a, b] = d
                    if np.isfinite(cost[a, b]):
                        cooc[objs[a], hyps[b]] += 1
            gm, hm, new = [-1] * G, [-1] * H, [False] * G
            for a in range(G):                                                   # 1. carry-over
                o = objs[a]
                if o in last:
                    b = next((b for b in range(H) if hyps[b] == last[o]), None)
                    if b is not None and hm[b] < 0 and np.isfinite(cost[a, b]):
                        gm[a], hm[b] = b, a
            rows = [a for a in range(G) if gm[a] < 0]                            # 2. assignment
            cols = [b for b in range(H) if hm[b] < 0]
            if rows and cols:
                sub = cost[np.ix_(rows, cols)]
                for i, j in zip(*linear_sum_assignment(expensive_edges(sub))):
                    if np.isfinite(sub[i, j]):
                        gm[rows[i]], hm[cols[j]], new[rows[i]] = cols[j], rows[i], True
            for a in range(G):                                                   # 3. events
                o = objs[a]
                present[o] += 1
                if gm[a] < 0:
                    n["num_misses"] += 1
                    history[o].append(False)
                    continue
                h = hyps[gm[a]]
                if new[a] and o in last and last[o] != h:
                    n["num_switches"] += 1
                else:
                    n["num_matches"] += 1
                last[o] = h
                tracked[o] += 1
                history[o].append(True)
                total_cost += cost[a, gm[a]]
            n["num_false_positives"] += H - sum(b >= 0 for b in gm)
            n["num_objects"] += G
            n["num_predictions"] += H
        for hist in history:                       # motmetrics' num_fragmentations
            hits = [t for t, x in enumerate(hist) if x]
            if hits:
                span = hist[hits[0]:hits[-1] + 1]
                n["num_fragmentations"] += sum(x and not y for x, y in zip(span, span[1:]))
        raw.append(SequenceCounts(np.array([n[k] for k in COUNTERS], np.int64), float(total_cost), present, tracked, cooc))
    return raw


def mot_reference(run, metric, threshold, dim=2, up_axis=(0, -1, 0)):
    """`mot_metrics` from `reference_counts`: the statement the tests hold the kernel to."""
    return _scores(reference_counts(run, metric, threshold, dim, up_axis), metric)
