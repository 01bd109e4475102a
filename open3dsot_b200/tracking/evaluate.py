"""Success / Precision of a tracker over a set of tracklets — what the reference's Lightning `test_step` /
`validation_step` accumulate (models/base_model.py:88-117: every frame's overlap and centre distance go into
TorchSuccess / TorchPrecision, whose `compute()` is the area under the curve)."""
from ..utils.metrics import Precision, Success


def evaluate(model, sequences, progress=None):
    """sequences: iterable of tracklets (lists of {"pc", "3d_bbox"}).  Returns {"success", "precision", "frames", "results"}."""
    succ, prec, results, frames = Success(), Precision(), [], 0
    for i, seq in enumerate(sequences):
        ious, dists, boxes = model.evaluate_one_sequence(seq)
        succ(ious)
        prec(dists)
        results.append(boxes)
        frames += len(seq)
        if progress is not None:
            progress(i, succ.compute(), prec.compute())
    return {"success": succ.compute(), "precision": prec.compute(), "frames": frames, "results": results}


def evaluate_batched(model, sequences, slots=64, seed=0, max_resident_bytes=16 << 30, use_graph=True, ids=None, precision="fp32"):
    """`evaluate()` with `slots` tracklets in flight on the device (tracking/batched_tracker.py): one graph replay per frame
    step for all of them, overlap and centre distance computed on the device, one device-to-host copy per chunk of tracklets
    whose padded frames fit `max_resident_bytes` (a tracklet is never split).  The random draws of a tracklet are keyed by
    (seed, its id, frame), so its result does not depend on `slots`.  `ids`: the tracklets' ids (default: their indices in
    `sequences`); a shard of a split passes the tracklets' indices in the whole split (`evaluate_sharded`).
    Returns the keys of `evaluate()` ("results": a data_classes.Box list per tracklet, in input order) plus the per-frame
    "overlaps" / "distances" (lists per tracklet).  Frame 0 of every tracklet is scored on the host, as the reference does:
    its ground truth against itself sits exactly on Success's top threshold.
    The model's shape_aggregation (including 'all': every past frame's crop, kept in a per-slot history whose bytes count
    against `max_resident_bytes`) and reference_BB ('previous_gt' / 'current_gt': the search area and the box update use the
    ground truth of the previous / current frame, and the result box takes its size) are honoured as the host loop does.
    `precision`: "fp32" or "bf16", the tensor-core operand precision of the network (BatchedDeviceTracker)."""
    import numpy as np

    from .. import runtime

    from ..datasets import data_classes
    from ..utils.metrics import estimateAccuracy, estimateOverlap
    from .batched_tracker import BatchedDeviceTracker, history_bytes, plan_chunks, pool_frame_bytes
    from .device_tracker import HISTORY_POINTS, tracking_modes

    runtime.check_precision(precision)
    sequences = list(sequences)
    cfg = model.config
    dim, up = cfg.IoU_space, cfg.up_axis
    n = len(sequences)
    ids = list(range(n)) if ids is None else [int(i) for i in ids]
    if len(ids) != n:
        raise ValueError(f"evaluate_batched: {len(ids)} ids for {n} tracklets")
    lengths = [len(s) for s in sequences]
    mode, ref_mode = tracking_modes(model)
    size_from = {"previous_result": lambda t: 0, "previous_gt": lambda t: t - 1, "current_gt": lambda t: t}[ref_mode]
    overlaps, distances, results = [[] for _ in range(n)], [[] for _ in range(n)], [[] for _ in range(n)]
    for j, seq in enumerate(sequences):
        if lengths[j]:
            gt0 = seq[0]["3d_bbox"]
            overlaps[j].append(estimateOverlap(gt0, gt0, dim=dim, up_axis=up))
            distances[j].append(estimateAccuracy(gt0, gt0, dim=dim, up_axis=up))
            results[j].append(gt0)
    if any(n_ > 1 for n_ in lengths):
        npts = max(f["pc"].points.shape[1] for s in sequences for f in s)
        fixed = history_bytes(min(slots, n), HISTORY_POINTS) if mode == "all" else 0
        for chunk in plan_chunks(lengths, pool_frame_bytes(npts), max_resident_bytes, fixed):
            if all(lengths[j] < 2 for j in chunk):
                continue
            trk = BatchedDeviceTracker(model, [sequences[j] for j in chunk], slots, seed=seed, ids=[ids[j] for j in chunk],
                                       max_points=npts, use_graph=use_graph, precision=precision)
            ov, di, cen, rot = trk.run()
            offsets = trk.plan["offsets"]
            del trk
            for i, j in enumerate(chunk):
                o, L = int(offsets[i]), lengths[j]
                # the fp32 state's size: the first box's, or in the ground-truth modes the reference box's
                wlh = [np.asarray(f["3d_bbox"].wlh, dtype=np.float32).astype(np.float64) for f in sequences[j]]
                overlaps[j] += ov[o + 1: o + L].tolist()
                distances[j] += di[o + 1: o + L].tolist()
                results[j] += [data_classes.Box(cen[o + t], wlh[size_from(t)], rot[o + t]) for t in range(1, L)]
    succ, prec = Success(), Precision()
    for j in range(n):
        succ(overlaps[j])
        prec(distances[j])
    return {"success": succ.compute(), "precision": prec.compute(), "frames": sum(lengths), "results": results,
            "overlaps": overlaps, "distances": distances}


def shard_plan(lengths, world):
    """The tracklets each of `world` ranks evaluates: longest first, each to the rank with the fewest frames so far (ties to
    the lowest rank), so every tracklet is evaluated exactly once and the ranks' frame counts stay balanced.  Each shard is
    in ascending index order."""
    shards, load = [[] for _ in range(world)], [0] * world
    for j in sorted(range(len(lengths)), key=lambda j: (-lengths[j], j)):
        r = min(range(world), key=lambda r: (load[r], r))
        shards[r].append(j)
        load[r] += lengths[j]
    return [sorted(s) for s in shards]


def gather_shards(n, ids, local):
    """All ranks' shard results (`local`: evaluate_batched's output over the tracklets `ids`) reassembled in global order on
    every rank, with Success / Precision over all `n` tracklets accumulated in that order."""
    import torch.distributed as dist
    parts = [None] * dist.get_world_size()
    dist.all_gather_object(parts, (list(ids), local["overlaps"], local["distances"], local["results"]))
    overlaps, distances, results = [None] * n, [None] * n, [None] * n
    for ids_r, ov, di, res in parts:
        for i, j in enumerate(ids_r):
            if overlaps[j] is not None:
                raise RuntimeError(f"gather_shards: tracklet {j} was evaluated by two ranks")
            overlaps[j], distances[j], results[j] = ov[i], di[i], res[i]
    missing = [j for j in range(n) if overlaps[j] is None]
    if missing:
        raise RuntimeError(f"gather_shards: tracklets {missing[:8]} were evaluated by no rank")
    succ, prec = Success(), Precision()
    for j in range(n):
        succ(overlaps[j])
        prec(distances[j])
    return {"success": succ.compute(), "precision": prec.compute(), "frames": sum(len(o) for o in overlaps),
            "results": results, "overlaps": overlaps, "distances": distances}


def evaluate_sharded(model, sequences, slots=64, seed=0, **kw):
    """`evaluate_batched` split across the ranks of a process group (shard_plan): each rank tracks its tracklets with their
    draws keyed by their index in `sequences`, and every rank returns the whole split's result.  With one rank it is
    `evaluate_batched`; `kw` (e.g. `precision`) goes to it."""
    from .. import ddp
    sequences = list(sequences)
    if not ddp.is_distributed():
        return evaluate_batched(model, sequences, slots=slots, seed=seed, **kw)
    import torch.distributed as dist
    mine = shard_plan([len(s) for s in sequences], dist.get_world_size())[dist.get_rank()]
    local = evaluate_batched(model, [sequences[j] for j in mine], slots=slots, seed=seed, ids=mine, **kw)
    return gather_shards(len(sequences), mine, local)
