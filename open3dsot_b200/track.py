"""`python -m open3dsot_b200.track --cfg <yaml> --checkpoint <ckpt> --path <dataset root> --split test --out results.jsonl`:
live multi-target tracking over the scans of every scene of a KITTI, nuScenes or Waymo split (tracking/multi_tracker.py).

The config's `dataset` picks the reader.  For every scene of the split, every scan from the first tracklet start to the last
tracklet end is streamed, whole (no `preload_offset` crop), in the reader's frame: KITTI in the config's `coordinate_mode`,
nuScenes and Waymo in the global frame.  Scenes are tracked together through `track_feeds`, one feed per scene in flight
(min(scenes, max_targets) feeds); the readers' transforms run on the device (`put_raw`, csrc/scan_ingest.cu) and the results do
not depend on the number of feeds.  A scene's frames are its scan files (KITTI, Waymo frame ids) or the positions of its key-frame
LIDAR_TOP scans in timestamp order (nuScenes).  Every tracklet of `category_name` starts on its first annotated
frame from its ground-truth box and is dropped after its last annotated frame; nothing else of the ground truth is used.  One
JSON line per (scene, frame) lists every active target's box; Success / Precision over the annotated frames are printed, with
the host metric path of `tracking.evaluate` (the first frame of a tracklet scored against its own ground truth).  A target's
draws are keyed by its tracklet's index in the split, as `evaluate_batched` keys them by default.

Several classes: `--add_class CFG [CKPT]` (repeatable) adds a class with its own model and weights, tracking its config's
`category_name`; every config shares the dataset and the reader's frame settings (`check_classes`).  Each class's reader lists
its tracklets, the scene plans are merged so that every scene streams once for all classes, and one `MultiClassTracker`
(tracking/multi_class.py) advances every class in one captured step per scan.  `--max_targets` is per class (`K`, or `NAME=K`
for one class).  Every JSON line's targets carry their "class"; Success / Precision are printed over all frames and per class,
and a class's boxes are those of a run with its config alone at the same --max_points and --max_targets.

Evidence and lost targets.  Every JSON line's targets carry "points", the points of that frame's scan in the box scaled by 1.25,
and "score", the model's confidence (BAT / P2B: the best proposal's score; M2-Track: the share of the current frame's sampled
points segmented as target); both are null on a tracklet's first frame.  `--lost MIN_POINTS PATIENCE` ends a tracklet once
PATIENCE consecutive frames had fewer than MIN_POINTS points in its box (tracking/multi_tracker.py, decided on the device): its
lines stop at that frame, its annotated frames after it are scored as failures (overlap 0, distance inf), and the printed
summary counts the tracklets ended early as "lost".  `--coast ALPHA` (with --lost) moves a missed target along its velocity
instead of writing the network's box (MultiTargetTracker's `coast=`): every JSON line's targets carry "coasting", whether that
frame's box was coasted, and the summary counts "coasted" (target-frames reported while coasting) and "reacquired" (coasting
spells that ended in a hit).  Success / Precision score the coasted boxes.

Detections.  `--detections FILE --detection_gate METRES --max_detections N` gives every scan a 3D detector's boxes: FILE has one
JSON line per {"scene", "frame", "class", "boxes": [[cx, cy, cz, w, l, h, qw, qx, qy, qz, score], ...]}, the scene id as the
reader lists it (`scene_list`), the frame as the scene's frames are numbered, the class a config's category_name and the
quaternion the box's orientation (data_classes.Box).  A scan without a line has no detections.  The tracker matches them to
its targets (MultiTargetTracker's `detections=`) and re-acquires a missed target at its detection; tracklets still start from
their first annotated box.  Every JSON line's targets carry "detection", the index of the detection matched on that frame in
its line's boxes (null: none), and "reacquired"; the summary counts "reacquired_at_detection", the target-frames re-acquired.

Multi-object scores.  `--mot {iou,distance} THRESHOLD` scores the run as multi-object tracking (tracking/mot.py: CLEAR MOT and
IDF1, on the device) with the config's IoU_space and up_axis: each scene is a sequence over its streamed frames, its ground
truth the split's annotations on the frame (object id: the tracklet's index) and its hypotheses every box the run reported on
the frame (id: the target's tracklet index).  A box reported on a frame where its tracklet has no annotation is a false positive
(nuScenes' min_points=1 filtering of the evaluation splits can leave such frames).  The summary gains "mot": {"total",
"sequences"}; with several classes, each class is scored against its own ground truth under "classes", and "mot": {"total"} at
the top sums them."""
import argparse
import json
import sys

import numpy as np


class _MaxTargets(argparse.Action):
    """--max_targets K (an int, every class) or NAME=K (repeatable): then a dict {NAME: K, None: the K of the other classes}."""

    def __call__(self, parser, namespace, value, option_string=None):
        name, eq, k = value.rpartition("=")
        try:
            k = int(k)
        except ValueError:
            parser.error(f"--max_targets {value}: expected K or NAME=K")
        cur = getattr(namespace, self.dest)
        if not eq:
            if isinstance(cur, dict):
                cur[None] = k
            else:
                setattr(namespace, self.dest, k)
        elif not name:
            parser.error(f"--max_targets {value}: expected K or NAME=K")
        else:
            if not isinstance(cur, dict):
                cur = {None: cur}
            cur[name] = k
            setattr(namespace, self.dest, cur)


def class_targets(max_targets, name):
    """A class's slots from --max_targets: the int, or the class's NAME=K entry (else the plain K, 64 by default)."""
    return max_targets.get(name, max_targets[None]) if isinstance(max_targets, dict) else max_targets


def parse_args(argv=None):
    p = argparse.ArgumentParser(prog="python -m open3dsot_b200.track")
    p.add_argument('--cfg', type=str, required=True, help='the config file')
    p.add_argument('--checkpoint', type=str, default=None, help='weights (a checkpoint of ours or of the reference)')
    p.add_argument('--path', type=str, required=True, help='dataset root (for KITTI: velodyne/, label_02/, calib/)')
    p.add_argument('--split', type=str, default='test', help='scene split (train / valid / test / *_tiny)')
    p.add_argument('--out', type=str, default='results.jsonl', help='per-frame results, one JSON line per (scene, frame)')
    p.add_argument('--add_class', action='append', nargs='+', metavar=('CFG', 'CKPT'), default=None,
                   help='track a further class: its config and, optionally, its weights (repeatable); the configs share the '
                        'dataset and its frame settings')
    p.add_argument('--max_targets', action=_MaxTargets, default=64,
                   help='tracker slots per class (targets in flight at once): K for every class, or NAME=K for the class whose '
                        'category_name is NAME (repeatable)')
    p.add_argument('--max_points', type=int, default=None, help='scan buffer size (default: the largest scan streamed)')
    p.add_argument('--seed', type=int, default=0, help='key of the random draws')
    p.add_argument('--precision', choices=('fp32', 'bf16'), default='fp32',
                   help='operand precision of the tensor-core layers (bf16: BF16 operands, FP32 accumulation)')
    # without --lost the namespace has no `lost` (argparse.SUPPRESS): the options of a run without the rule are what they were
    p.add_argument('--lost', type=int, nargs=2, metavar=('MIN_POINTS', 'PATIENCE'), default=argparse.SUPPRESS,
                   help='end a tracklet once PATIENCE consecutive frames had fewer than MIN_POINTS scan points in its box '
                        '(scaled by 1.25); its later annotated frames count as failures')
    # likewise --coast (SUPPRESS): a run without it has no `coast`
    p.add_argument('--coast', type=float, metavar='ALPHA', default=argparse.SUPPRESS,
                   help='with --lost: move a target whose frame is a miss along its velocity (ALPHA, in (0, 1]: the weight of the '
                        'newest velocity sample) instead of writing the network\'s box')
    # --detections and its two settings (SUPPRESS as well): a run without them keeps its options
    p.add_argument('--detections', type=str, metavar='FILE', default=argparse.SUPPRESS,
                   help='JSON lines of per-scan detections {"scene", "frame", "class", "boxes": [[cx, cy, cz, w, l, h, qw, qx, qy, '
                        'qz, score], ...]}: matched to the targets, re-acquiring missed ones')
    p.add_argument('--detection_gate', type=float, metavar='METRES', default=argparse.SUPPRESS,
                   help='with --detections: the largest centre distance of a match, in the plane orthogonal to up_axis')
    p.add_argument('--max_detections', type=int, metavar='N', default=argparse.SUPPRESS,
                   help='with --detections: the most detections of one scan (1 .. 1024)')
    # --mot as well (SUPPRESS): a run without it is scored as it always was
    p.add_argument('--mot', nargs=2, metavar=('METRIC', 'THRESHOLD'), default=argparse.SUPPRESS,
                   help='also score the run as multi-object tracking (CLEAR MOT, IDF1): METRIC iou (a pair matches when its '
                        'IoU >= THRESHOLD) or distance (centre distance <= THRESHOLD)')
    args = p.parse_args(argv)
    if hasattr(args, "lost"):
        from .tracking.multi_tracker import check_lost_rule
        try:
            args.lost = check_lost_rule(args.lost)
        except ValueError as e:
            p.error(f"--lost: {e}")
    if hasattr(args, "coast"):
        if not hasattr(args, "lost"):
            p.error("--coast needs --lost MIN_POINTS PATIENCE: the rule decides which frames are misses")
        from .tracking.multi_tracker import check_coast
        try:
            args.coast = check_coast(args.coast, args.lost)
        except ValueError as e:
            p.error(f"--coast: {e}")
    given = [hasattr(args, n) for n in ("detections", "detection_gate", "max_detections")]
    if any(given) and not all(given):
        p.error("--detections FILE needs --detection_gate METRES and --max_detections N, and they need it")
    if all(given):
        from .tracking.multi_tracker import check_detections
        try:
            args.detection_rule = check_detections((args.max_detections, args.detection_gate))
        except ValueError as e:
            p.error(f"--detection_gate / --max_detections: {e}")
    if hasattr(args, "mot"):
        try:
            args.mot = check_mot(args.mot)
        except ValueError as e:
            p.error(f"--mot: {e}")
    for extra in args.add_class or ():
        if len(extra) > 2:
            p.error(f"--add_class takes a config and at most one checkpoint, got {extra}")
    return args


def check_mot(mot):
    """--mot METRIC THRESHOLD as (metric, threshold): ValueError for an unknown metric or a threshold out of its range."""
    from .tracking.mot import check_scoring
    metric, threshold = mot
    return check_scoring(metric, threshold)[:2]


# reader settings that decide which scans a scene's frames are and in which frame their points are: the classes of one run share
# them, and with them every scan
FRAME_KEYS = {"kitti": (("coordinate_mode", "velodyne"),), "nuscenes": (("version", "v1.0-trainval"), ("key_frame_only", False)),
              "waymo": (("tiny", False),)}


def check_classes(cfgs, names):
    """Refuse (SystemExit) classes that cannot share one run: another dataset or other frame settings than the first config, or
    a category_name that another class already has.  `names`: the config files, for the messages."""
    first, dataset = cfgs[0], cfgs[0].get("dataset", "kitti")
    seen = {}
    for cfg, name in zip(cfgs, names):
        if cfg.get("dataset", "kitti") != dataset:
            raise SystemExit(f"{name}: dataset '{cfg.get('dataset', 'kitti')}' differs from {names[0]}'s '{dataset}'; the classes "
                             f"of one run track the same scans")
        for key, default in FRAME_KEYS.get(dataset, ()):
            if cfg.get(key, default) != first.get(key, default):
                raise SystemExit(f"{name}: {key}={cfg.get(key, default)} differs from {names[0]}'s {key}={first.get(key, default)}; "
                                 f"the classes of one run read the scans in the same frame")
        if cfg.category_name in seen:
            raise SystemExit(f"{name}: category_name '{cfg.category_name}' is already tracked by {seen[cfg.category_name]}")
        seen[cfg.category_name] = name


def scene_plan(dataset):
    """The streams of a split, in scene order: [{"scene", "first", "last", "frames", "tracklets": [{"index", "track_id", "start",
    "end", "frames"}]}] — `index` is the tracklet's index in the split (the reader's order), `frames` its annotated frames, and the
    stream runs over the scene's scans from `first` to `last` (their frame ids: the scene's "frames").  The reader provides
    `scene_list`, `scene_frames(scene)` and `anno_frame(anno)` -> (scene, frame)."""
    plans = {}
    for j, annos in enumerate(dataset.tracklet_anno_list):
        where = [dataset.anno_frame(a) for a in annos]
        scene, frames = where[0][0], [f for _, f in where]
        track_id = annos[0]["track_id"] if "track_id" in annos[0] else j
        plans.setdefault(scene, []).append({"index": j, "track_id": track_id, "start": frames[0], "end": frames[-1],
                                            "frames": frames})
    out = []
    for scene in dataset.scene_list:
        if scene in plans:
            tr = plans[scene]
            first, last = min(t["start"] for t in tr), max(t["end"] for t in tr)
            out.append({"scene": scene, "first": first, "last": last, "tracklets": tr,
                        "frames": [f for f in dataset.scene_frames(scene) if first <= f <= last]})
    return out


def class_scene_plan(datasets):
    """`scene_plan` over several classes' readers of one split, {class: reader}, merged by scene: a scene streams once, from the
    earliest start to the latest end over every class's tracklets, which carry their "class" (`index` stays the tracklet's index in
    its own reader).  A reader may know only the scenes and frames of its own class (Waymo indexes the scans its tracklets refer
    to; KITTI extends a scene to its own class's last labelled frame), so a merged scene's frames are those of every reader that
    plans the scene, and "reader_of" names, per frame, the class whose reader reads that scan: the first, in class order, that
    lists it.  Scenes in the first reader's order, then any other reader's."""
    merged = {}
    for cls, ds in datasets.items():
        for p in scene_plan(ds):
            m = merged.setdefault(p["scene"], {"scene": p["scene"], "first": p["first"], "last": p["last"], "tracklets": [],
                                               "reader_of": {}})
            m["first"], m["last"] = min(m["first"], p["first"]), max(m["last"], p["last"])
            m["tracklets"] += [dict(tr, **{"class": cls}) for tr in p["tracklets"]]
            for f in ds.scene_frames(p["scene"]):
                m["reader_of"].setdefault(f, cls)
    order = list(dict.fromkeys(s for ds in datasets.values() for s in ds.scene_list))
    out = []
    for scene in order:
        if scene in merged:
            m = merged[scene]
            m["reader_of"] = {f: c for f, c in sorted(m["reader_of"].items()) if m["first"] <= f <= m["last"]}
            m["frames"] = list(m["reader_of"])
            out.append(m)
    return out


def class_stream_max_points(datasets, plan):
    """`stream_max_points` of a merged plan: every frame's scan sized by the reader that reads it."""
    return max([1] + [datasets[p["reader_of"][f]].scan_size(p["scene"], f) for p in plan for f in p["frames"]])


def class_scenes(datasets, plan):
    """The `track_classes` scenes of a merged plan: targets named (class, tracklet index in its class's reader), starting from
    their first ground-truth box, every scan read as stored (`raw_scan`) by the reader `plan` assigns to its frame."""
    scenes = []
    for p in plan:
        pos = {f: t for t, f in enumerate(p["frames"])}
        starts, ends = {}, {}
        for tr in p["tracklets"]:
            c, j = tr["class"], tr["index"]
            starts.setdefault(pos[tr["start"]], []).append(((c, j), datasets[c].box_from_anno(datasets[c].tracklet_anno_list[j][0])))
            ends[(c, j)] = pos[tr["end"]]
        scenes.append({"frames": len(p["frames"]), "starts": starts, "ends": ends,
                       "scan": lambda t, p=p: datasets[p["reader_of"][p["frames"][t]]].raw_scan(p["scene"], p["frames"][t])})
    return scenes


def stream_max_points(dataset, plan):
    """The largest scan of the planned streams (`dataset.scan_size`: from the file sizes where the format allows)."""
    return max([1] + [dataset.scan_size(p["scene"], f) for p in plan for f in p["frames"]])


def _yaw(rot, up_axis):
    """Heading about the up axis: atan2 of the box's x axis in the ground plane (KITTI's rotation_y in camera coordinates)."""
    if up_axis[1] != 0:
        return float(np.arctan2(-rot[2, 0], rot[0, 0]))
    return float(np.arctan2(rot[1, 0], rot[0, 0]))


def _evidence(ev, detections=False):
    """A target's JSON evidence: {"points", "score"}, null where the frame has none (a tracklet's first frame), and "coasting"
    for a coasting tracker's evidence (points, score, coasted).  With `detections` the evidence ends with (reacquired,
    detection): "reacquired" and "detection", null when the frame matched none."""
    if detections:
        ev, (reacquired, det) = ev[:-2], ev[-2:]
    points, score = ev[:2]
    out = {"points": points if points >= 0 else None, "score": score if np.isfinite(score) else None}
    if len(ev) > 2:
        out["coasting"] = bool(ev[2])
    if detections:
        out.update(detection=det if det >= 0 else None, reacquired=bool(reacquired))
    return out


def read_detections(path):
    """The --detections file: {(scene, frame, class): (M, 16) float32 rows (tracking.multi_tracker.detection_rows)}; the scene
    id as a string.  Refuses (SystemExit) a malformed line or two lines for the same scan and class."""
    from .datasets.data_classes import Box
    from .datasets.nuscenes_data import quat_to_rot
    from .tracking.multi_tracker import detection_rows
    out = {}
    with open(path) as f:
        for n, line in enumerate(f, 1):
            if not line.strip():
                continue
            try:
                d = json.loads(line)
                key = (str(d["scene"]), int(d["frame"]), str(d["class"]))
                boxes = np.asarray(d["boxes"], np.float64).reshape(-1, 11)
            except (ValueError, KeyError, TypeError) as e:
                raise SystemExit(f"{path}:{n}: expected {{\"scene\", \"frame\", \"class\", \"boxes\": [[cx, cy, cz, w, l, h, qw, qx, qy, "
                                 f"qz, score], ...]}} ({e})") from None
            if key in out:
                raise SystemExit(f"{path}:{n}: a second line for scene {key[0]} frame {key[1]} class {key[2]}")
            if not np.isfinite(boxes).all() or (np.linalg.norm(boxes[:, 6:10], axis=1) == 0).any():
                raise SystemExit(f"{path}:{n}: every value must be finite and every quaternion non-zero")
            out[key] = detection_rows([Box(b[0:3], b[3:6], quat_to_rot(b[6:10])) for b in boxes], boxes[:, 10])
    return out


def _scan_detections(table, scene, frame, cls):
    """One scan's detection rows for a class from `read_detections`' table (none when the file has no line for it)."""
    return table.get((str(scene), int(frame), cls), np.zeros((0, 16), np.float32))


def _coast_counts(ev, min_points):
    """(frames reported while coasting, coasting spells that ended in a hit) of one target's evidence {t: (points, score,
    coasted)} over consecutive frames: a spell ends in a hit when the frame after it is not coasted and has min_points points
    (a spell can also end in the loss)."""
    frames = sorted(ev)
    coasted = sum(bool(ev[t][2]) for t in frames)
    reacquired = sum(bool(ev[a][2]) and not ev[b][2] and ev[b][0] >= min_points for a, b in zip(frames, frames[1:]))
    return coasted, reacquired


def _score_tracklet(boxes, gts, frames, dim, up):
    """(overlaps, distances) of one tracklet: `gts` its annotated boxes on stream frames `frames`, `boxes` {frame: result box}.
    The first frame is scored against its own ground truth; a frame with no result (after the tracklet was declared lost) is a
    failure: overlap 0, distance inf."""
    from .utils.metrics import estimateAccuracy, estimateOverlap
    overlaps, distances = [], []
    for i, (gt, t) in enumerate(zip(gts, frames)):
        box = gt if i == 0 else boxes.get(t)
        if box is None:
            overlaps.append(0.0)
            distances.append(float("inf"))
        else:
            overlaps.append(estimateOverlap(gt, box, dim=dim, up_axis=up))
            distances.append(estimateAccuracy(gt, box, dim=dim, up_axis=up))
    return overlaps, distances


def mot_sequences(plan, results, dataset, cls=None):
    """The scenes of a run as tracking.mot sequences, one per scene over its streamed frames: ground truth, the annotations of
    the scene's tracklets on the frame with the tracklet index as id; hypotheses, every box of `results` (track_feeds' per-scene
    {target: {frame: Box}}) on the frame with the target's tracklet index as id.  `cls`: one class of a run_classes plan and
    results (targets keyed (class, index))."""
    annos = dataset.tracklet_anno_list
    seqs = []
    for p, res in zip(plan, results):
        gt = {}
        for tr in p["tracklets"]:
            if cls is None or tr["class"] == cls:
                for a in annos[tr["index"]]:
                    gt.setdefault(dataset.anno_frame(a)[1], []).append((tr["index"], dataset.box_from_anno(a)))
        hyp = sorted((k, b) for k, b in res.items() if cls is None or k[0] == cls)
        seqs.append([(gt.get(fr, []), [(k if cls is None else k[1], b[t]) for k, b in hyp if t in b])
                     for t, fr in enumerate(p["frames"])])
    return seqs


def _mot(mot, seqs, dim, up):
    from .tracking.mot import mot_metrics
    return mot_metrics(seqs, mot[0], mot[1], dim, up)


def run(model, dataset, out_path, max_targets=64, max_points=None, seed=0, precision="fp32", lost=None, coast=None,
        detections=None, scan_detections=None, mot=None):
    """Track every scene of `dataset`'s split and write `out_path`; returns {"success", "precision", "frames", "scenes"},
    "lost" with a `lost` rule, and "coasted" / "reacquired" with `coast`.  `detections`: (max_per_scan, gate) and
    `scan_detections` the `read_detections` table: then also "reacquired_at_detection".  `mot`: (metric, threshold): then
    also "mot", the run's tracking.mot scores (mot_sequences)."""
    from .tracking.multi_tracker import track_feeds
    from .utils.metrics import Precision, Success

    cfg = model.config
    dim, up = cfg.IoU_space, cfg.up_axis
    plan = scene_plan(dataset)
    if max_points is None:
        max_points = stream_max_points(dataset, plan)
    annos = dataset.tracklet_anno_list
    scenes = []
    for p in plan:
        pos = {f: t for t, f in enumerate(p["frames"])}
        starts, ends = {}, {}
        for tr in p["tracklets"]:
            starts.setdefault(pos[tr["start"]], []).append((tr["index"], dataset.box_from_anno(annos[tr["index"]][0])))
            ends[tr["index"]] = pos[tr["end"]]
        scenes.append({"frames": len(p["frames"]), "starts": starts, "ends": ends,
                       "scan": lambda t, p=p: dataset.raw_scan(p["scene"], p["frames"][t])})
        if detections is not None:
            scenes[-1]["detections"] = lambda t, p=p: _scan_detections(scan_detections or {}, p["scene"], p["frames"][t],
                                                                       cfg.category_name)
    det = {} if detections is None else {"detections": detections}
    results, evidence = track_feeds(model, scenes, max(1, min(len(scenes), max_targets)), max_targets, seed=seed,
                                    max_points=max_points, precision=precision, lost=lost, evidence=True, coast=coast, **det)
    overlaps, distances = [[] for _ in annos], [[] for _ in annos]
    ended, coasted, reacquired, at_detection = 0, 0, 0, 0
    with open(out_path, "w") as f:
        for p, res, ev in zip(plan, results, evidence):
            scene, pos = p["scene"], {fr: t for t, fr in enumerate(p["frames"])}
            track_id = {tr["index"]: tr["track_id"] for tr in p["tracklets"]}
            for t, frame in enumerate(p["frames"]):
                targets = [{"id": track_id[j], "tracklet": j, "center": b[t].center.tolist(), "wlh": b[t].wlh.tolist(),
                            "yaw": _yaw(b[t].rotation_matrix, up), **_evidence(ev[j][t], detections is not None)}
                           for j, b in sorted(res.items()) if t in b]
                f.write(json.dumps({"scene": scene, "frame": frame, "targets": targets}) + "\n")
            for tr in p["tracklets"]:
                j = tr["index"]
                ended += max(res[j]) < pos[tr["end"]]
                if coast is not None:
                    c, r = _coast_counts(ev[j], lost[0])
                    coasted, reacquired = coasted + c, reacquired + r
                if detections is not None:
                    at_detection += sum(bool(e[-2]) for e in ev[j].values())
                overlaps[j], distances[j] = _score_tracklet(res[j], [dataset.box_from_anno(a) for a in annos[j]],
                                                            [pos[dataset.anno_frame(a)[1]] for a in annos[j]], dim, up)
    succ, prec = Success(), Precision()
    for j in range(len(annos)):
        succ(overlaps[j])
        prec(distances[j])
    out = {"success": succ.compute(), "precision": prec.compute(), "frames": sum(len(o) for o in overlaps), "scenes": len(plan)}
    if lost is not None:
        out["lost"] = ended
    if coast is not None:
        out.update(coasted=coasted, reacquired=reacquired)
    if detections is not None:
        out["reacquired_at_detection"] = at_detection
    if mot is not None:
        out["mot"] = _mot(mot, mot_sequences(plan, results, dataset), dim, up)
    return out


def run_classes(models, datasets, out_path, max_targets, max_points=None, seed=0, precision="fp32", lost=None, coast=None,
                detections=None, scan_detections=None, mot=None):
    """`run` for several classes in one pass over the scans: `models`, `datasets` and `max_targets` are {class: ...} (the class
    is its config's category_name).  Every scene streams once for all classes (class_scene_plan) through one MultiClassTracker;
    a target's draws are keyed by its tracklet's index in its class's reader, as in a one-class run.  Every JSON line's targets
    carry their "class".  Returns {"success", "precision", "frames", "scenes"} over every class's frames, and the same per class
    under "classes"; with a `lost` rule (every class's), "lost" counts the tracklets it ended early, overall and per class, and
    with `coast` (every class's), so do "coasted" and "reacquired"; with `detections` (every class's, and `scan_detections` the
    `read_detections` table), "reacquired_at_detection"; with `mot`, each class's tracking.mot scores against its own ground
    truth under "classes" and "mot": {"total"} over every class's sequences."""
    from .tracking.multi_class import track_classes
    from .utils.metrics import Precision, Success

    names = list(models)
    cfg = models[names[0]].config
    dim, up = cfg.IoU_space, cfg.up_axis
    plan = class_scene_plan(datasets)
    if max_points is None:
        max_points = class_stream_max_points(datasets, plan)
    annos = {c: datasets[c].tracklet_anno_list for c in names}
    scenes = class_scenes(datasets, plan)
    det = {}
    if detections is not None:
        det = {"detections": detections}
        for sc, p in zip(scenes, plan):
            sc["detections"] = lambda t, p=p: {c: _scan_detections(scan_detections or {}, p["scene"], p["frames"][t], c)
                                               for c in names}
    results, evidence = track_classes(models, scenes, max(1, min(len(scenes), sum(max_targets.values()))), max_targets,
                                      seed=seed, max_points=max_points, precision=precision, lost=lost, evidence=True,
                                      coast=coast, **det)
    overlaps = {c: [[] for _ in annos[c]] for c in names}
    distances = {c: [[] for _ in annos[c]] for c in names}
    ended = {c: 0 for c in names}
    coasted, reacquired = {c: 0 for c in names}, {c: 0 for c in names}
    at_detection = {c: 0 for c in names}
    rank = {c: i for i, c in enumerate(names)}
    with open(out_path, "w") as f:
        for p, res, ev in zip(plan, results, evidence):
            scene, pos = p["scene"], {fr: t for t, fr in enumerate(p["frames"])}
            track_id = {(tr["class"], tr["index"]): tr["track_id"] for tr in p["tracklets"]}
            for t, frame in enumerate(p["frames"]):
                targets = [{"class": c, "id": track_id[(c, j)], "tracklet": j, "center": b[t].center.tolist(),
                            "wlh": b[t].wlh.tolist(), "yaw": _yaw(b[t].rotation_matrix, up),
                            **_evidence(ev[(c, j)][t], detections is not None)}
                           for (c, j), b in sorted(res.items(), key=lambda kv: (rank[kv[0][0]], kv[0][1])) if t in b]
                f.write(json.dumps({"scene": scene, "frame": frame, "targets": targets}) + "\n")
            for tr in p["tracklets"]:
                c, j = tr["class"], tr["index"]
                ended[c] += max(res[(c, j)]) < pos[tr["end"]]
                if coast is not None:
                    n_coasted, n_reacquired = _coast_counts(ev[(c, j)], lost[0])
                    coasted[c] += n_coasted
                    reacquired[c] += n_reacquired
                if detections is not None:
                    at_detection[c] += sum(bool(e[-2]) for e in ev[(c, j)].values())
                ds = datasets[c]
                overlaps[c][j], distances[c][j] = _score_tracklet(res[(c, j)], [ds.box_from_anno(a) for a in annos[c][j]],
                                                                  [pos[ds.anno_frame(a)[1]] for a in annos[c][j]], dim, up)

    def scores(classes):
        succ, prec = Success(), Precision()
        for c in classes:
            for o, d in zip(overlaps[c], distances[c]):
                succ(o)
                prec(d)
        out = {"success": succ.compute(), "precision": prec.compute(), "frames": sum(len(o) for c in classes for o in overlaps[c])}
        if lost is not None:
            out["lost"] = sum(ended[c] for c in classes)
        if coast is not None:
            out.update(coasted=sum(coasted[c] for c in classes), reacquired=sum(reacquired[c] for c in classes))
        if detections is not None:
            out["reacquired_at_detection"] = sum(at_detection[c] for c in classes)
        return out

    out = scores(names)
    out.update({"scenes": len(plan), "classes": {c: scores([c]) for c in names}})
    if mot is not None:
        from .tracking.mot import total_scores
        for c in names:
            out["classes"][c]["mot"] = _mot(mot, mot_sequences(plan, results, datasets[c], cls=c), dim, up)
        out["mot"] = {"total": total_scores([s for c in names for s in out["classes"][c]["mot"]["sequences"]], mot[0])}
    return out


def reader(cfg, path, split):
    """The config's dataset reader over a split, for whole-scan tracking (no preloading, no crop)."""
    dataset = cfg.get("dataset", "kitti")
    if dataset == "kitti":
        from .datasets.kitti import kittiDataset
        return kittiDataset(path, split, category_name=cfg.category_name, coordinate_mode=cfg.get("coordinate_mode", "velodyne"),
                            preloading=False, preload_offset=-1)
    if dataset == "nuscenes":
        from .datasets.nuscenes_data import NuScenesDataset
        return NuScenesDataset(path, split, category_name=cfg.category_name, version=cfg.get("version", "v1.0-trainval"),
                               key_frame_only=cfg.get("key_frame_only", False), preloading=False, preload_offset=-1,
                               min_points=1 if split in (cfg.get("val_split"), cfg.get("test_split")) else -1)
    if dataset == "waymo":
        from .datasets.waymo_data import WaymoDataset
        return WaymoDataset(path, split, category_name=cfg.category_name, preloading=False, preload_offset=-1,
                            tiny=cfg.get("tiny", False))
    raise SystemExit(f"dataset '{dataset}': live tracking reads KITTI, nuScenes and Waymo")


def main(argv=None):
    import torch

    from .checkpoint import load_lightning_checkpoint
    from .config import load_config
    from .models import get_model
    from .trainer import load_weights

    args = parse_args(argv)
    rule = {"lost": args.lost} if hasattr(args, "lost") else {}           # without --lost, run / run_classes as they always were
    if hasattr(args, "coast"):
        rule["coast"] = args.coast
    if hasattr(args, "detections"):
        rule.update(detections=args.detection_rule, scan_detections=read_detections(args.detections))
    if hasattr(args, "mot"):
        rule["mot"] = args.mot
    classes = [(args.cfg, args.checkpoint)] + [(a[0], a[1] if len(a) > 1 else None) for a in args.add_class or ()]
    cfgs = [load_config(c) for c, _ in classes]
    check_classes(cfgs, [c for c, _ in classes])
    models, data = {}, {}
    for cfg, (_, ckpt) in zip(cfgs, classes):
        data[cfg.category_name] = reader(cfg, args.path, args.split)
        torch.manual_seed(0)
        model = models[cfg.category_name] = get_model(cfg.net_model)(cfg).cuda()
        if ckpt is not None:
            load_weights(model, load_lightning_checkpoint(ckpt)["state_dict"])
    if isinstance(args.max_targets, dict):
        unknown = set(args.max_targets) - set(models) - {None}
        if unknown:
            raise SystemExit(f"--max_targets: no class named {sorted(unknown)}; the classes are {list(models)}")
    if len(cfgs) == 1:
        name = cfgs[0].category_name
        out = run(models[name], data[name], args.out, max_targets=class_targets(args.max_targets, name), max_points=args.max_points,
                  seed=args.seed, precision=args.precision, **rule)
        out.update({"checkpoint": args.checkpoint, "split": args.split, "out": args.out})
    else:
        out = run_classes(models, data, args.out, {c: class_targets(args.max_targets, c) for c in models},
                          max_points=args.max_points, seed=args.seed, precision=args.precision, **rule)
        out.update({"checkpoint": [c for _, c in classes], "split": args.split, "out": args.out})
    print(json.dumps(out), flush=True)
    return out


if __name__ == "__main__":
    main(sys.argv[1:])
