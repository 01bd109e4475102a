"""`python -m open3dsot_b200.track --cfg <yaml> --checkpoint <ckpt> --path <KITTI root> --split test --out results.jsonl`:
live multi-target tracking over KITTI scan streams (tracking/multi_tracker.py).

For every scene of the split, every velodyne scan from the first tracklet start to the last tracklet end is streamed, whole (no
`preload_offset` crop), in the config's `coordinate_mode`.  Every tracklet of `category_name` starts on its first annotated
frame from its ground-truth box and is dropped after its last annotated frame; nothing else of the ground truth is used.  One
JSON line per (scene, frame) lists every active target's box; Success / Precision over the annotated frames are printed, with
the host metric path of `tracking.evaluate` (the first frame of a tracklet scored against its own ground truth).  A target's
draws are keyed by its tracklet's index in the split, as `evaluate_batched` keys them by default."""
import argparse
import json
import os
import sys

import numpy as np


def parse_args(argv=None):
    p = argparse.ArgumentParser(prog="python -m open3dsot_b200.track")
    p.add_argument('--cfg', type=str, required=True, help='the config file')
    p.add_argument('--checkpoint', type=str, default=None, help='weights (a checkpoint of ours or of the reference)')
    p.add_argument('--path', type=str, required=True, help='KITTI tracking root (velodyne/, label_02/, calib/)')
    p.add_argument('--split', type=str, default='test', help='scene split (train / valid / test / *_tiny)')
    p.add_argument('--out', type=str, default='results.jsonl', help='per-frame results, one JSON line per (scene, frame)')
    p.add_argument('--max_targets', type=int, default=64, help='tracker slots (targets in flight at once)')
    p.add_argument('--max_points', type=int, default=None, help='scan buffer size (default: the largest scan streamed)')
    p.add_argument('--seed', type=int, default=0, help='key of the random draws')
    return p.parse_args(argv)


def scene_plan(dataset):
    """The streams of a split, in scene order: [{"scene", "first", "last", "tracklets": [{"index", "track_id", "start", "end",
    "frames"}]}] — `index` is the tracklet's index in the split (the reader's order), `frames` its annotated frames, and the
    stream runs over the scans first .. last."""
    plans = {}
    for j, annos in enumerate(dataset.tracklet_anno_list):
        scene = annos[0]["scene"]
        frames = [a["frame"] for a in annos]
        plans.setdefault(scene, []).append({"index": j, "track_id": annos[0]["track_id"], "start": frames[0], "end": frames[-1],
                                            "frames": frames})
    out = []
    for scene in dataset.scene_list:
        if scene in plans:
            tr = plans[scene]
            out.append({"scene": scene, "first": min(t["start"] for t in tr), "last": max(t["end"] for t in tr), "tracklets": tr})
    return out


def stream_max_points(dataset, plan):
    """The largest scan of the planned streams, from the file sizes (16 bytes per point)."""
    n = 1
    for p in plan:
        for f in range(p["first"], p["last"] + 1):
            path = dataset.scan_path(p["scene"], f)
            if os.path.isfile(path):
                n = max(n, os.path.getsize(path) // 16)
    return n


def _yaw(rot, up_axis):
    """Heading about the up axis: atan2 of the box's x axis in the ground plane (KITTI's rotation_y in camera coordinates)."""
    if up_axis[1] != 0:
        return float(np.arctan2(-rot[2, 0], rot[0, 0]))
    return float(np.arctan2(rot[1, 0], rot[0, 0]))


def run(model, dataset, out_path, max_targets=64, max_points=None, seed=0):
    """Track every scene of `dataset`'s split and write `out_path`; returns {"success", "precision", "frames", "scenes"}."""
    import torch

    from .tracking.multi_tracker import track_stream
    from .utils.metrics import Precision, Success, estimateAccuracy, estimateOverlap

    cfg = model.config
    dim, up = cfg.IoU_space, cfg.up_axis
    plan = scene_plan(dataset)
    if max_points is None:
        max_points = stream_max_points(dataset, plan)
    annos = dataset.tracklet_anno_list
    overlaps, distances = [[] for _ in annos], [[] for _ in annos]
    with open(out_path, "w") as f:
        for p in plan:
            scene, first = p["scene"], p["first"]
            starts, ends = {}, {}
            for tr in p["tracklets"]:
                starts.setdefault(tr["start"] - first, []).append((tr["index"], dataset.box_from_anno(annos[tr["index"]][0])))
                ends[tr["index"]] = tr["end"] - first
            scans = (torch.from_numpy(np.ascontiguousarray(dataset.read_scan(scene, fr).points[:3].T, dtype=np.float32))
                     for fr in range(first, p["last"] + 1))
            res = track_stream(model, scans, starts, ends, max_targets, seed=seed, max_points=max_points)
            track_id = {tr["index"]: tr["track_id"] for tr in p["tracklets"]}
            for t in range(p["last"] - first + 1):
                targets = [{"id": track_id[j], "tracklet": j, "center": b[t].center.tolist(), "wlh": b[t].wlh.tolist(),
                            "yaw": _yaw(b[t].rotation_matrix, up)} for j, b in sorted(res.items()) if t in b]
                f.write(json.dumps({"scene": scene, "frame": first + t, "targets": targets}) + "\n")
            for tr in p["tracklets"]:
                j = tr["index"]
                for i, anno in enumerate(annos[j]):
                    gt = dataset.box_from_anno(anno)
                    box = gt if i == 0 else res[j][anno["frame"] - first]
                    overlaps[j].append(estimateOverlap(gt, box, dim=dim, up_axis=up))
                    distances[j].append(estimateAccuracy(gt, box, dim=dim, up_axis=up))
    succ, prec = Success(), Precision()
    for j in range(len(annos)):
        succ(overlaps[j])
        prec(distances[j])
    return {"success": succ.compute(), "precision": prec.compute(), "frames": sum(len(o) for o in overlaps), "scenes": len(plan)}


def main(argv=None):
    import torch

    from .checkpoint import load_lightning_checkpoint
    from .config import load_config
    from .datasets.kitti import kittiDataset
    from .models import get_model
    from .trainer import load_weights

    args = parse_args(argv)
    cfg = load_config(args.cfg)
    if cfg.get("dataset", "kitti") != "kitti":
        raise SystemExit(f"dataset '{cfg.dataset}': live stream tracking reads KITTI's per-scene scan directories only")
    torch.manual_seed(0)
    model = get_model(cfg.net_model)(cfg).cuda()
    if args.checkpoint is not None:
        load_weights(model, load_lightning_checkpoint(args.checkpoint)["state_dict"])
    data = kittiDataset(args.path, args.split, category_name=cfg.category_name, coordinate_mode=cfg.coordinate_mode,
                        preloading=False, preload_offset=-1)
    out = run(model, data, args.out, max_targets=args.max_targets, max_points=args.max_points, seed=args.seed)
    out.update({"checkpoint": args.checkpoint, "split": args.split, "out": args.out})
    print(json.dumps(out), flush=True)
    return out


if __name__ == "__main__":
    main(sys.argv[1:])
