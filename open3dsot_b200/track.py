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
draws are keyed by its tracklet's index in the split, as `evaluate_batched` keys them by default."""
import argparse
import json
import sys

import numpy as np


def parse_args(argv=None):
    p = argparse.ArgumentParser(prog="python -m open3dsot_b200.track")
    p.add_argument('--cfg', type=str, required=True, help='the config file')
    p.add_argument('--checkpoint', type=str, default=None, help='weights (a checkpoint of ours or of the reference)')
    p.add_argument('--path', type=str, required=True, help='dataset root (for KITTI: velodyne/, label_02/, calib/)')
    p.add_argument('--split', type=str, default='test', help='scene split (train / valid / test / *_tiny)')
    p.add_argument('--out', type=str, default='results.jsonl', help='per-frame results, one JSON line per (scene, frame)')
    p.add_argument('--max_targets', type=int, default=64, help='tracker slots (targets in flight at once)')
    p.add_argument('--max_points', type=int, default=None, help='scan buffer size (default: the largest scan streamed)')
    p.add_argument('--seed', type=int, default=0, help='key of the random draws')
    p.add_argument('--precision', choices=('fp32', 'bf16'), default='fp32',
                   help='operand precision of the tensor-core layers (bf16: BF16 operands, FP32 accumulation)')
    return p.parse_args(argv)


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


def stream_max_points(dataset, plan):
    """The largest scan of the planned streams (`dataset.scan_size`: from the file sizes where the format allows)."""
    return max([1] + [dataset.scan_size(p["scene"], f) for p in plan for f in p["frames"]])


def _yaw(rot, up_axis):
    """Heading about the up axis: atan2 of the box's x axis in the ground plane (KITTI's rotation_y in camera coordinates)."""
    if up_axis[1] != 0:
        return float(np.arctan2(-rot[2, 0], rot[0, 0]))
    return float(np.arctan2(rot[1, 0], rot[0, 0]))


def run(model, dataset, out_path, max_targets=64, max_points=None, seed=0, precision="fp32"):
    """Track every scene of `dataset`'s split and write `out_path`; returns {"success", "precision", "frames", "scenes"}."""
    from .tracking.multi_tracker import track_feeds
    from .utils.metrics import Precision, Success, estimateAccuracy, estimateOverlap

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
    results = track_feeds(model, scenes, max(1, min(len(scenes), max_targets)), max_targets, seed=seed, max_points=max_points,
                          precision=precision)
    overlaps, distances = [[] for _ in annos], [[] for _ in annos]
    with open(out_path, "w") as f:
        for p, res in zip(plan, results):
            scene, pos = p["scene"], {fr: t for t, fr in enumerate(p["frames"])}
            track_id = {tr["index"]: tr["track_id"] for tr in p["tracklets"]}
            for t, frame in enumerate(p["frames"]):
                targets = [{"id": track_id[j], "tracklet": j, "center": b[t].center.tolist(), "wlh": b[t].wlh.tolist(),
                            "yaw": _yaw(b[t].rotation_matrix, up)} for j, b in sorted(res.items()) if t in b]
                f.write(json.dumps({"scene": scene, "frame": frame, "targets": targets}) + "\n")
            for tr in p["tracklets"]:
                j = tr["index"]
                for i, anno in enumerate(annos[j]):
                    gt = dataset.box_from_anno(anno)
                    box = gt if i == 0 else res[j][pos[dataset.anno_frame(anno)[1]]]
                    overlaps[j].append(estimateOverlap(gt, box, dim=dim, up_axis=up))
                    distances[j].append(estimateAccuracy(gt, box, dim=dim, up_axis=up))
    succ, prec = Success(), Precision()
    for j in range(len(annos)):
        succ(overlaps[j])
        prec(distances[j])
    return {"success": succ.compute(), "precision": prec.compute(), "frames": sum(len(o) for o in overlaps), "scenes": len(plan)}


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
    cfg = load_config(args.cfg)
    data = reader(cfg, args.path, args.split)
    torch.manual_seed(0)
    model = get_model(cfg.net_model)(cfg).cuda()
    if args.checkpoint is not None:
        load_weights(model, load_lightning_checkpoint(args.checkpoint)["state_dict"])
    out = run(model, data, args.out, max_targets=args.max_targets, max_points=args.max_points, seed=args.seed,
              precision=args.precision)
    out.update({"checkpoint": args.checkpoint, "split": args.split, "out": args.out})
    print(json.dumps(out), flush=True)
    return out


if __name__ == "__main__":
    main(sys.argv[1:])
