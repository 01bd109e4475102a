"""Split evaluation throughput: `evaluate_batched`'s device tracker with K slots against the B=1 DeviceTracker and the host
`evaluate()` loop, on seeded synthetic tracklets (60,000 points per scan, as bench.py --track; lengths spread from 10 to 200
frames).  Prints one JSON line: frames/s of the whole evaluation per slot count (device events around every admission and
graph replay of the chunk), the B=1 DeviceTracker over the same tracklets (graph replay, one reset per tracklet), the host
`evaluate()` loop on a subset, and the card's name and power limit.  Frames counted are the tracked frames (frame 0 of a
tracklet is its ground truth and needs no network).
--shape-aggregation / --reference-bb override the config's template and reference-box modes.  With shape_aggregation 'all'
each slot count is first run once through `run()` (capture, warm-up and any growth of the history), then timed; the result
also gives the history's size at the end of the chunk and, at the largest slot count, the device time of one
o3d_crop_append (every slot appends a frame) and of one template resampling over the K x H history, against the step's time.

    python tools/bench_track_batched.py [--cfg BAT_Car.yaml] [--tracklets 144] [--points 60000] [--slots 1,8,32,64,128]
                                        [--shape-aggregation all] [--reference-bb previous_gt]"""
import argparse
import gc
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from open3dsot_b200.config import load_config  # noqa: E402
from open3dsot_b200.datasets.synthetic import synthetic_sequence  # noqa: E402
from open3dsot_b200.models import get_model  # noqa: E402
from open3dsot_b200.tracking import boxes as bx  # noqa: E402
from open3dsot_b200.tracking.batched_tracker import BatchedDeviceTracker  # noqa: E402
from open3dsot_b200.tracking.device_tracker import DeviceTracker, tracking_modes  # noqa: E402
from open3dsot_b200.tracking.evaluate import evaluate  # noqa: E402
from open3dsot_b200.tracking.sampling import resample_batched  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        name, power = (s.strip() for s in out[0].split(","))
        return name, power
    except Exception as e:                                     # the numbers stay usable without the label
        return f"unknown ({e.__class__.__name__})", "unknown"


def time_op(fn, iters=50):
    """Device milliseconds per call of `fn` (events around `iters` calls after two warm-up calls)."""
    for _ in range(2):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def history_ops(trk):
    """Per-step device time of the 'all' template's two history kernels at the tracker's K and H, on the histories the
    chunk left behind: the append of one frame per slot (on copies, so the histories stay as they are) and the resampling."""
    cfg, P, K = trk.cfg, trk.pool, trk.K
    frame = P.prev[torch.arange(K, device=P.scans.device) % P.num_frames]
    box = bx.Box(trk.box_c, trk.box_s, trk.box_r)
    hist, keep, count = trk.hist.clone(), trk.hist_keep.clone(), trk.hist_count.clone()

    def append():
        count.copy_(trk.hist_count)
        bx.crop_append(P.scans, box, cfg.model_bb_scale, cfg.model_bb_offset, frame, P.count, hist, keep, count)
    ms_append = time_op(append)
    ms_resample = time_op(lambda: resample_batched(trk.hist, trk.hist_keep, cfg.template_size, *trk.u_t))
    # the same resampling with every slot's history at 200 frames of ~700 points (the synthetic car's crop): a 200-frame
    # tracklet tracked on the object all along; an untrained network loses it after a few frames and leaves short histories
    counts = trk.hist_count.cpu().numpy()
    full = min(trk.H, 200 * 700)
    keep_full = torch.zeros_like(trk.hist_keep)
    keep_full[:, :full] = True
    ms_full = time_op(lambda: resample_batched(trk.hist, keep_full, cfg.template_size, *trk.u_t))
    return {"crop_append_ms": ms_append, "template_resample_ms": ms_resample, "H": trk.H,
            "history_points_mean": float(counts.mean()), "history_points_max": int(counts.max()),
            "template_resample_full_ms": ms_full, "full_history_points": full}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--cfg", default="BAT_Car.yaml")
    ap.add_argument("--tracklets", type=int, default=144)
    ap.add_argument("--points", type=int, default=60000)
    ap.add_argument("--slots", default="1,8,32,64,128")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--host-tracklets", type=int, default=2, help="tracklets (the shortest) of the host evaluate() subset")
    ap.add_argument("--shape-aggregation", default=None, help="override the config's shape_aggregation (e.g. all)")
    ap.add_argument("--reference-bb", default=None, help="override the config's reference_BB (previous_gt, current_gt)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_track_batched.py measures the GPU and needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    over = {"up_axis": [0, 0, 1]}
    if args.shape_aggregation:
        over["shape_aggregation"] = args.shape_aggregation
    if args.reference_bb:
        over["reference_BB"] = args.reference_bb
    cfg = load_config(os.path.join(ROOT, "cfgs", args.cfg), over)
    torch.manual_seed(0)
    net = get_model(cfg.net_model)(cfg).to(dev).eval()

    rng = np.random.default_rng(20261016)
    lengths = np.exp(rng.uniform(np.log(10), np.log(200), args.tracklets)).round().astype(int)
    lengths[:2] = (10, 200)                                     # both ends of the spread
    t0 = time.perf_counter()
    tracks = [synthetic_sequence(n_frames=int(n), n_points=args.points, seed=1000 + i, speed=0.3 + 0.4 * rng.random(),
                                 yaw_rate=4 * rng.random() - 2) for i, n in enumerate(lengths)]
    gen_s = time.perf_counter() - t0
    tracked = int(sum(n - 1 for n in lengths))
    res = {}
    for k in [int(s) for s in args.slots.split(",")]:
        trk = BatchedDeviceTracker(net, tracks, k, seed=args.seed, max_points=args.points)
        if trk.mode == "all":
            trk.run()                                            # the history's capacity settles on the first run
        else:
            trk._capture()                                       # capture + warm-up outside the timed window
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t = time.perf_counter()
        e0.record()
        trk.track()
        e1.record()
        torch.cuda.synchronize()
        wall = time.perf_counter() - t
        dev_s = e0.elapsed_time(e1) * 1e-3
        res[f"slots_{k}"] = {"frames_per_s": tracked / max(dev_s, wall), "device_s": dev_s, "wall_s": wall,
                             "steps": trk.plan["steps"], "slots_used": trk.plan["slots"]}
        if trk.mode == "all":
            res[f"slots_{k}"]["step_ms"] = dev_s * 1e3 / trk.plan["steps"]
            if k == int(args.slots.split(",")[-1]):
                res[f"slots_{k}"]["history_kernels"] = history_ops(trk)
        pool = trk.pool
        del trk
        if k != int(args.slots.split(",")[-1]):
            del pool
        gc.collect()
        torch.cuda.empty_cache()

    # B=1 DeviceTracker over the same tracklets: one captured frame, re-used across tracklets (reset only refills buffers)
    back = {"previous_gt": 1, "current_gt": 0}.get(tracking_modes(net)[1])
    ref = (lambda f: None) if back is None else (lambda f: pool.box(f - back))     # pool frame f's reference box
    offsets = np.concatenate([[0], np.cumsum(lengths)[:-1]])
    one = DeviceTracker(net, max_points=args.points)
    for j in range(2):                                          # warm-up and capture
        o = int(offsets[j])
        one.reset(pool.scans[o], tracks[j][0]["3d_bbox"].to_tensor(dev))
        for i in range(1, 4):
            one.step(pool.scans[o + i], n_valid=tracks[j][i]["pc"].points.shape[1], ref_box=ref(o + i))
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t = time.perf_counter()
    e0.record()
    for j, seq in enumerate(tracks):
        o = int(offsets[j])
        one.reset(pool.scans[o], seq[0]["3d_bbox"].to_tensor(dev))
        for i in range(1, len(seq)):
            one.step(pool.scans[o + i], n_valid=seq[i]["pc"].points.shape[1], ref_box=ref(o + i))
    e1.record()
    torch.cuda.synchronize()
    wall = time.perf_counter() - t
    dev_s = e0.elapsed_time(e1) * 1e-3
    res["device_tracker_b1"] = {"frames_per_s": tracked / max(dev_s, wall), "device_s": dev_s, "wall_s": wall}

    # the host evaluate() loop (one B=1 forward per frame, host metrics) on the shortest tracklets
    sub = [tracks[j] for j in np.argsort(lengths, kind="stable")[: args.host_tracklets]]
    evaluate(net, sub[:1])                                       # warm-up
    torch.cuda.synchronize()
    t = time.perf_counter()
    evaluate(net, sub)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t
    res["evaluate_host_loop"] = {"frames_per_s": sum(len(s) - 1 for s in sub) / wall, "wall_s": wall, "tracklets": len(sub)}

    name, power = card()
    best = max((v["frames_per_s"], k) for k, v in res.items() if k.startswith("slots_"))
    print(json.dumps({"metric": f"split evaluation frames/s, {cfg.net_model}, {args.tracklets} synthetic tracklets of "
                                f"{int(lengths.min())}-{int(lengths.max())} frames, {args.points} points per scan",
                      "shape_aggregation": cfg.get("shape_aggregation"), "reference_BB": cfg.get("reference_BB"),
                      "value": best[0], "best": best[1], "unit": "frames/s", "tracked_frames": tracked,
                      "results": res, "gpu": name, "power_limit": power, "tracklet_generation_s": gen_s}))


if __name__ == "__main__":
    main()
