"""Split evaluation throughput: `evaluate_batched`'s device tracker with K slots against the B=1 DeviceTracker and the host
`evaluate()` loop, on seeded synthetic tracklets (60,000 points per scan, as bench.py --track; lengths spread from 10 to 200
frames).  Prints one JSON line: frames/s of the whole evaluation per slot count (device events around every admission and
graph replay of the chunk), the B=1 DeviceTracker over the same tracklets (graph replay, one reset per tracklet), the host
`evaluate()` loop on a subset, and the card's name and power limit.  Frames counted are the tracked frames (frame 0 of a
tracklet is its ground truth and needs no network).

    python tools/bench_track_batched.py [--cfg BAT_Car.yaml] [--tracklets 144] [--points 60000] [--slots 1,8,32,64,128]"""
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
from open3dsot_b200.tracking.batched_tracker import BatchedDeviceTracker  # noqa: E402
from open3dsot_b200.tracking.device_tracker import DeviceTracker  # noqa: E402
from open3dsot_b200.tracking.evaluate import evaluate  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        name, power = (s.strip() for s in out[0].split(","))
        return name, power
    except Exception as e:                                     # the numbers stay usable without the label
        return f"unknown ({e.__class__.__name__})", "unknown"


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--cfg", default="BAT_Car.yaml")
    ap.add_argument("--tracklets", type=int, default=144)
    ap.add_argument("--points", type=int, default=60000)
    ap.add_argument("--slots", default="1,8,32,64,128")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--host-tracklets", type=int, default=2, help="tracklets (the shortest) of the host evaluate() subset")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_track_batched.py measures the GPU and needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    cfg = load_config(os.path.join(ROOT, "cfgs", args.cfg), {"up_axis": [0, 0, 1]})
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
        trk._capture()                                           # capture + warm-up outside the timed window
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
        pool = trk.pool
        del trk
        if k != int(args.slots.split(",")[-1]):
            del pool
        gc.collect()
        torch.cuda.empty_cache()

    # B=1 DeviceTracker over the same tracklets: one captured frame, re-used across tracklets (reset only refills buffers)
    offsets = np.concatenate([[0], np.cumsum(lengths)[:-1]])
    one = DeviceTracker(net, max_points=args.points)
    for j in range(2):                                          # warm-up and capture
        one.reset(pool.scans[int(offsets[j])], tracks[j][0]["3d_bbox"].to_tensor(dev))
        for i in range(1, 4):
            one.step(pool.scans[int(offsets[j]) + i], n_valid=tracks[j][i]["pc"].points.shape[1])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t = time.perf_counter()
    e0.record()
    for j, seq in enumerate(tracks):
        o = int(offsets[j])
        one.reset(pool.scans[o], seq[0]["3d_bbox"].to_tensor(dev))
        for i in range(1, len(seq)):
            one.step(pool.scans[o + i], n_valid=seq[i]["pc"].points.shape[1])
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
                      "value": best[0], "best": best[1], "unit": "frames/s", "tracked_frames": tracked,
                      "results": res, "gpu": name, "power_limit": power, "tracklet_generation_s": gen_s}))


if __name__ == "__main__":
    main()
