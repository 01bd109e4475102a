"""Cost and effect of coasting in the live tracker (MultiTargetTracker's `coast=`).

  python tools/bench_coast.py [--replays 2000] [--steps 20] [--warmup 3] [--reps 3] [--epochs 40] [--out results.json]

  * "write-back": the step's per-row write-back at buckets 1, 8, 32 and 128 (K = 128 slots, every row advancing, rule and coast
    on), once as the `o3d_track_update` kernel and once as its tensor formulation on CUDA (`track_update_tensors`), each captured
    on its own in a CUDA graph and timed with CUDA events over --replays replays;
  * "step": BAT-Car and M2-Track (untrained weights: the timing does not depend on them) at K = 1, 8, 32 and 128, every slot
    active, one feed of 60,000-point synthetic scans, in three settings (no rule, lost=(5, 10), lost=(5, 10) + coast=0.5), the
    settings alternated in one process, --steps CUDA-event-timed steps each after --warmup, --reps times;
  * "occlusion": BAT-Car trained with Trainer for --epochs seeded epochs on synthetic tracklets (the recipe of
    tools/bench_precision.py), then synthetic scenes (seeds 7000 + i) whose object 0 loses every point within 4 m of its centre
    for g = 1, 2 and 4 frames from frame 10, tracked with lost=(3, 6) alone and with coast=0.5: Success / Precision over every
    target-frame (frames after a loss score as failures), the share of occluded targets re-acquired (a frame with >= 3 points in
    the box and a centre within 1 m of the truth among the 3 frames after the gap), and the mean centre error over the gap frames.
    Synthetic data only: accuracy on KITTI / nuScenes weights is not measured here.
The card's name and power limit are printed with the numbers."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_multi_target import gpu_info, timed  # noqa: E402
from open3dsot_b200.config import load_config  # noqa: E402
from open3dsot_b200.datasets.synthetic import synthetic_scene, synthetic_sequence  # noqa: E402
from open3dsot_b200.models import get_model  # noqa: E402
from open3dsot_b200.tracking.multi_tracker import (MultiTargetTracker, Slots, coast_weights, track_feeds,  # noqa: E402
                                                   track_update, track_update_tensors)

MODELS = {"bat_car": "BAT_Car.yaml", "m2track": "M2_track_kitti.yaml"}
BUCKETS = (1, 8, 32, 128)
SETTINGS = {"none": {}, "lost": {"lost": (5, 10)}, "lost+coast": {"lost": (5, 10), "coast": 0.5}}
FAR = np.array([500.0, 500.0, -100.0], np.float32)


def _model(cfg_name, **over):
    cfg = load_config(os.path.join(ROOT, "cfgs", cfg_name), {"up_axis": [0, 0, 1], "degrees": True, **over})
    torch.manual_seed(0)
    return get_model(cfg.net_model)(cfg).cuda()


# ------------------------------------------------------------------ write-back
def bench_write_back(replays):
    K, rule, coast = 128, (5, 10), coast_weights(0.5)
    g = torch.Generator().manual_seed(0)
    rows = []
    for b in BUCKETS:
        row = {"bucket": b}
        for name, fn in (("kernel", track_update), ("tensors", track_update_tensors)):
            R = K + 2
            slots = Slots(torch.randn(R, 3), torch.randn(R, 3, 3), torch.randint(0, 9, (R,)), torch.zeros(R),
                          torch.randint(0, 50, (R,), dtype=torch.int32), torch.rand(R), torch.zeros(R, dtype=torch.int32),
                          torch.zeros(R, dtype=torch.bool), torch.randn(R, 3), torch.randn(R, 3), torch.zeros(R, dtype=torch.int64),
                          torch.zeros(R, dtype=torch.bool))
            slots = Slots(*(x.cuda() for x in slots))
            src = torch.randperm(K, generator=g)[:b].cuda()
            args = (src, src.clone(), torch.ones(b, dtype=torch.bool, device="cuda"), torch.randn(b, 3, device="cuda"),
                    torch.randn(b, 3, 3, device="cuda"), torch.randint(0, 10, (b,), dtype=torch.int32, device="cuda"),
                    torch.rand(b, device="cuda"))
            fn(slots, *args, rule, coast)                                     # warm-up outside the capture
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                fn(slots, *args, rule, coast)
            graph.replay()
            torch.cuda.synchronize()
            row[f"{name}_us"] = timed(lambda i: graph.replay(), replays) * 1e3 / replays
        rows.append(row)
        print(json.dumps({"write_back": row}), flush=True)
    return rows


# ------------------------------------------------------------------ step
def bench_step(steps, warmup, reps):
    out = []
    for name, cfg_name in MODELS.items():
        net = _model(cfg_name).eval()
        for K in BUCKETS:
            sc = synthetic_scene(n_frames=8, n_points=60_000, n_objects=min(K, 32), seed=11, extent=60.0)
            scans = [torch.from_numpy(s).cuda() for s in sc["scans"]]
            trks = {}
            for s, kw in SETTINGS.items():
                trk = trks[s] = MultiTargetTracker(net, 60_000, K, seed=0, **kw)
                trk.step(scans[0])
                for j in range(K):
                    trk.add(j, sc["boxes"][j % len(sc["boxes"])][0])
                for i in range(warmup):
                    trk.step(scans[1 + i % 7])
            torch.cuda.synchronize()
            ms = {s: [] for s in SETTINGS}
            for _ in range(reps):
                for s, trk in trks.items():
                    ms[s].append(timed(lambda i: trk.step(scans[1 + i % 7]), steps) / steps)
            row = {"model": name, "K": K, **{f"{s}_ms": v for s, v in ms.items()}}
            out.append(row)
            print(json.dumps({"step": row}), flush=True)
            del trks, scans
            torch.cuda.empty_cache()
    return out


# ------------------------------------------------------------------ occlusion accuracy
def _train(epochs):
    from open3dsot_b200.trainer import Trainer
    cfg_over = {"batch_size": 48, "epoch": 10 ** 6}
    net = _model("BAT_Car.yaml", **cfg_over)
    train = [synthetic_sequence(n_frames=20, n_points=20000, seed=20260924 + i) for i in range(48)]
    val = [synthetic_sequence(n_frames=20, n_points=20000, seed=1000 + i) for i in range(4)]
    tr = Trainer(net.train(), net.config, train, val, log_dir=None, slots=32)
    t0 = time.perf_counter()
    for _ in range(epochs):
        tr.train_epoch()
    return net.eval(), time.perf_counter() - t0


def _scenes(g, n_scenes=24, t0=10, frames=24, radius=4.0):
    scenes, truth = [], []
    for i in range(n_scenes):
        sc = synthetic_scene(n_frames=frames, n_points=20000, n_objects=4, seed=7000 + i, extent=20.0)
        scans = []
        for t, s in enumerate(sc["scans"]):
            s = s.copy()
            if t0 <= t < t0 + g:
                s[np.linalg.norm(s[:, :2] - sc["boxes"][0][t].center[None, :2], axis=1) < radius] = FAR
            scans.append(s)
        scenes.append({"frames": frames, "scan": (lambda t, s=scans: s[t]),
                       "starts": {0: [(10 * i + j, sc["boxes"][j][0]) for j in range(4)]}, "ends": {}})
        truth.append({10 * i + j: sc["boxes"][j] for j in range(4)})
    return scenes, truth


def bench_occlusion(net, lost=(3, 6), t0=10):
    from open3dsot_b200.utils.metrics import Precision, Success, estimateAccuracy, estimateOverlap
    out = []
    for g in (1, 2, 4):
        scenes, truth = _scenes(g, t0=t0)
        row = {"gap": g}
        for s, kw in (("lost", {}), ("lost+coast", {"coast": 0.5})):
            res, ev = track_feeds(net, scenes, 8, 32, seed=0, max_points=20000, lost=lost, evidence=True, **kw)
            succ, prec = Success(), Precision()
            gap_err, reacquired = [], 0
            for i, (r, e) in enumerate(zip(res, ev)):
                for tid, gt in truth[i].items():
                    boxes = r[tid]
                    o = [estimateOverlap(gt[t], boxes[t], dim=3, up_axis=[0, 0, 1]) if t in boxes else 0.0 for t in range(len(gt))]
                    d = [estimateAccuracy(gt[t], boxes[t], dim=3, up_axis=[0, 0, 1]) if t in boxes else float("inf")
                         for t in range(len(gt))]
                    succ(o)
                    prec(d)
                    if tid % 10 == 0:                                         # the occluded object
                        gap_err += [d[t] for t in range(t0, t0 + g)]
                        reacquired += any(t in boxes and e[tid][t][0] >= lost[0] and d[t] < 1.0
                                          for t in range(t0 + g, t0 + g + 3))
            row[s] = {"success": float(succ.compute()), "precision": float(prec.compute()),
                      "reacquired": reacquired / len(scenes), "gap_centre_error_m": float(np.mean(gap_err))}
        out.append(row)
        print(json.dumps({"occlusion": row}), flush=True)
    return out


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--replays", type=int, default=2000)
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--reps", type=int, default=3)
    p.add_argument("--epochs", type=int, default=40)
    p.add_argument("--skip", nargs="*", default=(), choices=("write_back", "step", "occlusion"))
    p.add_argument("--out", default=None)
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_coast: needs a CUDA device")
    res = {"gpu": gpu_info()}
    print(f"GPU: {res['gpu']}", flush=True)
    if "write_back" not in a.skip:
        res["write_back"] = bench_write_back(a.replays)
    if "step" not in a.skip:
        res["step"] = bench_step(a.steps, a.warmup, a.reps)
    if "occlusion" not in a.skip:
        net, secs = _train(a.epochs)
        res["train"] = {"epochs": a.epochs, "seconds": secs, "seeds": "train 20260924 + i (48), scenes 7000 + i (24)"}
        res["occlusion"] = bench_occlusion(net)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
