"""Cost and effect of detection matching in the live tracker (MultiTargetTracker's `detections=`).

  python tools/bench_associate.py [--replays 2000] [--steps 20] [--warmup 3] [--reps 3] [--epochs 40] [--out results.json]

  * "kernel": `o3d_box_associate` alone, captured in a CUDA graph and timed with CUDA events over --replays replays, for F = 1 and
    16 feeds, 8 / 32 / 128 advancing rows per feed and D = 64 / 256 / 1024 detections per feed, half of them within 0.5 m of a
    row's box (the rest spread over 40 m), gate 2 m, rule and coast on;
  * "step": BAT-Car (untrained weights: the timing does not depend on them) at K = 8, 32 and 128, every slot active, one feed
    of 60,000-point synthetic scans, lost=(5, 10) + coast=0.5, without detections and with detections=(64, 2.0) given 64
    detections per scan (the objects' boxes, the rest spread over the scene); the two settings alternated in one process,
    --steps CUDA-event-timed advances each after --warmup, --reps times;
  * "occlusion": tools/bench_coast.py's study (BAT-Car trained for --epochs seeded epochs on synthetic tracklets; object 0 of
    24 synthetic scenes loses every point within 4 m of its centre for g = 1, 2 and 4 frames from frame 10), tracked with
    lost=(3, 6) + coast=0.5 without and with detections=(64, 2.0).  Detections come from the ground truth of the visible
    objects (object 0 has none on its gap frames): centre noise N(0, 0.1 m) per axis, each dropped with probability 0.2, and
    2 false positives per scan placed uniformly over the scene.  Reported: Success / Precision over every target-frame,
    the share of occluded targets re-acquired (a frame with >= 3 points in the box and a centre within 1 m of the truth among
    the 3 frames after the gap, bench_coast's definition), and the mean centre error over those 3 frames.  Synthetic data
    only, with the same 40-epoch model.
The card's name and power limit are printed with the numbers."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_coast import _model, _scenes, _train  # noqa: E402
from bench_multi_target import gpu_info, timed  # noqa: E402
from open3dsot_b200 import ops  # noqa: E402
from open3dsot_b200.datasets.data_classes import Box  # noqa: E402
from open3dsot_b200.datasets.synthetic import synthetic_scene  # noqa: E402
from open3dsot_b200.tracking.multi_tracker import MultiTargetTracker, Slots, detection_gate2, detection_rows, track_feeds  # noqa: E402


# ------------------------------------------------------------------ the kernel alone
def bench_kernel(replays):
    rows = []
    g = np.random.default_rng(0)
    for F in (1, 16):
        for per_feed in (8, 32, 128):
            for D in (64, 256, 1024):
                b = F * per_feed
                K = b
                R = K + 2
                dev = "cuda"
                slots = Slots(*(x.to(dev) for x in (torch.zeros(R, 3), torch.eye(3).repeat(R, 1, 1), torch.full((R,), 5),
                                                    torch.zeros(R), torch.zeros(R, dtype=torch.int32), torch.zeros(R),
                                                    torch.zeros(R, dtype=torch.int32), torch.zeros(R, dtype=torch.bool),
                                                    torch.zeros(R, 3), torch.zeros(R, 3), torch.full((R,), 3),
                                                    torch.zeros(R, dtype=torch.bool))))
                src = torch.from_numpy(g.permutation(K)).to(dev)
                feed = torch.arange(b, device=dev) % F
                adv = torch.ones(b, dtype=torch.bool, device=dev)
                center = torch.from_numpy(g.uniform(-20, 20, (b, 3)).astype(np.float32)).to(dev)
                points = torch.from_numpy(g.integers(0, 10, b).astype(np.int32)).to(dev)
                det = g.uniform(-20, 20, (F, D, 16)).astype(np.float32)
                c = center.cpu().numpy()
                for f in range(F):
                    mine = c[f::F]
                    near = g.random(D) < 0.5
                    det[f, near, :3] = mine[g.integers(0, len(mine), near.sum())] + g.normal(0, 0.3, (near.sum(), 3))
                det = torch.from_numpy(det).to(dev)
                fed = torch.ones(F, dtype=torch.int64, device=dev)
                count = torch.full((F,), D, dtype=torch.int32, device=dev)
                rec = (torch.zeros(F, D, 16, device=dev), torch.zeros(F, dtype=torch.int32, device=dev),
                       torch.zeros(F, D, dtype=torch.int32, device=dev))
                run = lambda: ops.box_associate(src, feed, adv, center, points, slots, fed, count, det, rec, detection_gate2(2.0),
                                                (0, 1), (5, 10), True)
                _, match, _ = run()
                torch.cuda.synchronize()
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph):
                    run()
                graph.replay()
                torch.cuda.synchronize()
                us = timed(lambda i: graph.replay(), replays) * 1e3 / replays
                row = {"F": F, "rows_per_feed": per_feed, "D": D, "us": us, "matched": int((match >= 0).sum())}
                rows.append(row)
                print(json.dumps({"kernel": row}), flush=True)
    return rows


# ------------------------------------------------------------------ step time
def _step_detections(sc, t, n, extent, rng):
    boxes = [sc["boxes"][o][t] for o in range(len(sc["boxes"]))][:n]
    while len(boxes) < n:
        boxes.append(Box(np.append(rng.uniform(-extent, extent, 2), 0.0), np.array([1.8, 4.2, 1.6]), np.eye(3)))
    return detection_rows(boxes, rng.random(n))


def bench_step(steps, warmup, reps):
    out = []
    net = _model("BAT_Car.yaml").eval()
    rng = np.random.default_rng(0)
    for K in (8, 32, 128):
        sc = synthetic_scene(n_frames=8, n_points=60_000, n_objects=min(K, 32), seed=11, extent=60.0)
        scans = [torch.from_numpy(s).cuda() for s in sc["scans"]]
        dets = [_step_detections(sc, t, 64, 60.0, rng) for t in range(8)]
        trks = {}
        for s, kw in (("off", {}), ("detections", {"detections": (64, 2.0)})):
            trk = trks[s] = MultiTargetTracker(net, 60_000, K, seed=0, lost=(5, 10), coast=0.5, **kw)
            feed = (lambda t, trk=trk, on=bool(kw): trk.put(0, scans[t], **({"detections": dets[t]} if on else {})))
            feed(0)
            trk.advance()
            for j in range(K):
                trk.add(j, sc["boxes"][j % len(sc["boxes"])][0])
            for i in range(warmup):
                feed(1 + i % 7)
                trk.advance()
            trks[s] = (trk, feed)
        torch.cuda.synchronize()
        ms = {s: [] for s in trks}
        for _ in range(reps):
            for s, (trk, feed) in trks.items():
                ms[s].append(timed(lambda i: (feed(1 + i % 7), trk.advance()), steps) / steps)
        row = {"model": "bat_car", "K": K, **{f"{s}_ms": v for s, v in ms.items()}}
        out.append(row)
        print(json.dumps({"step": row}), flush=True)
        del trks, scans
        torch.cuda.empty_cache()
    return out


# ------------------------------------------------------------------ occlusion accuracy with detections
def _with_detections(scenes, truth, g, t0, seed, extent=20.0):
    """Each scene's "detections": the visible objects' ground truth (object 0 hidden on its gap frames), centre noise
    N(0, 0.1 m), each dropped with probability 0.2, and 2 uniform false positives per scan; drawn once, seeded."""
    rng = np.random.default_rng(seed)
    for sc, tr in zip(scenes, truth):
        table = []
        for t in range(sc["frames"]):
            boxes = [b[t] for tid, b in sorted(tr.items()) if not (tid % 10 == 0 and t0 <= t < t0 + g)]
            boxes = [b for b in boxes if rng.random() >= 0.2]
            rows = detection_rows(boxes, rng.uniform(0.5, 1.0, len(boxes)))
            rows[:, :3] += rng.normal(0, 0.1, (len(rows), 3)).astype(np.float32)
            fp = detection_rows([Box(np.append(rng.uniform(-extent, extent, 2), 0.0), np.array([1.8, 4.2, 1.6]), np.eye(3))
                                 for _ in range(2)], rng.uniform(0.1, 0.6, 2))
            table.append(np.concatenate([rows, fp]))
        sc["detections"] = lambda t, table=table: table[t]
    return scenes


def bench_occlusion(net, lost=(3, 6), t0=10):
    from open3dsot_b200.utils.metrics import Precision, Success, estimateAccuracy, estimateOverlap
    out = []
    for g in (1, 2, 4):
        scenes, truth = _scenes(g, t0=t0)
        scenes = _with_detections(scenes, truth, g, t0, seed=g)
        row = {"gap": g}
        for s, kw in (("lost+coast", {}), ("lost+coast+detections", {"detections": (64, 2.0)})):
            res, ev = track_feeds(net, scenes if kw else [{k: v for k, v in sc.items() if k != "detections"} for sc in scenes], 8, 32,
                                  seed=0, max_points=20000, lost=lost, coast=0.5, evidence=True, **kw)
            succ, prec = Success(), Precision()
            after_err, reacquired, at_det = [], 0, 0
            for i, (r, e) in enumerate(zip(res, ev)):
                for tid, gt in truth[i].items():
                    boxes = r[tid]
                    o = [estimateOverlap(gt[t], boxes[t], dim=3, up_axis=[0, 0, 1]) if t in boxes else 0.0 for t in range(len(gt))]
                    d = [estimateAccuracy(gt[t], boxes[t], dim=3, up_axis=[0, 0, 1]) if t in boxes else float("inf")
                         for t in range(len(gt))]
                    succ(o)
                    prec(d)
                    if tid % 10 == 0:                                         # the occluded object
                        after = range(t0 + g, t0 + g + 3)
                        after_err += [d[t] for t in after if t in boxes]
                        reacquired += any(t in boxes and e[tid][t][0] >= lost[0] and d[t] < 1.0 for t in after)
                        at_det += sum(bool(e[tid][t][3]) for t in after if t in boxes and kw)
            row[s] = {"success": float(succ.compute()), "precision": float(prec.compute()),
                      "reacquired": reacquired / len(scenes), "after_gap_centre_error_m": float(np.mean(after_err)),
                      "after_gap_frames_scored": len(after_err), "reacquired_at_detection_frames": at_det}
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
    p.add_argument("--skip", nargs="*", default=(), choices=("kernel", "step", "occlusion"))
    p.add_argument("--out", default=None)
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_associate: needs a CUDA device")
    res = {"gpu": gpu_info()}
    print(f"GPU: {res['gpu']}", flush=True)
    if "kernel" not in a.skip:
        res["kernel"] = bench_kernel(a.replays)
    if "step" not in a.skip:
        res["step"] = bench_step(a.steps, a.warmup, a.reps)
    if "occlusion" not in a.skip:
        net, secs = _train(a.epochs)
        res["train"] = {"epochs": a.epochs, "seconds": secs, "seeds": "train 20260924 + i (48), scenes 7000 + i (24)"}
        res["occlusion"] = bench_occlusion(net)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
