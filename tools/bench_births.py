"""Cost of starting targets on the device in the live tracker (MultiTargetTracker's `births=`), and of the host loop it replaces.

  python tools/bench_births.py [--replays 2000] [--steps 20] [--warmup 3] [--reps 3] [--loop_steps 12] [--out results.json]

  * "kernel": `o3d_track_birth` alone, captured in a CUDA graph with a reset of the matching's records in front of it (so every
    replay sees the same candidates), timed with CUDA events over --replays replays, for F = 1 and 16 feeds, D = 64 / 256 /
    1024 detections per feed spread over 80 m (none matched, score uniform in [0, 1), min_score 0.5), 32 advancing rows per
    feed, per_scan 8 (R = 8 F reserved slots), gate 2 m.  The reset alone is timed too;
  * "step": BAT-Car (untrained weights: the timing does not depend on them) at K = 8, 32 and 128, every slot active, one feed
    of 60,000-point synthetic scans with 64 detections each, detections=(64, 2.0) without and with births=(0.5, 4); with every
    slot taken no slot is reserved, so "births" is the cost of the step's birth stage (kernel and first-frame crop over R
    rows) when nothing is born.  The two settings alternate in one process, --steps CUDA-event-timed advances each after
    --warmup, --reps times;
  * "loop": a detection-driven online loop, F = 1, 4 and 16 feeds of 60,000-point synthetic scenes (6 objects each) put through
    put_raw as (n, 4) float32 rows, with detections from the ground truth: centre noise N(0, 0.2 m), each dropped with
    probability 0.2, and 2 false positives per scan.  BAT-Car, K = 8 F, detections=(16, 2.0); every target is dropped 8
    advances after the host learns of it.  "births": births=(0.5, 2) and births() after every advance (no sync); "add":
    unmatched() after every advance (one sync), then add() of up to 2 unmatched detections per feed scoring >= 0.5, in score
    order.  Host clock over --loop_steps advances after 2 warm-up advances, ending with a synchronize: scans/s and ms per
    advance.
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

from bench_associate import _step_detections  # noqa: E402
from bench_coast import _model  # noqa: E402
from bench_multi_target import gpu_info, timed  # noqa: E402
from open3dsot_b200.datasets.data_classes import Box  # noqa: E402
from open3dsot_b200.datasets.synthetic import synthetic_scene  # noqa: E402
from open3dsot_b200.tracking.multi_tracker import (BirthSlots, MultiTargetTracker, detection_gate2, detection_rows,  # noqa: E402
                                                   track_birth)


# ------------------------------------------------------------------ the kernel alone
def bench_kernel(replays):
    rows = []
    g = np.random.default_rng(0)
    dev = "cuda"
    for F in (1, 16):
        for D in (64, 256, 1024):
            b, per = 32 * F, 8
            K = max(b, per * F) + per * F
            R = per * F
            Rw = K + 2
            z = lambda *s, d=torch.float32: torch.zeros(*s, dtype=d, device=dev)
            slots = BirthSlots(z(Rw, 3), z(Rw, 3), z(Rw, 3, 3), z(Rw), z(Rw, d=torch.bool), z(Rw, d=torch.int64),
                               z(Rw, d=torch.int64), z(Rw, d=torch.int64), z(Rw, d=torch.int32), z(Rw), z(Rw, d=torch.int32),
                               z(Rw, d=torch.bool), z(Rw, 3), z(Rw, 3), z(Rw, d=torch.int64), z(Rw, d=torch.bool),
                               z(Rw, d=torch.int32), z(Rw, d=torch.bool))
            feed = torch.arange(b, device=dev) % F
            adv = torch.ones(b, dtype=torch.bool, device=dev)
            pred = torch.from_numpy(g.uniform(-40, 40, (b, 3)).astype(np.float32)).to(dev)
            det = g.uniform(-40, 40, (F, D, 16)).astype(np.float32)
            det[..., 15] = g.random((F, D))
            det = torch.from_numpy(det).to(dev)
            fed = torch.ones(F, dtype=torch.int64, device=dev)
            count = torch.full((F,), D, dtype=torch.int32, device=dev)
            rec0 = torch.full((F, D), -1, dtype=torch.int32, device=dev)
            rec = rec0.clone()
            bl = torch.tensor([list(range(b, b + R)), [f for f in range(F) for _ in range(per)]], device=dev)
            nxt = z(1, d=torch.int64)
            log = z(R, 4, d=torch.int64)

            def run():
                rec.copy_(rec0)
                track_birth(feed, adv, pred, fed, count, det, rec, bl, nxt, log, slots, detection_gate2(2.0), (0, 1), 0.5)
            run()
            torch.cuda.synchronize()
            born = int((log[:, 3] >= 0).sum())
            graphs = {}
            for name, fn in (("with_reset", run), ("reset", lambda: rec.copy_(rec0))):
                graphs[name] = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graphs[name]):
                    fn()
                graphs[name].replay()
            torch.cuda.synchronize()
            us = {n: timed(lambda i, gr=gr: gr.replay(), replays) * 1e3 / replays for n, gr in graphs.items()}
            row = {"F": F, "D": D, "rows_per_feed": 32, "R": R, "born": born, "us_with_reset": us["with_reset"],
                   "us_reset": us["reset"]}
            rows.append(row)
            print(json.dumps({"kernel": row}), flush=True)
    return rows


# ------------------------------------------------------------------ step time
def bench_step(steps, warmup, reps):
    out = []
    net = _model("BAT_Car.yaml").eval()
    rng = np.random.default_rng(0)
    for K in (8, 32, 128):
        sc = synthetic_scene(n_frames=8, n_points=60_000, n_objects=min(K, 32), seed=11, extent=60.0)
        scans = [torch.from_numpy(s).cuda() for s in sc["scans"]]
        dets = [_step_detections(sc, t, 64, 60.0, rng) for t in range(8)]
        trks = {}
        for s, kw in (("off", {}), ("births", {"births": (0.5, 4)})):
            trk = MultiTargetTracker(net, 60_000, K, seed=0, lost=(5, 10), coast=0.5, detections=(64, 2.0), **kw)
            feed = (lambda t, trk=trk: trk.put(0, scans[t], detections=dets[t]))
            trk.put(0, scans[0])
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


# ------------------------------------------------------------------ the online loop
def _loop_data(F, frames, seed=0):
    rng = np.random.default_rng(seed)
    feeds = []
    for f in range(F):
        sc = synthetic_scene(n_frames=frames, n_points=60_000, n_objects=6, seed=3000 + f, extent=40.0)
        scans = [np.concatenate([s, rng.random((len(s), 1), dtype=np.float32)], 1) for s in sc["scans"]]
        dets = []
        for t in range(frames):
            boxes = [sc["boxes"][o][t] for o in range(6) if rng.random() >= 0.2]
            rows = detection_rows(boxes, rng.uniform(0.5, 1.0, len(boxes)))
            rows[:, :3] += rng.normal(0, 0.2, (len(rows), 3)).astype(np.float32)
            fp = detection_rows([Box(np.append(rng.uniform(-40, 40, 2), 0.0), np.array([1.8, 4.2, 1.6]), np.eye(3))
                                 for _ in range(2)], rng.uniform(0.1, 0.7, 2))
            dets.append(np.concatenate([rows, fp]))
        feeds.append((scans, dets))
    return feeds


def _online(net, data, mode, steps, warmup=2, age=8, per=2, min_score=0.5):
    F = len(data)
    K = 8 * F
    kw = {"births": (min_score, per)} if mode == "births" else {}
    trk = MultiTargetTracker(net, 60_000, K, seed=0, feeds=F, detections=(16, 2.0), **kw)
    known, nxt, n_born = {}, 0, 0                                              # id -> advance the host learned of it
    t0 = None
    for s in range(warmup + steps):
        if s == warmup:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
        for f, (scans, dets) in enumerate(data):
            trk.put_raw(f, scans[s], detections=dets[s])
        trk.advance()
        if mode == "births":
            new = [tid for tid, *_ in trk.births()]
        else:
            new = []
            for f, um in trk.unmatched().items():
                um = sorted(um, key=lambda u: (-u[2], u[0]))
                for _, box, score in [u for u in um if u[2] >= min_score][:per]:
                    if len(trk.targets()) >= K:
                        break
                    trk.add(nxt, box, feed=f)
                    new.append(nxt)
                    nxt += 1
        n_born += len(new)
        for tid in new:
            known[tid] = s
        for tid in [t for t, s0 in known.items() if s - s0 >= age]:
            trk.drop(tid)
            del known[tid]
    torch.cuda.synchronize()
    sec = time.perf_counter() - t0
    return {"scans_per_s": F * steps / sec, "ms_per_advance": sec * 1e3 / steps, "targets_started": n_born}


def bench_loop(steps, reps):
    out = []
    net = _model("BAT_Car.yaml").eval()
    for F in (1, 4, 16):
        data = _loop_data(F, steps + 2)
        res = {m: [] for m in ("births", "add")}
        for _ in range(reps):
            for m in res:
                res[m].append(_online(net, data, m, steps))
        row = {"F": F, **res}
        out.append(row)
        print(json.dumps({"loop": row}), flush=True)
        del data
        torch.cuda.empty_cache()
    return out


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--replays", type=int, default=2000)
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--reps", type=int, default=3)
    p.add_argument("--loop_steps", type=int, default=12)
    p.add_argument("--skip", nargs="*", default=(), choices=("kernel", "step", "loop"))
    p.add_argument("--out", default=None)
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_births: needs a CUDA device")
    res = {"gpu": gpu_info()}
    print(f"GPU: {res['gpu']}", flush=True)
    if "kernel" not in a.skip:
        res["kernel"] = bench_kernel(a.replays)
    if "step" not in a.skip:
        res["step"] = bench_step(a.steps, a.warmup, a.reps)
    if "loop" not in a.skip:
        res["loop"] = bench_loop(a.loop_steps, a.reps)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
