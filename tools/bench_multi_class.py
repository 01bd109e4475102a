"""Live tracking of two object classes over shared scan feeds: one MultiClassTracker against two MultiTargetTrackers.

  python tools/bench_multi_class.py [--points 60000] [--feeds 4] [--targets 32] [--frames 20] [--warmup 3] [--trace out.json]

A synthetic scene of car-sized and pedestrian-sized moving boxes (datasets/synthetic.py: synthetic_scene, once per class, the
scans joined) is replayed on every feed as raw nuScenes-like rows ((n, 5) float32 and two affine transforms, `put_raw`).  For
each model pair (BAT-Car + BAT-Pedestrian, BAT-Car + M2-Track), with --targets slots per class spread over the feeds:
  * "multi": one MultiClassTracker: one packed copy, one `o3d_scan_ingest` and one graph replay per step for both classes;
  * "separate": two MultiTargetTrackers, each ingesting every scan itself, advanced one after the other per step.
Reported per step: scans/s (feed-scans), target-frames/s (both classes), and host milliseconds per step (Python time spent in
put_raw + advance, timed in the same run).  CUDA-event times over --frames steps after --warmup untimed ones.  Weights are
untrained (the timing does not depend on them).  With --trace, one replay of the multi-class step is profiled
(torch.profiler) and the trace written there; the kernels' streams and the time two or more streams ran kernels at once are
printed.  The card's name and power limit are printed with the numbers."""
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

from bench_multi_target import _inverse, _xf, gpu_info, timed  # noqa: E402
from open3dsot_b200.config import load_config  # noqa: E402
from open3dsot_b200.datasets.synthetic import CAR_WLH, PED_WLH, synthetic_scene  # noqa: E402
from open3dsot_b200.models import get_model  # noqa: E402
from open3dsot_b200.tracking.multi_class import MultiClassTracker  # noqa: E402
from open3dsot_b200.tracking.multi_tracker import MultiTargetTracker  # noqa: E402

PAIRS = {"bat_car+bat_ped": ("BAT_Car.yaml", "BAT_Pedestrian.yaml"), "bat_car+m2track": ("BAT_Car.yaml", "M2_track_kitti.yaml")}


def model(name):
    # one frame convention for both classes (M2-Track's config reads its rotation in radians)
    cfg = load_config(os.path.join(ROOT, "cfgs", name), {"up_axis": [0, 0, 1], "degrees": True})
    torch.manual_seed(0)
    return get_model(cfg.net_model)(cfg).cuda().eval()


def scene(n_points, n_frames, per_class):
    car = synthetic_scene(n_frames=n_frames, n_points=n_points // 2, n_objects=per_class, seed=7, wlh=CAR_WLH, extent=70.0)
    ped = synthetic_scene(n_frames=n_frames, n_points=n_points - n_points // 2, n_objects=per_class, seed=8, wlh=PED_WLH,
                          n_object=150, extent=70.0)
    to_ego, to_global = _xf(0.3, (1.0, 0.0, 1.8)), _xf(-1.1, (400.0, 1100.0, 0.0))
    to_sensor = _inverse(to_ego) @ np.vstack([_inverse(to_global), [0, 0, 0, 1]])
    rows = []
    for a, b in zip(car["scans"], ped["scans"]):
        s = np.concatenate([a, b])
        r = np.zeros((s.shape[0], 5), np.float32)
        r[:, :3] = (s.astype(np.float64) @ to_sensor[:, :3].T + to_sensor[:, 3]).astype(np.float32)
        rows.append(r)
    return rows, (to_ego, to_global), {"car": car["boxes"], "ped": ped["boxes"]}


def run(kind, models, rows, xfs, boxes, F, K, warmup, frames):
    """Steps per second and host seconds per step; K slots per class, K // F targets per class on every feed."""
    N = rows[0].shape[0]
    if kind == "multi":
        trk = MultiClassTracker(models, N, {c: K for c in models}, feeds=F, seed=0)
        trackers, adds = [trk], [lambda c, i, b, f: trk.add(c, i, b, feed=f)]
    else:
        trackers = [MultiTargetTracker(models[c], N, K, seed=0, feeds=F) for c in models]
        adds = [lambda c, i, b, f, t=t: t.add(i, b, feed=f) for t in trackers]
    host = [0.0]

    def one(t):
        t0 = time.perf_counter()
        for trk in trackers:
            for f in range(F):
                trk.put_raw(f, rows[t], xfs)
            trk.advance()
        host[0] += time.perf_counter() - t0

    one(0)
    per_feed = K // F
    for n, c in enumerate(models):
        add = adds[0] if kind == "multi" else adds[n]
        for f in range(F):
            for j in range(per_feed):
                add(c, f * per_feed + j, boxes[c][j][0], f)
    for i in range(warmup):
        one(1 + i)
    torch.cuda.synchronize()
    host[0] = 0.0
    ms = timed(lambda i: one(1 + warmup + i), frames)
    return frames / (ms / 1e3), host[0] / frames, trackers[0]


def overlap(trace_path):
    """Kernel streams of a chrome trace and the microseconds during which kernels of two or more streams ran at once."""
    with open(trace_path) as f:
        ev = [e for e in json.load(f)["traceEvents"] if e.get("cat") == "kernel"]
    streams = sorted({e["args"].get("stream") for e in ev})
    marks = sorted([(e["ts"], 1, e["args"].get("stream")) for e in ev] + [(e["ts"] + e["dur"], -1, e["args"].get("stream"))
                                                                           for e in ev])
    live, both, last, span = {}, 0.0, None, (min(e["ts"] for e in ev), max(e["ts"] + e["dur"] for e in ev)) if ev else (0, 0)
    for ts, d, s in marks:
        if last is not None and sum(1 for v in live.values() if v > 0) >= 2:
            both += ts - last
        live[s] = live.get(s, 0) + d
        last = ts
    return {"kernels": len(ev), "streams": len(streams), "span_us": span[1] - span[0], "concurrent_us": both}


def main(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--points", type=int, default=60000)
    p.add_argument("--feeds", type=int, default=4)
    p.add_argument("--targets", type=int, default=32, help="slots per class (every slot active)")
    p.add_argument("--frames", type=int, default=20)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--trace", default=None, help="write a torch.profiler trace of one multi-class replay here")
    p.add_argument("--out", default=None, help="also write the results as JSON here")
    a = p.parse_args(argv)
    torch.cuda.set_device(0)
    info = gpu_info()
    print(f"# {info}; {a.points} points per scan, {a.feeds} feeds, {a.targets} slots per class; {a.frames} timed steps after "
          f"{a.warmup} warm-up steps", flush=True)
    rows, xfs, boxes = scene(a.points, 2 + a.warmup + a.frames, a.targets // a.feeds)
    results = {"gpu": info, "points": a.points, "feeds": a.feeds, "targets_per_class": a.targets, "rows": []}
    for pair, (c0, c1) in PAIRS.items():
        models = {"car": model(c0), "ped": model(c1)}
        for kind in ("multi", "separate"):
            sps, host, trk = run(kind, models, rows, xfs, boxes, a.feeds, a.targets, a.warmup, a.frames)
            active = 2 * (a.targets // a.feeds) * a.feeds
            row = {"pair": pair, "tracker": kind, "steps_per_s": sps, "scans_per_s": sps * a.feeds,
                   "target_frames_per_s": sps * active, "host_ms_per_step": host * 1e3}
            results["rows"].append(row)
            print(f"{pair:16s} {kind:8s}: {sps * a.feeds:8.1f} scans/s  {sps * active:9.1f} target-frames/s  host "
                  f"{host * 1e3:6.2f} ms/step", flush=True)
            if kind == "multi" and a.trace and pair == "bat_car+m2track":
                torch.cuda.synchronize()
                with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                    for f in range(a.feeds):
                        trk.put_raw(f, rows[1], xfs)
                    trk.advance()
                    torch.cuda.synchronize()
                os.makedirs(os.path.dirname(os.path.abspath(a.trace)), exist_ok=True)
                prof.export_chrome_trace(a.trace)
                ov = overlap(a.trace)
                results["trace"] = {"pair": pair, **ov}
                print(f"trace {pair}: {ov['kernels']} kernels on {ov['streams']} streams over {ov['span_us']:.0f} us; two or more "
                      f"streams busy for {ov['concurrent_us']:.0f} us", flush=True)
            del trk
            torch.cuda.empty_cache()
    print(json.dumps(results))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
