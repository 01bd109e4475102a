"""Occupancy buckets of the live tracker: a step over the active targets only, against the full K-row step.

  python tools/bench_occupancy.py [--points 60000] [--slots 128] [--steps 20] [--warmup 3] [--out results.json]

For BAT-Car and M2-Track, one feed of synthetic 60,000-point scans (datasets/synthetic.py: synthetic_scene, device tensors, so
the step is timed and not the scan copy) and a tracker of --slots slots with 1, 8, 32, 64 and 128 active targets:
  * "bucketed": the tracker as it runs (one captured step per occupancy bucket);
  * "pinned": the same tracker with its buckets pinned to (K,), the full K-row step every advance.
The two are alternated in one process (blocks of 5 steps) over --steps CUDA-event-timed steps each after --warmup untimed ones.
Reported per point: steps/s and target-frames/s of both.  Also reported: the wall time of the first advance (planning and
capture), the peak device memory through it, the CUDA-event time of one step's gathers (the per-slot state with the first-frame
prefix rows, and that prefix alone) and scatters at bucket K, run on their own through the tracker's `_gather` / `_scatter`, as a
share of the step at full occupancy, and a track_feeds run over a synthetic multi-scene workload whose occupancy varies (16 feeds, 24 scenes of 1-12 targets and 30-200
frames, 20,000-point scans, 64 slots): seconds, bucketed against pinned.  Weights are untrained (the timing does not depend on
them).  The card's name and power limit are printed with the numbers."""
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
from open3dsot_b200.datasets.synthetic import synthetic_scene  # noqa: E402
from open3dsot_b200.models import get_model  # noqa: E402
from open3dsot_b200.tracking import multi_tracker as mt  # noqa: E402

MODELS = {"bat_car": "BAT_Car.yaml", "m2track": "M2_track_kitti.yaml"}
ACTIVE = (1, 8, 32, 64, 128)


def model(name):
    cfg = load_config(os.path.join(ROOT, "cfgs", name), {"up_axis": [0, 0, 1], "degrees": True})
    torch.manual_seed(0)
    return get_model(cfg.net_model)(cfg).cuda().eval()


def tracker(net, N, K, pinned):
    """A new tracker (pinned to the full step or not) and the device memory allocated before it; the peak counter is reset."""
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    trk = mt.MultiTargetTracker(net, N, K, seed=0)
    if pinned:
        trk._buckets = (K,)
    return trk, base


def first_advance(trk, scan, base):
    t0 = time.perf_counter()
    trk.step(scan)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, torch.cuda.max_memory_allocated() - base


def sweep(net, scans, boxes, K, warmup, steps):
    rows, extra = [], {}
    trks = {}
    for kind in ("pinned", "bucketed"):
        trk, base = tracker(net, scans[0].shape[0], K, kind == "pinned")
        sec, peak = first_advance(trk, scans[0], base)
        trks[kind] = trk
        extra[kind] = {"first_advance_s": sec, "peak_mib": peak / 2**20, "buckets": list(trk._buckets)}
    live = 0
    for n in ACTIVE:
        for trk in trks.values():
            for j in range(live, n):
                trk.add(j, boxes[j % len(boxes)][0])
        live = n
        for trk in trks.values():
            for i in range(warmup):
                trk.step(scans[1 + i % (len(scans) - 1)])
        ms = {k: 0.0 for k in trks}
        for r in range(steps // 5):
            for kind, trk in trks.items():
                ms[kind] += timed(lambda i, trk=trk: trk.step(scans[1 + (r * 5 + i) % (len(scans) - 1)]), 5)
        row = {"active": n}
        for kind in trks:
            sps = steps / (ms[kind] / 1e3)
            row[kind] = {"steps_per_s": sps, "target_frames_per_s": sps * n, "ms_per_step": ms[kind] / steps}
        rows.append(row)
        print(f"  active {n:4d}: bucketed {row['bucketed']['ms_per_step']:7.3f} ms/step ({row['bucketed']['steps_per_s']:7.1f} "
              f"steps/s, {row['bucketed']['target_frames_per_s']:8.1f} target-frames/s)   pinned "
              f"{row['pinned']['ms_per_step']:7.3f} ms/step ({row['pinned']['steps_per_s']:7.1f} steps/s)", flush=True)
    extra["gather_scatter"] = gather_scatter(trks["bucketed"])
    extra["gather_scatter"]["step_ms"] = rows[-1]["bucketed"]["ms_per_step"]
    return rows, extra


def gather_scatter(trk, reps=50):
    """CUDA-event milliseconds of one step's gathers (trk._gather: the per-slot state and the first-frame prefix rows), of the
    prefix rows' gather alone and of its scatters (trk._scatter), at bucket K with every slot in the work list; the tracker's
    state is put back afterwards."""
    K = trk.K
    snap = [t.clone() for t in trk._state()]
    trk._work.copy_(torch.from_numpy(mt.work_rows(list(range(K)), K)))
    src = trk._work[0]
    with torch.no_grad():
        r, box, dst = trk._gather(K)
        out = {"gather_ms": timed(lambda i: trk._gather(K), reps) / reps,
               "scatter_ms": timed(lambda i: trk._scatter(r, box, box, dst), reps) / reps}
        if "first" in r:
            out["prefix_gather_ms"] = timed(lambda i: (trk._first_local.index_select(0, src), trk._first_keep.index_select(0, src)),
                                            reps) / reps
            out["prefix_bytes"] = 2 * (r["first"][0].numel() * 4 + r["first"][1].numel())
    for t, v in zip(trk._state(), snap):
        t.copy_(v)
    torch.cuda.synchronize()
    return out


def feeds_workload(points):
    rng = np.random.default_rng(11)
    scenes, tid = [], 0
    for i in range(24):
        T, n = int(rng.integers(30, 201)), int(rng.integers(1, 13))
        sc = synthetic_scene(n_frames=T, n_points=points, n_objects=n, seed=500 + i, extent=40.0)
        starts, ends = {}, {}
        for j in range(n):
            a = int(rng.integers(0, T // 3))
            starts.setdefault(a, []).append((tid, sc["boxes"][j][a]))
            ends[tid] = int(rng.integers(a + (T - a) // 2, T))
            tid += 1
        scenes.append({"frames": T, "scan": (lambda t, s=sc["scans"]: s[t]), "starts": starts, "ends": ends})
    return scenes


def run_feeds(net, scenes, points, pinned):
    init = mt.MultiTargetTracker.__init__

    def pinned_init(self, *a, **k):
        init(self, *a, **k)
        self._buckets = (self.K,)
    if pinned:
        mt.MultiTargetTracker.__init__ = pinned_init
    try:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        mt.track_feeds(net, scenes, 16, 64, seed=0, max_points=points)
        torch.cuda.synchronize()
        return time.perf_counter() - t0
    finally:
        mt.MultiTargetTracker.__init__ = init


def main(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--points", type=int, default=60000)
    p.add_argument("--slots", type=int, default=128)
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--feeds_points", type=int, default=20000)
    p.add_argument("--out", default=None, help="also write the results as JSON here")
    a = p.parse_args(argv)
    torch.cuda.set_device(0)
    info = gpu_info()
    print(f"# {info}; {a.points} points per scan, one feed, {a.slots} slots; {a.steps} timed steps after {a.warmup} warm-up "
          f"steps per point", flush=True)
    sc = synthetic_scene(n_frames=8, n_points=a.points, n_objects=16, seed=7, extent=70.0)
    scans = [torch.tensor(s, device="cuda") for s in sc["scans"]]
    results = {"gpu": info, "points": a.points, "slots": a.slots, "models": {}}
    scenes = feeds_workload(a.feeds_points)
    for name, cfg in MODELS.items():
        net = model(cfg)
        print(f"{name}:", flush=True)
        rows, extra = sweep(net, scans, sc["boxes"], a.slots, a.warmup, a.steps)
        for kind in ("bucketed", "pinned"):
            e = extra[kind]
            print(f"  {kind}: buckets {e['buckets']}, first advance {e['first_advance_s']:.2f} s, peak {e['peak_mib']:.0f} MiB",
                  flush=True)
        g = extra["gather_scatter"]
        pre = (f", of which the first-frame prefix rows {g['prefix_gather_ms'] * 1e3:.1f} us ({g['prefix_bytes'] / 1e6:.0f} MB moved, "
               f"{100 * g['prefix_gather_ms'] / g['step_ms']:.2f} % of the step)" if "prefix_gather_ms" in g else ", no prefix")
        print(f"  at bucket {a.slots}: gathers {g['gather_ms'] * 1e3:.1f} us{pre}; scatters {g['scatter_ms'] * 1e3:.1f} us; together "
              f"{100 * (g['gather_ms'] + g['scatter_ms']) / g['step_ms']:.2f} % of the {g['step_ms']:.2f} ms step", flush=True)
        secs = {}
        for kind in ("pinned", "bucketed", "pinned", "bucketed"):
            secs.setdefault(kind, []).append(run_feeds(net, scenes, a.feeds_points, kind == "pinned"))
        feeds = {k: min(v) for k, v in secs.items()}
        print(f"  track_feeds (16 feeds, {len(scenes)} scenes, {sum(s['frames'] for s in scenes)} scene frames): bucketed "
              f"{feeds['bucketed']:.2f} s, pinned {feeds['pinned']:.2f} s (best of 2 each)", flush=True)
        results["models"][name] = {"sweep": rows, **extra, "track_feeds_s": feeds}
        del net
        torch.cuda.empty_cache()
    print(json.dumps(results))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
