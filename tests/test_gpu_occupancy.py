"""Occupancy buckets of the live tracker on the GPU: every box of every target bitwise the same as on a tracker pinned to the
full K-row step (three models, fp32 and bf16, K = 32 over 3 feeds with the active count passing 0, 1, 2, 3, 5, 9, 17 and 32 and
back, fragmented slots and held feeds; and K = 4), replay against eager and repeat runs, no host sync after the first advance
over every bucket, the crop kernel's grid of one replay and an advance with no target, several classes at different
occupancies, track_feeds, and the peak memory of capturing every bucket."""
import collections
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from open3dsot_b200.config import load_config
from open3dsot_b200.datasets.synthetic import synthetic_scene
from open3dsot_b200.models import get_model
from open3dsot_b200.tracking.multi_class import MultiClassTracker
from open3dsot_b200.tracking.multi_tracker import MultiTargetTracker, bucket_for, track_feeds, work_slots

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODELS = ["BAT_Car.yaml", "P2B_Car.yaml", "M2_track_kitti.yaml"]
N_POINTS = 4000
# targets live after each advance; the tracker's active count at an advance is the previous entry
COUNTS = {32: [0, 1, 2, 3, 5, 9, 17, 32, 32, 20, 17, 12, 9, 6, 5, 3, 2, 1, 0, 2, 4, 1, 0, 3, 1],
          4: [0, 1, 2, 3, 4, 4, 2, 1, 0, 3, 4, 1, 0, 2, 1]}
HOLD = {4: {2}, 5: {2}, 9: {1}, 12: {0, 2}, 20: {1}}                        # advance -> feeds that get no scan


def _model(cfg_name):
    cfg = load_config(os.path.join(ROOT, "cfgs", cfg_name), {"up_axis": [0, 0, 1], "degrees": True})
    torch.manual_seed(0)
    return get_model(cfg.net_model)(cfg).cuda().eval()


@pytest.fixture(scope="module")
def data():
    return [synthetic_scene(n_frames=26, n_points=N_POINTS, n_objects=4, seed=80 + f, extent=14.0) for f in range(3)]


def _drive(trk, data, counts, put=None, add=None, drop=None, targets=None, snapshot=None):
    """Run the schedule: every advance puts the next scan of each feed not held, then adds targets (id i on feed i % 3, object
    i % 4) or drops the ones in the lowest slots (so that the high slots stay occupied) until `counts[step]` are live.  Returns
    {id: (advances live, 15) float32 numpy} and the buckets the tracker's advances ran at."""
    put, add, drop = put or trk.put, add or (lambda i, b, f: trk.add(i, b, feed=f)), drop or trk.drop
    targets, snapshot = targets or trk.targets, snapshot or trk.snapshot
    seen, nxt, rec, used = [0, 0, 0], 0, {}, set()
    for s, c in enumerate(counts):
        fed = {f for f in range(3) if f not in HOLD.get(s, ())}
        for f in sorted(fed):
            put(f, data[f]["scans"][seen[f]])
            seen[f] += 1
        if isinstance(trk, MultiTargetTracker) and trk._buckets is not None:
            n = len(work_slots(trk._feed_of, fed))
            if n:
                used.add(bucket_for(n, trk._buckets))
        trk.advance()
        snap = snapshot()
        for tid, k in targets().items():
            rec.setdefault(tid, []).append(snap[k].clone())
        live = targets()
        for tid, _ in sorted(live.items(), key=lambda kv: kv[1])[:max(0, len(live) - c)]:
            drop(tid)
        while len(targets()) < c:
            f = nxt % 3
            add(nxt, data[f]["boxes"][nxt % 4][seen[f] - 1], f)
            nxt += 1
    return {tid: torch.stack(v).cpu().numpy() for tid, v in rec.items()}, used


def _run(net, data, K, precision="fp32", pinned=False, use_graph=True):
    trk = MultiTargetTracker(net, N_POINTS, K, seed=7, feeds=3, precision=precision, use_graph=use_graph)
    if pinned:
        trk._buckets = (K,)
    got, used = _drive(trk, data, COUNTS[K])
    return got, used, trk._buckets


def _same(a, b, what):
    assert sorted(a) == sorted(b), what
    for tid in a:
        assert np.isfinite(a[tid]).all() and np.array_equal(a[tid], b[tid]), (what, tid, float(np.abs(a[tid] - b[tid]).max()))


# ------------------------------------------------------------------ bitwise across buckets
@pytest.mark.parametrize("K", [32, 4])
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("cfg_name", MODELS)
def test_boxes_are_bitwise_the_full_step_at_every_bucket(cfg_name, precision, K, data):
    net = _model(cfg_name)
    got, used, buckets = _run(net, data, K, precision)
    want, _, pinned = _run(net, data, K, precision, pinned=True)
    assert pinned == (K,)
    one_row_stacks = cfg_name.startswith("M2")                               # its heads run one row per target
    assert buckets == ((16, 32) if one_row_stacks and K == 32 else tuple(b for b in (1, 2, 4, 8, 16, 32) if b < K) + (K,))
    assert used == set(buckets), (used, buckets)                            # the schedule visits every bucket
    _same(got, want, (cfg_name, precision, K))


# ------------------------------------------------------------------ replay against eager, repeat runs
@pytest.mark.parametrize("cfg_name", ["BAT_Car.yaml", "M2_track_kitti.yaml"])
def test_replay_equals_eager_and_repeats(cfg_name, data):
    net = _model(cfg_name)
    ref, _, _ = _run(net, data, 32)
    again, _, _ = _run(net, data, 32)
    eager, used, buckets = _run(net, data, 32, use_graph=False)
    assert used == set(buckets)
    _same(again, ref, "again")
    _same(eager, ref, "eager")


# ------------------------------------------------------------------ no host sync over every bucket
def test_no_sync_after_the_first_advance_whatever_the_occupancy(data):
    net = _model("BAT_Car.yaml")
    trk = MultiTargetTracker(net, N_POINTS, 8, seed=1, feeds=3)
    scans = [[torch.from_numpy(s) for s in data[f]["scans"]] for f in range(3)]
    for f in range(3):
        trk.put(f, scans[f][0])
    trk.advance()                                                            # plan and capture (synchronises once)
    assert trk._buckets == (1, 2, 4, 8) and sorted(trk.graphs) == [1, 2, 4, 8]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        ids = iter(range(100))
        for t, n_add in enumerate([1, 1, 2, 4], start=1):                    # 1, 2, 4 and 8 targets: every bucket
            for _ in range(n_add):
                i = next(ids)
                trk.add(i, data[i % 3]["boxes"][0][t - 1], feed=i % 3)
            for f in range(3):
                trk.put(f, scans[f][t])
            trk.advance()
        for tid in list(trk.targets())[:7]:
            trk.drop(tid)
        trk.put(0, scans[0][5])
        trk.put(1, scans[1][5])
        trk.put(2, scans[2][5])
        trk.advance()                                                        # one target: bucket 1
        trk.drop(next(iter(trk.targets())))
        trk.put(1, scans[1][6])
        trk.advance()                                                        # nothing to advance
        snap = trk.snapshot()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.isfinite(snap).all() and trk.targets() == {}


# ------------------------------------------------------------------ the kernels of one replay (child process, as in
# test_gpu_multi_target.py: a CUPTI session around a graph replay in the suite's process spoils later profiler-based tests)
_PROFILE_CHILD = r"""
import json, os, sys
import numpy as np, torch
sys.path.insert(0, sys.argv[1])
from open3dsot_b200.config import load_config
from open3dsot_b200.datasets.synthetic import synthetic_scene
from open3dsot_b200.models import get_model
from open3dsot_b200.tracking.multi_tracker import MultiTargetTracker
cfg = load_config(os.path.join(sys.argv[1], "cfgs", "BAT_Car.yaml"), {"up_axis": [0, 0, 1]})
torch.manual_seed(0)
net = get_model(cfg.net_model)(cfg).cuda().eval()
sc = synthetic_scene(n_frames=8, n_points=6000, n_objects=3, seed=900, extent=15.0)
xf = np.hstack([np.eye(3), np.zeros((3, 1))])
trk = MultiTargetTracker(net, 6000, 64, seed=2)
def step(t):
    trk.put_raw(0, sc["scans"][t], [xf])                 # host rows: the ingest kernel
    trk.advance()
step(0)
for j in range(3):
    trk.add(j, sc["boxes"][j][0])
step(1)
torch.cuda.synchronize()
def profiled(t, path):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        step(t)
        torch.cuda.synchronize()
    prof.export_chrome_trace(path)
    ev = [e for e in json.load(open(path))["traceEvents"] if e.get("cat") == "kernel"]
    return [(e["name"], e.get("args", {}).get("grid")) for e in ev]
out = {}
busy = profiled(2, sys.argv[2] + "/busy.json")
if not busy:
    busy = profiled(3, sys.argv[2] + "/busy.json")   # CUPTI now and then delivers no records for a short session
out["busy"] = busy
for j in range(3):
    trk.drop(j)
step(4)
torch.cuda.synchronize()
idle = profiled(5, sys.argv[2] + "/idle.json")
if not idle:
    idle = profiled(6, sys.argv[2] + "/idle.json")
out["idle"] = idle
with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:   # what advance() returns: boxes()
    trk.boxes()
    torch.cuda.synchronize()
prof.export_chrome_trace(sys.argv[2] + "/boxes.json")
out["boxes"] = [e["name"] for e in json.load(open(sys.argv[2] + "/boxes.json"))["traceEvents"] if e.get("cat") == "kernel"]
print(json.dumps(out))
"""


def test_one_replay_runs_on_its_bucket(tmp_path):
    r = subprocess.run([sys.executable, "-c", _PROFILE_CHILD, ROOT, str(tmp_path)], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
    crops = [grid for name, grid in got["busy"] if "crop_resample_kernel" in name]
    assert len(crops) == 2 and all(g == [4, 1, 1] for g in crops), got["busy"]          # 3 active of 64: bucket 4
    # an advance with nothing to advance: the ingest, and the device views advance() returns (boxes()), nothing else
    idle = collections.Counter(name for name, _ in got["idle"])
    idle.subtract(collections.Counter(got["boxes"]))
    ran = sorted(+idle)
    assert len(ran) == 1 and "scan_ingest_kernel" in ran[0] and idle[ran[0]] == 1, (got["idle"], got["boxes"])


# ------------------------------------------------------------------ several classes
def test_classes_are_bitwise_lone_pinned_trackers_and_never_sync(data):
    models = {"car": _model("BAT_Car.yaml"), "ped": _model("M2_track_kitti.yaml")}
    K = {"car": 32, "ped": 4}
    mc = MultiClassTracker(models, N_POINTS, K, feeds=3, seed=7)
    counts = {"car": COUNTS[32][:15], "ped": COUNTS[4]}
    # the car class follows COUNTS[32], the pedestrian class COUNTS[4]: ids of the two classes are tracked by one driver each
    got = {}
    for cls in ("car", "ped"):
        lone = MultiTargetTracker(models[cls], N_POINTS, K[cls], seed=7, feeds=3)
        lone._buckets = (K[cls],)
        got[cls] = _drive(lone, data, counts[cls])[0]
    rec = _drive_classes(mc, data, counts)
    for cls in ("car", "ped"):
        _same(rec[cls], got[cls], cls)
    assert mc.trackers["car"]._buckets == (1, 2, 4, 8, 16, 32) and mc.trackers["ped"]._buckets == (1, 2, 4)


def _drive_classes(mc, data, counts):
    """_drive for every class of `mc` at once: one put per feed and one advance for all classes, no sync after the first."""
    seen, nxt, rec = [0, 0, 0], {c: 0 for c in counts}, {c: {} for c in counts}
    calls = []
    from open3dsot_b200 import ops
    ingest = ops.scan_ingest
    for s in range(len(counts["ped"])):
        fed = {f for f in range(3) if f not in HOLD.get(s, ())}
        for f in sorted(fed):
            mc.put(f, data[f]["scans"][seen[f]])
            seen[f] += 1
        if s:
            torch.cuda.set_sync_debug_mode("error")
        ops.scan_ingest = lambda *a, **k: calls.append(s) or ingest(*a, **k)
        try:
            mc.advance()
            snap = mc.snapshot()
            for (cls, tid), k in mc.targets().items():
                rec[cls].setdefault(tid, []).append(snap[k].clone())
            for cls, trk in mc.trackers.items():
                live = trk.targets()
                for tid, _ in sorted(live.items(), key=lambda kv: kv[1])[:max(0, len(live) - counts[cls][s])]:
                    mc.drop(cls, tid)
                while len(trk.targets()) < counts[cls][s]:
                    i = nxt[cls]
                    mc.add(cls, i, data[i % 3]["boxes"][i % 4][seen[i % 3] - 1], feed=i % 3)
                    nxt[cls] += 1
        finally:
            torch.cuda.set_sync_debug_mode(0)
            ops.scan_ingest = ingest
    assert calls == list(range(len(counts["ped"])))                          # one ingest per advance
    return {c: {tid: torch.stack(v).cpu().numpy() for tid, v in r.items()} for c, r in rec.items()}


# ------------------------------------------------------------------ track_feeds
def test_track_feeds_is_bitwise_its_pinned_run(monkeypatch):
    from open3dsot_b200.tracking import multi_tracker as mt
    net = _model("BAT_Car.yaml")
    rng = np.random.default_rng(3)
    scenes = []
    for i, (T, n) in enumerate([(14, 5), (6, 1), (9, 3), (4, 2), (11, 4), (5, 1)]):
        sc = synthetic_scene(n_frames=T, n_points=3000, n_objects=n, seed=200 + i, extent=14.0)
        starts, ends = {}, {}
        for j in range(n):
            a = int(rng.integers(0, T // 2))
            starts.setdefault(a, []).append((100 * i + j, sc["boxes"][j][a]))
            ends[100 * i + j] = int(rng.integers(a, T))
        scenes.append({"frames": T, "scan": (lambda t, s=sc["scans"]: s[t]), "starts": starts, "ends": ends})

    def flat(res):
        return {tid: np.array([np.concatenate([b.center, b.wlh, b.rotation_matrix.ravel()]) for _, b in sorted(tr.items())])
                for scene in res for tid, tr in scene.items()}
    got = flat(track_feeds(net, scenes, 3, 8, seed=3, max_points=3000))
    init = mt.MultiTargetTracker.__init__

    def pinned_init(self, *a, **k):
        init(self, *a, **k)
        self._buckets = (self.K,)
    monkeypatch.setattr(mt.MultiTargetTracker, "__init__", pinned_init)
    want = flat(track_feeds(net, scenes, 3, 8, seed=3, max_points=3000))
    _same(got, want, "track_feeds")


# ------------------------------------------------------------------ memory
def _peak_through_first_advance(net, data, pinned):
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    trk = MultiTargetTracker(net, N_POINTS, 64, seed=1)
    if pinned:
        trk._buckets = (64,)
    trk.step(torch.from_numpy(data[0]["scans"][0]))
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    del trk
    return peak


def test_all_buckets_cost_about_the_memory_of_one(data):
    net = _model("BAT_Car.yaml")
    _peak_through_first_advance(net, data, True)                             # the weight caches, outside both measurements
    pinned = _peak_through_first_advance(net, data, True)
    bucketed = _peak_through_first_advance(net, data, False)
    print(f"peak through the first advance, K = 64: bucketed {bucketed / 2**20:.1f} MiB, pinned {pinned / 2**20:.1f} MiB, "
          f"ratio {bucketed / pinned:.3f}")
    assert bucketed <= 1.25 * pinned, (bucketed, pinned)
