"""Detection matching in the live tracker on the GPU: `o3d_box_associate` and `o3d_track_update` with matches bitwise against
their formulations (eager, repeated, graph replay); the feature off, or fed only detections beyond the gate, changes no box,
evidence or loss decision; every record bitwise across occupancy buckets with detections near the targets; a target re-acquired
at its detection after a synthetic occlusion (M2-Track, BAT-Car) without a host sync; births from `unmatched()`; two classes
as lone trackers; the kernels of one replay; track_feeds / track_classes and the command line with detections."""
import collections
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from open3dsot_b200 import track
from open3dsot_b200.datasets.data_classes import Box, PointCloud
from open3dsot_b200.datasets.kitti import kittiDataset
from open3dsot_b200.datasets.synthetic import synthetic_scene, synthetic_sequence
from open3dsot_b200.tracking.multi_class import MultiClassTracker, track_classes
from open3dsot_b200.tracking.multi_tracker import (MatchSlots, MultiTargetTracker, Slots, associate, coast_weights,
                                                   detection_gate2, detection_rows, track_feeds, track_update,
                                                   track_update_tensors)
from test_associate import associate_case, run_formulation
from test_coast import _bits, _random_case
from test_gpu_lost_targets import FAR, MODELS, _flat, _model
from test_gpu_occupancy import COUNTS, N_POINTS, _drive
from test_kitti_reader import _write_scene

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32


# ------------------------------------------------------------------ the kernels against their formulations
def _kernel_run(case, gate2, axes, rule, coast):
    state, src, feed, adv, center, points, fed, count, det = case
    F, D, _ = det.shape
    T = lambda x: torch.from_numpy(np.array(x, copy=True)).cuda()
    slots = Slots(*(T(x) for x in state))
    records = (torch.zeros(F, D, 16, device="cuda"), torch.zeros(F, dtype=torch.int32, device="cuda"),
               torch.full((F, D), -1, dtype=torch.int32, device="cuda"))
    args = [T(x) for x in (src, feed, adv, center, points)]
    extra = [T(x) for x in (fed, count, det)]
    return lambda: associate(*args, slots, *extra, records, gate2, axes, rule, coast), records


def _same_bits(a, b, what):
    a, b = a.cpu().numpy(), b.cpu().numpy()
    assert np.array_equal(_bits(a), _bits(b)), what


@pytest.mark.parametrize("F", [1, 16])
@pytest.mark.parametrize("D", [1, 64, 1024])
@pytest.mark.parametrize("b", [1, 7, 64, 300])
def test_associate_kernel_equals_the_formulation(b, D, F):
    rule, coast = (3, 2), True
    matched = 0
    for seed in range(2):
        case = associate_case(b + 5, b, F, D, 200 + seed, rule, grid=seed == 1)
        gate2, axes = detection_gate2(2.0 if seed == 1 else 3.0), ((0, 1), (0, 2))[seed]
        (want, want_rec) = run_formulation(case, gate2, axes, rule, coast)
        n = case[-2]
        runs = []
        for _ in range(2):                                                    # eager, then again
            fn, rec = _kernel_run(case, gate2, axes, rule, coast)
            runs.append((fn(), rec))
        fn, rec = _kernel_run(case, gate2, axes, rule, coast)
        init = [x.clone() for x in rec]
        fn()                                                                  # warm-up outside the capture
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            out = fn()
        for x, v in zip(rec, init):
            x.copy_(v)
        g.replay()
        runs.append((out, rec))
        torch.cuda.synchronize()
        for got, got_rec in runs:
            for w, x, name in zip(want, got, ("pred", "match", "match_box")):
                _same_bits(x, w, (b, D, F, seed, name))
            assert torch.equal(got_rec[1].cpu(), want_rec[1])
            for f in range(F):
                k = int(n[f]) if case[-3][f] else 0
                _same_bits(got_rec[0][f, :k], want_rec[0][f, :k], (f, "rec_det"))
                assert torch.equal(got_rec[2][f, :k].cpu(), want_rec[2][f, :k]), (f, "rec_slot")
        matched += int((want[1] >= 0).sum())
    assert matched > 0 or b < 64 or D < 64


@pytest.mark.parametrize("rule,alpha", [(None, None), ((3, 2), None), ((3, 2), 0.3), ((0, 1), 0.5)])
@pytest.mark.parametrize("b", [1, 7, 64, 300])
def test_track_update_with_matches_equals_the_formulation(b, rule, alpha):
    coast = coast_weights(alpha)
    for seed in range(3):
        case = _random_case(b + 5, b, 300 + seed, rule)
        rng = np.random.default_rng(seed)
        match = np.where(rng.random(b) < 0.5, rng.integers(0, 9, b), -1).astype(np.int32)
        match_box = rng.normal(0, 5, (b, 12)).astype(F32)
        det0 = rng.integers(-1, 5, b + 7).astype(np.int32)
        rq0 = rng.random(b + 7) < 0.3
        outs = []
        for dev in ("cpu", "cuda", "cuda"):
            T = lambda x: torch.from_numpy(np.array(x, copy=True)).to(dev)
            slots = Slots(*(T(x) for x in case[0]))
            ms = MatchSlots(T(det0), T(rq0))
            args = [T(x) for x in case[1:]]
            (track_update_tensors if dev == "cpu" else track_update)(slots, *args, rule, coast, (T(match), T(match_box)) + tuple(ms))
            outs.append(tuple(slots) + tuple(ms))
        for got in outs[1:]:
            for name, w, x in zip(Slots._fields + MatchSlots._fields, outs[0], got):
                _same_bits(x, w, (b, seed, name))


# ------------------------------------------------------------------ the live step
@pytest.fixture(scope="module")
def data():
    return [synthetic_scene(n_frames=26, n_points=N_POINTS, n_objects=4, seed=80 + f, extent=14.0) for f in range(3)]


def _near(data, f, t, noise=0.1, seed=0):
    """Detections of feed f's scan t: every object's ground-truth box, its centre moved by N(0, noise), in a shuffled order."""
    rng = np.random.default_rng(1000 * f + t + seed)
    boxes = [data[f]["boxes"][o][t] for o in range(len(data[f]["boxes"]))]
    rows = detection_rows(boxes, rng.random(len(boxes)))
    rows[:, :3] += rng.normal(0, noise, (len(boxes), 3)).astype(F32)
    return rows[rng.permutation(len(rows))]


def _far(data, f, t):
    rows = _near(data, f, t)
    rows[:, :3] += FAR
    return rows


def _run(net, data, precision, lost, coast, detections, dets=None, pinned=False, K=4):
    trk = MultiTargetTracker(net, N_POINTS, K, seed=7, feeds=3, precision=precision, lost=lost, coast=coast, detections=detections)
    if pinned:
        trk._buckets = (K,)
    seen = [0, 0, 0]

    def put(f, scan):
        kw = {} if dets is None else {"detections": dets(data, f, seen[f])}
        seen[f] += 1
        trk.put(f, scan, **kw)

    snap = lambda: torch.cat([trk._record(), trk._match_record(), trk.vel, trk.hit_c, trk.hit_t.float()[:, None],
                              trk.coasting.float()[:, None]], 1)
    return _drive(trk, data, COUNTS[K], put=put, snapshot=snap)[0]


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("cfg_name", MODELS)
def test_feature_off_and_detections_beyond_the_gate_change_nothing(cfg_name, precision, data):
    net = _model(cfg_name)
    plain = _run(net, data, precision, None, None, None)
    pts = np.concatenate([r[:, 15] for r in plain.values()])
    rule = (int(np.median(pts[pts >= 0])) + 1, 2)                            # a rule that fires
    for coast in (None, 0.5):
        off = _run(net, data, precision, rule, coast, None)
        never = _run(net, data, precision, rule, coast, (64, 2.0))
        beyond = _run(net, data, precision, rule, coast, (64, 2.0), dets=_far)
        assert sorted(off) == sorted(never) == sorted(beyond)
        for tid in off:
            assert np.array_equal(off[tid], never[tid], equal_nan=True), (coast, tid)
            assert np.array_equal(off[tid], beyond[tid], equal_nan=True), (coast, tid)
            assert (off[tid][:, 19] == -1).all() and not off[tid][:, 20].any()
        rec = np.concatenate(list(off.values()))
        assert rec[:, 18].any()                                               # the rule fired: some targets lost


@pytest.mark.parametrize("cfg_name", ["BAT_Car.yaml", "M2_track_kitti.yaml"])
def test_records_are_bitwise_across_buckets_with_detections(cfg_name, data):
    net = _model(cfg_name)
    plain = _run(net, data, "fp32", None, None, None, K=32)
    pts = np.concatenate([r[:, 15] for r in plain.values()])
    rule = (int(np.median(pts[pts >= 0])) + 1, 3)
    got = _run(net, data, "fp32", rule, 0.5, (64, 2.0), dets=_near, K=32)
    want = _run(net, data, "fp32", rule, 0.5, (64, 2.0), dets=_near, K=32, pinned=True)
    assert sorted(got) == sorted(want)
    for tid in got:
        assert np.array_equal(got[tid], want[tid], equal_nan=True), tid
    rec = np.concatenate(list(got.values()))
    assert (rec[:, 19] >= 0).any() and rec[:, 20].any()                       # matches, and some re-acquired misses


# ------------------------------------------------------------------ re-acquisition after a synthetic occlusion
T0, PATIENCE, MIN_POINTS, ALPHA = 4, 3, 1, 0.5


def _occluded(sc, obj, t0, g, radius=8.0):
    scans = []
    for t, s in enumerate(sc["scans"]):
        s = s.copy()
        if t0 <= t < t0 + g:
            s[np.linalg.norm(s[:, :2] - sc["boxes"][obj][t].center[None, :2], axis=1) < radius] = FAR
        scans.append(s)
    return scans


def _follow(net, scans, boxes, ids, K, detections=None, dets=None, sync_free=False, patience=PATIENCE):
    """One feed: add `ids` on scan 0 and advance through every scan, with `dets` {t: rows}; {id: (T, 19 + 2 + 1) records:
    _record(), detection, reacquired, coasting}."""
    trk = MultiTargetTracker(net, N_POINTS, K, seed=4, lost=(MIN_POINTS, patience), coast=ALPHA, detections=detections)
    rec = {i: [] for i in ids}

    def record():
        r = torch.cat([trk._record(), trk._match_record(), trk.coasting.float()[:, None]], 1)
        for i in ids:
            rec[i].append(r[trk.targets()[i]].clone())

    def put(t):
        kw = {} if detections is None else {"detections": (dets or {}).get(t, np.zeros((0, 16), F32))}
        trk.put(0, torch.from_numpy(scans[t]), **kw)
        trk.advance()

    put(0)
    for i in ids:
        trk.add(i, boxes[i][0])
    record()
    put(1)
    record()
    torch.cuda.synchronize()
    if sync_free:
        torch.cuda.set_sync_debug_mode("error")
    try:
        for t in range(2, len(scans)):
            put(t)
            record()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    return {i: torch.stack(v).cpu().numpy() for i, v in rec.items()}


@pytest.mark.parametrize("g", [1, 2])
@pytest.mark.parametrize("cfg_name", ["M2_track_kitti.yaml", "BAT_Car.yaml"])
def test_an_occluded_target_is_reacquired_at_its_detection(cfg_name, g):
    """Target 0's surroundings are emptied on frames T0 .. T0 + g - 1; on the last of them, where the network's box has no point
    and is a miss, the detector reports its ground-truth box."""
    net = _model(cfg_name)
    sc = synthetic_scene(n_frames=10, n_points=N_POINTS, n_objects=4, seed=300, extent=14.0)
    scans = _occluded(sc, 0, T0, g)
    at = T0 + g - 1
    truth = sc["boxes"][0][at]
    dets = {at: detection_rows([truth, Box(truth.center + FAR, truth.wlh, truth.rotation_matrix)], [0.9, 0.3])}
    # untrained BAT-Car boxes miss often before the occlusion: a long patience keeps target 0 advancing up to the detection
    patience = PATIENCE if cfg_name.startswith("M2") else 50
    base = _follow(net, scans, sc["boxes"], [0, 1, 2, 3], 8, patience=patience)
    assert not base[0][at, 18]                                                # still advancing on the detection's frame
    # the gate takes in target 0's box on that frame and no other target's (untrained BAT-Car boxes drift off their objects)
    dist = {i: float(np.linalg.norm(base[i][at, :2] - truth.center[:2].astype(F32))) for i in base}
    assert min(dist[i] for i in (1, 2, 3)) > dist[0], dist
    gate = dist[0] + 0.5 * (min(dist[i] for i in (1, 2, 3)) - dist[0])
    got = _follow(net, scans, sc["boxes"], [0, 1, 2, 3], 8, detections=(16, gate), dets=dets, sync_free=True, patience=patience)
    r0 = got[0]
    assert r0[at, 15] < MIN_POINTS                                            # the network's box is a miss
    assert np.array_equal(r0[at, :3], truth.center.astype(F32))              # the detection's centre and rotation
    assert np.array_equal(r0[at, 6:15], truth.rotation_matrix.astype(F32).reshape(9))
    assert np.array_equal(r0[at, 3:6], r0[at - 1, 3:6])                      # the slot keeps its wlh
    assert r0[at, 17] == 0 and r0[at, 19] == 0 and r0[at, 20] == 1 and r0[at, 21] == 0 and r0[at, 18] == 0
    assert not r0[:at, 20].any() and (r0[:at, 19] == -1).all()
    assert np.array_equal(r0[:at, :19], base[0][:at, :19], equal_nan=True)    # before it: the run without detections
    for i in (1, 2, 3):
        assert np.array_equal(got[i][:, :19], base[i][:, :19], equal_nan=True), i
        assert (got[i][:, 19] == -1).all() and not got[i][:, 20].any()


# ------------------------------------------------------------------ births from unmatched detections
def test_births_from_unmatched_detections():
    net = _model("M2_track_kitti.yaml")
    sc = synthetic_scene(n_frames=4, n_points=N_POINTS, n_objects=4, seed=300, extent=14.0)
    trk = MultiTargetTracker(net, N_POINTS, 8, seed=4, feeds=2, detections=(16, 2.0))
    first = detection_rows([sc["boxes"][o][0] for o in range(4)], [0.9, 0.8, 0.7, 0.6])
    trk.put(0, torch.from_numpy(sc["scans"][0]), detections=first)
    trk.put(1, torch.from_numpy(sc["scans"][0]))                             # fed without detections: none
    trk.advance()
    um = trk.unmatched()
    assert sorted(um) == [0, 1] and um[1] == [] and [d for d, _, _ in um[0]] == [0, 1, 2, 3]
    for d, box, score in um[0]:
        assert np.array_equal(box.center.astype(F32), first[d, :3]) and score == float(first[d, 15])
        trk.add(10 + d, box, feed=0)
    order = [2, 0, 3, 1]
    fp = Box(sc["boxes"][0][1].center + np.array([30.0, 30.0, 0.0]), sc["boxes"][0][1].wlh, np.eye(3))
    second = detection_rows([sc["boxes"][o][1] for o in order] + [fp], [0.5] * 5)
    trk.put(0, torch.from_numpy(sc["scans"][1]), detections=second)
    trk.advance()
    det = trk.boxes()["detection"].cpu().numpy()
    for d in range(4):
        assert det[trk.targets()[10 + d]] == order.index(d), (d, det)
    um = trk.unmatched()
    assert [d for d, _, _ in um[0]] == [4] and um[1] == []
    trk.put(1, torch.from_numpy(sc["scans"][1]))                             # feed 0 not fed: its records stay
    trk.advance()
    assert [d for d, _, _ in trk.unmatched()[0]] == [4]


# ------------------------------------------------------------------ classes
def test_classes_with_detections_are_lone_trackers(data):
    models = {"car": _model("BAT_Car.yaml"), "ped": _model("M2_track_kitti.yaml")}
    dets = {"car": _near, "ped": lambda d, f, t: _near(d, f, t, noise=0.3, seed=5)}
    rule = {"car": (5, 2), "ped": (5, 3)}

    def drive(add_put):
        seen, recs = [0, 0, 0], []
        for s in range(10):
            for f in range(3):
                add_put[0](f, data[f]["scans"][seen[f]], {c: dets[c](data, f, seen[f]) for c in models})
                seen[f] += 1
            add_put[2]()
            if s == 0:
                for f in range(3):
                    for o in range(2):
                        add_put[1](f, 10 * f + o, data[f]["boxes"][o][0])
            recs.append(add_put[3]())
        return torch.stack(recs).cpu().numpy()

    mc = MultiClassTracker(models, N_POINTS, {"car": 8, "ped": 8}, feeds=3, seed=7, lost=rule, coast={"ped": 0.5},
                           detections={"car": (16, 2.0), "ped": (16, 3.0)})
    both = drive((lambda f, s, d: mc.put(f, s, detections=d), lambda f, i, b: [mc.add(c, i, b, feed=f) for c in models],
                  mc.advance, lambda: torch.cat([mc._record(), mc._match_record()], 1)))
    for j, (c, coast, gate) in enumerate((("car", None, 2.0), ("ped", 0.5, 3.0))):
        trk = MultiTargetTracker(models[c], N_POINTS, 8, seed=7, feeds=3, lost=rule[c], coast=coast, detections=(16, gate))
        alone = drive((lambda f, s, d: trk.put(f, s, detections=d[c]), lambda f, i, b: trk.add(i, b, feed=f), trk.advance,
                       lambda: torch.cat([trk._record(), trk._match_record()], 1)))
        assert np.array_equal(both[:, 8 * j:8 * j + 8], alone, equal_nan=True), c
    assert (both[:, :, 19] >= 0).any()


# ------------------------------------------------------------------ the kernels of one replay (child process, as in
# test_gpu_coast.py)
_PROFILE_CHILD = r"""
import json, os, sys
import numpy as np
import torch
sys.path.insert(0, sys.argv[1])
from open3dsot_b200.config import load_config
from open3dsot_b200.datasets.synthetic import synthetic_scene
from open3dsot_b200.models import get_model
from open3dsot_b200.tracking.multi_tracker import MultiTargetTracker, detection_rows
cfg = load_config(os.path.join(sys.argv[1], "cfgs", "BAT_Car.yaml"), {"up_axis": [0, 0, 1]})
torch.manual_seed(0)
net = get_model(cfg.net_model)(cfg).cuda().eval()
sc = synthetic_scene(n_frames=6, n_points=6000, n_objects=3, seed=900, extent=15.0)
trk = MultiTargetTracker(net, 6000, 8, seed=2, lost=(5, 3), coast=0.5, detections=(64, 2.0))
scans = [torch.from_numpy(s).cuda() for s in sc["scans"]]
dets = lambda t: detection_rows([sc["boxes"][o][t] for o in range(3)], [0.5] * 3)
trk.put(0, scans[0], detections=dets(0)); trk.advance()
for j in range(3):
    trk.add(j, sc["boxes"][j][0])
trk.put(0, scans[1], detections=dets(1)); trk.advance()
torch.cuda.synchronize()
names = []
for t in (2, 3):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        trk.put(0, scans[t], detections=dets(t)); trk.advance()
        torch.cuda.synchronize()
    prof.export_chrome_trace(sys.argv[2] + "/step.json")
    names = [e["name"] for e in json.load(open(sys.argv[2] + "/step.json"))["traceEvents"] if e.get("cat") == "kernel"]
    if names:
        break
print(json.dumps(names))
"""


def test_one_replay_associates_in_one_kernel(tmp_path):
    r = subprocess.run([sys.executable, "-c", _PROFILE_CHILD, ROOT, str(tmp_path)], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    names = json.loads(r.stdout.strip().splitlines()[-1])
    count = collections.Counter(names)
    assert sum(v for k, v in count.items() if "associate_kernel" in k) == 1, names
    assert sum(v for k, v in count.items() if "track_update_kernel" in k) == 1, names
    assert not [k for k in count if "index_copy" in k], names


# ------------------------------------------------------------------ track_feeds, track_classes and the command line
def _det_scenes(near=True):
    rng = np.random.default_rng(3)
    scenes = []
    for i, (T, n) in enumerate([(9, 3), (7, 2)]):
        sc = synthetic_scene(n_frames=T, n_points=3000, n_objects=n, seed=500 + i, extent=14.0)
        starts = {0: [(100 * i + j, sc["boxes"][j][0]) for j in range(n)]}
        ends = {100 * i + j: T - 1 for j in range(n)}

        def dets(t, sc=sc, n=n):
            rows = detection_rows([sc["boxes"][j][t] for j in range(n)], rng.random(n))
            if not near:
                rows[:, :3] += FAR
            return rows
        scenes.append({"frames": T, "scan": (lambda t, s=sc["scans"]: s[t]), "starts": starts, "ends": ends, "detections": dets})
    return scenes


def test_track_feeds_and_track_classes_with_detections():
    net = _model("M2_track_kitti.yaml")
    plain, plain_ev = track_feeds(net, _det_scenes(), 2, 6, seed=3, max_points=3000, lost=(1, 2), evidence=True)
    far, far_ev = track_feeds(net, _det_scenes(False), 2, 6, seed=3, max_points=3000, lost=(1, 2), evidence=True,
                              detections=(8, 2.0))
    near, near_ev = track_feeds(net, _det_scenes(), 2, 6, seed=3, max_points=3000, lost=(1, 2), evidence=True,
                                detections=(8, 2.0))
    plain, far = _flat(plain), _flat(far)
    far_ev = {tid: tr for scene in far_ev for tid, tr in scene.items()}
    near_ev = {tid: tr for scene in near_ev for tid, tr in scene.items()}
    for tid in plain:
        for t in plain[tid]:
            assert np.array_equal(plain[tid][t], far[tid][t]), (tid, t)
            assert len(far_ev[tid][t]) == 4 and far_ev[tid][t][2:] == (False, -1)
    assert sum(e[3] >= 0 for tr in near_ev.values() for e in tr.values()) > 0
    models = {"car": _model("BAT_Car.yaml"), "ped": net}
    cls_scenes = []
    for s in _det_scenes():
        cls_scenes.append({"frames": s["frames"], "scan": s["scan"], "ends": {(c, tid): e for tid, e in s["ends"].items() for c in models},
                           "starts": {t: [((c, tid), b) for tid, b in g for c in models] for t, g in s["starts"].items()},
                           "detections": lambda t, d=s["detections"]: {"ped": d(t)}})
    both, both_ev = track_classes(models, cls_scenes, 2, {"car": 8, "ped": 8}, seed=3, max_points=3000, lost=(1, 2),
                                  evidence=True, detections={"ped": (8, 2.0)})
    both_ev = {key: tr for scene in both_ev for key, tr in scene.items()}
    assert all(len(e) == 2 for key, tr in both_ev.items() if key[0] == "car" for e in tr.values())
    assert all(len(e) == 4 for key, tr in both_ev.items() if key[0] == "ped" for e in tr.values())
    assert sum(e[3] >= 0 for key, tr in both_ev.items() if key[0] == "ped" for e in tr.values()) > 0


def test_command_line_with_detections(tmp_path, capsys):
    root = str(tmp_path / "kitti")
    seqs = [synthetic_sequence(n_frames=n, n_points=1500, seed=40 + i, n_object=300, speed=0.3 + 0.1 * i, yaw_rate=1.0 + i)
            for i, n in enumerate([8, 6])]
    for f in seqs[1]:
        f["pc"] = PointCloud(f["pc"].points + np.array([[0.0], [12.0], [0.0]], np.float32))
        b = f["3d_bbox"]
        f["3d_bbox"] = Box(b.center + np.array([0.0, 12.0, 0.0]), b.wlh, b.rotation_matrix)
    for t in range(3, 5):                                       # the first car's surroundings are emptied on frames 3 and 4
        p = seqs[0][t]["pc"].points.copy()
        p[:, np.linalg.norm(p[:2] - seqs[0][t]["3d_bbox"].center[:2, None], axis=0) < 6.0] = FAR[:, None]
        seqs[0][t]["pc"] = PointCloud(p)
    _write_scene(root, "0019", [((5, "Pedestrian"), seqs[0]), ((8, "Pedestrian"), seqs[1])], extra_dontcare=False)
    ds = kittiDataset(root, "test", "Pedestrian", preloading=False, preload_offset=-1)
    npts = max(f["pc"].points.shape[1] for t in ds.tracklets() for f in t)
    lines = []
    for t in range(8):
        boxes = [ds.box_from_anno(a) for annos in ds.tracklet_anno_list for a in annos if a["frame"] == t]
        rows = []
        for b in boxes:
            w = np.sqrt(max(1e-12, 1 + np.trace(b.rotation_matrix))) / 2          # the rotation's quaternion (no half turn here)
            q = [w, (b.rotation_matrix[2, 1] - b.rotation_matrix[1, 2]) / (4 * w), (b.rotation_matrix[0, 2] - b.rotation_matrix[2, 0]) / (4 * w),
                 (b.rotation_matrix[1, 0] - b.rotation_matrix[0, 1]) / (4 * w)]
            rows.append(list(b.center) + list(b.wlh) + q + [0.9])
        lines.append({"scene": "0019", "frame": t, "class": "Pedestrian", "boxes": rows})
    (tmp_path / "d.jsonl").write_text("\n".join(json.dumps(l) for l in lines) + "\n")
    cfg_path = os.path.join(ROOT, "cfgs", "M2_track_kitti.yaml")
    base = ["--cfg", cfg_path, "--path", root, "--split", "test", "--max_targets", "3", "--max_points", str(npts), "--lost", "1",
            "3", "--coast", "0.5"]
    plain = track.main(base + ["--out", str(tmp_path / "plain.jsonl")])
    got = track.main(base + ["--out", str(tmp_path / "det.jsonl"), "--detections", str(tmp_path / "d.jsonl"),
                             "--detection_gate", "2.0", "--max_detections", "8"])
    printed = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert "reacquired_at_detection" not in plain and printed["reacquired_at_detection"] == got["reacquired_at_detection"]
    out = [json.loads(l) for l in open(tmp_path / "det.jsonl")]
    targets = [t for l in out for t in l["targets"]]
    assert all("detection" in t and isinstance(t["reacquired"], bool) for t in targets)
    assert sum(t["detection"] is not None for t in targets) > 0
    assert got["reacquired_at_detection"] == sum(t["reacquired"] for t in targets)
