"""Coasting in the live tracker on the GPU: `o3d_track_update` bitwise against its tensor formulation (eager, graph replay, repeat
runs); boxes and evidence unchanged by coasting under a rule that never fires; every record bitwise across occupancy buckets
with a rule that fires; a target coasted through an occlusion and re-acquired (M2-Track, synthetic scene); track_feeds /
track_classes with coasting; the command line with --coast; and the kernels of one coasting replay."""
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
from open3dsot_b200.tracking.multi_class import track_classes
from open3dsot_b200.tracking.multi_tracker import MultiTargetTracker, Slots, coast_weights, track_feeds, track_update
from test_coast import _bits, _formulation, _random_case
from test_gpu_lost_targets import FAR, MODELS, _flat, _model, _scenes
from test_gpu_occupancy import COUNTS, N_POINTS, _drive
from test_kitti_reader import _write_scene

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32


# ------------------------------------------------------------------ the kernel
def _kernel(case, rule, coast):
    state, src, dst, adv, center, rot, points, score = case
    slots = Slots(*(torch.from_numpy(np.array(x, copy=True)).cuda() for x in state))
    args = [torch.from_numpy(x).cuda() for x in (src, dst, adv, center, rot, points, score)]
    return slots, args


@pytest.mark.parametrize("rule,alpha", [(None, None), ((3, 2), None), ((3, 2), 0.3), ((3, 2), 1.0), ((0, 1), 0.5)])
@pytest.mark.parametrize("b", [1, 7, 64, 300])
def test_kernel_equals_the_formulation(b, rule, alpha):
    coast = coast_weights(alpha)
    for seed in range(3):
        case = _random_case(b + 5, b, 100 + seed, rule)
        want = _formulation(*case, rule, coast)
        slots, args = _kernel(case, rule, coast)
        track_update(slots, *args, rule, coast)
        again, args2 = _kernel(case, rule, coast)
        track_update(again, *args2, rule, coast)
        graphed, args3 = _kernel(case, rule, coast)
        init = [x.clone() for x in graphed]
        track_update(graphed, *args3, rule, coast)                            # warm-up outside the capture
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            track_update(graphed, *args3, rule, coast)
        for x, v in zip(graphed, init):
            x.copy_(v)
        g.replay()
        torch.cuda.synchronize()
        for k in Slots._fields:
            w = _bits(getattr(want, k).numpy())
            for got in (slots, again, graphed):
                assert np.array_equal(_bits(getattr(got, k).cpu().numpy()), w), (b, seed, k)


# ------------------------------------------------------------------ the live step: unchanged boxes, records across buckets
@pytest.fixture(scope="module")
def data():
    return [synthetic_scene(n_frames=26, n_points=N_POINTS, n_objects=4, seed=80 + f, extent=14.0) for f in range(3)]


def _run(net, data, precision, lost, coast=None, pinned=False, K=32):
    trk = MultiTargetTracker(net, N_POINTS, K, seed=7, feeds=3, precision=precision, lost=lost, coast=coast)
    if pinned:
        trk._buckets = (K,)
    snap = lambda: torch.cat([trk._record(), trk.vel, trk.hit_c, trk.hit_t.float()[:, None], trk.coasting.float()[:, None]], 1)
    return _drive(trk, data, COUNTS[K], snapshot=snap)[0]


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("cfg_name", MODELS)
def test_coast_is_bitwise_across_buckets_and_changes_nothing_under_a_rule_that_never_fires(cfg_name, precision, data):
    net = _model(cfg_name)
    plain = _run(net, data, precision, None)
    never = _run(net, data, precision, (0, 1), coast=0.5)
    assert sorted(plain) == sorted(never)
    for tid in plain:
        assert np.array_equal(plain[tid][:, :17], never[tid][:, :17], equal_nan=True), tid     # boxes and evidence
        assert not never[tid][:, 17:19].any() and not never[tid][:, -1].any(), tid            # no miss, no loss, no coast
    pts = np.concatenate([r[:, 15] for r in plain.values()])
    rule = (int(np.median(pts[pts >= 0])) + 1, 2)
    fires = _run(net, data, precision, rule, coast=0.5)
    fires_pinned = _run(net, data, precision, rule, coast=0.5, pinned=True)
    for tid in fires:
        assert np.array_equal(fires[tid], fires_pinned[tid], equal_nan=True), tid
    rec = np.concatenate(list(fires.values()))
    assert rec[:, -1].any() and rec[:, 18].any()                              # some frames coasted, some targets lost
    assert np.array_equal(rec[:, -1] != 0, (rec[:, 17] > 0) & (rec[:, 18] == 0))


# ------------------------------------------------------------------ an occlusion on a synthetic scene
T0, PATIENCE, MIN_POINTS, ALPHA = 4, 3, 1, 0.5


def _occluded(sc, obj, t0, g, radius=8.0):
    """The scene's scans with every point within `radius` m of object `obj`'s centre moved far away on frames t0 .. t0 + g - 1."""
    scans = []
    for t, s in enumerate(sc["scans"]):
        s = s.copy()
        if t0 <= t < t0 + g:
            s[np.linalg.norm(s[:, :2] - sc["boxes"][obj][t].center[None, :2], axis=1) < radius] = FAR
        scans.append(s)
    return scans


def _follow(net, scans, boxes, ids, K, coast=ALPHA, sync_free=False):
    """One feed: add `ids` on scan 0 and advance through every scan; {id: (T, 19 + 4) records: _record(), velocity, coasting}."""
    trk = MultiTargetTracker(net, N_POINTS, K, seed=4, lost=(MIN_POINTS, PATIENCE), coast=coast)
    rec = {i: [] for i in ids}

    def record():
        r = torch.cat([trk._record(), trk.vel, trk.coasting.float()[:, None]], 1)
        for i in ids:
            rec[i].append(r[trk.targets()[i]].clone())

    trk.step(torch.from_numpy(scans[0]))
    for i in ids:
        trk.add(i, boxes[i][0])
    record()
    trk.step(torch.from_numpy(scans[1]))                                      # plan and capture: the one sync
    record()
    torch.cuda.synchronize()
    if sync_free:
        torch.cuda.set_sync_debug_mode("error")
    try:
        for t in range(2, len(scans)):
            trk.step(torch.from_numpy(scans[t]))
            record()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    return {i: torch.stack(v).cpu().numpy() for i, v in rec.items()}


def _host_coast(r):
    """Target records (T, 23): the centres a coasting tracker reports, recomputed in float32 from the recorded hit boxes, and the
    velocity after every frame."""
    alpha, beta = (F32(w) for w in coast_weights(ALPHA))
    hit_c, hit_t, vel = r[0, :3].astype(F32), 0, np.zeros(3, F32)
    centres, vels = [hit_c], [vel]
    for t in range(1, len(r)):
        if r[t - 1, 18]:                                                      # lost before: held
            centres.append(centres[-1])
        elif r[t, 15] >= MIN_POINTS:
            v = (r[t, :3] - hit_c) / F32(t - hit_t)
            vel = v if hit_t == 0 else alpha * v + beta * vel
            hit_c, hit_t = r[t, :3].astype(F32), t
            centres.append(hit_c)
        else:
            centres.append(hit_c + vel * F32(t - hit_t))
        vels.append(vel)
    return np.stack(centres), np.stack(vels)


@pytest.fixture(scope="module")
def occlusion():
    # M2-Track: its untrained boxes stay on their objects over this scene (test_gpu_lost_targets.py relies on it too)
    net = _model("M2_track_kitti.yaml")
    sc = synthetic_scene(n_frames=10, n_points=N_POINTS, n_objects=4, seed=300, extent=14.0)
    clean = _follow(net, sc["scans"], sc["boxes"], [0, 1, 2, 3], 8)
    # target 0 is a hit on every frame the occlusion tests look at when nothing is occluded
    assert (clean[0][1:T0 + 6, 15] >= MIN_POINTS).all(), {i: r[:, 15] for i, r in clean.items()}
    return net, sc, clean


def test_an_occluded_target_coasts_and_is_reacquired(occlusion):
    net, sc, clean = occlusion
    g = 2
    scans = _occluded(sc, 0, T0, g)
    got = _follow(net, scans, sc["boxes"], [0, 1, 2, 3], 8, sync_free=True)
    r0 = got[0]
    gap = list(range(T0, T0 + g))
    assert (r0[gap, 15] == 0).all()
    centres, vels = _host_coast(r0)
    assert np.array_equal(_bits(r0[:, :3]), _bits(centres)), (r0[:, :3], centres)
    assert np.array_equal(_bits(r0[:, 19:22]), _bits(vels))
    assert np.array_equal(np.flatnonzero(r0[:, 22]), gap), r0[:, 22]         # coasting exactly on the gap
    assert not r0[:, 18].any()                                                # never lost
    assert list(r0[gap, 17]) == list(range(1, g + 1))
    after = T0 + g
    assert r0[after, 15] >= MIN_POINTS and r0[after, 17] == 0 and r0[after, 22] == 0   # a hit again
    for t in gap:                                                             # coasted rotation: the previous one
        assert np.array_equal(r0[t, 6:15], r0[t - 1, 6:15])
    assert np.array_equal(r0[:T0], clean[0][:T0], equal_nan=True)             # before the gap: the clean run
    for i in (1, 2, 3):
        assert np.array_equal(got[i], clean[i], equal_nan=True), i
    alone = _follow(net, scans, sc["boxes"], [0], 1)
    assert np.array_equal(alone[0], r0, equal_nan=True)


def test_an_occlusion_past_patience_is_lost_holding_the_coasted_box(occlusion):
    net, sc, _ = occlusion
    scans = _occluded(sc, 0, T0, 4)
    r0 = _follow(net, scans, sc["boxes"], [0, 1], 2)[0]
    lost_at = T0 + PATIENCE - 1
    assert not r0[:lost_at, 18].any() and r0[lost_at:, 18].all(), r0[:, 17:]
    assert np.array_equal(np.flatnonzero(r0[:, 22]), np.arange(T0, lost_at))
    centres, _ = _host_coast(r0)
    assert np.array_equal(_bits(r0[:, :3]), _bits(centres))                  # the loss frame's box is the coasted one
    assert (r0[lost_at:] == r0[lost_at]).all()                                # held from the loss on


# ------------------------------------------------------------------ track_feeds and track_classes with coasting
def test_track_feeds_coasts_through_misses_and_ends_at_the_loss():
    net = _model("M2_track_kitti.yaml")
    scenes = _scenes()
    free = _flat(track_feeds(net, scenes, 2, 6, seed=3, max_points=3000))
    cut, cut_ev = track_feeds(net, scenes, 2, 6, seed=3, max_points=3000, lost=(1, 2), evidence=True)
    co, co_ev = track_feeds(net, scenes, 2, 6, seed=3, max_points=3000, lost=(1, 2), coast=0.5, evidence=True)
    cut, co = _flat(cut), _flat(co)
    cut_ev = {tid: tr for scene in cut_ev for tid, tr in scene.items()}
    co_ev = {tid: tr for scene in co_ev for tid, tr in scene.items()}
    assert all(len(e) == 2 for tr in cut_ev.values() for e in tr.values())  # no coast: the evidence as it was
    coasted = 0
    for tid in free:
        frames = sorted(co[tid])
        assert frames == sorted(free[tid])[:len(frames)], tid
        assert sorted(co_ev[tid]) == frames
        flags = [co_ev[tid][t][2] for t in frames]
        coasted += sum(flags)
        assert all(co_ev[tid][t][0] < 1 for t in frames if co_ev[tid][t][2])   # a coasted frame is a miss
        first_miss = next((t for t in frames[1:] if co_ev[tid][t][0] < 1), None)
        for t in frames:                                                      # up to the first miss: the lost-only run
            if first_miss is not None and t >= first_miss:
                break
            assert np.array_equal(co[tid][t], cut[tid][t]), (tid, t)
        if len(frames) < len(free[tid]):                                      # ended at the loss: two misses in a row
            assert [co_ev[tid][t][0] < 1 for t in frames[-2:]] == [True, True] and flags[-2:] == [True, False], tid
    assert len(co[0]) < len(free[0])                                         # the emptied target still ends
    assert coasted > 0


def test_track_classes_coasting_classes_are_lone_trackers():
    models = {"car": _model("BAT_Car.yaml"), "ped": _model("M2_track_kitti.yaml")}
    scenes = _scenes()
    rules, coasts = {"car": (1, 2), "ped": (30, 3)}, {"ped": 0.5}
    cls_scenes = [{"frames": s["frames"], "scan": s["scan"], "ends": {(c, tid): e for tid, e in s["ends"].items() for c in models},
                   "starts": {t: [((c, tid), b) for tid, b in g for c in models] for t, g in s["starts"].items()}} for s in scenes]
    both, both_ev = track_classes(models, cls_scenes, 2, {"car": 8, "ped": 8}, seed=3, max_points=3000, lost=rules,
                                  coast=coasts, evidence=True)
    both = _flat(both)
    both_ev = {key: tr for scene in both_ev for key, tr in scene.items()}
    for c in models:
        alone, alone_ev = track_feeds(models[c], scenes, 2, 8, seed=3, max_points=3000, lost=rules[c], coast=coasts.get(c),
                                      evidence=True)
        alone = _flat(alone)
        alone_ev = {tid: tr for scene in alone_ev for tid, tr in scene.items()}
        for tid in alone:
            assert sorted(both[(c, tid)]) == sorted(alone[tid]), (c, tid)
            for t in alone[tid]:
                assert np.array_equal(both[(c, tid)][t], alone[tid][t]), (c, tid, t)
                a, b = both_ev[(c, tid)][t], alone_ev[tid][t]
                assert len(a) == len(b) == (3 if c == "ped" else 2)
                assert a[0] == b[0] and a[2:] == b[2:] and (a[1] == b[1] or (np.isnan(a[1]) and np.isnan(b[1]))), (c, tid, t)
    assert any(e[2] for key, tr in both_ev.items() if key[0] == "ped" for e in tr.values())


# ------------------------------------------------------------------ the command line
def test_command_line_with_coast(tmp_path, capsys):
    root = str(tmp_path / "kitti")
    seqs = [synthetic_sequence(n_frames=n, n_points=1500, seed=40 + i, n_object=300, speed=0.3 + 0.1 * i, yaw_rate=1.0 + i)
            for i, n in enumerate([8, 6])]
    for f in seqs[1]:                                           # the second car drives 12 m to the left
        f["pc"] = PointCloud(f["pc"].points + np.array([[0.0], [12.0], [0.0]], np.float32))
        b = f["3d_bbox"]
        f["3d_bbox"] = Box(b.center + np.array([0.0, 12.0, 0.0]), b.wlh, b.rotation_matrix)
    for t in range(3, 8):                                       # the first car's surroundings are emptied from frame 3 on
        p = seqs[0][t]["pc"].points.copy()
        p[:, np.linalg.norm(p[:2] - seqs[0][t]["3d_bbox"].center[:2, None], axis=0) < 6.0] = FAR[:, None]
        seqs[0][t]["pc"] = PointCloud(p)
    _write_scene(root, "0019", [((5, "Pedestrian"), seqs[0]), ((8, "Pedestrian"), seqs[1])], extra_dontcare=False)
    ds = kittiDataset(root, "test", "Pedestrian", preloading=False, preload_offset=-1)
    npts = max(f["pc"].points.shape[1] for t in ds.tracklets() for f in t)
    cfg_path = os.path.join(ROOT, "cfgs", "M2_track_kitti.yaml")
    base = ["--cfg", cfg_path, "--path", root, "--split", "test", "--max_targets", "3", "--max_points", str(npts), "--lost", "1",
            "3"]
    plain = track.main(base + ["--out", str(tmp_path / "plain.jsonl")])
    got = track.main(base + ["--out", str(tmp_path / "coast.jsonl"), "--coast", "0.5"])
    printed = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert "coasted" not in plain and "reacquired" not in plain and "lost" in plain
    assert printed["coasted"] == got["coasted"] and printed["reacquired"] == got["reacquired"]
    plain_lines = [json.loads(l) for l in open(tmp_path / "plain.jsonl")]
    lines = [json.loads(l) for l in open(tmp_path / "coast.jsonl")]
    assert all("coasting" not in t for l in plain_lines for t in l["targets"])
    assert all(isinstance(t["coasting"], bool) for l in lines for t in l["targets"])
    by = {(l["frame"], t["id"]): t for l in lines for t in l["targets"]}
    assert got["coasted"] == sum(t["coasting"] for t in by.values()) >= 1, by
    ends_in_hit = [(f, i) for (f, i), t in by.items() if t["coasting"] and (f + 1, i) in by and not by[(f + 1, i)]["coasting"]
                   and by[(f + 1, i)]["points"] >= 1]
    assert got["reacquired"] == len(ends_in_hit)
    assert all(not t["coasting"] for l in lines if l["frame"] < 3 for t in l["targets"])
    for l, pl in zip(lines, plain_lines):                                     # before the occlusion: the run without --coast
        if l["frame"] < 3:
            assert [{k: v for k, v in t.items() if k != "coasting"} for t in l["targets"]] == pl["targets"]


# ------------------------------------------------------------------ the kernels of one replay (child process, as in
# test_gpu_occupancy.py: a CUPTI session around a graph replay in the suite's process spoils later profiler-based tests)
_PROFILE_CHILD = r"""
import json, os, sys
import torch
sys.path.insert(0, sys.argv[1])
from open3dsot_b200.config import load_config
from open3dsot_b200.datasets.synthetic import synthetic_scene
from open3dsot_b200.models import get_model
from open3dsot_b200.tracking.multi_tracker import MultiTargetTracker
cfg = load_config(os.path.join(sys.argv[1], "cfgs", "BAT_Car.yaml"), {"up_axis": [0, 0, 1]})
torch.manual_seed(0)
net = get_model(cfg.net_model)(cfg).cuda().eval()
sc = synthetic_scene(n_frames=6, n_points=6000, n_objects=3, seed=900, extent=15.0)
trk = MultiTargetTracker(net, 6000, 8, seed=2, lost=(5, 3), coast=0.5)
scans = [torch.from_numpy(s).cuda() for s in sc["scans"]]
trk.step(scans[0])
for j in range(3):
    trk.add(j, sc["boxes"][j][0])
trk.step(scans[1])
torch.cuda.synchronize()
names = []
for t in (2, 3):                                   # CUPTI now and then delivers no records for a short session
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        trk.step(scans[t])
        torch.cuda.synchronize()
    prof.export_chrome_trace(sys.argv[2] + "/step.json")
    names = [e["name"] for e in json.load(open(sys.argv[2] + "/step.json"))["traceEvents"] if e.get("cat") == "kernel"]
    if names:
        break
print(json.dumps(names))
"""


def test_one_coasting_replay_writes_back_in_one_kernel(tmp_path):
    r = subprocess.run([sys.executable, "-c", _PROFILE_CHILD, ROOT, str(tmp_path)], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    names = json.loads(r.stdout.strip().splitlines()[-1])
    count = collections.Counter(names)
    assert sum(v for k, v in count.items() if "track_update_kernel" in k) == 1, names
    assert not [k for k in count if "index_copy" in k], names
    assert any("box_points_kernel" in k for k in count), names
