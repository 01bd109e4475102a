"""Target births in the live tracker on the GPU: `o3d_track_birth` bitwise against its formulation (eager, repeated, graph
replay); births that never happen change no box, evidence, record or `unmatched()` result; a tracker with births equals one
that add()s the same detections after every advance, boxes, evidence and first-frame crops; no host sync; scarce slots; two
classes as lone trackers; a first scan without targets; the kernels of one replay."""
import collections
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from open3dsot_b200.datasets.data_classes import Box
from open3dsot_b200.tracking.multi_class import MultiClassTracker
from open3dsot_b200.tracking.multi_tracker import BIRTH_ID_BASE, BirthSlots, MultiTargetTracker, detection_gate2, detection_rows
from test_births import birth_case, check_case, run_births
from test_coast import _bits
from test_gpu_associate import _near
from test_gpu_lost_targets import MODELS, _model
from test_gpu_occupancy import COUNTS, HOLD, N_POINTS

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32


def _same(a, b, what):
    a, b = a.cpu().numpy(), b.cpu().numpy()
    assert np.array_equal(_bits(a), _bits(b)), what


# ------------------------------------------------------------------ the kernel against its formulation
@pytest.mark.parametrize("F", [1, 16])
@pytest.mark.parametrize("D", [1, 64, 1024])
@pytest.mark.parametrize("R", ["1", "per_scan", "K"])
def test_birth_kernel_equals_the_formulation(F, D, R):
    K, b, per = 128, 96, 8
    born = 0
    for seed in range(2):
        case = birth_case(K, b, F, D, 400 + seed, per=per, grid=seed == 1)
        R_n = {"1": 1, "per_scan": per, "K": K}[R]
        bl = case[-1]
        if bl.shape[1] < R_n:                                                  # pad the birth list to R entries
            bl = np.concatenate([bl, np.array([[K] * (R_n - bl.shape[1]), [-1] * (R_n - bl.shape[1])])], 1)
        else:
            keep = bl[:, :R_n].copy()
            bl = keep
        case = case[:-1] + (bl,)
        gate2, axes = detection_gate2(2.0), ((0, 1), (0, 2))[seed]
        want = check_case(case, K, gate2, axes, 0.5, n0=3)                    # the formulation, checked against the loop
        born += len(want)
        w_slots, w_rec, w_next, w_log = run_births(case, K, gate2, axes, 0.5, n0=3)
        runs = [run_births(case, K, gate2, axes, 0.5, n0=3, device="cuda") for _ in range(2)]   # eager, then again
        feed, adv, pred, fed, count, det, rec_slot, bl = case
        T = lambda x: torch.from_numpy(np.array(x, copy=True)).cuda()
        from test_births import _slots
        from open3dsot_b200.tracking import multi_tracker as mt
        slots = BirthSlots(*(x.cuda() for x in _slots(K, 0)))
        init = [x.clone() for x in slots]
        args = [T(x) for x in (feed, adv, pred, fed, count, det)]
        rec, nxt, blt = T(rec_slot), torch.tensor([3], device="cuda"), T(bl)
        log = torch.zeros(bl.shape[1], 4, dtype=torch.int64, device="cuda")
        fn = lambda: mt.track_birth(*args, rec, blt, nxt, log, slots, gate2, axes, 0.5)
        fn()                                                                  # warm-up outside the capture
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            fn()
        for x, v in zip(slots, init):
            x.copy_(v)
        rec.copy_(T(rec_slot))
        nxt.fill_(3)
        g.replay()
        runs.append((slots, rec, nxt, log))
        torch.cuda.synchronize()
        for s, r, n, l in runs:
            for name, w, x in zip(BirthSlots._fields, w_slots, s):
                _same(x, w, (F, D, R, seed, name))
            assert torch.equal(r.cpu(), w_rec) and torch.equal(n.cpu(), w_next) and torch.equal(l.cpu(), w_log)
    assert born > 0 or D == 1


# ------------------------------------------------------------------ the live step
@pytest.fixture(scope="module")
def data():
    from open3dsot_b200.datasets.synthetic import synthetic_scene
    return [synthetic_scene(n_frames=26, n_points=N_POINTS, n_objects=4, seed=80 + f, extent=14.0) for f in range(3)]


def _drive_run(net, data, precision, births, K=12, gate=2.0, lost=(3, 2), tracked_only=False):
    """test_gpu_occupancy's schedule over K slots (its at most 4 targets, plus the slots a per_scan = 1 rule keeps pending: 3
    feeds, BIRTH_LAG advances), dropping the oldest targets (lowest ids) rather than those in the lowest slots, since a tracker
    with births gives add() other slots.  Every fed feed gets detections near its objects (`tracked_only`: only a feed with a
    target).  Returns {id: records} and the last unmatched()."""
    trk = MultiTargetTracker(net, N_POINTS, K, seed=7, feeds=3, precision=precision, lost=lost, detections=(16, gate),
                             births=births)
    seen, nxt, rec = [0, 0, 0], 0, {}
    for s, c in enumerate(COUNTS[4]):
        tracked = set(trk._feed_of.values())
        for f in sorted(f for f in range(3) if f not in HOLD.get(s, ())):
            dets = _near(data, f, seen[f]) if f in tracked or not tracked_only else np.zeros((0, 16), F32)
            trk.put(f, data[f]["scans"][seen[f]], detections=dets)
            seen[f] += 1
        trk.advance()
        snap = torch.cat([trk._record(), trk._match_record()], 1)
        for tid, k in trk.targets().items():
            rec.setdefault(tid, []).append(snap[k].clone())
        live = sorted(trk.targets())
        for tid in live[:max(0, len(live) - c)]:
            trk.drop(tid)
        while len(trk.targets()) < c:
            f = nxt % 3
            trk.add(nxt, data[f]["boxes"][nxt % 4][seen[f] - 1], feed=f)
            nxt += 1
    return {tid: torch.stack(v).cpu().numpy() for tid, v in rec.items()}, trk.unmatched()


def _same_runs(a, b):
    (ra, ua), (rb, ub) = a, b
    assert sorted(ra) == sorted(rb)
    for tid in ra:
        assert np.array_equal(_bits(ra[tid]), _bits(rb[tid])), tid
    assert sorted(ua) == sorted(ub)
    for f in ua:
        assert [(d, s) for d, _, s in ua[f]] == [(d, s) for d, _, s in ub[f]]
        for (_, x, _), (_, y, _) in zip(ua[f], ub[f]):
            assert np.array_equal(x.center, y.center) and np.array_equal(x.rotation_matrix, y.rotation_matrix)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("cfg_name", MODELS)
def test_births_that_never_happen_change_nothing(cfg_name, precision, data):
    net = _model(cfg_name)
    # every score is below min_score
    _same_runs(_drive_run(net, data, precision, None), _drive_run(net, data, precision, (2.0, 1)))
    # every detection within the gate of a row of its feed: only feeds with targets (none lost) get detections, wide gate
    kw = dict(gate=50.0, lost=None, tracked_only=True)
    plain = _drive_run(net, data, precision, None, **kw)
    _same_runs(plain, _drive_run(net, data, precision, (0.0, 1), **kw))
    assert sum((r[:, 19] >= 0).sum() for r in plain[0].values()) > 0


def _staggered(data, f, t):
    """Feed f's detections on scan t: none on some scans, the objects' boxes with noise (and a false positive) on others."""
    if (t + f) % 3 == 2:
        return np.zeros((0, 16), F32)
    rows = _near(data, f, t, noise=0.3)
    fp = detection_rows([Box(np.array([30.0 + t, -30.0 + f, 0.0]), np.array([1.6, 4.0, 1.5]), np.eye(3))], [0.95])
    return np.concatenate([rows[:1 + (t % 4)], fp])


def _born_vs_added(net, data, precision, n_adv=9, K=16):
    kw = dict(seed=7, feeds=3, precision=precision, lost=(3, 3), coast=0.5, detections=(16, 2.0))
    born = MultiTargetTracker(net, N_POINTS, K, births=(0.2, 2), **kw)
    added = MultiTargetTracker(net, N_POINTS, K, **kw)
    recs = {"born": {}, "added": {}}
    prefix = {}
    all_births = []
    for t in range(n_adv):
        dets = {f: _staggered(data, f, t) for f in range(3)}
        for trk in (born, added):
            for f in range(3):
                trk.put(f, data[f]["scans"][t], detections=dets[f])
            trk.advance()
        new = born.births(wait=True)
        all_births += new
        for tid, f, k, d in new:
            r = dets[f][d]
            added.add(tid, Box(r[0:3].astype(np.float64), r[3:6].astype(np.float64), r[6:15].reshape(3, 3).astype(np.float64)),
                      feed=f)
        for name, trk in (("born", born), ("added", added)):
            snap = torch.cat([trk._record(), trk._match_record(), trk.vel, trk.hit_c, trk.t.float()[:, None]], 1)
            for tid, k in trk.targets().items():
                recs[name].setdefault(tid, []).append(snap[k].clone())
                if trk.mode in ("firstandprevious", "first"):
                    prefix.setdefault((name, tid), (trk.first_local[k].clone(), trk.first_keep[k].clone()))
    return all_births, recs, prefix


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("cfg_name", MODELS)
def test_births_equal_add_after_every_advance(cfg_name, precision, data):
    net = _model(cfg_name)
    births, recs, prefix = _born_vs_added(net, data, precision)
    assert len(births) >= 6 and len({f for _, f, _, _ in births}) == 3
    assert [tid for tid, *_ in births] == [BIRTH_ID_BASE + n for n in range(len(births))]
    assert sorted(recs["born"]) == sorted(recs["added"])
    for tid in recs["born"]:
        a, b = torch.stack(recs["born"][tid]).cpu().numpy(), torch.stack(recs["added"][tid]).cpu().numpy()
        assert np.array_equal(_bits(a), _bits(b)), tid
    for (name, tid), (local, keep) in prefix.items():
        if name == "born":
            l2, k2 = prefix[("added", tid)]
            assert torch.equal(keep, k2) and np.array_equal(_bits(local.cpu().numpy()), _bits(l2.cpu().numpy())), tid


def _stream(net, data, sync, debug=False, K=16):
    trk = MultiTargetTracker(net, N_POINTS, K, seed=7, feeds=3, lost=(3, 3), detections=(16, 2.0), births=(0.2, 2))
    births, boxes = [], []
    dets = [{f: _staggered(data, f, t) for f in range(3)} for t in range(10)]
    for t in range(10):
        if t == 2 and debug:
            torch.cuda.set_sync_debug_mode("error")
        try:
            for f in range(3):
                trk.put(f, data[f]["scans"][t], detections=dets[t][f])
            trk.advance()
            births += trk.births()
            boxes.append(torch.cat([trk.snapshot(), trk.key.float()[:, None], trk.active.float()[:, None]], 1))
        finally:
            torch.cuda.set_sync_debug_mode(0)
        if sync:
            torch.cuda.synchronize()
    births += trk.births(wait=True)
    return births, torch.stack(boxes).cpu().numpy()


def test_no_host_sync_and_the_same_births_however_far_the_device_lags(data):
    net = _model("BAT_Car.yaml")
    free, free_boxes = _stream(net, data, sync=False, debug=True)
    synced, synced_boxes = _stream(net, data, sync=True)
    assert len(free) > 0 and free == synced
    assert np.array_equal(_bits(free_boxes), _bits(synced_boxes))


def test_scarce_slots_take_the_top_ranked_candidates(data):
    net = _model("M2_track_kitti.yaml")
    trk = MultiTargetTracker(net, N_POINTS, 3, seed=4, detections=(16, 2.0), births=(0.0, 8))
    boxes = [Box(np.array([6.0 * i - 20.0, 25.0, 0.0]), np.array([1.6, 4.0, 1.5]), np.eye(3)) for i in range(6)]
    scores = [0.2, 0.9, 0.4, 0.9, 0.7, 0.1]
    trk.put(0, data[0]["scans"][0], detections=detection_rows(boxes, scores))
    trk.advance()
    got = trk.births(wait=True)
    assert [(tid - BIRTH_ID_BASE, d) for tid, _, _, d in got] == [(0, 1), (1, 3), (2, 4)]
    assert [d for d, _, _ in trk.unmatched()[0]] == [0, 2, 5]
    trk.drop(BIRTH_ID_BASE + 1)
    far = Box(np.array([40.0, 40.0, 0.0]), np.array([1.6, 4.0, 1.5]), np.eye(3))          # beyond every target's gate
    trk.put(0, data[0]["scans"][1], detections=detection_rows([far], [0.5]))
    trk.advance()
    assert [(tid - BIRTH_ID_BASE, d) for tid, _, _, d in trk.births(wait=True)] == [(3, 0)]


def test_a_first_scan_starts_targets_through_the_birth_only_graph(data):
    net = _model("P2B_Car.yaml")
    trk = MultiTargetTracker(net, N_POINTS, 8, seed=4, feeds=2, detections=(16, 2.0), births=(0.0, 4))
    trk.put(0, data[0]["scans"][0], detections=_near(data, 0, 0))
    trk.put(1, data[1]["scans"][0])
    trk.advance()
    assert trk._birth_graph is not None and trk.targets() == {}
    got = trk.births(wait=True)
    assert 1 <= len(got) <= 4 and {f for _, f, _, _ in got} == {0}
    ids = trk.boxes()["ids"].cpu().numpy()
    for tid, f, k, d in got:
        assert ids[k] == tid and np.array_equal(trk.box_c[k].cpu().numpy(), _near(data, 0, 0)[d, :3])
        assert trk.first_keep[k].any()


def test_classes_with_births_are_lone_trackers(data):
    models = {"car": _model("BAT_Car.yaml"), "ped": _model("M2_track_kitti.yaml")}
    rules = {"car": (0.2, 2), "ped": (0.5, 1)}
    gates = {"car": 2.0, "ped": 3.0}

    def drive(put, advance, births, record):
        out, recs = [], []
        for t in range(8):
            for f in range(3):
                put(f, data[f]["scans"][t], {c: _staggered(data, f, t + j) for j, c in enumerate(models)})
            advance()
            out.append(births())
            recs.append(record())
        return out, torch.stack(recs).cpu().numpy()

    mc = MultiClassTracker(models, N_POINTS, {"car": 8, "ped": 8}, feeds=3, seed=7, lost=(3, 3),
                           detections={c: (16, g) for c, g in gates.items()}, births=rules)
    both_b, both = drive(lambda f, s, d: mc.put(f, s, detections=d), mc.advance, mc.births,
                         lambda: torch.cat([mc._record(), mc._match_record()], 1))
    for j, c in enumerate(models):
        trk = MultiTargetTracker(models[c], N_POINTS, 8, seed=7, feeds=3, lost=(3, 3), detections=(16, gates[c]), births=rules[c])
        alone_b, alone = drive(lambda f, s, d: trk.put(f, s, detections=d[c]), trk.advance, trk.births,
                               lambda: torch.cat([trk._record(), trk._match_record()], 1))
        assert [b[c] for b in both_b] == alone_b, c
        assert np.array_equal(both[:, 8 * j:8 * j + 8], alone, equal_nan=True), c
        assert sum(len(b) for b in alone_b) > 0


# ------------------------------------------------------------------ the kernels of one replay (child process)
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
trk = MultiTargetTracker(net, 6000, 8, seed=2, lost=(5, 3), coast=0.5, detections=(64, 2.0), births=(0.3, 2))
scans = [torch.from_numpy(s).cuda() for s in sc["scans"]]
dets = lambda t: detection_rows([sc["boxes"][o][t] for o in range(3)], [0.5] * 3)
trk.put(0, scans[0], detections=dets(0)); trk.advance()
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


def test_one_replay_starts_targets_in_one_kernel(tmp_path):
    r = subprocess.run([sys.executable, "-c", _PROFILE_CHILD, ROOT, str(tmp_path)], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    names = json.loads(r.stdout.strip().splitlines()[-1])
    count = collections.Counter(names)
    assert sum(v for k, v in count.items() if "birth_kernel" in k) == 1, names
    assert sum(v for k, v in count.items() if "associate_kernel" in k) == 1, names
    assert sum(v for k, v in count.items() if "track_update_kernel" in k) == 1, names
