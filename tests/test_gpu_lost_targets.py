"""Evidence and lost targets of the live tracker on the GPU: `o3d_box_points` exactly against its tensor formulation (shapes,
counts, shared scans, rotated boxes, points on the faces, repeat runs, graph replay) and within face-rounding of the fp64 oracle;
boxes unchanged by a rule that never fires; evidence and loss decisions bitwise across occupancy buckets, K and the other
targets; the rule on a synthetic scene; track_feeds / track_classes with rules; and the command line with --lost."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import tracking_ref as R
from open3dsot_b200 import ops, track
from open3dsot_b200.config import load_config
from open3dsot_b200.datasets.data_classes import Box, PointCloud
from open3dsot_b200.datasets.kitti import kittiDataset
from open3dsot_b200.datasets.synthetic import synthetic_scene, synthetic_sequence
from open3dsot_b200.models import get_model
from open3dsot_b200.tracking import boxes as bx
from open3dsot_b200.tracking.multi_class import track_classes
from open3dsot_b200.tracking.multi_tracker import EVIDENCE_WLH_FACTOR, MultiTargetTracker, track_feeds
from test_gpu_occupancy import COUNTS, N_POINTS, _drive
from test_kitti_reader import _write_scene

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODELS = ["BAT_Car.yaml", "P2B_Car.yaml", "M2_track_kitti.yaml"]
FAR = np.array([500.0, 500.0, -100.0], np.float32)        # where "removed" points go: indices, and so every draw, stay put


def _model(cfg_name):
    cfg = load_config(os.path.join(ROOT, "cfgs", cfg_name), {"up_axis": [0, 0, 1], "degrees": True})
    torch.manual_seed(0)
    return get_model(cfg.net_model)(cfg).cuda().eval()


# ------------------------------------------------------------------ the kernel
def _rot(yaw, pitch=0.0):
    rz = np.array([[np.cos(yaw), -np.sin(yaw), 0], [np.sin(yaw), np.cos(yaw), 0], [0, 0, 1]])
    ry = np.array([[np.cos(pitch), 0, np.sin(pitch)], [0, 1, 0], [-np.sin(pitch), 0, np.cos(pitch)]])
    return rz @ ry


def _kernel_inputs(K, N, seed):
    """4 scans (counts 0, 1, N // 3, N) shared by the rows (row k reads scan k % 4); rotated boxes, except rows 3, 11, 19, .., an
    axis-aligned box (yaw 0 or 90 degrees, exact in fp32) at the origin with scan points planted exactly on its faces."""
    g = torch.Generator().manual_seed(seed)
    scans = torch.rand(4, N, 3, generator=g) * 16 - 8
    count = torch.tensor([0, 1, N // 3, N])
    frame = torch.arange(K) % 4
    rng = np.random.default_rng(seed)
    rot = np.stack([_rot(rng.uniform(-np.pi, np.pi), rng.uniform(-0.2, 0.2)) for _ in range(K)])
    center = rng.uniform(-3, 3, (K, 3))
    half = rng.uniform(1.0, 5.0, (K, 3))
    planted = 0
    for k in range(3, K, 8):                                                  # rows of scan 3, whose count is N
        rot[k] = np.eye(3) if k % 16 == 3 else np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])
        center[k] = 0.0
        half[k] = [1.5, 0.75, 0.5]
        h = half[k] if k % 16 == 3 else np.array([0.75, 1.5, 0.5])          # the faces in the scan's frame
        faces = np.array([[sx * h[0], sy * h[1] * 0.5, sz * h[2]] for sx in (-1, 1) for sy in (-1, 1) for sz in (-1, 1)]
                         + [[0.0, h[1], 0.0], [0.0, -h[1], 0.0]], np.float32)
        at = 100 + 20 * planted
        scans[frame[k], at:at + len(faces)] = torch.from_numpy(faces)
        planted += 1
    t = lambda a: torch.tensor(a, dtype=torch.float32)
    return scans, count, frame, t(center), t(rot), t(half)


def _both(scans, count, frame, center, rot, half):
    dev = [x.cuda() for x in (scans, count, frame, center, rot, half)]
    got = ops.box_points(*dev)
    want = bx.box_point_counts(scans, count, frame, center, rot, half)
    return got, want, dev


@pytest.mark.parametrize("N", [60_000, 120_000])
@pytest.mark.parametrize("K", [1, 7, 64, 300])
def test_kernel_equals_the_tensor_formulation(K, N):
    scans, count, frame, center, rot, half = _kernel_inputs(K, N, 11 + K)
    got, want, dev = _both(scans, count, frame, center, rot, half)
    assert got.dtype == torch.int32 and got.shape == (K,)
    assert torch.equal(got.cpu(), want), (got.cpu() - want).abs().max()
    c = want.numpy()
    assert (c[frame.numpy() == 0] == 0).all() and (c[frame.numpy() == 1] <= 1).all()
    if K >= 7:
        assert (c[frame.numpy() >= 2] > 0).all()                              # boxes that hold points
    for k in range(3, K, 8):                                                  # points exactly on the faces count
        assert c[k] >= 10, (k, c[k])
    again = ops.box_points(*dev)
    assert torch.equal(again, got)


def test_face_points_count_and_just_outside_do_not():
    scans = torch.zeros(1, 8, 3)
    scans[0, :4] = torch.tensor([[1.5, 0.75, 0.5], [-1.5, -0.75, -0.5], [1.5, 0.0, 0.0], [0.0, 0.0, 0.0]])
    scans[0, 4:] = torch.tensor([[np.nextafter(np.float32(1.5), np.float32(2)), 0.0, 0.0], [0.0, -0.75000006, 0.0],
                                 [0.0, 0.0, 0.50000006], [9.0, 9.0, 9.0]])
    args = (scans, torch.tensor([8]), torch.zeros(1, dtype=torch.int64), torch.zeros(1, 3), torch.eye(3)[None],
            torch.tensor([[1.5, 0.75, 0.5]]))
    got, want, _ = _both(*args)
    assert int(got) == int(want) == 4


def test_graph_replay_equals_the_eager_call():
    scans, count, frame, center, rot, half = (x.cuda() for x in _kernel_inputs(64, 60_000, 5))
    eager = ops.box_points(scans, count, frame, center, rot, half)
    out = torch.full((64,), 12345, dtype=torch.int32, device="cuda")
    ops.box_points(scans, count, frame, center, rot, half, out=out)             # warm-up outside the capture
    out.fill_(777)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ops.box_points(scans, count, frame, center, rot, half, out=out)
    for _ in range(3):                                                        # the memset inside the graph zeroes every replay
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, eager)


def test_kernel_against_the_fp64_oracle():
    scans, count, frame, center, rot, half = _kernel_inputs(7, 60_000, 3)
    got = ops.box_points(*(x.cuda() for x in (scans, count, frame, center, rot, half))).cpu().numpy()
    near_total = 0
    for k in range(7):
        n = int(min(count[frame[k]], scans.shape[1]))
        pts = scans[frame[k], :n].double().numpy()
        h = half[k].double().numpy()
        box = R.Box(center[k].double().numpy(), np.array([2 * h[1], 2 * h[0], 2 * h[2]]), rot[k].double().numpy())
        want = int(R._in_box_inclusive(pts, box, 1.0).sum())
        local = (pts - box.center) @ box.rot
        near = int((np.abs(np.abs(local) - h) < 1e-5).any(1).sum())
        near_total += near
        assert abs(int(got[k]) - want) <= near, (k, got[k], want, near)
    print(f"points within 1e-5 m of a face: {near_total}")


# ------------------------------------------------------------------ the live step: unchanged boxes, evidence across buckets
@pytest.fixture(scope="module")
def data():
    return [synthetic_scene(n_frames=26, n_points=N_POINTS, n_objects=4, seed=80 + f, extent=14.0) for f in range(3)]


def _run(net, data, precision, lost, pinned=False, K=32):
    trk = MultiTargetTracker(net, N_POINTS, K, seed=7, feeds=3, precision=precision, lost=lost)
    if pinned:
        trk._buckets = (K,)
    return _drive(trk, data, COUNTS[K], snapshot=trk._record)[0]


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("cfg_name", MODELS)
def test_rule_that_never_fires_changes_no_box_and_evidence_is_bitwise_across_buckets(cfg_name, precision, data):
    net = _model(cfg_name)
    plain = _run(net, data, precision, None)
    never = _run(net, data, precision, (0, 1))
    pinned = _run(net, data, precision, (0, 1), pinned=True)
    assert sorted(plain) == sorted(never) == sorted(pinned)
    for tid in plain:
        assert np.array_equal(plain[tid][:, :15], never[tid][:, :15]), tid            # boxes
        assert np.array_equal(plain[tid][:, 15:17], never[tid][:, 15:17], equal_nan=True), tid
        assert np.array_equal(never[tid], pinned[tid], equal_nan=True), tid             # evidence at every bucket
        assert not never[tid][:, 18].any()
    pts = np.concatenate([r[:, 15] for r in plain.values()])
    score = np.concatenate([r[:, 16] for r in plain.values()])
    assert (pts > 0).any() and np.isfinite(score).any()
    if cfg_name.startswith("M2"):
        s = score[np.isfinite(score)]
        assert ((s >= 0) & (s <= 1)).all()
    # a rule that fires (below the median count, twice in a row): its decisions are the same at every bucket
    rule = (int(np.median(pts[pts >= 0])) + 1, 2)
    fires = _run(net, data, precision, rule)
    fires_pinned = _run(net, data, precision, rule, pinned=True)
    for tid in fires:
        assert np.array_equal(fires[tid], fires_pinned[tid], equal_nan=True), tid
    assert any(r[:, 18].any() for r in fires.values())


# ------------------------------------------------------------------ the rule on a synthetic scene
T0, PATIENCE, MIN_POINTS = 4, 3, 1


def _emptied(sc, obj, t0, radius=8.0):
    """The scene's scans with every point within `radius` m of object `obj`'s centre moved far away from frame t0 on."""
    scans = []
    for t, s in enumerate(sc["scans"]):
        s = s.copy()
        if t >= t0:
            near = np.linalg.norm(s[:, :2] - sc["boxes"][obj][t].center[None, :2], axis=1) < radius
            s[near] = FAR
        scans.append(s)
    return scans


def _follow(net, scans, boxes, ids, K, lost, check_points=False, sync_free=False):
    """One feed: add `ids` (object i) on scan 0, advance through every scan; returns {id: (T, 19) records} and the tracker."""
    trk = MultiTargetTracker(net, N_POINTS, K, seed=4, lost=lost)
    dev = [torch.from_numpy(s) for s in scans]
    trk.step(dev[0])
    for i in ids:
        trk.add(i, boxes[i][0])
    rec = {i: [trk._record()[trk.targets()[i]].clone()] for i in ids}
    if sync_free:
        trk.step(dev[1])                                                      # plan and capture: the one sync
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        for i in ids:
            rec[i].append(trk._record()[trk.targets()[i]].clone())
    try:
        for t in range(2 if sync_free else 1, len(scans)):
            trk.step(dev[t])
            r = trk._record()
            for i in ids:
                rec[i].append(r[trk.targets()[i]].clone())
            if check_points:                                                  # points: the formulation on the returned box
                cur = trk.scan_feeds.fcur[0]
                k = torch.tensor([trk.targets()[i] for i in ids], device="cuda")
                adv = torch.tensor([not bool(rec[i][-2][18]) for i in ids])   # not lost before this advance
                want = bx.box_point_counts(trk.scans[0, cur][None].cpu(), trk.count[0, cur][None].cpu(),
                                           torch.zeros(len(ids), dtype=torch.int64), trk.box_c[k].cpu(), trk.box_r[k].cpu(),
                                           bx.inclusive_half(trk.box_s[k].cpu(), EVIDENCE_WLH_FACTOR))
                got = trk.points[k].cpu()
                assert torch.equal(got[adv], want[adv]), (t, got, want)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    return {i: torch.stack(v).cpu().numpy() for i, v in rec.items()}, trk


def test_rule_declares_an_emptied_target_lost_on_time():
    # M2-Track: with untrained weights its boxes stay on their objects over these scenes, which the rule needs before t0 (the
    # untrained BAT-Car's proposals carry its boxes off their objects within a frame or two)
    net = _model("M2_track_kitti.yaml")
    sc = synthetic_scene(n_frames=10, n_points=N_POINTS, n_objects=4, seed=300, extent=14.0)
    clean, _ = _follow(net, sc["scans"], sc["boxes"], [0, 1, 2, 3], 8, (MIN_POINTS, PATIENCE), check_points=True)
    assert all((r[1:T0, 15] >= MIN_POINTS).all() for r in clean.values()), {i: r[:, 15] for i, r in clean.items()}
    scans = _emptied(sc, 0, T0)
    got, trk = _follow(net, scans, sc["boxes"], [0, 1, 2, 3], 8, (MIN_POINTS, PATIENCE), sync_free=True)
    r0 = got[0]
    lost_at = T0 + PATIENCE - 1
    assert (r0[T0:, 15] == 0).all()
    assert not r0[:lost_at, 18].any() and r0[lost_at:, 18].all(), r0[:, 17:]
    assert list(r0[T0:lost_at + 1, 17]) == list(range(1, PATIENCE + 1))
    assert (r0[lost_at:] == r0[lost_at]).all()                                # box, evidence held from the loss on
    assert int(trk.t[trk.targets()[0]]) == lost_at
    for i in (1, 2, 3):                                                       # the other targets: bitwise unchanged
        assert np.array_equal(got[i][:, :15], clean[i][:, :15]), i
        assert np.array_equal(got[i][:, 15:], clean[i][:, 15:], equal_nan=True), i
    # K and the other targets: target 0 alone in a one-slot tracker records the same
    alone, _ = _follow(net, scans, sc["boxes"], [0], 1, (MIN_POINTS, PATIENCE))
    assert np.array_equal(alone[0], r0, equal_nan=True)
    # read back, drop, and the slot is reused
    k0 = trk.targets()[0]
    assert trk.lost_targets() == [0]
    torch.cuda.set_sync_debug_mode("error")
    try:
        trk.drop(0)
        trk.add(9, sc["boxes"][1][len(scans) - 1])
        trk.step(torch.from_numpy(scans[-1]))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert trk.targets()[9] == k0 and trk.lost_targets() == [] and int(trk.points[k0]) > 0
    assert trk.drop_lost() == []


# ------------------------------------------------------------------ track_feeds and track_classes with rules
def _scenes(emptied=True):
    rng = np.random.default_rng(3)
    scenes = []
    for i, (T, n) in enumerate([(12, 3), (7, 2), (9, 3)]):
        sc = synthetic_scene(n_frames=T, n_points=3000, n_objects=n, seed=500 + i, extent=14.0)
        scans = _emptied(sc, 0, 3) if emptied and i == 0 else sc["scans"]
        starts, ends = {}, {}
        for j in range(n):
            a = 0 if j == 0 else int(rng.integers(0, T // 2))
            starts.setdefault(a, []).append((100 * i + j, sc["boxes"][j][a]))
            ends[100 * i + j] = int(rng.integers(max(a, T - 3), T))
        scenes.append({"frames": T, "scan": (lambda t, s=scans: s[t]), "starts": starts, "ends": ends})
    return scenes


def _flat(res):
    return {tid: {t: np.concatenate([b.center, b.wlh, b.rotation_matrix.ravel()]) for t, b in tr.items()}
            for scene in res for tid, tr in scene.items()}


def test_track_feeds_results_end_at_the_loss():
    net = _model("BAT_Car.yaml")
    scenes = _scenes()
    free, free_ev = track_feeds(net, scenes, 2, 6, seed=3, max_points=3000, evidence=True)
    plain = track_feeds(net, scenes, 2, 6, seed=3, max_points=3000)
    assert _flat(plain).keys() == _flat(free).keys()
    cut, cut_ev = track_feeds(net, scenes, 2, 6, seed=3, max_points=3000, lost=(1, 2), evidence=True)
    free, cut = _flat(free), _flat(cut)
    free_ev = {tid: tr for scene in free_ev for tid, tr in scene.items()}
    cut_ev = {tid: tr for scene in cut_ev for tid, tr in scene.items()}
    ended = []
    for tid in free:
        frames = sorted(cut[tid])
        assert frames == sorted(free[tid])[:len(frames)], tid                  # a prefix of the run without the rule
        for t in frames:
            assert np.array_equal(cut[tid][t], free[tid][t]), (tid, t)
            assert cut_ev[tid][t] == free_ev[tid][t] or (np.isnan(cut_ev[tid][t][1]) and np.isnan(free_ev[tid][t][1]))
        if len(frames) < len(free[tid]):
            ended.append(tid)
            pts = [free_ev[tid][t][0] for t in frames[-2:]]
            assert all(p < 1 for p in pts), (tid, pts)                          # two misses in a row
    assert 0 in ended, ended                                                  # the emptied target ends early


def test_track_classes_rules_per_class_are_lone_trackers():
    models = {"car": _model("BAT_Car.yaml"), "ped": _model("M2_track_kitti.yaml")}
    scenes = _scenes()
    rules = {"car": (1, 2), "ped": (30, 1)}
    cls_scenes = [{"frames": s["frames"], "scan": s["scan"], "ends": {(c, tid): e for tid, e in s["ends"].items() for c in models},
                   "starts": {t: [((c, tid), b) for tid, b in g for c in models] for t, g in s["starts"].items()}} for s in scenes]
    both, both_ev = track_classes(models, cls_scenes, 2, {"car": 8, "ped": 8}, seed=3, max_points=3000, lost=rules, evidence=True)
    both = _flat(both)
    both_ev = {key: tr for scene in both_ev for key, tr in scene.items()}
    for c in models:
        alone, alone_ev = track_feeds(models[c], scenes, 2, 8, seed=3, max_points=3000, lost=rules[c], evidence=True)
        alone = _flat(alone)
        alone_ev = {tid: tr for scene in alone_ev for tid, tr in scene.items()}
        for tid in alone:
            assert sorted(both[(c, tid)]) == sorted(alone[tid]), (c, tid)
            for t in alone[tid]:
                assert np.array_equal(both[(c, tid)][t], alone[tid][t]), (c, tid, t)
                a, b = both_ev[(c, tid)][t], alone_ev[tid][t]
                assert a[0] == b[0] and (a[1] == b[1] or (np.isnan(a[1]) and np.isnan(b[1]))), (c, tid, t)


# ------------------------------------------------------------------ the command line
def test_command_line_ends_a_lost_tracklet(tmp_path, capsys):
    from open3dsot_b200.utils.metrics import Precision, Success, estimateAccuracy, estimateOverlap
    root = str(tmp_path / "kitti")
    seqs = [synthetic_sequence(n_frames=n, n_points=1500, seed=40 + i, n_object=300, speed=0.3 + 0.1 * i, yaw_rate=1.0 + i)
            for i, n in enumerate([8, 6])]
    for f in seqs[1]:                                           # the second car drives 12 m to the left
        f["pc"] = PointCloud(f["pc"].points + np.array([[0.0], [12.0], [0.0]], np.float32))
        b = f["3d_bbox"]
        f["3d_bbox"] = Box(b.center + np.array([0.0, 12.0, 0.0]), b.wlh, b.rotation_matrix)
    for t in range(3, 8):                                       # the first car's surroundings are emptied from frame 3 on
        p = seqs[0][t]["pc"].points.copy()
        near = np.linalg.norm(p[:2] - seqs[0][t]["3d_bbox"].center[:2, None], axis=0) < 6.0
        p[:, near] = FAR[:, None]
        seqs[0][t]["pc"] = PointCloud(p)
    # M2-Track, whose untrained boxes stay on their objects here (the config tracks the "Pedestrian" class)
    _write_scene(root, "0019", [((5, "Pedestrian"), seqs[0]), ((8, "Pedestrian"), seqs[1])], extra_dontcare=False)
    ds = kittiDataset(root, "test", "Pedestrian", preloading=False, preload_offset=-1)
    npts = max(f["pc"].points.shape[1] for t in ds.tracklets() for f in t)
    cfg_path = os.path.join(ROOT, "cfgs", "M2_track_kitti.yaml")
    cfg = load_config(cfg_path)
    base = ["--cfg", cfg_path, "--path", root, "--split", "test", "--max_targets", "3", "--max_points", str(npts)]
    free = track.main(base + ["--out", str(tmp_path / "free.jsonl")])
    got = track.main(base + ["--out", str(tmp_path / "lost.jsonl"), "--lost", "1", "2"])
    printed = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert printed["lost"] == got["lost"] == 1 and "lost" not in free
    free_lines = [json.loads(l) for l in open(tmp_path / "free.jsonl")]
    lines = [json.loads(l) for l in open(tmp_path / "lost.jsonl")]
    frames_of = lambda ls, i: [l["frame"] for l in ls for t in l["targets"] if t["id"] == i]
    assert frames_of(free_lines, 5) == list(range(8)) and frames_of(free_lines, 8) == list(range(6))
    end = frames_of(lines, 5)[-1]
    assert frames_of(lines, 5) == list(range(end + 1)) and 3 <= end < 7, end      # lines stop at the loss frame
    assert frames_of(lines, 8) == list(range(6))
    for l, fl in zip(lines, free_lines):                                       # up to the loss, the same lines
        ft = {t["id"]: t for t in fl["targets"]}
        for t in l["targets"]:
            assert t == ft[t["id"]] and "points" in t and "score" in t
    first = [t for l in lines for t in l["targets"] if l["frame"] == 0]
    assert all(t["points"] is None and t["score"] is None for t in first)
    # Success / Precision: the lost tracklet's remaining annotated frames are failures
    by = {(l["frame"], t["tracklet"]): t for l in lines for t in l["targets"]}
    succ, prec = Success(), Precision()
    dim, up = cfg.IoU_space, cfg.up_axis
    for j, annos in enumerate(ds.tracklet_anno_list):
        o, d = [], []
        for t, anno in enumerate(annos):
            gt = ds.box_from_anno(anno)
            tid = j
            if t == 0:
                box = gt
            elif (t, tid) in by:
                b = by[(t, tid)]
                yaw = b["yaw"]
                rot = _rot(yaw) if up[1] == 0 else np.array([[np.cos(yaw), 0, np.sin(yaw)], [0, 1, 0], [-np.sin(yaw), 0, np.cos(yaw)]])
                box = Box(np.array(b["center"]), np.array(b["wlh"]), rot)
            else:
                o.append(0.0)
                d.append(float("inf"))
                continue
            o.append(estimateOverlap(gt, box, dim=dim, up_axis=up))
            d.append(estimateAccuracy(gt, box, dim=dim, up_axis=up))
        succ(o)
        prec(d)
    assert abs(succ.compute() - got["success"]) < 1e-3 and abs(prec.compute() - got["precision"]) < 1e-3, (got, succ.compute())
    assert got["success"] <= free["success"] + 1e-9
