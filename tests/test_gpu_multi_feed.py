"""Many scan feeds through one live tracker, on the GPU: `o3d_scan_ingest` against the readers' host transforms (at most one
float32 ulp, the count of non-identical values reported), scenes tracked together against each scene alone, reproducibility and
replay against eager, holding feeds, no host sync, the kernels one advance runs, and the command line over KITTI, nuScenes and
Waymo fixtures against evaluate_batched."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from open3dsot_b200 import ops, track
from open3dsot_b200.config import load_config
from open3dsot_b200.datasets.data_classes import Box, PointCloud
from open3dsot_b200.datasets.kitti import kittiDataset
from open3dsot_b200.datasets.nuscenes_data import NuScenesDataset
from open3dsot_b200.datasets.synthetic import synthetic_scene, synthetic_sequence
from open3dsot_b200.datasets.waymo_data import WaymoDataset
from open3dsot_b200.models import get_model
from open3dsot_b200.tracking.evaluate import evaluate_batched
from open3dsot_b200.tracking.multi_tracker import MultiTargetTracker, track_feeds, track_stream
from test_kitti_reader import _write_scene
from test_multi_feed import _write_waymo
from test_nuscenes_waymo_readers import _write_nuscenes

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODELS = ["BAT_Car.yaml", "P2B_Car.yaml", "M2_track_kitti.yaml"]


def _model(cfg_name, **over):
    cfg = load_config(os.path.join(ROOT, "cfgs", cfg_name), {"up_axis": [0, 0, 1], **over})
    torch.manual_seed(0)
    return cfg, get_model(cfg.net_model)(cfg).cuda().eval()


# ------------------------------------------------------------------ the ingest kernel against the readers
def _ingest(items, feeds, N):
    """Run one o3d_scan_ingest over `items` [(feed, half, rows, transforms)] into NaN-filled buffers."""
    scans = torch.full((feeds, 2, N, 3), float("nan"), device="cuda")
    count = torch.full((feeds, 2), -1, dtype=torch.int64, device="cuda")
    buf, desc, d0, s0 = ops.pack_scans(items)
    ops.scan_ingest(scans, count, desc, buf.to("cuda", non_blocking=True), d0, s0)
    return scans.cpu().numpy(), count.cpu().numpy()


def _within_one_ulp(got, want, what):
    """At most one float32 ulp apart; reports how many values are not bit-identical."""
    assert got.shape == want.shape and got.dtype == want.dtype == np.float32, (what, got.shape, want.shape)
    diff = got != want
    ulp = np.spacing(np.maximum(np.abs(got), np.abs(want)))
    assert (np.abs(got.astype(np.float64) - want) <= ulp).all(), (what, float(np.abs(got - want).max()))
    print(f"{what}: {int(diff.sum())} of {diff.size} values not bit-identical")
    return int(diff.sum())


def _reader_cases(tmp_path):
    """(name, reader, [(scene, frame)]) over the three fixtures, KITTI in both coordinate modes."""
    root = str(tmp_path / "kitti")
    seqs = [synthetic_sequence(n_frames=3, n_points=700 + 100 * i, seed=60 + i, n_object=200) for i in range(2)]
    _write_scene(root, "0019", [((1, "Car"), seqs[0]), ((2, "Car"), seqs[1])])
    out = []
    for mode in ("velodyne", "camera"):
        ds = kittiDataset(root, "test", "Car", coordinate_mode=mode, preloading=False, preload_offset=-1)
        out.append((f"kitti-{mode}", ds, [("0019", f) for f in range(3)] + [("0019", 50)]))      # frame 50: a missing file
    _write_nuscenes(str(tmp_path / "nusc"))
    ds = NuScenesDataset(str(tmp_path / "nusc"), "x", "Car", version="v1.0-mini", scenes=["scene-0061", "scene-0103"],
                         preload_offset=-1)
    out.append(("nuscenes", ds, [(s, f) for s in ds.scene_list for f in ds.scene_frames(s)]))
    _write_waymo(str(tmp_path / "waymo"))
    ds = WaymoDataset(str(tmp_path / "waymo"), "val", "VEHICLE", preloading=False, preload_offset=-1)
    out.append(("waymo", ds, [(s, f) for s in ds.scene_list for f in ds.scene_frames(s)]))
    return out


def test_ingest_matches_the_readers(tmp_path):
    for name, ds, frames in _reader_cases(tmp_path):
        feeds = len(frames)
        items = [(i, i % 2, *ds.raw_scan(s, f)) for i, (s, f) in enumerate(frames)]
        N = max(r.shape[0] for _, _, r, _ in items)
        scans, count = _ingest(items, feeds, N)
        for i, (s, f) in enumerate(frames):
            want = np.ascontiguousarray(ds.read_scan(s, f).points.T, dtype=np.float32)
            n = want.shape[0]
            assert count[i, i % 2] == n and count[i, 1 - i % 2] == -1, (name, s, f)
            _within_one_ulp(scans[i, i % 2, :n], want, f"{name} {s}/{f}")
            assert np.isnan(scans[i, i % 2, n:]).all() and np.isnan(scans[i, 1 - i % 2]).all()   # nothing else written


def _random_xf(rng):
    q = np.linalg.qr(rng.normal(size=(3, 3)))[0]
    return np.hstack([q, rng.uniform(-500, 500, (3, 1))])


def test_ingest_random_rows_and_transforms_at_120k_points():
    rng = np.random.default_rng(1)
    N = 120_000
    a = rng.uniform(-80, 80, (N, 5)).astype(np.float32)                   # nuScenes-like rows, two transforms
    b = rng.uniform(-80, 80, (N - 7, 3))                                   # float64 rows, one transform
    c = rng.uniform(-80, 80, (N // 3, 4)).astype(np.float32)               # no transform: a plain copy
    xa, xb = [_random_xf(rng), _random_xf(rng)], [_random_xf(rng)]
    empty = np.zeros((0, 4), np.float32)
    # feed 3 gets an empty scan, feed 4 nothing at all
    scans, count = _ingest([(0, 1, a, xa), (1, 0, b, xb), (2, 0, c, []), (3, 1, empty, xb)], 5, N)
    assert count.tolist() == [[-1, N], [N - 7, -1], [N // 3, -1], [-1, 0], [-1, -1]]
    for feed, half, rows, xfs in ((0, 1, a, xa), (1, 0, b, xb)):
        p = rows[:, :3].T.astype(np.float64)
        for m in xfs:
            p = m[:, :3] @ p + m[:, 3][:, None]
        _within_one_ulp(scans[feed, half, :rows.shape[0]], np.ascontiguousarray(p.T, dtype=np.float32), f"random feed {feed}")
    assert np.array_equal(scans[2, 0, :N // 3], c[:, :3])
    assert np.isnan(scans[3]).all() and np.isnan(scans[4]).all()


# ------------------------------------------------------------------ scenes together against each scene alone
SCENES = [  # (frames, seed, [(start, end)] per target): staggered starts, unequal lengths; six scenes on four feeds
    (9, 31, [(0, 8), (2, 6)]), (5, 32, [(1, 4)]), (7, 33, [(0, 3), (0, 6), (4, 6)]),
    (4, 34, [(0, 3)]), (6, 35, [(2, 5), (0, 1)]), (3, 36, [(0, 2)]),
]


def _scenes(transformed=()):
    """Synthetic scenes as track_feeds input; scene i in `transformed` is given as raw float64 rows in a sensor frame with the
    transform back to the scene's frame (the ingest's float64 path)."""
    out = []
    for i, (T, seed, targets) in enumerate(SCENES):
        sc = synthetic_scene(n_frames=T, n_points=5000, n_objects=len(targets), seed=seed, extent=14.0)
        starts, ends = {}, {}
        for j, (a, e) in enumerate(targets):
            tid = 100 * i + j
            starts.setdefault(a, []).append((tid, sc["boxes"][j][a]))
            ends[tid] = e
        if i in transformed:
            xf = np.hstack([np.eye(3), [[1.0], [-2.0], [0.5]]])
            scan = (lambda t, s=sc["scans"], xf=xf: ((s[t].astype(np.float64) - xf[:, 3]), [xf]))
        else:
            scan = (lambda t, s=sc["scans"]: s[t])
        out.append({"frames": T, "scan": scan, "starts": starts, "ends": ends})
    return out


def _flat(res):
    return {tid: np.array([np.concatenate([b.center, b.rotation_matrix.ravel()]) for _, b in sorted(tr.items())])
            for scene in res for tid, tr in scene.items()}


@pytest.fixture(scope="module", params=MODELS)
def together(request):
    cfg, net = _model(request.param)
    scenes = _scenes(transformed=(2,))
    return request.param, net, scenes, track_feeds(net, scenes, 4, 6, seed=3, max_points=5000)


def test_scenes_on_feeds_match_each_scene_alone(together):
    name, net, scenes, res = together
    got = _flat(res)
    for i, sc in enumerate(scenes):
        alone = _flat(track_feeds(net, [sc], 1, 3, seed=3, max_points=5000))
        for (a, e), tid in zip(SCENES[i][2], (100 * i + j for j in range(len(SCENES[i][2])))):
            assert sorted(res[i][tid]) == list(range(a, e + 1)), (name, tid)
            d = float(np.abs(got[tid] - alone[tid]).max())
            assert d < 1e-4, (name, tid, d)


def test_feeds_repeat_bitwise_and_replay_equals_eager(together):
    name, net, scenes, res = together
    again = _flat(track_feeds(net, scenes, 4, 6, seed=3, max_points=5000))
    eager = _flat(track_feeds(net, scenes, 4, 6, seed=3, max_points=5000, use_graph=False))
    for tid, v in _flat(res).items():
        assert np.array_equal(again[tid], v) and np.array_equal(eager[tid], v), (name, tid)


def test_one_feed_tracks_as_track_stream(together):
    """track_feeds with one scene on one feed (host scans through the ingest kernel) against track_stream (device scans)."""
    name, net, scenes, res = together
    sc = scenes[0]
    ref = track_stream(net, [torch.tensor(sc["scan"](t), device="cuda") for t in range(sc["frames"])], sc["starts"], sc["ends"], 3,
                       seed=3, max_points=5000)
    got = track_feeds(net, [sc], 1, 3, seed=3, max_points=5000)[0]
    for tid in ref:
        assert np.array_equal(_flat([{tid: got[tid]}])[tid], _flat([{tid: ref[tid]}])[tid]), (name, tid)


# ------------------------------------------------------------------ holding feeds, no host sync
def test_feed_without_a_scan_holds_and_nothing_syncs():
    cfg, net = _model("BAT_Car.yaml")
    sc = [synthetic_scene(n_frames=5, n_points=5000, n_objects=2, seed=50 + i, extent=14.0) for i in range(3)]
    trk = MultiTargetTracker(net, 5000, 6, seed=1, feeds=3)
    for f in range(3):
        trk.put(f, sc[f]["scans"][0])                                      # host arrays: the ingest path
    trk.advance()                                                           # capture (synchronises once)
    for f in range(3):
        trk.add(10 * f, sc[f]["boxes"][0][0], feed=f)
    on_device = torch.tensor(sc[0]["scans"][2], device="cuda")
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        trk.put(0, sc[0]["scans"][1])
        trk.put_raw(1, np.concatenate([sc[1]["scans"][1], np.ones((5000, 1), np.float32)], 1),
                    [np.hstack([np.eye(3), np.zeros((3, 1))])])
        trk.advance()                                                       # feed 2 holds
        held = trk.snapshot()
        t_held = trk.t.clone()
        trk.put(0, on_device)                                               # a device scan: copied straight in
        trk.advance()                                                       # feeds 1 and 2 hold
        trk.drop(0)
        trk.add(11, sc[1]["boxes"][1][1], feed=1)
        after = trk.snapshot()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    k0, k1, k2 = 0, 1, 2
    assert trk.targets() == {11: 0, 10: 1, 20: 2}
    assert torch.equal(held[k2], after[k2]) and torch.equal(held[k1], after[k1])     # holding slots keep their box ...
    assert int(trk.t[k2]) == int(t_held[k2]) == 0 and int(trk.t[k1]) == 1          # ... and their frame counter
    assert trk.feed_seen == [3, 2, 1] and trk._fcur == [0, 1, 0]


# ------------------------------------------------------------------ the kernels of one advance (child process, as in
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
sc = [synthetic_scene(n_frames=5, n_points=5000, n_objects=1, seed=70 + i, extent=14.0) for i in range(3)]
xf = np.hstack([np.eye(3), np.zeros((3, 1))])
trk = MultiTargetTracker(net, 5000, 4, seed=2, feeds=3)
def put(t):
    for f in range(3):
        trk.put_raw(f, sc[f]["scans"][t], [xf])
put(0); trk.advance()
for f in range(3):
    trk.add(f, sc[f]["boxes"][0][0], feed=f)
put(1); trk.advance()
torch.cuda.synchronize()
def profiled(t):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        put(t); trk.advance()
        torch.cuda.synchronize()
    return [e.name for e in prof.events()]
names = profiled(2)
if not any("kernel" in n for n in names):
    names = profiled(3)
print(json.dumps(names))
"""


def test_one_advance_runs_one_ingest_and_one_crop_kernel_per_crop():
    r = subprocess.run([sys.executable, "-c", _PROFILE_CHILD, ROOT], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    names = json.loads(r.stdout.strip().splitlines()[-1])
    ingest = [n for n in names if "scan_ingest_kernel" in n]
    crops = [n for n in names if "crop_resample_kernel" in n]
    assert len(ingest) == 1, sorted(set(names))
    assert len(crops) == 2, sorted(set(names))                            # BAT: the search crop and the template crop
    assert not any("crop_box_frame_kernel" in n for n in names)


# ------------------------------------------------------------------ the command line over the three fixture trees
def _cli(tmp_path, cfg_name, root, split, ds, max_targets=4):
    out = str(tmp_path / f"{cfg_name}.jsonl")
    cfg_path = os.path.join(ROOT, "cfgs", cfg_name)
    got = track.main(["--cfg", cfg_path, "--path", root, "--split", split, "--out", out, "--max_targets", str(max_targets)])
    cfg = load_config(cfg_path)
    torch.manual_seed(0)
    net = get_model(cfg.net_model)(cfg).cuda()
    ref = evaluate_batched(net, ds.tracklets(), slots=3, seed=0)
    assert got["frames"] == ref["frames"] == ds.get_num_frames_total()
    assert abs(got["success"] - ref["success"]) < 1e-4 and abs(got["precision"] - ref["precision"]) < 1e-4, (cfg_name, got, ref)
    return [json.loads(l) for l in open(out)], net


def test_command_line_on_kitti_matches_evaluate_batched_and_one_feed(tmp_path, capsys):
    root = str(tmp_path / "kitti")
    seqs = [synthetic_sequence(n_frames=n, n_points=1500, seed=80 + i, n_object=300, speed=0.3 + 0.1 * i, yaw_rate=1.0 + i)
            for i, n in enumerate([6, 4, 5])]
    for f in seqs[1]:
        f["pc"] = PointCloud(f["pc"].points + np.array([[0.0], [12.0], [0.0]], np.float32))
        b = f["3d_bbox"]
        f["3d_bbox"] = Box(b.center + np.array([0.0, 12.0, 0.0]), b.wlh, b.rotation_matrix)
    _write_scene(root, "0019", [((5, "Car"), seqs[0]), ((8, "Car"), seqs[1])], extra_dontcare=False)
    _write_scene(root, "0020", [((2, "Car"), seqs[2])], extra_dontcare=False)
    ds = kittiDataset(root, "test", "Car", preloading=False, preload_offset=-1)
    lines, net = _cli(tmp_path, "BAT_Car.yaml", root, "test", ds)
    assert [(l["scene"], l["frame"]) for l in lines] == [("0019", f) for f in range(6)] + [("0020", f) for f in range(5)]
    # the single-feed run: each scene streamed alone from device scans
    plan = track.scene_plan(ds)
    npts = track.stream_max_points(ds, plan)                             # the draws' layout follows the scan buffer's size
    annos = ds.tracklet_anno_list
    by_line = {(l["scene"], l["frame"], t["tracklet"]): t for l in lines for t in l["targets"]}
    for p in plan:
        starts, ends = {}, {}
        for tr in p["tracklets"]:
            starts.setdefault(tr["start"] - p["first"], []).append((tr["index"], ds.box_from_anno(annos[tr["index"]][0])))
            ends[tr["index"]] = tr["end"] - p["first"]
        scans = [torch.tensor(np.ascontiguousarray(ds.read_scan(p["scene"], f).points[:3].T, np.float32), device="cuda")
                 for f in p["frames"]]
        res = track_stream(net, scans, starts, ends, 4, seed=0, max_points=npts)
        for j, tr in res.items():
            for t, b in tr.items():
                line = by_line[(p["scene"], p["frames"][t], j)]
                assert np.abs(np.array(line["center"]) - b.center).max() < 1e-4, (p["scene"], j, t)


def test_command_line_on_nuscenes_matches_evaluate_batched(tmp_path, capsys):
    root = str(tmp_path / "nusc")
    _write_nuscenes(root, version="v1.0-trainval")
    os.makedirs(os.path.join(root, "splits"))
    with open(os.path.join(root, "splits", "val.txt"), "w") as f:
        f.write("scene-0061\nscene-0103\n")
    cfg = load_config(os.path.join(ROOT, "cfgs", "BAT_CAR_NUSCENES.yaml"))
    ds = track.reader(cfg, root, "val")
    assert ds.get_num_tracklets() == 2
    lines, _ = _cli(tmp_path, "BAT_CAR_NUSCENES.yaml", root, "val", ds)
    assert [(l["scene"], l["frame"]) for l in lines] == [(s, f) for s in ("scene-0061", "scene-0103") for f in range(3)]


def test_command_line_on_waymo_matches_evaluate_batched(tmp_path, capsys):
    root = str(tmp_path / "waymo")
    _write_waymo(root)
    cfg = load_config(os.path.join(ROOT, "cfgs", "BAT_Car_Waymo.yaml"))
    ds = track.reader(cfg, root, "test")
    lines, _ = _cli(tmp_path, "BAT_Car_Waymo.yaml", root, "test", ds)
    assert [(l["scene"], l["frame"]) for l in lines] == [("0", f) for f in range(4)] + [("1", f) for f in range(3)]
