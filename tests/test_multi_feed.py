"""Many scan feeds through one live tracker, CPU part: the argument checks of `o3d_scan_ingest` through the built library (no
launch), the tracker's feed refusals, the scheduler's invariants, and the command line's scene plans over nuScenes and Waymo
fixtures (every annotation mapped to a (scene, frame) whose whole scan and box are the reader's)."""
import os
import pickle

import numpy as np
import pytest
import torch

from open3dsot_b200 import _lib, ops
from open3dsot_b200.datasets import data_classes as dc
from open3dsot_b200.datasets.nuscenes_data import NuScenesDataset
from open3dsot_b200.datasets.waymo_data import WaymoDataset
from open3dsot_b200.track import scene_plan, stream_max_points
from open3dsot_b200.tracking.multi_tracker import MultiTargetTracker, feed_schedule, scene_peak
from test_nuscenes_waymo_readers import _write_nuscenes
from test_tracking_host import _cfg, _Echo


# ------------------------------------------------------------------ o3d_scan_ingest's argument checks
def _desc(n=1, **kw):
    d = np.zeros(n, ops.SCAN_DESC)
    d["rows"], d["stride"], d["n_xf"] = 100, 4, 1
    d["feed"] = np.arange(n)
    for k, v in kw.items():
        d[k][0] = v
    return d


def _ingest(desc, n_desc=None, desc_dev=16, slab=16, slab_bytes=1 << 20, feeds=4, max_points=1000, scans=16, count=16):
    """Non-null placeholders for the device pointers: never dereferenced, every call here fails before a launch."""
    L = _lib.lib()
    host = desc.ctypes.data if desc is not None else None
    return L.o3d_scan_ingest(host, desc_dev, len(desc) if n_desc is None else n_desc, slab, slab_bytes, feeds, max_points, scans,
                             count, None), L.o3d_last_error()


def test_scan_ingest_argument_errors_return_status():
    for kw in (dict(desc_dev=None), dict(scans=None), dict(count=None), dict(slab=None)):
        st, msg = _ingest(_desc(), **kw)
        assert st < 0 and b"null" in msg, kw
    st, msg = _ingest(None, n_desc=1)
    assert st < 0 and b"null" in msg
    st, msg = _ingest(_desc(stride=2))
    assert st < 0 and b"stride 2" in msg
    st, msg = _ingest(_desc(stride=17))
    assert st < 0 and b"stride 17" in msg
    st, msg = _ingest(_desc(rows=1001))                                     # more rows than the scan buffer holds
    assert st < 0 and b"rows 1001" in msg
    st, msg = _ingest(_desc(rows=-1))
    assert st < 0 and b"rows -1" in msg
    st, msg = _ingest(_desc(feed=4))                                        # feed out of range
    assert st < 0 and b"feed 4" in msg
    st, msg = _ingest(_desc(feed=-1))
    assert st < 0 and b"feed -1" in msg
    st, msg = _ingest(_desc(half=2))
    assert st < 0 and b"half 2" in msg
    st, msg = _ingest(_desc(n_xf=3))
    assert st < 0 and b"n_xf 3" in msg
    st, msg = _ingest(_desc(is_f64=2))
    assert st < 0 and b"is_f64" in msg
    st, msg = _ingest(_desc(offset=2))                                      # not aligned to a float
    assert st < 0 and b"outside the slab" in msg
    st, msg = _ingest(_desc(), slab_bytes=100 * 16 - 4)                     # rows past the end of the slab
    assert st < 0 and b"outside the slab" in msg
    st, msg = _ingest(_desc(is_f64=1), slab_bytes=100 * 16)                 # the same rows as float64 need twice the bytes
    assert st < 0 and b"outside the slab" in msg
    d = _desc(2)
    d["feed"] = 1
    st, msg = _ingest(d)                                                    # two descriptors writing one buffer
    assert st < 0 and b"both write feed 1" in msg
    st, msg = _ingest(_desc(9), feeds=4)
    assert st < 0 and b"n_desc" in msg
    st, msg = _ingest(_desc(), feeds=0)
    assert st < 0 and b"feeds=0" in msg
    assert _ingest(_desc(), n_desc=0)[0] == 0                               # nothing to do: no launch


def test_pack_scans_lays_out_descriptors_and_rows():
    a = np.arange(12, dtype=np.float32).reshape(3, 4)
    b = np.arange(10, dtype=np.float64).reshape(2, 5)
    xf = np.hstack([np.eye(3) * 2, np.ones((3, 1))])
    buf, desc, d0, s0 = ops.pack_scans([(2, 1, a, []), (0, 0, b, [xf, np.vstack([xf, [0, 0, 0, 1]])])], head=24)
    host = buf.numpy()
    assert d0 == 32 and s0 == d0 + 2 * 224 and np.shares_memory(desc, host[d0:s0])
    assert list(desc["feed"]) == [2, 0] and list(desc["half"]) == [1, 0] and list(desc["rows"]) == [3, 2]
    assert list(desc["stride"]) == [4, 5] and list(desc["is_f64"]) == [0, 1] and list(desc["n_xf"]) == [0, 2]
    assert np.array_equal(desc["xf"][1, 0], xf.reshape(-1)) and np.array_equal(desc["xf"][1, 1], xf.reshape(-1))
    o = desc["offset"]
    assert o[0] % 16 == 0 and o[1] % 16 == 0
    assert np.array_equal(host[s0 + o[0]:s0 + o[0] + a.nbytes].view(np.float32).reshape(3, 4), a)
    assert np.array_equal(host[s0 + o[1]:s0 + o[1] + b.nbytes].view(np.float64).reshape(2, 5), b)
    with pytest.raises(ValueError, match="at most two"):
        ops.pack_scans([(0, 0, a, [xf] * 3)])


# ------------------------------------------------------------------ the tracker's feed refusals
def test_tracker_refuses_bad_feeds():
    box = dc.Box(np.zeros(3), np.array([1.5, 4.0, 1.5]), np.eye(3))
    with pytest.raises(ValueError, match="feeds=0"):
        MultiTargetTracker(_Echo(_cfg()), 100, 4, feeds=0)
    trk = MultiTargetTracker(_Echo(_cfg()), 100, 4, use_graph=False, feeds=3)
    assert trk.scans.shape == (3, 2, 100, 3) and trk.count.shape == (3, 2)
    with pytest.raises(ValueError, match="step"):
        trk.step(torch.zeros(5, 3))                                         # step() is the one-feed form
    with pytest.raises(ValueError, match="feed 3"):
        trk.put(3, torch.zeros(5, 3))
    with pytest.raises(ValueError, match="max_points"):
        trk.put(1, torch.zeros(101, 3))
    trk.put(1, torch.ones(5, 3))
    with pytest.raises(ValueError, match="already has a scan staged"):
        trk.put(1, torch.zeros(5, 3))
    with pytest.raises(RuntimeError, match="GPU"):
        trk.put_raw(0, np.zeros((5, 4), np.float32))                        # ingest runs on the device only
    with pytest.raises(RuntimeError, match="feed 2"):
        trk.add(7, box, feed=2)                                             # no scan on that feed yet
    with pytest.raises(ValueError, match="feed -1"):
        trk.add(7, box, feed=-1)
    trk.feed_seen[2] = 1                                                    # as after an advance with a scan of feed 2
    trk.add(7, box, feed=2)
    assert int(trk.slot_feed[0]) == 2
    trk.drop(7)
    assert int(trk.slot_feed[0]) == 0


# ------------------------------------------------------------------ the scheduler
def _check_schedule(lengths, peaks, feeds, max_targets):
    sched = feed_schedule(lengths, peaks, feeds, max_targets)
    assert sorted(i for i, _, _ in sched) == list(range(len(lengths)))     # every scene runs once
    assert [lengths[i] for i, _, _ in sched] == sorted(lengths, reverse=True)   # admitted longest first
    assert [s for _, _, s in sched] == sorted(s for _, _, s in sched)
    end = max(s + lengths[i] for i, _, s in sched)
    for step in range(end):
        run = [(i, f) for i, f, s in sched if s <= step < s + lengths[i]]
        assert sum(peaks[i] for i, _ in run) <= max_targets                # the reserved slots never exceed max_targets
        assert len({f for _, f in run}) == len(run) and all(0 <= f < feeds for _, f in run)   # one scene per feed at a time
    by_feed = {}
    for i, f, s in sched:
        by_feed.setdefault(f, []).append((s, s + lengths[i]))
    for spans in by_feed.values():                                         # a feed is reused only after its scene ended
        assert all(a[1] <= b[0] for a, b in zip(spans, spans[1:]))
    return sched


def test_schedule_invariants():
    rng = np.random.default_rng(4)
    for trial in range(40):
        n = int(rng.integers(1, 30))
        feeds, max_targets = int(rng.integers(1, 9)), int(rng.integers(1, 20))
        lengths = [int(x) for x in rng.integers(1, 50, n)]
        peaks = [int(x) for x in rng.integers(0, max_targets + 1, n)]
        _check_schedule(lengths, peaks, feeds, max_targets)
    # the second scene's feed is reused once it ends ...
    assert _check_schedule([10, 6, 3], [3, 2, 2], feeds=3, max_targets=5) == [(0, 0, 0), (1, 1, 0), (2, 1, 6)]
    # ... but here slots, not feeds, hold the third scene back until the first one ends
    assert _check_schedule([10, 6, 3], [3, 2, 3], feeds=3, max_targets=5) == [(0, 0, 0), (1, 1, 0), (2, 0, 10)]


def test_schedule_refuses_a_scene_that_never_fits():
    with pytest.raises(ValueError, match="max_targets=4"):
        feed_schedule([5, 5], [2, 5], feeds=2, max_targets=4)
    with pytest.raises(ValueError, match="no frames"):
        feed_schedule([0], [0], feeds=1, max_targets=4)


def test_scene_peak():
    box = None
    starts = {0: [(1, box), (2, box)], 3: [(3, box)], 5: [(4, box)]}
    assert scene_peak(8, starts, {1: 2, 2: 3, 3: 4}) == 2                  # target 3 starts on target 2's last frame
    assert scene_peak(8, starts, {1: 3, 2: 5, 3: 4}) == 3
    assert scene_peak(8, starts, {}) == 4                                  # no end: to the scene's last frame


# ------------------------------------------------------------------ scene plans over nuScenes and Waymo fixtures
def _check_plan(ds):
    plan = scene_plan(ds)
    where = {}
    for p in plan:
        assert p["frames"] == [f for f in ds.scene_frames(p["scene"]) if p["first"] <= f <= p["last"]]
        for tr in p["tracklets"]:
            assert tr["frames"] == sorted(tr["frames"]) and set(tr["frames"]) <= set(p["frames"])
            where[tr["index"]] = (p["scene"], tr["frames"])
    assert sorted(where) == list(range(ds.get_num_tracklets()))            # every tracklet is in some scene's stream
    for j, annos in enumerate(ds.tracklet_anno_list):
        scene, frames = where[j]
        got = ds.get_frames(j, range(len(annos)))
        for a, fr, frame in zip(annos, got, frames):
            assert ds.anno_frame(a) == (scene, frame)
            assert np.array_equal(ds.read_scan(scene, frame).points, fr["pc"].points)   # the whole scan of that frame
            b = ds.box_from_anno(a)
            assert np.array_equal(b.center, fr["3d_bbox"].center) and np.array_equal(b.rotation_matrix, fr["3d_bbox"].rotation_matrix)
            assert np.array_equal(b.wlh, fr["3d_bbox"].wlh)
            rows, xfs = ds.raw_scan(scene, frame)
            assert rows.shape[0] == fr["pc"].points.shape[1] == ds.scan_size(scene, frame)
    assert stream_max_points(ds, plan) == max(ds.scan_size(p["scene"], f) for p in plan for f in p["frames"])
    return plan


def test_nuscenes_plan_maps_every_annotation(tmp_path):
    _write_nuscenes(str(tmp_path))
    ds = NuScenesDataset(str(tmp_path), "x", "Pedestrian", version="v1.0-mini", scenes=["scene-0061", "scene-0103"],
                         preload_offset=-1)
    plan = _check_plan(ds)
    assert [p["scene"] for p in plan] == ["scene-0061", "scene-0103"]
    assert [(p["first"], p["last"]) for p in plan] == [(1, 2), (1, 2)]     # the pedestrians appear in the second sample
    assert ds.scene_frames("scene-0061") == [0, 1, 2]
    rows, xfs = ds.raw_scan("scene-0061", 1)
    assert rows.shape == (200, 5) and rows.dtype == np.float32 and len(xfs) == 2 and all(x.shape == (3, 4) for x in xfs)
    car = NuScenesDataset(str(tmp_path), "x", "Car", version="v1.0-mini", scenes=["scene-0061", "scene-0103"], preload_offset=-1)
    assert [(p["first"], p["last"]) for p in _check_plan(car)] == [(0, 2), (0, 2)]


def _write_waymo(root, split="val"):
    """Two converter-format Waymo segments: lidar/seq_<s>_frame_<f>.pkl with the points (float64 in segment 0, float32 in
    segment 1), annos/... with veh_to_global, and the sot_infos index: three tracklets, one starting late, and an unannotated
    last frame in segment 1."""
    os.makedirs(os.path.join(root, "lidar"), exist_ok=True)
    os.makedirs(os.path.join(root, "annos"), exist_ok=True)
    rng = np.random.default_rng(11)
    infos = {}
    tracks = {("0", "a"): range(0, 4), ("0", "b"): range(1, 3), ("1", "a"): range(0, 3)}
    for s, n_frames, dtype in (("0", 4, np.float64), ("1", 4, np.float32)):
        for f in range(n_frames):
            lp = os.path.join(root, "lidar", f"seq_{s}_frame_{f}.pkl")
            with open(lp, "wb") as fh:
                pickle.dump({"lidars": {"points_xyz": rng.uniform(-40, 40, (300 + 10 * f, 3)).astype(dtype)}, "frame_id": f,
                             "scene_name": f"segment-{s}"}, fh)
            c, si = np.cos(0.3 + 0.05 * f), np.sin(0.3 + 0.05 * f)
            pose = np.array([[c, -si, 0, 1000.0 + 2 * f], [si, c, 0, -500.0 + f], [0, 0, 1, 3.0], [0, 0, 0, 1]])
            with open(lp.replace("lidar", "annos"), "wb") as fh:
                pickle.dump({"veh_to_global": pose.reshape(-1)}, fh)
    for (s, obj), frames in tracks.items():
        infos[f"seg{s}_{obj}"] = [{"PC": os.path.join(root, "lidar", f"seq_{s}_frame_{f}.pkl"),
                                   "Box": np.array([5.0 + f, 2.0 * (obj == "b"), 0.8, 4.5, 1.9, 1.6, 1.0, 0.0, 0.1 * f]),
                                   "Class": "VEHICLE"} for f in frames]
    with open(os.path.join(root, f"sot_infos_vehicle_{split}.pkl"), "wb") as fh:
        pickle.dump(infos, fh)


def test_waymo_plan_maps_every_annotation(tmp_path):
    _write_waymo(str(tmp_path))
    ds = WaymoDataset(str(tmp_path), "val", "VEHICLE", preloading=False, preload_offset=-1)
    plan = _check_plan(ds)
    assert [p["scene"] for p in plan] == ["0", "1"] and ds.scene_frames("1") == [0, 1, 2, 3]
    assert [(p["first"], p["last"]) for p in plan] == [(0, 3), (0, 2)]
    assert [[t["frames"] for t in p["tracklets"]] for p in plan] == [[[0, 1, 2, 3], [1, 2]], [[0, 1, 2]]]
    assert ds.raw_scan("0", 0)[0].dtype == np.float64 and ds.raw_scan("1", 0)[0].dtype == np.float32   # rows as stored
    assert ds._scene_and_frame(str(tmp_path / "lidar" / "seq_1_frame_3.pkl")) == ("1", 3)
