"""Several object classes over shared scan feeds, CPU part: per-class scene peaks and the feed schedule, the multi-class
tracker's refusals and bookkeeping (stand-in models on the CPU), the merged scene plan of two readers over a KITTI fixture, and
the command line's class arguments."""
import os
import pickle

import numpy as np
import pytest
import torch

from open3dsot_b200 import track
from open3dsot_b200.config import load_config
from open3dsot_b200.datasets import data_classes as dc
from open3dsot_b200.datasets.kitti import kittiDataset
from open3dsot_b200.datasets.waymo_data import WaymoDataset
from open3dsot_b200.datasets.synthetic import synthetic_sequence
from open3dsot_b200.tracking.multi_class import MultiClassTracker, track_classes
from open3dsot_b200.tracking.multi_tracker import MultiTargetTracker, ScanFeeds, class_peaks, feed_schedule, scene_peak
from test_kitti_reader import _write_scene
from test_multi_feed import _write_waymo
from test_tracking_host import _cfg, _Echo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BOX = dc.Box(np.zeros(3), np.array([1.5, 4.0, 1.5]), np.eye(3))


# ------------------------------------------------------------------ per-class peaks and the schedule
def test_class_peaks():
    starts = {0: [(("Car", 1), BOX), (("Car", 2), BOX), (("Ped", 1), BOX)], 3: [(("Ped", 2), BOX)], 5: [(("Car", 3), BOX)]}
    ends = {("Car", 1): 2, ("Car", 2): 6, ("Ped", 1): 4, ("Car", 3): 7}
    assert class_peaks(8, starts, ends) == {"Car": 2, "Ped": 2}
    # each class's peak is scene_peak over that class's targets alone
    cars = {t: [(k, b) for k, b in g if k[0] == "Car"] for t, g in starts.items()}
    assert scene_peak(8, cars, ends) == 2
    assert class_peaks(8, {}, {}) == {}


def _check_class_schedule(lengths, peaks, feeds, max_targets):
    sched = feed_schedule(lengths, peaks, feeds, max_targets)
    assert sorted(i for i, _, _ in sched) == list(range(len(lengths)))
    assert [lengths[i] for i, _, _ in sched] == sorted(lengths, reverse=True)
    end = max(s + lengths[i] for i, _, s in sched)
    for step in range(end):
        run = [(i, f) for i, f, s in sched if s <= step < s + lengths[i]]
        for c, k in max_targets.items():                                   # every class's peaks fit at every step
            assert sum(peaks[i].get(c, 0) for i, _ in run) <= k, (step, c)
        assert len({f for _, f in run}) == len(run) and all(0 <= f < feeds for _, f in run)
    # no scene is admitted early: one step sooner, its feed or some class's slots were still taken
    for n, (i, f, s) in enumerate(sched):
        if s == 0:
            continue
        before = [(j, g) for j, g, t in sched[:n] if t <= s - 1 < t + lengths[j]]
        feeds_busy = len(before) >= feeds
        slots_busy = any(sum(peaks[j].get(c, 0) for j, _ in before) + peaks[i].get(c, 0) > k for c, k in max_targets.items())
        held_by_queue = n > 0 and sched[n - 1][2] == s                    # admitted in order: the one before it waited too
        assert feeds_busy or slots_busy or held_by_queue, (i, s)
    return sched


def test_class_schedule_invariants():
    rng = np.random.default_rng(9)
    for _ in range(40):
        n = int(rng.integers(1, 25))
        feeds = int(rng.integers(1, 8))
        cap = {"Car": int(rng.integers(1, 12)), "Ped": int(rng.integers(1, 12))}
        lengths = [int(x) for x in rng.integers(1, 40, n)]
        peaks = [{"Car": int(rng.integers(0, cap["Car"] + 1)), "Ped": int(rng.integers(0, cap["Ped"] + 1))} for _ in range(n)]
        _check_class_schedule(lengths, peaks, feeds, cap)
    # the Car slots are free but the pedestrians of scene 2 wait for scene 0's to end
    sched = _check_class_schedule([10, 6, 3], [{"Car": 1, "Ped": 2}, {"Car": 1}, {"Car": 1, "Ped": 1}], 3, {"Car": 5, "Ped": 2})
    assert sched == [(0, 0, 0), (1, 1, 0), (2, 0, 10)]
    # one class per scene: the two classes' slots are counted apart
    sched = _check_class_schedule([10, 6, 3], [{"Car": 2}, {"Ped": 2}, {"Car": 2}], 3, {"Car": 4, "Ped": 2})
    assert sched == [(0, 0, 0), (1, 1, 0), (2, 2, 0)]


def test_class_schedule_refuses_a_scene_that_never_fits():
    with pytest.raises(ValueError, match=r"max_targets\['Ped'\]=2: scene 1 has 3 targets of class 'Ped'"):
        feed_schedule([5, 5], [{"Car": 1}, {"Ped": 3}], 2, {"Car": 4, "Ped": 2})
    with pytest.raises(ValueError, match="'Cyclist'"):
        feed_schedule([5], [{"Cyclist": 1}], 1, {"Car": 4})
    with pytest.raises(ValueError, match="no frames"):
        feed_schedule([0], [{"Car": 1}], 1, {"Car": 4})


# ------------------------------------------------------------------ the tracker: refusals and bookkeeping
def _models(**per_class):
    return {n: _Echo(_cfg(**kw)) for n, kw in per_class.items()}


def test_refuses_mismatched_frame_conventions_and_bad_classes():
    for key, val in (("up_axis", [0, -1, 0]), ("IoU_space", 2), ("degrees", False)):
        with pytest.raises(ValueError, match=f"class 'Ped': {key}="):
            MultiClassTracker(_models(Car={}, Ped={key: val}), 100, {"Car": 2, "Ped": 2})
    with pytest.raises(ValueError, match="no classes"):
        MultiClassTracker({}, 100, {})
    with pytest.raises(ValueError, match="'Ped' has no slot count"):
        MultiClassTracker(_models(Car={}, Ped={}), 100, {"Car": 2})
    # each class's own refusals apply, naming the class
    with pytest.raises(ValueError, match="class 'Ped': reference_BB"):
        MultiClassTracker(_models(Car={}, Ped={"reference_BB": "previous_gt"}), 100, {"Car": 2, "Ped": 2})
    with pytest.raises(ValueError, match="class 'Ped': shape_aggregation 'all'"):
        MultiClassTracker(_models(Car={}, Ped={"shape_aggregation": "all"}), 100, {"Car": 2, "Ped": 2})
    with pytest.raises(ValueError, match="class 'Car': max_points=100, max_targets=0"):
        MultiClassTracker(_models(Car={}, Ped={}), 100, {"Car": 0, "Ped": 2})


def test_add_drop_targets_and_shared_feeds():
    trk = MultiClassTracker(_models(Car={}, Ped={"shape_aggregation": "previous"}), 100, {"Car": 2, "Ped": 3}, feeds=2,
                            use_graph=False)
    feeds = trk.scan_feeds
    assert all(t.scan_feeds is feeds for t in trk.trackers.values()) and feeds.scans.shape == (2, 2, 100, 3)
    with pytest.raises(ValueError, match="class 'Cyclist' is not tracked"):
        trk.add("Cyclist", 1, BOX)
    trk.put(0, torch.ones(7, 3))
    feeds.ingest()                                                         # advance()'s ingest (its step needs the GPU)
    # the feed state is one: both class trackers see the same parity and counters
    assert feeds.feed_seen == [1, 0] and all(t.feed_seen == [1, 0] and t._fcur == [0, 1] for t in trk.trackers.values())
    assert int(feeds.count[0, 0]) == 7 and feeds.fstate.tolist() == [[1, 0], [0, 1], [1, 0]]
    trk.add("Car", 3, BOX)
    trk.add("Ped", 3, BOX)                                                 # the same id in another class
    with pytest.raises(ValueError, match="target_id 3 is already active"):
        trk.add("Car", 3, BOX)                                             # a duplicate (class, id)
    with pytest.raises(RuntimeError, match="feed 1"):
        trk.add("Car", 4, BOX, feed=1)                                     # no scan on that feed yet
    trk.add("Ped", 9, BOX)
    assert trk.targets() == {("Car", 3): 0, ("Ped", 3): 2, ("Ped", 9): 3}   # rows of snapshot(): Car's 2 slots, then Ped's
    assert trk.snapshot().shape == (5, 15)
    trk.drop("Ped", 3)
    with pytest.raises(ValueError, match="target_id 3 is not active"):
        trk.drop("Ped", 3)
    assert trk.targets() == {("Car", 3): 0, ("Ped", 9): 3}
    with pytest.raises(ValueError, match="use put"):
        trk.step(torch.zeros(5, 3))


def test_track_classes_refuses_bad_scenes():
    models = _models(Car={}, Ped={})
    scene = {"frames": 3, "scan": lambda t: np.zeros((5, 3), np.float32), "starts": {0: [(("Ped", 1), BOX), (("Ped", 2), BOX)]},
             "ends": {}}
    with pytest.raises(ValueError, match=r"max_targets\['Ped'\]=1"):
        track_classes(models, [scene], 1, {"Car": 1, "Ped": 1}, max_points=5, use_graph=False)
    cyc = dict(scene, starts={0: [(("Cyclist", 1), BOX)]})
    with pytest.raises(ValueError, match="'Cyclist', which has no model"):
        track_classes(models, [cyc], 1, {"Car": 1, "Ped": 2}, max_points=5, use_graph=False)
    with pytest.raises(ValueError, match="ids must be unique"):
        track_classes(models, [scene, scene], 1, {"Car": 1, "Ped": 2}, max_points=5, use_graph=False)


def test_store_refuses_a_tracker_of_another_size():
    feeds = ScanFeeds(100, 2, "cpu")
    with pytest.raises(ValueError, match="max_points=50"):
        MultiTargetTracker(_Echo(_cfg()), 50, 2, feeds=feeds)
    trk = MultiTargetTracker(_Echo(_cfg()), 100, 2, feeds=feeds, use_graph=False)
    assert trk.F == 2 and trk.scans is feeds.scans


# ------------------------------------------------------------------ the merged scene plan over a KITTI fixture
def test_class_scene_plan_merges_two_readers(tmp_path):
    root = str(tmp_path)
    a = synthetic_sequence(n_frames=5, n_points=900, seed=1, n_object=200)
    b = synthetic_sequence(n_frames=3, n_points=700, seed=2, n_object=200)
    c = synthetic_sequence(n_frames=4, n_points=800, seed=3, n_object=200)
    d = synthetic_sequence(n_frames=2, n_points=600, seed=4, n_object=200)
    # scene 0019: car 4 over frames 0-4, a pedestrian over frames 0-2; scene 0020: car 7 over frames 0-3, a pedestrian over 0-1
    # (each merged stream runs to the last frame of either class)
    _write_scene(root, "0019", [((4, "Car"), a), ((2, "Pedestrian"), b)])
    _write_scene(root, "0020", [((7, "Car"), c), ((1, "Pedestrian"), d)])
    cars = kittiDataset(root, "test", "Car", preloading=False, preload_offset=-1)
    peds = kittiDataset(root, "test", "Pedestrian", preloading=False, preload_offset=-1)
    plan = track.class_scene_plan({"Car": cars, "Pedestrian": peds})
    assert [p["scene"] for p in plan] == ["0019", "0020"]
    assert [(p["first"], p["last"], p["frames"]) for p in plan] == [(0, 4, [0, 1, 2, 3, 4]), (0, 3, [0, 1, 2, 3])]
    got = [[(t["class"], t["index"], t["track_id"], t["start"], t["end"]) for t in p["tracklets"]] for p in plan]
    assert got == [[("Car", 0, 4, 0, 4), ("Pedestrian", 0, 2, 0, 2)], [("Car", 1, 7, 0, 3), ("Pedestrian", 1, 1, 0, 1)]]
    assert [(p["first"], p["last"]) for p in track.scene_plan(peds)] == [(0, 2), (0, 1)]
    # each class's tracklets are its own reader's, in that reader's plan
    for cls, ds in (("Car", cars), ("Pedestrian", peds)):
        alone = {(p["scene"], t["index"]): (t["start"], t["end"], t["frames"]) for p in track.scene_plan(ds) for t in p["tracklets"]}
        merged = {(p["scene"], t["index"]): (t["start"], t["end"], t["frames"]) for p in plan for t in p["tracklets"]
                  if t["class"] == cls}
        assert merged == alone


def _check_class_scenes(datasets, plan):
    """Every frame of the merged plan is read by a reader that lists it, and its scan is that reader's whole scan."""
    scenes = track.class_scenes(datasets, plan)
    sizes = []
    for p, sc in zip(plan, scenes):
        assert sc["frames"] == len(p["frames"]) == len(p["reader_of"])
        for t, f in enumerate(p["frames"]):
            ds = datasets[p["reader_of"][f]]
            assert f in ds.scene_frames(p["scene"])
            rows, xfs = sc["scan"](t)
            want_rows, want_xfs = ds.raw_scan(p["scene"], f)
            assert np.array_equal(rows, want_rows) and all(np.array_equal(a, b) for a, b in zip(xfs, want_xfs))
            sizes.append(ds.scan_size(p["scene"], f))
    assert track.class_stream_max_points(datasets, plan) == max(sizes)
    return scenes


def test_class_plan_reads_scenes_the_first_class_is_absent_from_on_waymo(tmp_path):
    root = str(tmp_path)
    _write_waymo(root)                                                     # vehicles in segments 0 and 1
    lidar = os.path.join(root, "lidar")
    peds = {"seg0_p": [{"PC": os.path.join(lidar, f"seq_0_frame_{f}.pkl"), "Class": "PEDESTRIAN",
                        "Box": np.array([-3.0 + 0.2 * f, 4.0, 0.9, 0.8, 0.7, 1.8, 1.0, 0.0, 0.05 * f])} for f in (1, 2)]}
    with open(os.path.join(root, "sot_infos_pedestrian_val.pkl"), "wb") as fh:
        pickle.dump(peds, fh)
    ped = WaymoDataset(root, "val", "PEDESTRIAN", preloading=False, preload_offset=-1)
    veh = WaymoDataset(root, "val", "VEHICLE", preloading=False, preload_offset=-1)
    assert ped.scene_list == ["0"]                                        # the pedestrian reader knows segment 0 only
    with pytest.raises(KeyError):
        ped.raw_scan("1", 0)
    datasets = {"PEDESTRIAN": ped, "VEHICLE": veh}
    plan = track.class_scene_plan(datasets)
    assert [(p["scene"], p["first"], p["last"]) for p in plan] == [("0", 0, 3), ("1", 0, 2)]
    assert plan[0]["reader_of"] == {f: "PEDESTRIAN" for f in range(4)}     # the first class's reader lists segment 0 ...
    assert plan[1]["reader_of"] == {f: "VEHICLE" for f in range(3)}        # ... and only the vehicle reader segment 1
    scenes = _check_class_scenes(datasets, plan)
    starts = {k for sc in scenes for g in sc["starts"].values() for k, _ in g}
    assert starts == {("PEDESTRIAN", 0), ("VEHICLE", 0), ("VEHICLE", 1), ("VEHICLE", 2)}
    assert scenes[0]["ends"][("PEDESTRIAN", 0)] == 2 and scenes[1]["ends"][("VEHICLE", 2)] == 2


def test_class_plan_reads_scenes_the_first_class_is_absent_from_on_kitti(tmp_path):
    root = str(tmp_path)
    car = synthetic_sequence(n_frames=3, n_points=900, seed=11, n_object=200)
    ped = synthetic_sequence(n_frames=4, n_points=700, seed=12, n_object=200)
    _write_scene(root, "0019", [((4, "Car"), car)])
    _write_scene(root, "0020", [((1, "Pedestrian"), ped)])                 # no car in scene 0020
    datasets = {c: kittiDataset(root, "test", c, preloading=False, preload_offset=-1) for c in ("Car", "Pedestrian")}
    plan = track.class_scene_plan(datasets)
    assert [(p["scene"], p["frames"]) for p in plan] == [("0019", [0, 1, 2]), ("0020", [0, 1, 2, 3])]
    assert plan[0]["reader_of"] == {f: "Car" for f in range(3)}
    assert plan[1]["reader_of"] == {f: "Pedestrian" for f in range(4)}
    _check_class_scenes(datasets, plan)


# ------------------------------------------------------------------ who advances shared feeds
def test_only_the_owner_advances_shared_feeds():
    feeds = ScanFeeds(100, 2, "cpu")
    first = MultiTargetTracker(_Echo(_cfg()), 100, 2, feeds=feeds, use_graph=False)
    other = MultiTargetTracker(_Echo(_cfg()), 100, 2, feeds=feeds, use_graph=False)
    assert feeds.owner is first
    other.put(0, torch.ones(3, 3))
    with pytest.raises(RuntimeError, match="another tracker owns"):
        other.advance()                                                    # would move first's scans without stepping it
    assert feeds.feed_seen == [0, 0] and feeds.staged                     # refused before anything moved
    with pytest.raises(ValueError, match="already belong to another tracker"):
        MultiClassTracker(_models(Car={}), 100, {"Car": 2}, feeds=feeds)
    trk = MultiClassTracker(_models(Car={}, Ped={}), 100, {"Car": 2, "Ped": 2}, use_graph=False)
    assert trk.scan_feeds.owner is trk
    with pytest.raises(RuntimeError, match="another tracker owns"):
        trk.trackers["Car"].advance()
    free = ScanFeeds(100, 1, "cpu")
    with pytest.raises(ValueError, match="class 'Ped'"):
        MultiClassTracker(_models(Car={}, Ped={"shape_aggregation": "all"}), 100, {"Car": 2, "Ped": 2}, feeds=free)
    assert free.owner is None                                              # a failed build leaves the store free


# ------------------------------------------------------------------ the command line
def test_command_line_class_arguments():
    base = ["--cfg", "a.yaml", "--path", "/data"]
    a = track.parse_args(base)
    assert a.add_class is None and a.max_targets == 64 and track.class_targets(a.max_targets, "Car") == 64
    a = track.parse_args(base + ["--add_class", "b.yaml", "--add_class", "c.yaml", "c.ckpt", "--max_targets", "Pedestrian=8"])
    assert a.add_class == [["b.yaml"], ["c.yaml", "c.ckpt"]]
    assert a.max_targets == {None: 64, "Pedestrian": 8}
    assert track.class_targets(a.max_targets, "Pedestrian") == 8 and track.class_targets(a.max_targets, "Car") == 64
    a = track.parse_args(base + ["--max_targets", "Car=16", "--max_targets", "32"])
    assert track.class_targets(a.max_targets, "Car") == 16 and track.class_targets(a.max_targets, "Van") == 32
    assert track.parse_args(base + ["--max_targets", "12"]).max_targets == 12
    for bad in (["--max_targets", "Car=x"], ["--max_targets", "=4"], ["--add_class", "b.yaml", "b.ckpt", "extra"]):
        with pytest.raises(SystemExit):
            track.parse_args(base + bad)


def test_single_class_arguments_unchanged():
    a = track.parse_args(["--cfg", "x.yaml", "--path", "/data", "--max_targets", "4", "--seed", "3", "--precision", "bf16"])
    assert vars(a) == {"cfg": "x.yaml", "checkpoint": None, "path": "/data", "split": "test", "out": "results.jsonl",
                       "add_class": None, "max_targets": 4, "max_points": None, "seed": 3, "precision": "bf16"}


def test_command_line_refuses_classes_that_cannot_share_scans():
    cfg = lambda name, **over: load_config(os.path.join(ROOT, "cfgs", name), over)
    track.check_classes([cfg("BAT_Car.yaml"), cfg("BAT_Pedestrian.yaml")], ["car", "ped"])           # compatible
    with pytest.raises(SystemExit, match="dataset 'nuscenes' differs"):
        track.check_classes([cfg("BAT_Car.yaml"), cfg("BAT_PEDESTRIAN_NUSCENES.yaml")], ["car", "ped"])
    with pytest.raises(SystemExit, match="coordinate_mode=camera"):
        track.check_classes([cfg("BAT_Car.yaml"), cfg("BAT_Pedestrian.yaml", coordinate_mode="camera")], ["car", "ped"])
    with pytest.raises(SystemExit, match="key_frame_only=False"):
        track.check_classes([cfg("BAT_CAR_NUSCENES.yaml"), cfg("BAT_PEDESTRIAN_NUSCENES.yaml")], ["car", "ped"])
    with pytest.raises(SystemExit, match="category_name 'Car' is already tracked"):
        track.check_classes([cfg("BAT_Car.yaml"), cfg("P2B_Car.yaml", coordinate_mode="velodyne")], ["bat", "p2b"])
    with pytest.raises(SystemExit, match="dataset"):
        track.main(["--cfg", os.path.join(ROOT, "cfgs", "BAT_Car.yaml"), "--path", "/nonexistent",
                    "--add_class", os.path.join(ROOT, "cfgs", "BAT_PEDESTRIAN_NUSCENES.yaml")])


def test_single_class_command_line_runs_the_one_class_path(tmp_path, monkeypatch):
    """One --cfg: main() calls run() (the one-class path, unchanged) with the arguments it always had, never run_classes."""
    root = str(tmp_path)
    _write_scene(root, "0019", [((4, "Car"), synthetic_sequence(n_frames=3, n_points=500, seed=1, n_object=100))])
    calls = []
    monkeypatch.setattr(torch.nn.Module, "cuda", lambda self, *a, **k: self)   # build the model on the CPU
    monkeypatch.setattr(track, "run", lambda *a, **k: calls.append(("run", a, k)) or {"success": 1.0, "precision": 2.0})
    monkeypatch.setattr(track, "run_classes", lambda *a, **k: calls.append(("run_classes", a, k)))
    out = str(tmp_path / "r.jsonl")
    got = track.main(["--cfg", os.path.join(ROOT, "cfgs", "BAT_Car.yaml"), "--path", root, "--out", out, "--max_targets", "5",
                      "--seed", "2", "--precision", "bf16"])
    assert [c[0] for c in calls] == ["run"]
    _, (model, ds, path), kw = calls[0]
    assert type(model).__name__ == "BAT" and isinstance(ds, kittiDataset) and ds.category_name == "Car" and path == out
    assert kw == {"max_targets": 5, "max_points": None, "seed": 2, "precision": "bf16"}
    assert got == {"success": 1.0, "precision": 2.0, "checkpoint": None, "split": "test", "out": out}
