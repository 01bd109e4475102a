"""Live multi-target tracking, CPU part: the argument checks of `o3d_crop_resample` through the built library (no launch), the
tracker's refusals, the stream driver's bookkeeping and the command line's scene plan over a KITTI fixture."""
import numpy as np
import pytest
import torch

from open3dsot_b200 import _lib
from open3dsot_b200.datasets import data_classes as dc
from open3dsot_b200.datasets.kitti import kittiDataset
from open3dsot_b200.datasets.synthetic import synthetic_scene, synthetic_sequence
from open3dsot_b200.track import parse_args, scene_plan, stream_max_points
from open3dsot_b200.tracking.multi_tracker import MultiTargetTracker
from test_kitti_reader import _write_scene
from test_tracking_host import _cfg, _Echo


def _args(**kw):
    """o3d_crop_resample's arguments with non-null placeholders (never dereferenced: every call here fails before a launch)."""
    a = dict(scans=16, count=16, frame=16, center=16, rot=16, half=16, N=100, prefix=None, prefix_keep=None, Np=0, seed=0, key=16,
             key_frame=16, perm=0, pick=1, K=4, size=512, scratch=16, out=16, n_out=None, stream=None)
    a.update(kw)
    return list(a.values())


def test_crop_resample_argument_errors_return_status():
    L = _lib.lib()
    f = L.o3d_crop_resample
    assert f(*_args(key=None)) < 0 and b"null" in L.o3d_last_error()
    assert f(*_args(out=None)) < 0 and b"null" in L.o3d_last_error()
    assert f(*_args(scratch=None)) < 0
    assert f(*_args(scans=None)) < 0 and b"scan crop" in L.o3d_last_error()
    assert f(*_args(frame=None)) < 0
    assert f(*_args(Np=8)) < 0 and b"prefix" in L.o3d_last_error()               # a prefix needs its points and keep mask
    assert f(*_args(K=70000)) < 0 and b"K=" in L.o3d_last_error()                  # K > 65535
    assert f(*_args(K=-1)) < 0
    assert f(*_args(N=-5)) < 0 and b"N=" in L.o3d_last_error()
    assert f(*_args(Np=-1)) < 0
    assert f(*_args(size=0)) < 0 and b"size" in L.o3d_last_error()
    assert f(*_args(size=4096)) < 0 and b"size" in L.o3d_last_error()             # size > RESAMPLE_MAX_SIZE
    assert f(*_args(perm=-1)) < 0 and b"stream" in L.o3d_last_error()
    assert f(*_args(K=0)) == 0                                                      # nothing to do: no launch
    assert f(*_args(K=0, N=0, scans=None, frame=None, center=None, rot=None, half=None)) == 0   # prefix-only form: no scan needed


def test_tracker_refuses_what_a_live_stream_cannot_do():
    with pytest.raises(ValueError, match="reference_BB"):
        MultiTargetTracker(_Echo(_cfg(reference_BB="previous_gt")), 100, 4)
    with pytest.raises(ValueError, match="reference_BB"):
        MultiTargetTracker(_Echo(_cfg(reference_BB="current_gt")), 100, 4)
    with pytest.raises(ValueError, match="shape_aggregation"):
        MultiTargetTracker(_Echo(_cfg(shape_aggregation="all")), 100, 4)
    with pytest.raises(ValueError, match="max_targets"):
        MultiTargetTracker(_Echo(_cfg()), 100, 0)


def test_tracker_refuses_bad_targets_and_scans():
    trk = MultiTargetTracker(_Echo(_cfg()), 100, 2, use_graph=False)
    box = dc.Box(np.zeros(3), np.array([1.5, 4.0, 1.5]), np.eye(3))
    with pytest.raises(RuntimeError, match="step"):
        trk.add(3, box)                                    # no scan yet
    with pytest.raises(ValueError, match="max_points"):
        trk.step(torch.zeros(101, 3))                     # larger than the scan buffer: refused before anything is copied
    trk.scans_seen = 1                                     # as after a first step: the (empty) scan buffer is the current scan
    trk.add(3, box)
    with pytest.raises(ValueError, match="target_id 3"):
        trk.add(3, box)                                    # a duplicate active id
    trk.add(8, box)
    with pytest.raises(ValueError, match="max_targets"):
        trk.add(9, box)                                    # beyond capacity
    with pytest.raises(ValueError, match="target_id 4"):
        trk.drop(4)                                        # unknown id
    assert trk.targets() == {3: 0, 8: 1}
    trk.drop(3)
    trk.add(9, box)                                        # the freed slot is reused
    assert trk.targets() == {8: 1, 9: 0}
    ids = trk.boxes()["ids"]
    assert ids.tolist() == [9, 8]
    trk.drop(9)
    assert trk.boxes()["ids"].tolist() == [-1, 8]
    assert torch.equal(trk.box_c[0], torch.zeros(3)) and torch.equal(trk.box_r[0], torch.eye(3))   # back to the dummy box


def test_synthetic_scene_is_a_stream_of_moving_boxes():
    s = synthetic_scene(n_frames=4, n_points=5000, n_objects=6, seed=3)
    assert len(s["scans"]) == 4 and all(x.shape == (5000, 3) and x.dtype == np.float32 for x in s["scans"])
    assert len(s["boxes"]) == 6 and all(len(b) == 4 for b in s["boxes"])
    for boxes in s["boxes"]:
        assert np.linalg.norm(boxes[3].center - boxes[0].center) > 0.5          # every object moves
        n_in = [int(((x - b.center) @ b.rotation_matrix).__abs__().__lt__(b.wlh[[1, 0, 2]] / 2 + 0.05).all(1).sum())
                for x, b in zip(s["scans"], boxes)]
        assert min(n_in) >= 250                                                  # its surface points are in its box


def test_scene_plan_groups_tracklets_by_scene(tmp_path):
    root = str(tmp_path)
    a = synthetic_sequence(n_frames=5, n_points=900, seed=1, n_object=200)
    b = synthetic_sequence(n_frames=3, n_points=700, seed=2, n_object=200)
    c = synthetic_sequence(n_frames=4, n_points=800, seed=3, n_object=200)
    # scene 0019: car 4 over frames 0-4, car 2 over frames 0-2 (then absent); scene 0020: car 7 over frames 0-3, a pedestrian
    _write_scene(root, "0019", [((4, "Car"), a), ((2, "Car"), b)])
    _write_scene(root, "0020", [((7, "Car"), c), ((1, "Pedestrian"), b)])
    ds = kittiDataset(root, "test", "Car", preloading=False, preload_offset=-1)
    plan = scene_plan(ds)
    assert [p["scene"] for p in plan] == ["0019", "0020"]
    assert [(p["first"], p["last"]) for p in plan] == [(0, 4), (0, 3)]
    got = [[(t["index"], t["track_id"], t["start"], t["end"], t["frames"]) for t in p["tracklets"]] for p in plan]
    assert got == [[(0, 4, 0, 4, [0, 1, 2, 3, 4]), (1, 2, 0, 2, [0, 1, 2])], [(2, 7, 0, 3, [0, 1, 2, 3])]]
    assert stream_max_points(ds, plan) == 900 + 700                     # frames 0-2 of scene 0019 hold both cars' scans
    scan = ds.read_scan("0019", 1)
    assert scan.points.shape == (3, 1600)                              # the whole scan
    assert ds.read_scan("0019", 99).points.shape == (3, 1)             # a missing scan: the reader's placeholder
    assert ds.velos == {} or all(not v for v in ds.velos.values())     # streaming does not fill the reader's cache
    box = ds.box_from_anno(ds.tracklet_anno_list[2][1])
    assert np.abs(box.center - c[1]["3d_bbox"].center).max() < 1e-4


def test_command_line_defaults():
    a = parse_args(["--cfg", "x.yaml", "--path", "/data"])
    assert (a.split, a.out, a.max_targets, a.max_points, a.seed, a.checkpoint) == ("test", "results.jsonl", 64, None, 0, None)
