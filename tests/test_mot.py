"""Multi-object tracking scores on the host (tracking/mot.py): the reference `mot_reference` against hand-worked sequences, one
per rule of the module docstring; `mot_metrics` input refusals; `o3d_mot_clear`'s argument checks through the C ABI (refused
before any launch, so no device is needed); `--mot` parsing and the command line passing it to `run` / `run_classes`.

motmetrics itself is not installed here: these cases, not motmetrics, pin the semantics the kernel is held to."""
import ctypes
import json
import math
import os

import numpy as np
import pytest
import torch

from open3dsot_b200 import _lib, track
from open3dsot_b200.datasets.data_classes import Box
from open3dsot_b200.datasets.kitti import kittiDataset
from open3dsot_b200.datasets.synthetic import synthetic_sequence
from open3dsot_b200.tracking.mot import MAX_BOXES, check_run, mot_metrics, mot_reference, pack_run
from open3dsot_b200.utils.metrics import _footprint, estimateAccuracy, estimateOverlap
from test_kitti_reader import _write_scene

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
UP = (0, 0, 1)


def B(x, y=0.0, wlh=(1.0, 1.0, 1.0), yaw=0.0):
    return Box([x, y, 0.0], wlh, yaw_degrees=yaw)


def dist(seqs, thr=1.0):
    """The reference with centre distance in 3-D (cost = |dx| for boxes on the x axis)."""
    return mot_reference(seqs, "distance", thr, dim=3, up_axis=UP)


def seq0(r):
    return r["sequences"][0]


def test_estimate_overlap_takes_precomputed_footprints():
    rng = np.random.default_rng(0)
    for _ in range(20):
        a = Box(rng.normal(size=3), rng.uniform(0.5, 3, 3), yaw_degrees=rng.uniform(-180, 180))
        b = Box(a.center + rng.normal(scale=0.8, size=3), rng.uniform(0.5, 3, 3), yaw_degrees=rng.uniform(-180, 180))
        for dim in (2, 3):
            for up in ((0, 0, 1), (0, -1, 0)):
                fp = (_footprint(a, up), _footprint(b, up))
                assert estimateOverlap(a, b, dim, up, footprints=fp) == estimateOverlap(a, b, dim, up)


def test_carry_over_beats_a_cheaper_new_pair():
    seqs = [[([(1, B(0))], [(10, B(0.5))]),
             ([(1, B(0))], [(10, B(0.9)), (11, B(0.1))])]]
    s = seq0(dist(seqs))
    assert (s["num_matches"], s["num_switches"], s["num_false_positives"], s["num_misses"]) == (2, 0, 1, 0)
    assert s["total_cost"] == 0.5 + 0.9


@pytest.mark.parametrize("order", ["o2 first", "o1 first"])
def test_two_objects_with_the_same_last_match_are_decided_by_frame_order(order):
    # o1 - h7, then o2 takes h7 (o1 absent): both have m[o] = h7.  On frame 2 the first of them in the frame carries h7; h8 is
    # valid with o2 only
    a, b = (1, B(0.0)), (2, B(3.0))
    f2 = [b, a] if order == "o2 first" else [a, b]
    seqs = [[([a], [(7, B(0.0))]),
             ([b], [(7, B(3.0))]),
             (f2, [(7, B(1.4)), (8, B(2.2))])]]
    s = seq0(dist(seqs, thr=2.0))
    got = (s["num_matches"], s["num_switches"], s["num_misses"], s["num_false_positives"])
    if order == "o2 first":          # o2 keeps h7; o1 has no valid partner left
        assert got == (3, 0, 1, 1) and math.isclose(s["total_cost"], 3.0 - 1.4, abs_tol=1e-12)
    else:                            # o1 keeps h7; o2 switches to h8
        assert got == (3, 1, 0, 0) and math.isclose(s["total_cost"], 1.4 + (3.0 - 2.2), abs_tol=1e-12)


def test_maximum_cardinality_beats_greedy_by_cost():
    # greedy takes o1-h1 (0.1) and leaves o2 without a partner; the maximum matching pairs o1-h2 and o2-h1
    seqs = [[([(1, B(0.0)), (2, B(1.1))], [(10, B(0.1)), (11, B(-1.0))])]]
    s = seq0(dist(seqs, thr=1.05))
    assert (s["num_matches"], s["num_misses"], s["num_false_positives"]) == (2, 0, 0)
    assert math.isclose(s["total_cost"], 1.0 + 1.0, abs_tol=1e-12)


def test_switch_then_switch_back():
    o = (1, B(0.0))
    seqs = [[([o], [(10, B(0.1))]), ([o], [(10, B(0.1))]), ([o], [(11, B(0.2))]), ([o], [(10, B(0.1))])]]
    s = seq0(dist(seqs))
    assert (s["num_matches"], s["num_switches"]) == (2, 2)
    assert s["mota"] == 1 - 2 / 4


def test_misses_and_false_positives_in_one_sided_and_empty_frames():
    seqs = [[([(1, B(0.0)), (2, B(5.0))], []), ([], [(10, B(0.0))]), ([], []), ([(1, B(0.0))], [(10, B(3.0))])]]
    s = seq0(dist(seqs))
    assert (s["num_objects"], s["num_predictions"], s["num_matches"], s["num_misses"], s["num_false_positives"]) == (3, 2, 0, 3, 2)
    assert s["mota"] == 1 - 5 / 3 and math.isnan(s["motp"]) and s["idf1"] == 0.0
    empty = seq0(dist([[([], [])]]))
    assert math.isnan(empty["mota"]) and math.isnan(empty["idf1"]) and math.isnan(empty["idp"])


def test_fragmentations_count_gaps_between_tracked_frames_only():
    # tracked T T M T M M T M: gaps after frames 1 and 3 count; the miss after the last tracked frame does not
    o = (1, B(0.0))
    hit, miss = ([o], [(10, B(0.1))]), ([o], [])
    seqs = [[hit, hit, miss, hit, miss, miss, hit, miss]]
    s = seq0(dist(seqs))
    assert s["num_fragmentations"] == 2 and s["num_misses"] == 4
    assert seq0(dist([[miss, hit, hit, miss]]))["num_fragmentations"] == 0


def test_mostly_tracked_and_lost_at_exactly_0_8_and_0_2():
    objs = {1: 4, 2: 1, 3: 0, 4: 3}          # tracked frames of 5: 0.8 (MT), 0.2 (PT), 0 (ML), 0.6 (PT)
    frames = []
    for t in range(5):
        gt = [(o, B(10.0 * o)) for o in objs]
        hyp = [(100 + o, B(10.0 * o)) for o, k in objs.items() if t < k]
        frames.append((gt, hyp))
    s = seq0(dist([frames]))
    assert (s["mostly_tracked"], s["partially_tracked"], s["mostly_lost"]) == (1, 2, 1)


def test_idf1_takes_the_global_assignment():
    # o1 ~ h1 on frames 0-1, o1 ~ h2 on frames 2-4: per frame 4 matches and a switch, but one identity: idtp = 3
    o = (1, B(0.0))
    seqs = [[([o], [(10, B(0.1))])] * 2 + [([o], [(11, B(0.2))])] * 3]
    s = seq0(dist(seqs))
    assert (s["num_matches"], s["num_switches"], s["idtp"], s["idfn"], s["idfp"]) == (4, 1, 3, 2, 2)
    assert s["idf1"] == 2 * 3 / 10 and s["idp"] == 3 / 5 and s["idr"] == 3 / 5


def test_thresholds_are_inclusive():
    # IoU: squares of side 3 one apart in x: intersection 6, union 12, IoU exactly 0.5
    gt, hyp = B(0.0, wlh=(3.0, 3.0, 1.0)), B(1.0, wlh=(3.0, 3.0, 1.0))
    assert estimateOverlap(gt, hyp, 2, UP) == 0.5
    at = mot_reference([[([(1, gt)], [(2, hyp)])]], "iou", 0.5, dim=2, up_axis=UP)
    s = seq0(at)
    assert s["num_matches"] == 1 and s["total_cost"] == 0.5 and s["mean_iou"] == 0.5
    above = seq0(mot_reference([[([(1, gt)], [(2, hyp)])]], "iou", np.nextafter(0.5, 1.0), dim=2, up_axis=UP))
    assert above["num_matches"] == 0 and above["num_misses"] == 1 and above["num_false_positives"] == 1
    # distance: (3, 4, 0) from the origin is exactly 5
    far = Box([3.0, 4.0, 0.0], (1.0, 1.0, 1.0))
    assert estimateAccuracy(B(0.0), far, 3, UP) == 5.0
    assert seq0(dist([[([(1, B(0.0))], [(2, far)])]], thr=5.0))["num_matches"] == 1
    assert seq0(dist([[([(1, B(0.0))], [(2, far)])]], thr=np.nextafter(5.0, 0.0)))["num_matches"] == 0


def test_totals_sum_the_sequences_and_recompute_the_ratios():
    o = (1, B(0.0))
    a = [([o], [(10, B(0.1))]), ([o], [(11, B(0.2))])]
    b = [([o, (2, B(4.0))], [(10, B(0.3))]), ([o], [(12, B(9.0))])]
    r = dist([a, b])
    sa, sb = r["sequences"]
    t = r["total"]
    for k in ("num_objects", "num_predictions", "num_matches", "num_switches", "num_misses", "num_false_positives",
              "num_fragmentations", "mostly_tracked", "partially_tracked", "mostly_lost", "idtp"):
        assert t[k] == sa[k] + sb[k], k
    assert t["total_cost"] == sa["total_cost"] + sb["total_cost"]
    assert t["mota"] == 1 - (t["num_misses"] + t["num_switches"] + t["num_false_positives"]) / t["num_objects"]
    assert t["idf1"] == 2 * t["idtp"] / (t["num_objects"] + t["num_predictions"])
    # ids never cross sequences: object 1 of b is not object 1 of a
    assert sb["num_switches"] == 0 and sa["num_switches"] == 1


def test_pack_run_round_trip_and_dense_indices():
    seqs = [[([(5, B(0.0)), (9, B(1.0))], [(3, B(0.0))])], [([(5, B(2.0))], [])]]
    run = pack_run(seqs)
    assert run.seq_frame.tolist() == [0, 1, 2] and run.frame_gt.tolist() == [0, 2, 3] and run.frame_hyp.tolist() == [0, 1, 1]
    _, dense = check_run(run)
    assert dense.obj_off.tolist() == [0, 2, 3] and dense.hyp_off.tolist() == [0, 1, 1] and dense.cooc_off.tolist() == [0, 2, 2]
    assert (dense.max_gt, dense.max_hyp) == (2, 1)
    assert json.dumps(dist(run)) == json.dumps(dist(seqs))        # NaN ratios compare equal as text


def test_mot_metrics_refusals():
    ok = [[([(1, B(0.0))], [(2, B(0.0))])]]
    bad_scoring = [("mota", 0.5, 2, UP), ("iou", 0.0, 2, UP), ("iou", 1.5, 2, UP), ("iou", float("nan"), 2, UP),
                   ("distance", 0.0, 2, UP), ("distance", float("inf"), 2, UP), ("distance", -1.0, 2, UP),
                   ("iou", "x", 2, UP), ("iou", 0.5, 4, UP), ("iou", 0.5, 2, (0, 0, 0))]
    for metric, thr, dim, up in bad_scoring:
        for fn in (mot_metrics, mot_reference):
            with pytest.raises(ValueError, match="mot:"):
                fn(ok, metric, thr, dim, up)
    bad_runs = [[[([(1, B(0.0)), (1, B(3.0))], [])]],                            # an id twice in one frame
                [[([], [(4, B(0.0)), (4, B(3.0))])]],
                [[([(i, B(float(i))) for i in range(MAX_BOXES + 1)], [])]],       # too many boxes in a frame
                [[([], [(i, B(float(i))) for i in range(MAX_BOXES + 1)])]],
                [[([(1, Box([np.nan, 0, 0], (1, 1, 1)))], [])]],                  # not finite
                [[([(1, B(0.0))],)]],                                             # not a (gt, hyp) pair
                [[([1], [])]]]                                                    # not (id, Box)
    for run in bad_runs:
        for fn in (mot_metrics, mot_reference):
            with pytest.raises(ValueError, match="mot:"):
                fn(run, "iou", 0.5, 2, UP)
    run = pack_run(ok)
    with pytest.raises(ValueError, match="frame_gt"):
        check_run(run._replace(frame_gt=np.array([0, 2])))
    with pytest.raises(ValueError, match="seq_frame"):
        check_run(run._replace(seq_frame=np.array([1, 1])))
    with pytest.raises(ValueError, match="gt_box"):
        check_run(run._replace(gt_box=np.zeros((1, 14))))
    # the largest frame is accepted
    check_run([[([(i, B(float(i))) for i in range(MAX_BOXES)], [(i, B(float(i))) for i in range(MAX_BOXES)])]])


def _desc(**over):
    d = _lib.MotClearDesc(1, 0, 0.5, 2, 4, 4, 4, 1, *([16] * 15))
    for k, v in over.items():
        setattr(d, k, v)
    return d


def test_c_abi_refusals():
    L = _lib.lib()
    assert L.o3d_mot_clear(None, None) < 0 and b"null" in L.o3d_last_error()
    assert L.o3d_mot_clear(ctypes.byref(_desc(S=0)), None) == 0                  # nothing to launch
    bad = [dict(S=-1), dict(max_gt=257), dict(max_hyp=-1), dict(max_gt=-1), dict(work_rows=0), dict(metric=2), dict(metric=-1),
           dict(threshold=0.0), dict(threshold=1.5), dict(threshold=float("nan")), dict(metric=1, threshold=0.0),
           dict(metric=1, threshold=float("inf")), dict(metric=1, threshold=-2.0), dict(dim=1), dict(dim=4), dict(up_mask=0),
           dict(up_mask=8), dict(seq_frame=None), dict(work=None), dict(cooc=None), dict(hyp_box=None)]
    for over in bad:
        assert L.o3d_mot_clear(ctypes.byref(_desc(**over)), None) < 0, over
    assert b"o3d_mot_clear" in L.o3d_last_error()


# ------------------------------------------------------------------ the command line
def test_mot_option_parsing():
    base = ["--cfg", "a.yaml", "--path", "/data"]
    assert not hasattr(track.parse_args(base), "mot")
    assert track.parse_args(base + ["--mot", "iou", "0.5"]).mot == ("iou", 0.5)
    assert track.parse_args(base + ["--mot", "distance", "2"]).mot == ("distance", 2.0)
    for bad in (["foo", "0.5"], ["iou", "0"], ["iou", "1.5"], ["iou", "x"], ["distance", "-1"], ["distance", "inf"], ["iou"]):
        with pytest.raises(SystemExit):
            track.parse_args(base + ["--mot", *bad])


def _tree(tmp_path):
    root = str(tmp_path)
    _write_scene(root, "0019", [((4, "Car"), synthetic_sequence(n_frames=3, n_points=500, seed=1, n_object=100))])
    return root


def test_command_lines_pass_mot_to_run_and_run_classes(tmp_path, monkeypatch):
    root = _tree(tmp_path)
    calls = []
    monkeypatch.setattr(torch.nn.Module, "cuda", lambda self, *a, **k: self)
    monkeypatch.setattr(track, "run", lambda *a, **k: calls.append(("run", k)) or {"success": 1.0})
    monkeypatch.setattr(track, "run_classes", lambda *a, **k: calls.append(("run_classes", k)) or {"success": 1.0})
    out = str(tmp_path / "r.jsonl")
    car = os.path.join(ROOT, "cfgs", "BAT_Car.yaml")
    track.main(["--cfg", car, "--path", root, "--out", out, "--mot", "iou", "0.5"])
    track.main(["--cfg", car, "--path", root, "--out", out, "--mot", "distance", "2", "--lost", "1", "2", "--coast", "0.5"])
    track.main(["--cfg", car, "--path", root, "--out", out, "--mot", "iou", "0.7",
                "--add_class", os.path.join(ROOT, "cfgs", "BAT_Pedestrian.yaml")])
    assert [c[0] for c in calls] == ["run", "run", "run_classes"]
    assert calls[0][1] == {"max_targets": 64, "max_points": None, "seed": 0, "precision": "fp32", "mot": ("iou", 0.5)}
    assert calls[1][1]["mot"] == ("distance", 2.0) and calls[1][1]["lost"] == (1, 2) and calls[1][1]["coast"] == 0.5
    assert calls[2][1]["mot"] == ("iou", 0.7)


def test_mot_sequences_of_a_run(tmp_path):
    """The ground truth of a scene is its annotations with the tracklet index as id; a run that reports every annotated box
    scores perfectly, and a box on a frame without its annotation is a false positive."""
    root = _tree(tmp_path)
    ds = kittiDataset(root, "test", "Car", preloading=False, preload_offset=-1)
    plan = track.scene_plan(ds)
    results = [{tr["index"]: {t: ds.box_from_anno(a) for t, a in enumerate(ds.tracklet_anno_list[tr["index"]])}
                for tr in p["tracklets"]} for p in plan]
    seqs = track.mot_sequences(plan, results, ds)
    assert len(seqs) == 1 and len(seqs[0]) == 3 and all(len(gt) == len(hyp) == 1 for gt, hyp in seqs[0])
    s = mot_reference(seqs, "iou", 0.5, 2, UP)["total"]
    assert (s["num_matches"], s["mota"], s["idf1"], s["mean_iou"]) == (3, 1.0, 1.0, 1.0)
    j = plan[0]["tracklets"][0]["index"]
    results[0][j][3] = results[0][j][2]                      # a box on a frame past the annotations
    plan[0]["frames"].append(plan[0]["frames"][-1] + 1)
    s = mot_reference(track.mot_sequences(plan, results, ds), "iou", 0.5, 2, UP)["total"]
    assert (s["num_matches"], s["num_false_positives"]) == (3, 1)
