"""Evidence and lost targets of the live tracker, without a GPU: `o3d_box_points`' argument checks through the C ABI, the tensor
formulation of the in-box count against the reference's points_in_box and the fp64 oracle, the `lost=` refusals of
MultiTargetTracker / MultiClassTracker / track_feeds, what `add` / `drop` do to the evidence, and `--lost` parsing."""
import os

import numpy as np
import pytest
import torch

from oracle import tracking_ref as R
from open3dsot_b200 import _lib, track
from open3dsot_b200.datasets.data_classes import Box
from open3dsot_b200.datasets.synthetic import synthetic_sequence
from open3dsot_b200.tracking import boxes as bx
from open3dsot_b200.tracking.multi_class import MultiClassTracker
from open3dsot_b200.tracking.multi_tracker import MultiTargetTracker, check_lost_rule, track_feeds
from test_tracking_host import _cfg, _Echo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = np.load(os.path.join(ROOT, "tests", "golden", "ref_tracking.npz"))


# ------------------------------------------------------------------ the C entry's argument checks
def test_box_points_refuses_bad_arguments():
    L = _lib.lib()
    p = 16                                                                  # never dereferenced: every call is refused or K = 0
    full = [p, p, p, p, p, p, 100, 4, p, None]
    for i in (0, 2, 3, 4, 5, 8):                                             # count (1) may be NULL
        args = list(full)
        args[i] = None
        assert L.o3d_box_points(*args) < 0, i
        assert b"null" in L.o3d_last_error()
    for N, K in ((100, -1), (100, 65536), (-1, 4), (-5, 0)):
        assert L.o3d_box_points(p, p, p, p, p, p, N, K, p, None) < 0, (N, K)
        assert b"bad sizes" in L.o3d_last_error()
    assert L.o3d_box_points(p, None, p, p, p, p, 100, 0, p, None) == 0     # K = 0: nothing to do, nothing launched


# ------------------------------------------------------------------ the tensor formulation
def _counts(points, center, rot, wlh, factor, count=None):
    scans = torch.as_tensor(points, dtype=torch.float32)[None]
    c = torch.as_tensor(center, dtype=torch.float32)[None]
    r = torch.as_tensor(rot, dtype=torch.float32)[None]
    half = bx.inclusive_half(torch.as_tensor(wlh, dtype=torch.float32)[None], factor)
    n = None if count is None else torch.tensor([count])
    return int(bx.box_point_counts(scans, n, torch.zeros(1, dtype=torch.int64), c, r, half)[0])


def test_count_equals_the_reference_points_in_box():
    seq = synthetic_sequence(n_frames=int(G["meta.n_frames"]), n_points=int(G["meta.n_points"]), seed=int(G["meta.tracklet_seeds"][0]),
                             n_object=int(G["meta.n_object"]))
    pts = seq[1]["pc"].points.T
    mask = G["points_in_box_1.25"]
    assert 0 < mask.sum() < mask.size
    assert _counts(pts, G["box_in.center"], G["box_in.rot"], G["box_in.wlh"], 1.25) == int(mask.sum())


def test_count_equals_the_oracle_on_random_rotated_boxes():
    rng = np.random.default_rng(5)
    for trial in range(40):
        pts = rng.uniform(-6, 6, size=(3000, 3)).astype(np.float32)
        yaw, pitch = rng.uniform(-np.pi, np.pi), rng.uniform(-0.3, 0.3)
        rz = np.array([[np.cos(yaw), -np.sin(yaw), 0], [np.sin(yaw), np.cos(yaw), 0], [0, 0, 1]])
        ry = np.array([[np.cos(pitch), 0, np.sin(pitch)], [0, 1, 0], [-np.sin(pitch), 0, np.cos(pitch)]])
        rot = (rz @ ry).astype(np.float32).astype(np.float64)
        center = rng.uniform(-2, 2, 3).astype(np.float32).astype(np.float64)
        wlh = rng.uniform(0.5, 5, 3).astype(np.float32).astype(np.float64)
        box = R.Box(center, wlh, rot)
        count = int(rng.integers(0, 3001))
        want = int(R._in_box_inclusive(pts[:count].astype(np.float64), box, 1.25).sum())
        got = _counts(pts, center, rot, wlh, 1.25, count)
        # fp32 box-frame coordinates against fp64 ones: only points within rounding distance of a face may differ
        local = (pts[:count].astype(np.float64) - center) @ rot
        half = np.array([wlh[1], wlh[0], wlh[2]]) * 1.25 / 2
        near = int((np.abs(np.abs(local) - half) < 1e-5).any(1).sum())
        assert abs(got - want) <= near, (trial, got, want, near)
        if near == 0:
            assert got == want


def test_count_includes_points_on_the_faces_and_respects_count():
    half = torch.tensor([[1.5, 0.75, 0.5]])
    face = torch.tensor([[1.5, 0.0, 0.0], [-1.5, 0.75, -0.5], [0.0, -0.75, 0.5], [1.5000001, 0.0, 0.0], [0.0, 0.0, 0.0]])
    scans = torch.cat([face, torch.full((3, 3), 9.0)])[None]
    eye = torch.eye(3)[None]
    frame = torch.zeros(1, dtype=torch.int64)
    assert int(bx.box_point_counts(scans, None, frame, torch.zeros(1, 3), eye, half)[0]) == 4     # 1.5000001 is outside
    for n, want in ((0, 0), (1, 1), (4, 3), (8, 4), (100, 4), (-3, 0)):
        assert int(bx.box_point_counts(scans, torch.tensor([n]), frame, torch.zeros(1, 3), eye, half)[0]) == want, n


# ------------------------------------------------------------------ lost= refusals
def test_lost_rule_refusals():
    assert check_lost_rule(None) is None
    assert check_lost_rule((0, 1)) == (0, 1) and check_lost_rule([30, 5]) == (30, 5)
    for bad, msg in (((-1, 3), "min_points=-1"), ((5, 0), "patience=0"), ((5, -2), "patience=-2"), ((5,), "expected None"),
                     (5, "expected None"), ((1.5, 2), "integers"), ((True, 2), "integers")):
        with pytest.raises(ValueError, match=msg):
            check_lost_rule(bad)
        with pytest.raises(ValueError, match=msg):
            MultiTargetTracker(_Echo(_cfg()), 100, 2, use_graph=False, lost=bad)
        with pytest.raises(ValueError, match=msg):
            track_feeds(None, [], 1, 4, max_points=100, lost=bad)


def test_multi_class_lost_rules():
    models = {n: _Echo(_cfg()) for n in ("Car", "Ped")}
    mc = MultiClassTracker(models, 100, {"Car": 2, "Ped": 3}, use_graph=False, lost={"Car": (10, 2)})
    assert mc.trackers["Car"].lost_rule == (10, 2) and mc.trackers["Ped"].lost_rule is None
    mc = MultiClassTracker(models, 100, {"Car": 2, "Ped": 3}, use_graph=False, lost=(4, 3))
    assert mc.trackers["Car"].lost_rule == mc.trackers["Ped"].lost_rule == (4, 3)
    with pytest.raises(ValueError, match="lost: class 'Cyclist' has no model"):
        MultiClassTracker(models, 100, {"Car": 2, "Ped": 3}, use_graph=False, lost={"Cyclist": (1, 1)})
    with pytest.raises(ValueError, match="patience=0"):
        MultiClassTracker(models, 100, {"Car": 2, "Ped": 3}, use_graph=False, lost={"Ped": (1, 0)})


def test_add_and_drop_reset_the_evidence():
    trk = MultiTargetTracker(_Echo(_cfg(shape_aggregation="previous")), 100, 3, use_graph=False, lost=(5, 2))
    trk.scan_feeds.feed_seen[0] = 1
    trk.scans_seen = 1                                                      # as after a first advance
    trk.points.fill_(7)
    trk.score.fill_(0.5)
    trk.misses.fill_(2)
    trk.lost.fill_(True)
    trk.add(4, Box(np.zeros(3), np.array([1.5, 4.0, 1.5]), np.eye(3)))
    k = trk.targets()[4]
    b = trk.boxes()
    assert int(b["points"][k]) == -1 and torch.isnan(b["score"][k]) and int(trk.misses[k]) == 0 and not bool(b["lost"][k])
    assert b["points"].dtype == torch.int32 and b["score"].dtype == torch.float32 and b["lost"].dtype == torch.bool
    ev = trk.evidence()
    assert ev.shape == (3, 4) and ev.dtype == torch.float32 and ev[k, 0] == -1 and torch.isnan(ev[k, 1])
    assert trk.snapshot().shape == (3, 15)
    assert trk.lost_targets() == []
    trk.lost[k].fill_(True)                                                 # as the rule leaves it
    assert trk.lost_targets() == [4]
    assert trk.drop_lost() == [4] and trk.targets() == {}
    assert int(trk.points[k]) == -1 and not bool(trk.lost[k]) and int(trk.misses[k]) == 0


# ------------------------------------------------------------------ the command line
def test_lost_option_parsing(capsys):
    base = ["--cfg", "c.yaml", "--path", "p"]
    assert not hasattr(track.parse_args(base), "lost")                    # a run without the rule keeps its options
    assert track.parse_args(base + ["--lost", "20", "3"]).lost == (20, 3)
    for bad in (["--lost", "20"], ["--lost", "a", "3"], ["--lost", "-1", "3"], ["--lost", "5", "0"]):
        with pytest.raises(SystemExit):
            track.parse_args(base + bad)
    assert "--lost" in capsys.readouterr().err


def test_tracklet_scoring_counts_frames_after_a_loss_as_failures():
    gts = [Box(np.array([float(i), 0.0, 0.0]), np.array([1.5, 4.0, 1.5]), np.eye(3)) for i in range(4)]
    got = {0: gts[0], 1: gts[1]}                                            # lost on frame 1
    o, d = track._score_tracklet(got, gts, [0, 1, 2, 3], 3, [0, 0, 1])
    assert min(o[:2]) > 0.999 and max(d[:2]) < 1e-9 and o[2:] == [0.0, 0.0] and d[2:] == [float("inf")] * 2
    assert track._evidence((-1, float("nan"))) == {"points": None, "score": None}
    assert track._evidence((12, 0.25)) == {"points": 12, "score": 0.25}
