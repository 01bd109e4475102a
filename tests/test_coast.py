"""Coasting in the live tracker, without a GPU: the write-back's tensor formulation (`track_update_tensors`) bitwise against a
plain per-row float32 loop, `o3d_track_update`'s argument checks through the C ABI, the `coast=` refusals of MultiTargetTracker /
MultiClassTracker / track_feeds, the coast state `add` / `drop` set, and `--coast` parsing."""
import ctypes

import numpy as np
import pytest
import torch

from open3dsot_b200 import _lib, track
from open3dsot_b200.datasets.data_classes import Box
from open3dsot_b200.tracking.multi_class import MultiClassTracker
from open3dsot_b200.tracking.multi_tracker import (MultiTargetTracker, Slots, check_coast, coast_weights, track_feeds,
                                                   track_update_tensors)
from test_tracking_host import _cfg, _Echo

F32 = np.float32


# ------------------------------------------------------------------ the tensor formulation against a per-row loop
def _random_case(K, b, seed, rule, min_points=3):
    """Slot state of K + 2 rows and a b-row work list: the first n rows random distinct slots, the rest padding (read K, write
    K + 1).  Rows advance or hold (held: not fed, or lost); first samples (hit_t == 0), gaps > 1, counts around min_points and
    NaN scores all occur."""
    rng = np.random.default_rng(seed)
    R = K + 2
    t = rng.integers(0, 12, R)
    hit_t = np.where(rng.random(R) < 0.3, 0, rng.integers(0, 12, R) % (t + 1))
    patience = rule[1] if rule else 3
    misses = np.minimum(rng.integers(0, patience + 1, R), np.maximum(t - hit_t, 0)).astype(np.int32)
    lost = misses >= patience
    state = Slots(box_c=rng.normal(0, 5, (R, 3)).astype(F32), box_r=rng.normal(0, 1, (R, 3, 3)).astype(F32), t=t,
                  first_flag=(rng.random(R) < 0.5).astype(F32), points=rng.integers(-1, 8, R).astype(np.int32),
                  score=np.where(rng.random(R) < 0.2, np.nan, rng.random(R)).astype(F32), misses=misses, lost=lost,
                  vel=rng.normal(0, 1, (R, 3)).astype(F32), hit_c=rng.normal(0, 5, (R, 3)).astype(F32), hit_t=hit_t,
                  coasting=(misses > 0) & ~lost)
    state.box_c[K] = 0.0                                                      # the idle row
    n = int(rng.integers(0, b + 1))
    slots = rng.permutation(K)[:n]
    src = np.concatenate([slots, np.full(b - n, K)]).astype(np.int64)
    dst = np.concatenate([slots, np.full(b - n, K + 1)]).astype(np.int64)
    adv = (rng.random(b) < 0.8) & ~lost[src] & (src < K)
    center = rng.normal(0, 5, (b, 3)).astype(F32)
    rot = rng.normal(0, 1, (b, 3, 3)).astype(F32)
    points = rng.integers(0, 2 * min_points + 1, b).astype(np.int32)
    score = np.where(rng.random(b) < 0.2, np.nan, rng.random(b)).astype(F32)
    return state, src, dst, adv, center, rot, points, score


def _loop(state, src, dst, adv, center, rot, points, score, rule, coast):
    """The write-back row by row in numpy float32, as the semantics state it."""
    out = Slots(*(np.array(x, copy=True) for x in state))
    for i in range(len(src)):
        s, d = src[i], dst[i]
        row = {k: np.array(getattr(state, k)[s], copy=True) for k in Slots._fields}
        if adv[i]:
            row["t"] = row["t"] + 1
            row["first_flag"] = F32(0)
            row["points"], row["score"] = points[i], score[i]
            row["box_c"], row["box_r"] = center[i].copy(), rot[i].copy()
            if rule is not None:
                hit = points[i] >= rule[0]
                row["misses"] = np.int32(0) if hit else row["misses"] + 1
                if coast is not None:
                    alpha, beta = F32(coast[0]), F32(coast[1])
                    gap = F32(row["t"] - row["hit_t"])
                    if hit:
                        v = (center[i] - row["hit_c"]) / gap
                        row["vel"] = v if row["hit_t"] == 0 else alpha * v + beta * row["vel"]
                        row["hit_c"], row["hit_t"] = center[i].copy(), row["t"]
                    else:
                        row["box_c"] = row["hit_c"] + row["vel"] * gap
                        row["box_r"] = getattr(state, "box_r")[s].copy()
        if rule is not None:
            row["lost"] = row["lost"] | (row["misses"] >= rule[1])
            if adv[i] and coast is not None:
                row["coasting"] = not hit and not row["lost"]
        for k in Slots._fields:
            getattr(out, k)[d] = row[k]
    return out


def _bits(x):
    x = np.asarray(x)
    return x.view(np.int32) if x.dtype == np.float32 else x


def _formulation(state, src, dst, adv, center, rot, points, score, rule, coast):
    slots = Slots(*(torch.from_numpy(np.array(x, copy=True)) for x in state))
    track_update_tensors(slots, torch.from_numpy(src), torch.from_numpy(dst), torch.from_numpy(adv), torch.from_numpy(center),
                         torch.from_numpy(rot), torch.from_numpy(points), torch.from_numpy(score), rule, coast)
    return slots


@pytest.mark.parametrize("rule,alpha", [(None, None), ((3, 2), None), ((3, 2), 0.3), ((3, 2), 1.0), ((0, 1), 0.3)])
@pytest.mark.parametrize("K,b", [(1, 1), (9, 7), (70, 64)])
def test_formulation_equals_the_row_loop(K, b, rule, alpha):
    coast = coast_weights(alpha)
    for seed in range(6):
        case = _random_case(K, b, seed, rule)
        got = _formulation(*case, rule, coast)
        want = _loop(*case, rule, coast)
        for k in Slots._fields:
            assert np.array_equal(_bits(getattr(got, k).numpy()), _bits(getattr(want, k))), (seed, k)


def test_the_cases_cover_every_branch():
    rule, coast = (3, 2), coast_weights(0.5)
    seen = set()
    for seed in range(6):
        state, src, dst, adv, center, rot, points, score = case = _random_case(70, 64, seed, rule)
        hit = points >= rule[0]
        new_misses = state.misses[src] + 1
        seen |= {"pad"} if (src == 70).any() else set()
        seen |= {"held"} if (~adv & (src < 70)).any() else set()
        seen |= {"first"} if (adv & hit & (state.hit_t[src] == 0)).any() else set()
        seen |= {"gap"} if (adv & hit & (state.t[src] + 1 - state.hit_t[src] > 1) & (state.hit_t[src] > 0)).any() else set()
        seen |= {"miss"} if (adv & ~hit).any() else set()
        seen |= {"loss"} if (adv & ~hit & (new_misses >= rule[1])).any() else set()
        seen |= {"nan"} if np.isnan(score[adv]).any() else set()
        got = _formulation(*case, rule, coast)
        seen |= {"coasting"} if got.coasting[torch.from_numpy(dst[adv & ~hit])].any() else set()
    assert seen == {"pad", "held", "first", "gap", "miss", "loss", "nan", "coasting"}, seen


def test_coasted_centre_and_velocity_by_hand():
    # a target at x = 0 (frame 0), hit at x = 2 on frame 1, missed on frames 2 and 3, hit at x = 9 on frame 4
    z = lambda *s, d=torch.float32: torch.zeros(*s, dtype=d)
    slots = Slots(z(3, 3), torch.eye(3).repeat(3, 1, 1), z(3, d=torch.int64), z(3), z(3, d=torch.int32), z(3), z(3, d=torch.int32),
                  z(3, d=torch.bool), z(3, 3), z(3, 3), z(3, d=torch.int64), z(3, d=torch.bool))
    one = torch.zeros(1, dtype=torch.int64)
    rot = (torch.eye(3) * 2)[None]
    coast = coast_weights(0.5)
    xs = []
    for x, n in ((2.0, 5), (7.0, 0), (8.0, 0), (9.0, 5)):
        track_update_tensors(slots, one, one, torch.ones(1, dtype=torch.bool), torch.tensor([[x, 0.0, 0.0]]), rot,
                             torch.tensor([n], dtype=torch.int32), torch.tensor([0.5]), (1, 3), coast)
        xs.append((float(slots.box_c[0, 0]), bool(slots.coasting[0]), float(slots.vel[0, 0]), int(slots.misses[0])))
    v = float(F32(0.5) * (F32(7) / F32(3)) + F32(0.5) * F32(2))              # (9 - 2) / 3 weighed against 2
    assert xs == [(2.0, False, 2.0, 0), (4.0, True, 2.0, 1), (6.0, True, 2.0, 2), (9.0, False, v, 0)]
    assert int(slots.hit_t[0]) == 4 and float(slots.hit_c[0, 0]) == 9.0


# ------------------------------------------------------------------ the C entry's argument checks
_PTRS = ("src", "dst", "adv", "center", "rot", "points", "score", "box_c", "box_r", "t", "first_flag", "slot_points", "slot_score",
         "misses", "lost", "vel", "hit_c", "hit_t", "coasting")


def _desc(**kw):
    d = dict(b=4, rule=1, min_points=1, patience=2, coast=1, alpha=0.5, beta=0.5, **{n: 16 for n in _PTRS})   # never dereferenced
    d.update(kw)
    return _lib.TrackUpdateDesc(**d)


def test_track_update_refuses_bad_arguments():
    L = _lib.lib()
    call = lambda d: L.o3d_track_update(ctypes.byref(d), None)
    assert L.o3d_track_update(None, None) < 0 and b"null" in L.o3d_last_error()
    for n in _PTRS:
        assert call(_desc(**{n: None})) < 0, n
        assert b"null" in L.o3d_last_error()
    for b in (-1, 65536):
        assert call(_desc(b=b)) < 0 and b"bad sizes" in L.o3d_last_error()
    for kw in (dict(rule=2), dict(coast=-1), dict(rule=0), dict(min_points=-1), dict(patience=0), dict(alpha=0.0),
               dict(alpha=1.5), dict(alpha=float("nan"))):
        assert call(_desc(**kw)) < 0, kw
    assert call(_desc(b=0)) == 0                                              # nothing to do, nothing launched
    assert call(_desc(b=0, rule=0, coast=0)) == 0


# ------------------------------------------------------------------ coast= refusals and the state add / drop set
def test_coast_refusals():
    assert check_coast(None, None) is None and check_coast(0.5, (1, 2)) == 0.5 and check_coast(1, (0, 1)) == 1.0
    assert coast_weights(0.3) == (float(np.float32(0.3)), float(np.float32(0.7)))
    for bad, msg in ((0.0, "0 < alpha"), (1.5, "0 < alpha"), (-0.2, "0 < alpha"), (float("nan"), "0 < alpha"), (True, "0 < alpha"),
                     ("0.5", "0 < alpha"), ((0.5,), "0 < alpha")):
        with pytest.raises(ValueError, match=msg):
            check_coast(bad, (1, 2))
        with pytest.raises(ValueError, match=msg):
            MultiTargetTracker(_Echo(_cfg()), 100, 2, use_graph=False, lost=(1, 2), coast=bad)
        with pytest.raises(ValueError, match=msg):
            track_feeds(None, [], 1, 4, max_points=100, lost=(1, 2), coast=bad)
    for where in (lambda: MultiTargetTracker(_Echo(_cfg()), 100, 2, use_graph=False, coast=0.5),
                  lambda: track_feeds(None, [], 1, 4, max_points=100, coast=0.5)):
        with pytest.raises(ValueError, match="lost="):
            where()


def test_multi_class_coast():
    models = {n: _Echo(_cfg()) for n in ("Car", "Ped")}
    mc = MultiClassTracker(models, 100, {"Car": 2, "Ped": 3}, use_graph=False, lost=(1, 2), coast={"Car": 0.25})
    assert mc.trackers["Car"].coast == 0.25 and mc.trackers["Ped"].coast is None
    assert list(mc._coast_rows()) == [True, True, False, False, False]
    mc = MultiClassTracker(models, 100, {"Car": 2, "Ped": 3}, use_graph=False, lost=(1, 2), coast=0.5)
    assert mc.trackers["Car"].coast == mc.trackers["Ped"].coast == 0.5
    with pytest.raises(ValueError, match="coast: class 'Cyclist' has no model"):
        MultiClassTracker(models, 100, {"Car": 2, "Ped": 3}, use_graph=False, lost=(1, 2), coast={"Cyclist": 0.5})
    with pytest.raises(ValueError, match="class 'Ped'.*lost="):                   # Ped has no rule
        MultiClassTracker(models, 100, {"Car": 2, "Ped": 3}, use_graph=False, lost={"Car": (1, 2)}, coast=0.5)
    with pytest.raises(ValueError, match="class 'Car'.*0 < alpha"):
        MultiClassTracker(models, 100, {"Car": 2, "Ped": 3}, use_graph=False, lost=(1, 2), coast={"Car": 2.0})


def test_add_and_drop_set_the_coast_state():
    trk = MultiTargetTracker(_Echo(_cfg(shape_aggregation="previous")), 100, 3, use_graph=False, lost=(5, 2), coast=0.5)
    trk.scan_feeds.feed_seen[0] = 1
    trk.scans_seen = 1                                                      # as after a first advance
    for x in (trk.vel, trk.hit_c):
        x.fill_(3.0)
    trk.hit_t.fill_(4)
    trk.coasting.fill_(True)
    trk.add(4, Box(np.array([1.0, 2.0, 3.0]), np.array([1.5, 4.0, 1.5]), np.eye(3)))
    k = trk.targets()[4]
    b = trk.boxes()
    assert b["coasting"].data_ptr() == trk._coasting.data_ptr() and b["velocity"].data_ptr() == trk._vel.data_ptr()  # views
    assert torch.equal(trk.hit_c[k], torch.tensor([1.0, 2.0, 3.0])) and int(trk.hit_t[k]) == 0
    assert not bool(b["coasting"][k]) and not b["velocity"][k].any()
    assert trk.evidence().shape == (3, 4) and trk._record().shape == (3, 19) and trk.snapshot().shape == (3, 15)
    trk.coasting[k].fill_(True)
    trk.drop(4)
    assert not bool(trk.coasting[k]) and not trk.hit_c[k].any() and not trk.vel[k].any()


# ------------------------------------------------------------------ the command line
def test_coast_option_parsing(capsys):
    base = ["--cfg", "c.yaml", "--path", "p"]
    assert not hasattr(track.parse_args(base + ["--lost", "1", "3"]), "coast")      # a run without it keeps its options
    assert track.parse_args(base + ["--lost", "1", "3", "--coast", "0.5"]).coast == 0.5
    with pytest.raises(SystemExit):
        track.parse_args(base + ["--coast", "0.5"])
    assert "--coast needs --lost" in capsys.readouterr().err
    for bad in (["--coast", "0"], ["--coast", "1.5"], ["--coast", "nan"], ["--coast", "x"], ["--coast"]):
        with pytest.raises(SystemExit):
            track.parse_args(base + ["--lost", "1", "3"] + bad)
        assert "--coast" in capsys.readouterr().err


def test_coast_counts_and_json_evidence():
    ev = {0: (-1, float("nan"), False), 1: (4, 0.5, False), 2: (0, 0.1, True), 3: (0, 0.1, True), 4: (6, 0.7, False),
          5: (0, 0.2, True), 6: (0, 0.1, False)}                            # frame 6: the loss
    assert track._coast_counts(ev, 1) == (3, 1)
    assert track._evidence((3, 0.5, True)) == {"points": 3, "score": 0.5, "coasting": True}
    assert track._evidence((3, 0.5)) == {"points": 3, "score": 0.5}
