"""Detection matching in the live tracker, without a GPU: the matching's formulation (`associate_tensors`) against a per-feed
numpy float32 greedy loop, the write-back's re-acquisition (`track_update_tensors` with matches) against a per-row loop and by
hand, `o3d_box_associate` / `o3d_track_update`'s argument checks through the C ABI, the `detections=` and `put(...,
detections=)` refusals, and `--detections` parsing."""
import ctypes
import json

import numpy as np
import pytest
import torch

from open3dsot_b200 import _lib, track
from open3dsot_b200.datasets.data_classes import Box
from open3dsot_b200.tracking.multi_class import MultiClassTracker
from open3dsot_b200.tracking.multi_tracker import (MatchSlots, MultiTargetTracker, Slots, associate_tensors, check_detections,
                                                   coast_weights, detection_gate2, detection_rows, plane_axes, track_feeds,
                                                   track_update_tensors)
from test_coast import _bits, _loop, _random_case
from test_tracking_host import _cfg, _Echo

F32 = np.float32
NAN = F32("nan")


# ------------------------------------------------------------------ a matching case and its numpy greedy loop
def associate_case(K, b, F, D, seed, rule=(3, 2), grid=False, n_det=None):
    """Slot state of K + 2 rows, a b-row work list over F feeds (padding rows read K, feed 0) and each feed's detections
    (F, D, 16).  `grid`: every centre on an integer grid, so that exact distance ties and pairs exactly at an integer gate
    occur.  `n_det`: detections per fed feed (default random in 0 .. D)."""
    rng = np.random.default_rng(seed)
    state, src, dst, adv, center, rot, points, score = _random_case(K, b, seed, rule)
    R = K + 2
    feed_of_slot = rng.integers(0, F, R)
    feed_of_slot[K] = 0
    feed = feed_of_slot[src].astype(np.int64)
    fed = (rng.random(F) < 0.85).astype(np.int64)
    adv = adv & (fed[feed] != 0)
    count = np.array([(rng.integers(0, D + 1) if n_det is None else min(n_det, D)) if fed[f] else 0 for f in range(F)], np.int32)
    det = rng.normal(0, 1, (F, D, 16)).astype(F32)
    if grid:
        center = rng.integers(-1, 2, (b, 3)).astype(F32)
        det[..., :3] = rng.integers(-1, 2, (F, D, 3)).astype(F32)
        state = state._replace(hit_c=rng.integers(-1, 2, (R, 3)).astype(F32), vel=np.zeros((R, 3), F32))
    else:
        det[..., :3] = rng.normal(0, 5, (F, D, 3)).astype(F32)
        near = rng.random((F, D)) < 0.5                                       # half the detections near some row's box
        if b:
            det[..., :3] = np.where(near[..., None], center[rng.integers(0, b, (F, D))] + rng.normal(0, 0.5, (F, D, 3)).astype(F32),
                                    det[..., :3])
    return state, src, feed, adv, center, points, fed, count, det


def _pred_loop(state, src, adv, center, points, rule, coast):
    b = len(src)
    pred = np.full((b, 3), NAN, F32)
    for i in range(b):
        if adv[i]:
            s = src[i]
            hit = rule is None or points[i] >= rule[0]
            if coast and not hit:
                pred[i] = state.hit_c[s] + state.vel[s] * F32(state.t[s] + 1 - state.hit_t[s])
            else:
                pred[i] = center[i]
    return pred


def greedy_loop(state, src, feed, adv, center, points, fed, count, det, gate2, axes, rule, coast):
    """The matching as the semantics state it, in numpy float32: per fed feed, every pair within the gate in ascending
    (d2, row, detection) order, accepted when both are free."""
    b, (F, D, _) = len(src), det.shape
    pred = _pred_loop(state, src, adv, center, points, rule, coast)
    match, match_box = np.full(b, -1, np.int32), np.zeros((b, 12), F32)
    rec_slot = {}
    for f in range(F):
        if not fed[f]:
            continue
        pairs = []
        for i in range(b):
            if not adv[i] or feed[i] != f:
                continue
            for d in range(count[f]):
                dx = pred[i, axes[0]] - det[f, d, axes[0]]
                dy = pred[i, axes[1]] - det[f, d, axes[1]]
                d2 = dx * dx + dy * dy
                if d2 <= F32(gate2):
                    pairs.append((float(d2), i, d))
        slot = np.full(count[f], -1, np.int32)
        for _, i, d in sorted(pairs):
            if match[i] < 0 and slot[d] < 0:
                match[i] = d
                match_box[i] = np.concatenate([det[f, d, 0:3], det[f, d, 6:15]])
                slot[d] = src[i]
        rec_slot[f] = slot
    return pred, match, match_box, rec_slot


def run_formulation(case, gate2, axes, rule, coast, device="cpu"):
    state, src, feed, adv, center, points, fed, count, det = case
    F, D, _ = det.shape
    T = lambda x: torch.from_numpy(np.array(x, copy=True)).to(device)
    slots = Slots(*(T(x) for x in state))
    records = (torch.zeros(F, D, 16, device=device), torch.zeros(F, dtype=torch.int32, device=device),
               torch.full((F, D), -1, dtype=torch.int32, device=device))
    out = associate_tensors(T(src), T(feed), T(adv), T(center), T(points), slots, T(fed), T(count), T(det), records, gate2, axes,
                            rule, coast)
    return out, records


def _check(case, gate2, axes, rule, coast):
    (pred, match, match_box), (rec_det, rec_count, rec_slot) = run_formulation(case, gate2, axes, rule, coast)
    want_pred, want_match, want_box, want_slot = greedy_loop(*case, gate2, axes, rule, coast)
    assert np.array_equal(_bits(pred.numpy()), _bits(want_pred))
    assert np.array_equal(match.numpy(), want_match)
    assert np.array_equal(_bits(match_box.numpy()), _bits(want_box))
    det, fed, count = case[-1], case[-3], case[-2]
    for f in range(det.shape[0]):
        n = int(rec_count[f])
        assert n == (count[f] if fed[f] else 0)
        if fed[f]:
            assert np.array_equal(rec_slot[f, :n].numpy(), want_slot[f])
            assert np.array_equal(_bits(rec_det[f, :n].numpy()), _bits(det[f, :n]))
    return want_match


@pytest.mark.parametrize("rule,alpha", [(None, None), ((3, 2), None), ((3, 2), 0.5)])
@pytest.mark.parametrize("K,b,F,D", [(1, 1, 1, 1), (9, 7, 2, 5), (70, 64, 3, 40), (40, 32, 16, 3)])
def test_formulation_equals_the_greedy_loop(K, b, F, D, rule, alpha):
    coast = alpha is not None
    matched = 0
    for seed in range(4):
        for axes in ((0, 1), (0, 2)):
            want = _check(associate_case(K, b, F, D, seed, rule), detection_gate2(2.0), axes, rule, coast)
            matched += (want >= 0).sum()
    assert matched > 0 or b == 1


@pytest.mark.parametrize("K,b,F,D", [(9, 7, 1, 9), (70, 64, 2, 64), (12, 12, 1, 3), (16, 8, 1, 12)])
def test_ties_and_pairs_exactly_at_the_gate(K, b, F, D):
    """Integer centres: equal distances are broken by row, then by detection, and d2 == gate2 = 4 is inside the gate."""
    ties = at_gate = 0
    for seed in range(6):
        case = associate_case(K, b, F, D, seed, (3, 2), grid=True)
        gate2 = detection_gate2(2.0)
        assert gate2 == 4.0
        want = _check(case, gate2, (0, 1), (3, 2), True)
        pred, _, _, _ = greedy_loop(*case, gate2, (0, 1), (3, 2), True)
        state, src, feed, adv, center, points, fed, count, det = case
        for f in range(F):
            rows = [i for i in range(b) if adv[i] and feed[i] == f]
            d2 = [[float((pred[i, 0] - det[f, d, 0]) ** 2 + (pred[i, 1] - det[f, d, 1]) ** 2) for d in range(count[f])]
                  for i in rows]
            flat = [v for r in d2 for v in r if v <= 4.0]
            ties += len(flat) - len(set(flat))
            at_gate += flat.count(4.0)
    assert ties > 0 and at_gate > 0


def test_rows_and_detections_on_either_side():
    rule = (3, 2)
    for seed in range(4):
        more_rows = associate_case(40, 32, 1, 3, seed, rule, n_det=3)
        want = _check(more_rows, detection_gate2(50.0), (0, 1), rule, False)
        assert (want >= 0).sum() == min(3, more_rows[3].sum())                 # every detection is within a huge gate
        more_dets = associate_case(6, 3, 1, 64, seed, rule, n_det=64)
        want = _check(more_dets, detection_gate2(50.0), (0, 1), rule, False)
        assert (want >= 0).sum() == more_dets[3].sum()
        none = associate_case(9, 7, 2, 8, seed, rule, n_det=0)
        assert (_check(none, detection_gate2(2.0), (0, 1), rule, False) < 0).all()


def test_rows_that_do_not_advance_never_match():
    state, src, feed, adv, center, points, fed, count, det = associate_case(70, 64, 1, 64, 3, (3, 2), n_det=64)
    lost = state.lost[src] & (src < 70)
    assert lost.any() and (~adv & (src < 70) & ~lost).any() and (src == 70).any()
    det[0, :, :3] = center[np.arange(64) % len(center)]                          # a detection on every row's box
    case = state, src, feed, adv, center, points, np.array([1]), np.array([64], np.int32), det
    want = _check(case, detection_gate2(1.0), (0, 1), (3, 2), False)
    assert (want[~adv] == -1).all() and (want[adv] >= 0).all()


# ------------------------------------------------------------------ the write-back with matches
def _match_loop(case, match, match_box, detection, reacquired, rule, coast):
    """test_coast's per-row loop with the matched misses' P replaced by their detection; detection / reacquired row by row."""
    state, src, dst, adv, center, rot, points, score = case
    hit = np.ones(len(src), bool) if rule is None else points >= rule[0]
    re = adv & (match >= 0) & ~hit
    center = np.where(re[:, None], match_box[:, :3], center)
    rot = np.where(re[:, None, None], match_box[:, 3:].reshape(-1, 3, 3), rot)
    points = np.where(re, max(rule[0], 0) if rule else points, points).astype(np.int32)   # the loop's hit test sees a hit
    out = _loop(state, src, dst, adv, center, rot, points, score, rule, coast)
    out.points[dst[re]] = case[6][re]                                         # the evidence stays the network's proposal
    det, rq = detection.copy(), reacquired.copy()
    for i in range(len(src)):
        s, d = src[i], dst[i]
        det[d], rq[d] = (match[i], re[i]) if adv[i] else (detection[s], reacquired[s])
    return out, det, rq, re


@pytest.mark.parametrize("rule,alpha", [(None, None), ((3, 2), None), ((3, 2), 0.3), ((0, 1), 0.5)])
@pytest.mark.parametrize("K,b", [(9, 7), (70, 64)])
def test_write_back_with_matches_equals_the_row_loop(K, b, rule, alpha):
    coast = coast_weights(alpha)
    reacq = 0
    for seed in range(6):
        case = _random_case(K, b, seed, rule)
        rng = np.random.default_rng(50 + seed)
        match = np.where(rng.random(b) < 0.5, rng.integers(0, 9, b), -1).astype(np.int32)
        match_box = rng.normal(0, 5, (b, 12)).astype(F32)
        detection = rng.integers(-1, 5, K + 2).astype(np.int32)
        reacquired = rng.random(K + 2) < 0.3
        want, want_det, want_rq, re = _match_loop(case, match, match_box, detection, reacquired, rule, coast)
        reacq += re.sum()
        slots = Slots(*(torch.from_numpy(np.array(x, copy=True)) for x in case[0]))
        ms = MatchSlots(torch.from_numpy(detection.copy()), torch.from_numpy(reacquired.copy()))
        _, src, dst, adv, center, rot, points, score = (torch.from_numpy(np.asarray(x)) if i else x for i, x in enumerate(case))
        track_update_tensors(slots, src, dst, adv, center, rot, points, score, rule, coast,
                             (torch.from_numpy(match), torch.from_numpy(match_box)) + tuple(ms))
        for k in Slots._fields:
            assert np.array_equal(_bits(getattr(slots, k).numpy()), _bits(getattr(want, k))), (seed, k)
        assert np.array_equal(ms.detection.numpy(), want_det) and np.array_equal(ms.reacquired.numpy(), want_rq)
    assert reacq > 0 or rule is None or rule[0] == 0


def test_no_match_is_the_write_back_without_matches():
    for rule, alpha in (((3, 2), 0.5), ((3, 2), None), (None, None)):
        case = _random_case(70, 64, 9, rule)
        plain = Slots(*(torch.from_numpy(np.array(x, copy=True)) for x in case[0]))
        matched = Slots(*(torch.from_numpy(np.array(x, copy=True)) for x in case[0]))
        args = [torch.from_numpy(np.asarray(x)) for x in case[1:]]
        track_update_tensors(plain, *args, rule, coast_weights(alpha))
        ms = MatchSlots(torch.full((72,), 7, dtype=torch.int32), torch.ones(72, dtype=torch.bool))
        track_update_tensors(matched, *args, rule, coast_weights(alpha),
                             (torch.full((64,), -1, dtype=torch.int32), torch.zeros(64, 12)) + tuple(ms))
        for k in Slots._fields:
            assert torch.equal(getattr(plain, k).view(-1).view(torch.uint8) if getattr(plain, k).is_floating_point()
                               else getattr(plain, k), getattr(matched, k).view(-1).view(torch.uint8)
                               if getattr(matched, k).is_floating_point() else getattr(matched, k)), k


@pytest.mark.parametrize("alpha", [None, 0.5])
def test_a_reacquired_row_by_hand(alpha):
    # a target at x = 0 (frame 0), hit at x = 2 on frame 1, missed on frame 2, missed on frame 3 with a detection at x = 7.5
    z = lambda *s, d=torch.float32: torch.zeros(*s, dtype=d)
    slots = Slots(z(3, 3), torch.eye(3).repeat(3, 1, 1), z(3, d=torch.int64), z(3), z(3, d=torch.int32), z(3), z(3, d=torch.int32),
                  z(3, d=torch.bool), z(3, 3), z(3, 3), z(3, d=torch.int64), z(3, d=torch.bool))
    ms = MatchSlots(torch.full((3,), -1, dtype=torch.int32), z(3, d=torch.bool))
    one = torch.zeros(1, dtype=torch.int64)
    coast = coast_weights(alpha)
    det_rot = torch.tensor([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])
    out = []
    for x, n, m in ((2.0, 5, -1), (7.0, 0, -1), (8.0, 0, 4)):
        box = torch.cat([torch.tensor([7.5, 1.0, 0.0]), det_rot.reshape(9)])[None]
        track_update_tensors(slots, one, one, torch.ones(1, dtype=torch.bool), torch.tensor([[x, 0.0, 0.0]]), (torch.eye(3) * 2)[None],
                             torch.tensor([n], dtype=torch.int32), torch.tensor([0.5]), (1, 3), coast,
                             (torch.tensor([m], dtype=torch.int32), box) + tuple(ms))
        out.append((slots.box_c[0].tolist(), int(slots.misses[0]), bool(ms.reacquired[0]), int(ms.detection[0]),
                    bool(slots.coasting[0])))
    coasted_x = 4.0 if alpha is not None else 7.0
    assert out[0] == ([2.0, 0.0, 0.0], 0, False, -1, False)
    assert out[1] == ([coasted_x, 0.0, 0.0], 1, False, -1, alpha is not None)
    assert out[2] == ([7.5, 1.0, 0.0], 0, True, 4, False)                   # re-acquired: the detection's box, no miss
    assert torch.equal(slots.box_r[0], det_rot) and int(slots.points[0]) == 0   # evidence: the network's proposal
    if alpha is not None:
        a, b = (F32(w) for w in coast)
        v = a * ((F32(7.5) - F32(2.0)) / F32(2)) + b * F32(2.0)
        assert float(slots.vel[0, 0]) == float(v) and float(slots.vel[0, 1]) == float(a * (F32(1.0) / F32(2)) + b * F32(0))
        assert slots.hit_c[0].tolist() == [7.5, 1.0, 0.0] and int(slots.hit_t[0]) == 3


# ------------------------------------------------------------------ the C entries' argument checks
_APTRS = ("src", "feed", "adv", "center", "points", "t", "hit_t", "hit_c", "vel", "fed", "count", "det", "pred", "match",
          "match_box", "rec_det", "rec_count", "rec_slot")


def _adesc(**kw):
    d = dict(b=4, F=2, D=8, axis0=0, axis1=1, gate2=4.0, rule=1, min_points=1, coast=1, **{n: 16 for n in _APTRS})  # never read
    d.update(kw)
    return _lib.AssociateDesc(**d)


def test_box_associate_refuses_bad_arguments():
    L = _lib.lib()
    call = lambda d: L.o3d_box_associate(ctypes.byref(d), None)
    assert L.o3d_box_associate(None, None) < 0 and b"null" in L.o3d_last_error()
    for n in _APTRS:
        assert call(_adesc(**{n: None})) < 0, n
        assert b"null" in L.o3d_last_error()
    for kw in (dict(b=-1), dict(b=65536), dict(F=0), dict(D=0), dict(D=1025)):
        assert call(_adesc(**kw)) < 0 and b"bad sizes" in L.o3d_last_error(), kw
    for g in (0.0, -1.0, float("nan"), float("inf")):
        assert call(_adesc(gate2=g)) < 0 and b"gate2" in L.o3d_last_error(), g
    for a0, a1 in ((0, 0), (1, 1), (-1, 1), (0, 3), (3, 2)):
        assert call(_adesc(axis0=a0, axis1=a1)) < 0 and b"axes" in L.o3d_last_error(), (a0, a1)
    for kw in (dict(rule=2), dict(coast=2), dict(rule=0, coast=1), dict(min_points=-1)):
        assert call(_adesc(**kw)) < 0, kw
    assert call(_adesc(b=0)) == 0                                             # nothing to do, nothing launched
    assert call(_adesc(b=0, D=1024, axis0=2, axis1=0, rule=0, coast=0)) == 0


def test_track_update_refuses_some_match_pointers_null():
    from test_coast import _desc
    L = _lib.lib()
    names = ("match", "match_box", "slot_detection", "slot_reacquired")
    for n in names:
        d = _desc(b=0, **{m: 16 for m in names if m != n})
        assert L.o3d_track_update(ctypes.byref(d), None) < 0 and b"null" in L.o3d_last_error(), n
    assert L.o3d_track_update(ctypes.byref(_desc(b=0, **{m: 16 for m in names})), None) == 0
    assert L.o3d_track_update(ctypes.byref(_desc(b=0)), None) == 0


# ------------------------------------------------------------------ detections= and put(..., detections=)
def test_detections_refusals_and_helpers():
    assert check_detections(None) is None and check_detections((64, 2)) == (64, 2.0) and check_detections((1024, 0.5)) == (1024, 0.5)
    for bad, msg in (((0, 2.0), "max_per_scan"), ((1025, 2.0), "max_per_scan"), ((2.5, 2.0), "max_per_scan"),
                     ((True, 2.0), "max_per_scan"), ((64, 0.0), "gate"), ((64, -1.0), "gate"), ((64, float("nan")), "gate"),
                     ((64, float("inf")), "gate"), ((64, "2"), "gate"), ((64, 1e-46), "gate"), ((64,), "expected"),
                     (64, "expected")):
        with pytest.raises(ValueError, match=msg):
            check_detections(bad)
        with pytest.raises(ValueError, match=msg):
            MultiTargetTracker(_Echo(_cfg()), 100, 2, use_graph=False, detections=bad)
        with pytest.raises(ValueError, match=msg):
            track_feeds(None, [], 1, 4, max_points=100, detections=bad)
    assert detection_gate2(0.1) == float(np.float32(0.1) * np.float32(0.1))
    assert plane_axes([0, 0, 1]) == (0, 1) and plane_axes([0, -1, 0]) == (0, 2) and plane_axes([1, 0, 0]) == (1, 2)
    with pytest.raises(ValueError, match="up_axis"):
        plane_axes([0, 1, 1])
    with pytest.raises(ValueError, match="up_axis"):
        MultiTargetTracker(_Echo(_cfg(up_axis=[1, 1, 0])), 100, 2, use_graph=False, detections=(4, 1.0))
    rot = np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])
    rows = detection_rows([Box(np.array([1.0, 2.0, 3.0]), np.array([1.5, 4.0, 1.6]), rot)], [0.75])
    assert rows.dtype == np.float32 and rows.shape == (1, 16)
    assert rows[0].tolist() == np.float32([1.0, 2.0, 3.0, 1.5, 4.0, 1.6] + rot.reshape(-1).tolist() + [0.75]).tolist()
    assert detection_rows([], []).shape == (0, 16)
    with pytest.raises(ValueError, match="scores"):
        detection_rows([Box(np.zeros(3), np.ones(3), rot)], [])


def test_put_refuses_bad_detections_and_stages_nothing():
    trk = MultiTargetTracker(_Echo(_cfg()), 100, 2, use_graph=False, feeds=2, detections=(4, 1.0))
    pts = torch.zeros(10, 3)
    good = np.zeros((2, 16), np.float32)
    for bad, msg in ((np.zeros((5, 16)), "max_per_scan=4"), (np.zeros((2, 15)), "shape"), (np.zeros(16), "shape"),
                     (np.full((1, 16), np.nan), "finite"), (np.full((1, 16), np.inf), "finite"), ([["a"] * 16], "numbers")):
        with pytest.raises(ValueError, match=msg):
            trk.put(0, pts, detections=bad)
        assert not trk.scan_feeds.staged and not trk._det_staged
    with pytest.raises(ValueError, match="feed 2 out of range"):
        trk.put(2, pts, detections=good)
    trk.put(1, pts, detections=torch.from_numpy(good))
    trk.put(0, pts, detections=[])
    assert set(trk.scan_feeds.staged) == {0, 1} and trk._det_staged[1].shape == (2, 16) and trk._det_staged[0].shape == (0, 16)
    plain = MultiTargetTracker(_Echo(_cfg()), 100, 2, use_graph=False)
    with pytest.raises(ValueError, match="built without"):
        plain.put(0, pts, detections=good)
    assert not plain.scan_feeds.staged
    with pytest.raises(ValueError, match="built without"):
        plain.unmatched()
    b = trk.boxes()
    assert b["detection"].data_ptr() == trk._detection.data_ptr() and (b["detection"] == -1).all() and not b["reacquired"].any()
    assert trk.evidence().shape == (2, 4) and trk._record().shape == (2, 19) and trk.snapshot().shape == (2, 15)
    assert trk.unmatched() == {0: [], 1: []}                                 # nothing advanced yet


def test_add_and_drop_reset_the_detection_state():
    trk = MultiTargetTracker(_Echo(_cfg(shape_aggregation="previous")), 100, 3, use_graph=False, detections=(8, 2.0))
    trk.scan_feeds.feed_seen[0] = 1
    trk.scans_seen = 1
    trk.detection.fill_(5)
    trk.reacquired.fill_(True)
    trk.add(4, Box(np.array([1.0, 2.0, 3.0]), np.array([1.5, 4.0, 1.5]), np.eye(3)))
    k = trk.targets()[4]
    assert int(trk.detection[k]) == -1 and not bool(trk.reacquired[k])
    trk.detection[k].fill_(2)
    trk.reacquired[k].fill_(True)
    trk.drop(4)
    assert int(trk.detection[k]) == -1 and not bool(trk.reacquired[k])


def test_multi_class_detections():
    models = {n: _Echo(_cfg()) for n in ("Car", "Ped")}
    mc = MultiClassTracker(models, 100, {"Car": 2, "Ped": 3}, use_graph=False, detections={"Car": (16, 2.0)})
    assert mc.trackers["Car"].detections == (16, 2.0) and mc.trackers["Ped"].detections is None
    assert list(mc._detect_rows()) == [True, True, False, False, False]
    mc = MultiClassTracker(models, 100, {"Car": 2, "Ped": 3}, use_graph=False, detections=(16, 2.0))
    assert mc.trackers["Car"].detections == mc.trackers["Ped"].detections == (16, 2.0)
    with pytest.raises(ValueError, match="detections: class 'Cyclist' has no model"):
        MultiClassTracker(models, 100, {"Car": 2, "Ped": 3}, use_graph=False, detections={"Cyclist": (16, 2.0)})
    with pytest.raises(ValueError, match="class 'Car'.*max_per_scan"):
        MultiClassTracker(models, 100, {"Car": 2, "Ped": 3}, use_graph=False, detections={"Car": (0, 2.0)})
    mc = MultiClassTracker(models, 100, {"Car": 2, "Ped": 3}, use_graph=False, detections={"Car": (16, 2.0)})
    pts, rows = torch.zeros(10, 3), np.zeros((3, 16), np.float32)
    for bad, msg in (({"Ped": rows}, "class 'Ped'.*built without"), ({"Bus": rows}, "class 'Bus'"), (rows, "class: ")):
        with pytest.raises(ValueError, match=msg):
            mc.put(0, pts, detections=bad)
        assert not mc.scan_feeds.staged
    mc.put(0, pts, detections={"Car": rows})
    assert mc.trackers["Car"]._det_staged[0].shape == (3, 16)
    assert mc.unmatched() == {"Car": {0: []}}


# ------------------------------------------------------------------ the command line
def test_detections_option_parsing(tmp_path, capsys):
    base = ["--cfg", "c.yaml", "--path", "p"]
    plain = track.parse_args(base)
    assert not any(hasattr(plain, n) for n in ("detections", "detection_gate", "max_detections"))
    args = track.parse_args(base + ["--detections", "d.jsonl", "--detection_gate", "2.5", "--max_detections", "64"])
    assert args.detections == "d.jsonl" and args.detection_rule == (64, 2.5)
    for bad in (["--detections", "d.jsonl"], ["--detections", "d.jsonl", "--detection_gate", "2"], ["--detection_gate", "2"],
                ["--max_detections", "4", "--detection_gate", "2"]):
        with pytest.raises(SystemExit):
            track.parse_args(base + bad)
        assert "--detections FILE needs" in capsys.readouterr().err
    for bad in (["--detection_gate", "0", "--max_detections", "4"], ["--detection_gate", "nan", "--max_detections", "4"],
                ["--detection_gate", "2", "--max_detections", "0"], ["--detection_gate", "2", "--max_detections", "2000"]):
        with pytest.raises(SystemExit):
            track.parse_args(base + ["--detections", "d.jsonl"] + bad)
        assert "--detection_gate / --max_detections" in capsys.readouterr().err


def test_read_detections(tmp_path):
    path = tmp_path / "d.jsonl"
    lines = [{"scene": "0019", "frame": 3, "class": "Car", "boxes": [[1, 2, 3, 1.5, 4, 1.6, 1, 0, 0, 0, 0.9],
                                                                      [5, 6, 7, 1, 1, 1, 0, 0, 0, 2, 0.2]]},
             {"scene": 19, "frame": 4, "class": "Car", "boxes": []}]
    path.write_text("\n".join(json.dumps(l) for l in lines) + "\n\n")
    table = track.read_detections(str(path))
    assert sorted(table) == [("0019", 3, "Car"), ("19", 4, "Car")]
    a = table[("0019", 3, "Car")]
    assert a.shape == (2, 16) and a[0, :6].tolist() == np.float32([1, 2, 3, 1.5, 4, 1.6]).tolist() and a[0, 6:15].tolist() == np.eye(3).reshape(-1).tolist()
    assert np.allclose(a[1, 6:15], np.diag([-1.0, -1.0, 1.0]).reshape(-1)) and a[1, 15] == np.float32(0.2)   # 180 deg about z
    assert table[("19", 4, "Car")].shape == (0, 16)
    assert track._scan_detections(table, "0019", 5, "Car").shape == (0, 16)
    for bad in ('{"scene": "0", "frame": 1, "class": "Car", "boxes": [[1, 2, 3]]}', '{"scene": "0", "frame": 1}', "not json",
                '{"scene": "0", "frame": 1, "class": "Car", "boxes": [[1, 2, 3, 1, 1, 1, 0, 0, 0, 0, 1]]}',
                '{"scene": "0", "frame": 1, "class": "Car", "boxes": [[1, 2, 3, 1, 1, 1, 1, 0, 0, 0, NaN]]}'):
        path.write_text(bad + "\n")
        with pytest.raises(SystemExit, match="d.jsonl:1"):
            track.read_detections(str(path))
    path.write_text(json.dumps(lines[1]) + "\n" + json.dumps(lines[1]) + "\n")
    with pytest.raises(SystemExit, match="second line"):
        track.read_detections(str(path))


def test_json_evidence_with_detections():
    assert track._evidence((3, 0.5, True, 2), detections=True) == {"points": 3, "score": 0.5, "detection": 2, "reacquired": True}
    assert track._evidence((3, 0.5, False, True, 1), detections=True) == {"points": 3, "score": 0.5, "coasting": False,
                                                                          "detection": 1, "reacquired": True}
    assert track._evidence((-1, float("nan"), False, -1), detections=True) == {"points": None, "score": None, "detection": None,
                                                                              "reacquired": False}
