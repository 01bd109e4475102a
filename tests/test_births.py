"""Target births in the live tracker, without a GPU: the births' formulation (`birth_tensors`) against a per-feed numpy loop, a
birth's slot state and first-frame crop against what `add()` writes for the same box, `o3d_track_birth`'s argument checks
through the C ABI, the `births=` refusals, and the host's bookkeeping (reservations, pending slots in the work list and the
bucket, resolution BIRTH_LAG advances later, `births(wait=True)`, MultiClassTracker) over a stand-in step."""
import ctypes

import numpy as np
import pytest
import torch

from open3dsot_b200 import _lib
from open3dsot_b200.datasets.data_classes import Box
from open3dsot_b200.tracking import multi_tracker as mt
from open3dsot_b200.tracking.multi_class import MultiClassTracker, track_classes
from open3dsot_b200.tracking.multi_tracker import (BIRTH_ID_BASE, BIRTH_LAG, BirthSlots, MultiTargetTracker, associate,
                                                   check_births, detection_gate2, detection_rows, track_feeds)
from test_coast import _bits
from test_tracking_host import _cfg, _Echo

F32 = np.float32


# ------------------------------------------------------------------ a births case and its numpy loop
def birth_case(K, b, F, D, seed, per=3, grid=False, n_det=None, reserve=None):
    """A b-row step over F feeds (rows' pred centres, NaN where a row does not advance), each feed's detections and matching
    records, and a birth list of up to `per` reserved slots per fed feed (`reserve`: {feed: rows} instead).  `grid`: integer
    centres, so that pairs exactly at the integer gate occur; scores from a few values, so that ties and scores exactly at
    min_score = 0.5 occur."""
    rng = np.random.default_rng(seed)
    feed = rng.integers(0, F, b).astype(np.int64)
    adv = rng.random(b) < 0.7
    if grid:
        pred = rng.integers(-3, 4, (b, 3)).astype(F32)
    else:
        pred = rng.normal(0, 6, (b, 3)).astype(F32)
    pred[~adv] = np.nan
    fed = (rng.random(F) < 0.8).astype(np.int64)
    count = np.array([(rng.integers(0, D + 1) if n_det is None else min(n_det, D)) if fed[f] else 0 for f in range(F)], np.int32)
    det = rng.normal(0, 1, (F, D, 16)).astype(F32)
    det[..., :3] = rng.integers(-3, 4, (F, D, 3)).astype(F32) if grid else rng.normal(0, 6, (F, D, 3)).astype(F32)
    det[..., 15] = rng.choice(F32([0.1, 0.5, 0.5, 0.7, 0.9, 0.9, -0.0, 0.0]), (F, D))
    rec_slot = np.where(rng.random((F, D)) < 0.2, rng.integers(0, K, (F, D)), -1).astype(np.int32)
    free = list(rng.permutation(K))
    entries = []
    for f in range(F):
        r = reserve.get(f, 0) if reserve is not None else (rng.integers(0, per + 1) if fed[f] else 0)
        r = min(r, len(free))
        entries += [(int(free.pop(0)), f) for _ in range(r)]
    R = max(1, min(K, per * F))
    entries = entries[:R]
    bl = np.array([[k for k, _ in entries] + [K] * (R - len(entries)), [f for _, f in entries] + [-1] * (R - len(entries))], np.int64)
    return feed, adv, pred, fed, count, det, rec_slot, bl


def birth_loop(case, gate2, axes, min_score, n0=0):
    """The births as the semantics state them, one feed and one candidate at a time: [(entry, slot, id, feed, detection)]."""
    feed, adv, pred, fed, count, det, rec_slot, bl = case
    a0, a1 = axes
    g2 = F32(gate2)
    d2 = lambda p, q: (F32(p[a0]) - F32(q[a0])) * (F32(p[a0]) - F32(q[a0])) + (F32(p[a1]) - F32(q[a1])) * (F32(p[a1]) - F32(q[a1]))
    out, n = [], n0
    for f in range(det.shape[0]):
        entries = [e for e in range(bl.shape[1]) if bl[1, e] == f]
        if not fed[f] or not entries:
            continue
        cands = []
        for d in range(count[f]):
            q = det[f, d]
            if rec_slot[f, d] >= 0 or not q[15] >= F32(min_score):
                continue
            if any(adv[i] and feed[i] == f and d2(pred[i], q) <= g2 for i in range(len(feed))):
                continue
            cands.append(d)
        cands.sort(key=lambda d: (-float(det[f, d, 15]), d))
        born = []
        for d in cands:
            if len(born) == len(entries):
                break
            if any(d2(det[f, d], det[f, e]) <= g2 for e in born):
                continue
            born.append(d)
        for e, d in zip(entries, born):
            out.append((e, int(bl[0, e]), BIRTH_ID_BASE + n, f, d))
            n += 1
    return out


def _slots(K, seed):
    rng = np.random.default_rng(seed)
    R = K + 2
    T = torch.from_numpy
    return BirthSlots(T(rng.normal(0, 3, (R, 3)).astype(F32)), T(rng.random((R, 3)).astype(F32)),
                      T(rng.normal(0, 1, (R, 3, 3)).astype(F32)), T(rng.random(R).astype(F32)), T(rng.random(R) < 0.5),
                      T(rng.integers(0, 99, R)), T(rng.integers(0, 9, R)), T(rng.integers(0, 3, R)),
                      T(rng.integers(-1, 9, R).astype(np.int32)), T(rng.random(R).astype(F32)),
                      T(rng.integers(0, 3, R).astype(np.int32)), T(rng.random(R) < 0.3), T(rng.normal(0, 1, (R, 3)).astype(F32)),
                      T(rng.normal(0, 1, (R, 3)).astype(F32)), T(rng.integers(0, 9, R)), T(rng.random(R) < 0.3),
                      T(rng.integers(-1, 9, R).astype(np.int32)), T(rng.random(R) < 0.3))


def run_births(case, K, gate2, axes, min_score, n0=0, device="cpu", seed=0):
    feed, adv, pred, fed, count, det, rec_slot, bl = case
    T = lambda x: torch.from_numpy(np.array(x, copy=True)).to(device)
    slots = BirthSlots(*(x.to(device) for x in _slots(K, seed)))
    rec, nxt = T(rec_slot), torch.tensor([n0], device=device)
    log = torch.zeros(bl.shape[1], 4, dtype=torch.int64, device=device)
    mt.track_birth(T(feed), T(adv), T(pred), T(fed), T(count), T(det), rec, T(bl), nxt, log, slots, gate2, axes, min_score)
    return slots, rec, nxt, log


def want_state(case, K, births, seed=0):
    """_slots(K, seed) with the loop's births written as add() writes them."""
    det, rec_slot = case[5], case[6].copy()
    s = [x.numpy().copy() for x in _slots(K, seed)]
    names = BirthSlots._fields
    for _, k, tid, f, d in births:
        row = det[f, d]
        vals = dict(box_c=row[0:3], box_s=row[3:6], box_r=row[6:15].reshape(3, 3), first_flag=1.0, active=True, key=tid, t=0,
                    slot_feed=f, points=-1, score=np.nan, misses=0, lost=False, vel=0.0, hit_c=row[0:3], hit_t=0, coasting=False,
                    detection=-1, reacquired=False)
        for i, n in enumerate(names):
            s[i][k] = vals[n]
        rec_slot[f, d] = k
    return s, rec_slot


def check_case(case, K, gate2, axes, min_score, n0=0):
    want = birth_loop(case, gate2, axes, min_score, n0)
    slots, rec, nxt, log = run_births(case, K, gate2, axes, min_score, n0)
    s, rec_slot = want_state(case, K, want)
    for n, w, g in zip(BirthSlots._fields, s, slots):
        assert np.array_equal(_bits(g.numpy()), _bits(w)), n
    assert np.array_equal(rec.numpy(), rec_slot)
    wl = np.full((case[-1].shape[1], 4), -1, np.int64)
    for e, k, tid, f, d in want:
        wl[e] = (k, tid, f, d)
    assert np.array_equal(log.numpy(), wl) and int(nxt[0]) == n0 + len(want)
    return want


@pytest.mark.parametrize("K,b,F,D,per", [(1, 1, 1, 1, 1), (9, 7, 2, 5, 3), (70, 64, 3, 40, 8), (40, 32, 16, 12, 2),
                                         (8, 0, 3, 16, 4)])
def test_formulation_equals_the_loop(K, b, F, D, per):
    born = 0
    for seed in range(6):
        for axes in ((0, 1), (0, 2)):
            case = birth_case(K, b, F, D, seed, per=per)
            born += len(check_case(case, K, detection_gate2(2.0), axes, 0.5, n0=seed * 7))
    assert born > 0 or K == 1


def test_ties_scores_at_min_score_and_pairs_at_the_gate():
    """Integer centres and a gate of 2 (gate2 = 4 exactly): detections exactly at the gate of a row are no candidates and those
    exactly at the gate of a born one are passed over; equal scores rank by index; a score equal to min_score is a candidate."""
    at_row = at_born = ties = at_min = 0
    for seed in range(40):
        case = birth_case(24, 16, 2, 24, seed, per=6, grid=True)
        want = check_case(case, 24, detection_gate2(2.0), (0, 1), 0.5)
        feed, adv, pred, fed, count, det, rec_slot, bl = case
        for f in range(2):
            q = det[f, :count[f]]
            rows = pred[adv & (feed == f)]
            at_row += int(((rows[:, None, 0] - q[None, :, 0]) ** 2 + (rows[:, None, 1] - q[None, :, 1]) ** 2 == 4).sum())
            born = [d for _, _, _, g, d in want if g == f]
            at_born += sum(int(((q[d, :2] - q[:, :2]) ** 2).sum(-1).__eq__(4).sum()) for d in born)
            at_min += sum(q[d, 15] == F32(0.5) for d in born)
            ties += len(born) - len({float(q[d, 15]) for d in born})
    assert at_row > 0 and at_born > 0 and at_min > 0 and ties > 0


def test_fewer_and_more_candidates_than_reserved_rows():
    for seed in range(4):
        for n, r, born in ((32, 3, 3), (2, 6, 2)):
            case = birth_case(40, 0, 1, 32, seed, n_det=n, reserve={0: r})
            case[3][:], case[4][:], case[6][:] = 1, n, -1                    # fed, n detections, none matched
            want = check_case(case, 40, detection_gate2(0.01), (0, 1), -1.0)  # every detection a candidate, far apart
            assert [e for e, *_ in want] == list(range(born))


def test_feeds_without_reservation_or_not_fed_start_nothing():
    for seed in range(4):
        case = birth_case(30, 20, 3, 16, seed, n_det=16, reserve={0: 2, 2: 3})
        feed, adv, pred, fed, count, det, rec_slot, bl = case
        fed[:] = [1, 1, 0]
        count[:] = [16, 16, 0]
        want = check_case(case, 30, detection_gate2(1.0), (0, 1), -1.0)
        assert {f for _, _, _, f, _ in want} <= {0}
        fed[2], count[2] = 0, 16                                               # a count on a feed that is not fed is ignored
        check_case(case, 30, detection_gate2(1.0), (0, 1), -1.0)


# ------------------------------------------------------------------ the C entry's argument checks
_BPTRS = ("feed", "adv", "pred", "fed", "count", "det", "rec_slot", "birth_slot", "birth_feed", "next", "log") + \
         tuple(n for n, _, _ in __import__("open3dsot_b200.ops", fromlist=["BIRTH_SLOTS"]).BIRTH_SLOTS)


def _bdesc(**kw):
    d = dict(b=4, F=2, D=8, R=4, axis0=0, axis1=1, gate2=4.0, min_score=0.5, id_base=BIRTH_ID_BASE,
             **{n: 16 for n in _BPTRS})                                                  # never dereferenced
    d.update(kw)
    return _lib.BirthDesc(**d)


def test_track_birth_refuses_bad_arguments():
    L = _lib.lib()
    call = lambda d: L.o3d_track_birth(ctypes.byref(d), None)
    assert L.o3d_track_birth(None, None) < 0 and b"null" in L.o3d_last_error()
    for n in _BPTRS:
        assert call(_bdesc(**{n: None})) < 0, n
        assert b"null" in L.o3d_last_error()
    for kw in (dict(b=-1), dict(b=65536), dict(F=0), dict(D=0), dict(D=1025), dict(R=0), dict(R=65536)):
        assert call(_bdesc(**kw)) < 0 and b"bad sizes" in L.o3d_last_error(), kw
    for g in (0.0, -1.0, float("nan"), float("inf")):
        assert call(_bdesc(gate2=g)) < 0 and b"gate2" in L.o3d_last_error(), g
    for m in (float("nan"), float("inf"), -float("inf")):
        assert call(_bdesc(min_score=m)) < 0 and b"min_score" in L.o3d_last_error(), m
    for a0, a1 in ((0, 0), (-1, 1), (0, 3)):
        assert call(_bdesc(axis0=a0, axis1=a1)) < 0 and b"axes" in L.o3d_last_error(), (a0, a1)
    assert call(_bdesc(id_base=-1)) < 0 and b"id_base" in L.o3d_last_error()


# ------------------------------------------------------------------ births= and add()
def test_births_refusals():
    assert check_births(None, None) is None and check_births((0.3, 2), (8, 1.0)) == (float(F32(0.3)), 2)
    assert check_births((-5, 8), (8, 1.0)) == (-5.0, 8)
    for bad, msg in (((0.5, 0), "per_scan"), ((0.5, 9), "per_scan"), ((0.5, 2.0), "per_scan"), ((0.5, True), "per_scan"),
                     ((float("nan"), 2), "min_score"), ((float("inf"), 2), "min_score"), ((1e39, 2), "min_score"),
                     (("a", 2), "min_score"), ((0.5,), "expected"), (0.5, "expected")):
        with pytest.raises(ValueError, match=msg):
            check_births(bad, (8, 1.0))
        with pytest.raises(ValueError, match=msg):
            MultiTargetTracker(_Echo(_cfg()), 100, 4, use_graph=False, detections=(8, 1.0), births=bad)
    with pytest.raises(ValueError, match="detections="):
        MultiTargetTracker(_Echo(_cfg()), 100, 4, use_graph=False, births=(0.5, 2))
    for fn, args in ((track_feeds, (None, [], 1, 4)), (track_classes, ({}, [], 1, {}))):
        with pytest.raises(ValueError, match="births= is not supported"):
            fn(*args, max_points=100, detections=(8, 1.0), births=(0.5, 2))
    plain = MultiTargetTracker(_Echo(_cfg()), 100, 4, use_graph=False, detections=(8, 1.0))
    with pytest.raises(ValueError, match="built without births"):
        plain.births()


def test_add_refuses_born_ids():
    trk = MultiTargetTracker(_Echo(_cfg()), 100, 4, use_graph=False, detections=(8, 1.0), births=(0.5, 2))
    trk.scan_feeds.feed_seen[0] = trk.scans_seen = 1
    box = Box(np.zeros(3), np.ones(3), np.eye(3))
    for tid in (BIRTH_ID_BASE, BIRTH_ID_BASE + 5, -1):
        with pytest.raises(ValueError, match="ids 0 .. "):
            trk.add(tid, box)
    trk.add(BIRTH_ID_BASE - 1, box)
    plain = MultiTargetTracker(_Echo(_cfg()), 100, 4, use_graph=False)          # without births every id is taken as before
    plain.scan_feeds.feed_seen[0] = plain.scans_seen = 1
    plain.add(BIRTH_ID_BASE + 5, box)


# ------------------------------------------------------------------ the host's bookkeeping over a stand-in step
def _stand_in(trk, calls):
    """Replace the network step with one that matches and starts targets exactly as the step does, taking each advancing row's
    box as the network's (no network, no crops: runs on the CPU); `calls` records the bucket of every step."""
    def step(b):
        calls.append(b)
        with torch.no_grad():
            r, box, dst = trk._gather(b)
            points = torch.full((b,), 100, dtype=torch.int32)
            pred, m, m_box = associate(trk._work[0, :b], r["feed"], r["adv"], box.center, points, trk._slots, trk.fstate[0],
                                       trk._det_n, trk._det_in, (trk._det_rec, trk._det_count, trk._det_slot), trk._gate2,
                                       trk._axes)
            mt.track_update(trk._slots, trk._work[0, :b], dst, r["adv"], box.center, box.rot, points, torch.zeros(b), None, None,
                            (m, m_box) + tuple(trk._match_slots))
            if trk.birth_rule is not None:
                trk._birth_stage(r["feed"], r["adv"], pred)
    trk._step = step
    return trk


def _tracker(K=8, F=2, births=(0.5, 2), mode="firstandprevious", calls=None):
    trk = MultiTargetTracker(_Echo(_cfg(shape_aggregation=mode)), 400, K, use_graph=False, feeds=F, detections=(16, 1.0),
                             births=births)
    return _stand_in(trk, [] if calls is None else calls)


def _scan(seed, n=300):
    return torch.from_numpy(np.random.default_rng(seed).uniform(-20, 20, (n, 3)).astype(F32))


def _dets(xs, score=0.9):
    return detection_rows([Box(np.array([x, 0.0, 0.0]), np.array([1.5, 4.0, 1.5]), np.eye(3)) for x in xs], [score] * len(xs))


def test_reservations_pending_slots_and_resolution_lag():
    calls = []
    trk = _tracker(K=8, calls=calls)
    trk.put(0, _scan(0), detections=_dets([0.0, 5.0, 10.0]))                   # 3 staged: 2 reserved (per_scan)
    trk.put(1, _scan(1), detections=_dets([-7.0]))
    trk.advance()                                                             # advance 0: births into slots 0, 1 (feed 0), 2 (feed 1)
    assert trk._pending == {0: 0, 1: 0, 2: 1} and trk.targets() == {} and trk.births() == []
    assert calls == [8, 1, 2, 4, 8]                                           # the plan's steps (every bucket); nothing to step
    box = Box(np.array([-3.0, 0.0, 0.0]), np.array([1.5, 4.0, 1.5]), np.eye(3))
    trk.add(7, box, feed=1)                                                   # add() takes the lowest slot neither a target's nor pending
    assert trk.targets() == {7: 3}
    trk.put(0, _scan(2))
    trk.put(1, _scan(3))
    trk.advance()                                                             # advance 1: pending slots step (3 + 1 target)
    assert calls[-1] == 4 and trk.targets() == {7: 3} and trk.births() == []
    trk.put(0, _scan(4), detections=_dets([20.0]))
    trk.advance()                                                             # advance 2: advance 0 resolved at its start
    born = trk.births()
    assert [(tid - BIRTH_ID_BASE, f, k, d) for tid, f, k, d in born] == [(0, 0, 0, 0), (1, 0, 1, 1), (2, 1, 2, 0)]
    assert trk.targets() == {7: 3, BIRTH_ID_BASE: 0, BIRTH_ID_BASE + 1: 1, BIRTH_ID_BASE + 2: 2}
    assert trk._pending == {4: 0} and calls[-1] == 2                          # feed 0's two born targets step
    assert trk.births(wait=True) == [(BIRTH_ID_BASE + 3, 0, 4, 0)] and trk._pending == {}
    assert sorted(d for d, _, _ in trk.unmatched()[0]) == [] and trk.unmatched()[1] == []
    st = trk.boxes()
    assert st["ids"].tolist()[:5] == [BIRTH_ID_BASE, BIRTH_ID_BASE + 1, BIRTH_ID_BASE + 2, 7, BIRTH_ID_BASE + 3]
    trk.drop(BIRTH_ID_BASE + 1)                                               # born targets are ordinary targets once resolved
    assert BIRTH_ID_BASE + 1 not in trk.targets() and not bool(trk.active[1])


def test_unborn_reservations_are_freed_and_stay_unmatched():
    trk = _tracker(K=8, births=(0.95, 2))                                     # every score below min_score
    trk.put(0, _scan(0), detections=_dets([0.0, 5.0]))
    trk.advance()
    assert trk._pending == {0: 0, 1: 0}
    for i in range(BIRTH_LAG):
        trk.put(0, _scan(1 + i))
        trk.advance()
    assert trk._pending == {} and trk.births() == [] and trk.targets() == {}
    assert not trk.active.any()


def test_scarce_slots_and_the_id_counter():
    trk = _tracker(K=3, births=(0.0, 4), F=1)
    rows = detection_rows([Box(np.array([4.0 * i, 0, 0]), np.ones(3), np.eye(3)) for i in range(5)], [0.1, 0.9, 0.5, 0.7, 0.3])
    trk.put(0, _scan(0), detections=rows)
    trk.advance()
    assert sorted(trk._pending) == [0, 1, 2]
    got = trk.births(wait=True)
    assert [(tid - BIRTH_ID_BASE, d) for tid, _, _, d in got] == [(0, 1), (1, 3), (2, 2)]   # descending score
    assert [d for d, _, _ in trk.unmatched()[0]] == [0, 4]
    with pytest.raises(ValueError, match="all 3 slots"):
        trk.add(1, Box(np.zeros(3), np.ones(3), np.eye(3)))
    trk.drop(BIRTH_ID_BASE + 1)
    trk.put(0, _scan(1), detections=rows)
    trk.advance()
    assert [(tid - BIRTH_ID_BASE, k) for tid, _, k, _ in trk.births(wait=True)] == [(3, 1)]


def test_a_birth_writes_what_add_writes():
    """The same detection box, born on the device (the formulation here) and add()ed after the advance, gives bitwise the same
    slot state and first-frame crop."""
    for mode in ("firstandprevious", "first", "previous"):
        scan = _scan(5, n=400)
        scan[:40] = torch.from_numpy(np.random.default_rng(1).uniform(-1, 1, (40, 3)).astype(F32)) + torch.tensor([3.0, 1.0, 0.0])
        rot = np.array([[0.6, -0.8, 0.0], [0.8, 0.6, 0.0], [0.0, 0.0, 1.0]])
        box = Box(np.array([3.1, 0.9, 0.2]), np.array([1.7, 3.9, 1.4]), rot)
        rows = detection_rows([box], [0.9])
        born = _tracker(K=4, F=1, mode=mode, births=(0.5, 1))
        born.put(0, scan.clone(), n_valid=350, detections=rows)
        born.advance()
        (tid, _, k, _), = born.births(wait=True)
        added = _tracker(K=4, F=1, mode=mode, births=None)
        added.put(0, scan.clone(), n_valid=350, detections=rows)
        added.advance()
        (d, b, _), = added.unmatched()[0]
        added.add(tid, b)
        j = added.targets()[tid]
        for name in BirthSlots._fields:
            assert np.array_equal(_bits(getattr(born, "_" + name)[k].numpy()), _bits(getattr(added, "_" + name)[j].numpy())), \
                (mode, name)
        if mode != "previous":
            assert torch.equal(born.first_keep[k], added.first_keep[j]) and born.first_keep[k].any()
            assert np.array_equal(_bits(born.first_local[k].numpy()), _bits(added.first_local[j].numpy()))


def test_feature_off_keeps_the_upload_and_the_step():
    trk = _tracker(births=None)
    assert trk.R == 0 and trk._det_at == 16 * 8 + 16 and trk._n_at == 16 * 8
    assert len(trk._state()) == 12 + 2 + 3 and not hasattr(trk, "_birth_list")
    on = _tracker(births=(0.5, 3))
    assert on.R == 6 and on._n_at == 16 * 8 + 16 * 6 and on._birth_list.data_ptr() == on._upload.data_ptr() + 16 * 8


def test_multi_class_births():
    models = {n: _Echo(_cfg()) for n in ("Car", "Ped")}
    mc = MultiClassTracker(models, 400, {"Car": 4, "Ped": 4}, use_graph=False, detections=(8, 1.0), births={"Car": (0.5, 2)})
    assert mc.trackers["Car"].birth_rule == (0.5, 2) and mc.trackers["Ped"].birth_rule is None
    with pytest.raises(ValueError, match="births: class 'Bus' has no model"):
        MultiClassTracker(models, 400, {"Car": 4, "Ped": 4}, use_graph=False, detections=(8, 1.0), births={"Bus": (0.5, 2)})
    with pytest.raises(ValueError, match="class 'Ped'.*detections="):
        MultiClassTracker(models, 400, {"Car": 4, "Ped": 4}, use_graph=False, detections={"Car": (8, 1.0)}, births=(0.5, 2))
    with pytest.raises(ValueError, match="no class was built with births"):
        MultiClassTracker(models, 400, {"Car": 4, "Ped": 4}, use_graph=False, detections=(8, 1.0)).births()
    mc = MultiClassTracker(models, 400, {"Car": 4, "Ped": 4}, use_graph=False, detections=(8, 1.0), births=(0.5, 2))
    for trk in mc.trackers.values():
        _stand_in(trk, [])
    mc.put(0, _scan(0), detections={"Car": _dets([0.0, 5.0, 9.0]), "Ped": _dets([2.0])})
    mc.advance()
    assert mc.births() == {"Car": [], "Ped": []}
    got = mc.births(wait=True)
    assert [(t - BIRTH_ID_BASE, d) for t, _, _, d in got["Car"]] == [(0, 0), (1, 1)]
    assert [(t - BIRTH_ID_BASE, d) for t, _, _, d in got["Ped"]] == [(0, 0)]
    assert sorted(mc.targets()) == [("Car", BIRTH_ID_BASE), ("Car", BIRTH_ID_BASE + 1), ("Ped", BIRTH_ID_BASE)]
