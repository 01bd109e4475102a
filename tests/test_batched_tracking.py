"""Split evaluation with many tracklets in flight, host side: the slot schedule and chunking, the keyed-draw restatement
against Philox4x32-10 known-answer vectors, and the argument checks of the two C-ABI entry points (no GPU needed)."""
import numpy as np
import pytest

from _philox import keyed_uniform, philox4x32_10
from open3dsot_b200 import _lib
from open3dsot_b200.tracking.batched_tracker import plan_chunks, plan_schedule


def _replay(plan, lengths):
    """Simulate the schedule: per step, which tracklet each slot tracks; returns (admitted order, frames tracked per tracklet)."""
    occupant, left, admitted, tracked = {}, {}, [], {}
    for t in range(plan["steps"]):
        for k, j in plan["admissions"][t]:
            assert left.get(k, 0) == 0, f"slot {k} re-filled while tracklet {occupant[k]} still runs"
            occupant[k], left[k] = j, lengths[j] - 1
            admitted.append(j)
        for k in list(left):
            if left[k]:
                tracked[occupant[k]] = tracked.get(occupant[k], 0) + 1
                left[k] -= 1
    assert all(v == 0 for v in left.values())
    return admitted, tracked


@pytest.mark.parametrize("slots", [1, 3, 8, 64])
def test_schedule_admits_every_tracklet_once_longest_first(slots):
    rng = np.random.default_rng(slots)
    lengths = [int(x) for x in rng.integers(1, 30, size=25)] + [1, 1, 2]
    plan = plan_schedule(lengths, slots)
    admitted, tracked = _replay(plan, lengths)
    multi = [j for j, n in enumerate(lengths) if n > 1]
    assert sorted(admitted) == multi                                         # each multi-frame tracklet exactly once
    assert [lengths[j] for j in admitted] == sorted((lengths[j] for j in multi), reverse=True)   # longest first
    assert all(tracked[j] == lengths[j] - 1 for j in multi)
    assert plan["slots"] == min(slots, len(multi))
    assert all(k < plan["slots"] for step in plan["admissions"] for k, _ in step)
    # record offsets are pool frame indices: tracklet j's frame i lives at offsets[j] + i in the concatenated pool
    pool = [(j, i) for j, n in enumerate(lengths) for i in range(n)]
    for j, n in enumerate(lengths):
        assert [pool[plan["offsets"][j] + i] for i in range(n)] == [(j, i) for i in range(n)]


def test_schedule_edge_cases():
    empty = plan_schedule([], 8)
    assert empty["steps"] == 0 and empty["admissions"] == [] and len(empty["offsets"]) == 0 and empty["slots"] == 0
    ones = plan_schedule([1, 1, 1], 4)                                        # 1-frame tracklets never take a slot
    assert ones["steps"] == 0 and ones["slots"] == 0 and list(ones["offsets"]) == [0, 1, 2]
    wide = plan_schedule([5, 3, 1, 7], 100)                                   # more slots than tracklets
    assert wide["slots"] == 3 and wide["steps"] == 6
    assert wide["admissions"][0] == [(0, 3), (1, 0), (2, 1)]
    narrow = plan_schedule([5, 3, 1, 7], 1)                                   # one slot: back to back, longest first
    assert narrow["steps"] == 6 + 4 + 2
    assert [a for a in narrow["admissions"] if a] == [[(0, 3)], [(0, 0)], [(0, 1)]]


def test_chunks_keep_tracklets_whole():
    lengths = [4, 6, 3, 9, 1, 2]
    chunks = plan_chunks(lengths, 10, 100)
    assert [j for c in chunks for j in c] == list(range(len(lengths)))
    assert all(sum(lengths[j] for j in c) * 10 <= 100 for c in chunks)
    assert plan_chunks([], 10, 100) == []
    with pytest.raises(ValueError, match="max_resident_bytes"):
        plan_chunks([3, 20], 10, 100)


def test_philox_known_answers():
    """Random123's kat_vectors for philox4x32_10 (the generator cuRAND's Philox4_32_10 implements)."""
    kat = [((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
           ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
           ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
            (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1))]
    for ctr, key, want in kat:
        got = philox4x32_10(np.array(ctr, dtype=np.uint32), np.array(key, dtype=np.uint32))
        assert [int(x) for x in got] == list(want)


def test_keyed_draw_mapping():
    """element e of (seed, tracklet, frame, stream) = word e % 4 of Philox(counter (e // 4, frame, stream, 0), key (seed, tracklet))."""
    u = keyed_uniform(7, 3, 5, 2, 11)
    assert u.dtype == np.float32 and u.shape == (11,) and (u >= 0).all() and (u < 1).all()
    for e in (0, 3, 4, 10):
        w = philox4x32_10(np.array([e // 4, 5, 2, 0], dtype=np.uint32), np.array([7, 3], dtype=np.uint32))[e % 4]
        assert u[e] == np.float32(int(w) >> 8) * np.float32(2.0 ** -24)
    assert np.array_equal(keyed_uniform(7, 3, 5, 2, 6), u[:6])               # a prefix does not depend on the length
    assert not np.array_equal(keyed_uniform(7, 4, 5, 2, 11), u)                # another tracklet, another stream of draws
    assert not np.array_equal(keyed_uniform(7, 3, 6, 2, 11), u)
    assert not np.array_equal(keyed_uniform(8, 3, 5, 2, 11), u)


def test_argument_errors_return_status():
    L = _lib.lib()
    assert L.o3d_keyed_uniform(None, 16, 4, 0, 0, 8, 16, None) < 0
    assert b"null" in L.o3d_last_error()
    assert L.o3d_keyed_uniform(16, 16, 70000, 0, 0, 8, 16, None) < 0          # K > 65535
    assert b"K=" in L.o3d_last_error()
    assert L.o3d_keyed_uniform(16, 16, 4, 0, -1, 8, 16, None) < 0             # negative stream
    assert L.o3d_keyed_uniform(16, 16, 0, 0, 0, 8, 16, None) == 0             # nothing to do: no launch
    ptrs = [16] * 7
    assert L.o3d_track_metrics(*ptrs, 4, 3, 4, None, 16, None) < 0
    assert b"null" in L.o3d_last_error()
    assert L.o3d_track_metrics(*ptrs, 4, 1, 4, 16, 16, None) < 0              # dim not 2 / 3
    assert b"dim" in L.o3d_last_error()
    assert L.o3d_track_metrics(*ptrs, 4, 3, 0, 16, 16, None) < 0              # no up axis
    assert b"up_mask" in L.o3d_last_error()
    assert L.o3d_track_metrics(*ptrs, -1, 3, 4, 16, 16, None) < 0
