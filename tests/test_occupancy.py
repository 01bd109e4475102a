"""Occupancy buckets of the live tracker, CPU part: the bucket list for a range of slot counts and smallest buckets, the smallest
bucket derived from the stacks' row counts, the work list of one advance (slot order, padding, no work, held feeds), the host
mirror of the slots' feeds through add / drop, and the threshold the library exports."""
import ctypes

import numpy as np
import pytest
import torch

from open3dsot_b200 import _lib
from open3dsot_b200.datasets import data_classes as dc
from open3dsot_b200.tracking.multi_tracker import (MultiTargetTracker, bucket_for, occupancy_buckets, smallest_bucket,
                                                   work_rows, work_slots)
from test_tracking_host import _cfg, _Echo


@pytest.mark.parametrize("K, smallest, want", [
    (1, 1, (1,)), (2, 1, (1, 2)), (3, 1, (1, 2, 3)), (4, 1, (1, 2, 4)), (5, 1, (1, 2, 4, 5)),
    (32, 1, (1, 2, 4, 8, 16, 32)), (33, 1, (1, 2, 4, 8, 16, 32, 33)), (128, 1, (1, 2, 4, 8, 16, 32, 64, 128)),
    (128, 16, (16, 32, 64, 128)), (128, 3, (4, 8, 16, 32, 64, 128)), (20, 16, (16, 20)), (16, 16, (16,)),
    (8, 16, (8,)), (4, 16, (4,)), (64, 64, (64,)), (64, 65, (64,)), (100, 40, (64, 100))])
def test_bucket_list(K, smallest, want):
    assert occupancy_buckets(K, smallest) == want


def test_bucket_for_is_the_smallest_that_holds():
    buckets = occupancy_buckets(48, 4)
    assert buckets == (4, 8, 16, 32, 48)
    assert [bucket_for(n, buckets) for n in (0, 1, 4, 5, 9, 16, 17, 33, 48)] == [4, 4, 4, 8, 16, 16, 32, 48, 48]
    with pytest.raises(StopIteration):
        bucket_for(49, buckets)


def test_smallest_bucket_keeps_every_stack_on_its_side_of_every_threshold():
    T = 16
    # BAT / P2B: at least 64 rows per target in every stack
    assert smallest_bucket(32, {(64 * 32, T), (128 * 32, T), (1024 * 32, T)}) == 1
    # one row per target (M2-Track's heads): with K >= 16 the smallest bucket is 16
    assert smallest_bucket(32, {(32, T), (512 * 32, T)}) == 16
    assert smallest_bucket(16, {(16, T), (512 * 16, T)}) == 16
    assert occupancy_buckets(128, smallest_bucket(128, {(128, T), (512 * 128, T)})) == (16, 32, 64, 128)
    # every stack below the threshold at K stays below it at every smaller size: all buckets
    assert smallest_bucket(4, {(4, T), (4 * 512, T)}) == 1
    # a stack at 8 rows per target with K = 4 (P = 32) must keep P >= 16: bucket 2 and up
    assert smallest_bucket(4, {(4, T), (32, T), (4 * 512, T)}) == 2
    # 3 rows per target: ceil(16 / 3) = 6 targets, so the buckets start at 8
    assert occupancy_buckets(64, smallest_bucket(64, {(3 * 64, T)})) == (8, 16, 32, 64)
    # the skinny forward's threshold: 2048 rows per target at K = 4 (P = 8192 >= 4096) needs 2 targets; at K = 1 nothing
    assert smallest_bucket(4, {(8192, T), (8192, 4096), (4, T)}) == 2
    assert smallest_bucket(1, {(2048, 4096)}) == 1
    assert smallest_bucket(7, set()) == 1


def _stack(n_layers, K0, cout, S=0, lift=False):
    d = _lib.StackDesc()
    d.n_layers, d.P, d.K0, d.S = n_layers, 1000, K0, S
    for l, c in enumerate(cout):
        d.cout[l] = c
    if lift:
        d.lift = ctypes.pointer(_lib.LiftDesc())
    return d


def _thresholds(d):
    out = (ctypes.c_int * 4)()
    n = _lib.lib().o3d_stack_plan_thresholds(ctypes.byref(d), out)
    return None if n < 0 else sorted(out[:n])


def test_plan_thresholds_of_a_stack():
    """The row counts at which a stack's eval-mode plan can change, from the library (no launch)."""
    assert _thresholds(_stack(3, 64, [64, 128, 256])) == [16]                       # the tensor-core test only
    assert _thresholds(_stack(2, 8, [64, 64])) == [16, 4096]                        # an xyz-sized first layer: skinny forward
    assert _thresholds(_stack(1, 4, [64], S=32)) == [16]                            # ... unless it is the pooled last layer
    assert _thresholds(_stack(2, 4, [64, 64], S=32)) == [16, 4096]
    assert _thresholds(_stack(3, 64, [64, 8, 32])) == [16, 4096]                    # a layer after one 8 channels wide
    assert _thresholds(_stack(2, 12, [64, 64])) == [16]
    assert _thresholds(_stack(2, 0, [64, 128], lift=True)) == [16, 128]              # a lifted stack's virtual first layer
    assert _thresholds(_stack(0, 8, [])) is None


def test_work_list_slot_order_padding_and_held_feeds():
    slot_feed = {5: 0, 1: 2, 3: 0, 0: 1}
    assert work_slots(slot_feed, {0, 1, 2}) == [0, 1, 3, 5]
    assert work_slots(slot_feed, {0}) == [3, 5]                            # feeds 1 and 2 hold this advance
    assert work_slots(slot_feed, {2, 7}) == [1]
    assert work_slots(slot_feed, set()) == []                              # n = 0
    assert work_slots({}, {0}) == []
    rows = work_rows([3, 5], 6)
    assert rows.dtype == np.int64 and rows.shape == (2, 6)
    assert rows[0].tolist() == [3, 5, 6, 6, 6, 6]                          # padding reads the idle row K
    assert rows[1].tolist() == [3, 5, 7, 7, 7, 7]                          # and writes row K + 1
    assert work_rows([], 2).tolist() == [[2, 2], [3, 3]]
    assert work_rows([0, 1], 2).tolist() == [[0, 1], [0, 1]]


def test_tracker_work_list_follows_add_and_drop():
    box = dc.Box(np.zeros(3), np.array([1.5, 4.0, 1.5]), np.eye(3))
    trk = MultiTargetTracker(_Echo(_cfg()), 100, 6, use_graph=False, feeds=3)
    trk.feed_seen[:] = [1, 1, 1]                                           # as after an advance with a scan of every feed
    for tid, f in ((10, 2), (11, 0), (12, 1), (13, 0)):
        trk.add(tid, box, feed=f)
    assert trk.targets() == {10: 0, 11: 1, 12: 2, 13: 3}
    assert work_slots(trk._feed_of, {0}) == [1, 3]
    trk.drop(11)
    trk.drop(10)
    assert work_slots(trk._feed_of, {0, 1, 2}) == [2, 3]                  # only high slots left: no slot moves
    trk.add(14, box, feed=2)                                               # the lowest free slot
    assert trk.targets() == {12: 2, 13: 3, 14: 0}
    assert work_slots(trk._feed_of, {0, 2}) == [0, 3]
    # the public slot state keeps its K rows; the idle row K still holds the dummy box
    assert trk.box_c.shape == (6, 3) and trk.box_r.shape == (6, 3, 3) and trk.t.shape == (6,) and trk.active.shape == (6,)
    assert trk.snapshot().shape == (6, 15)
    assert not bool(trk._active[6]) and torch.equal(trk._box_r[6], torch.eye(3)) and (trk._box_s[6] == 1).all()
