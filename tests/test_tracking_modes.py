"""shape_aggregation 'all' and reference_BB 'previous_gt' / 'current_gt' on the device trackers, CPU part: the history append's
tensor formulation against numpy, the B=1 tracker's history and search area against the host frame loop's crops, the chunk
plan's history bytes, and the argument checks (no GPU needed)."""
import numpy as np
import pytest
import torch

from open3dsot_b200 import _lib
from open3dsot_b200.datasets import data_classes as dc
from open3dsot_b200.datasets.synthetic import synthetic_sequence
from open3dsot_b200.tracking import boxes as bx
from open3dsot_b200.tracking import device_tracker as dtm
from open3dsot_b200.tracking.batched_tracker import BatchedDeviceTracker, history_bytes, plan_chunks
from open3dsot_b200.tracking.device_tracker import DeviceTracker
from test_tracking_host import _cfg, _Echo


def _np_crop(scan, n_valid, c, R, half):
    local = (scan[:n_valid].astype(np.float64) - c) @ R
    return local[(np.abs(local) < half).all(1)]


def _random_boxes(rng, B):
    yaw = rng.uniform(-np.pi, np.pi, B)
    rot = np.stack([[[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]] for a in yaw])
    return bx.Box(torch.tensor(rng.normal(0, 0.5, (B, 3))), torch.tensor(rng.uniform(1.0, 3.0, (B, 3))), torch.tensor(rot))


def test_crop_append_tensor_formulation_matches_numpy():
    rng = np.random.default_rng(0)
    F, N, B, H, scale, offset = 5, 400, 4, 700, 1.25, 0.1
    scans = torch.tensor(rng.normal(0, 1.5, (F, N, 3)))
    count = torch.tensor([400, 0, 250, 37, 400])                       # full, empty and partial prefixes
    hist = torch.full((B, H, 3), -9.0, dtype=torch.float64)
    keep = torch.zeros(B, H, dtype=torch.bool)
    cnt = torch.zeros(B, dtype=torch.int64)
    want = [[] for _ in range(B)]
    frames_per_step = [[0, 2, -1, 4], [1, 3, -1, 0], [4, -1, -1, 2], [2, 0, 3, 3]]   # slot 2 idle until the last step
    for step in frames_per_step:
        box = _random_boxes(rng, B)
        frame = torch.tensor(step)
        before = hist.clone(), keep.clone(), cnt.clone()
        bx.crop_append(scans, box, scale, offset, frame, count, hist, keep, cnt)
        half = (torch.stack([box.wlh[:, 1], box.wlh[:, 0], box.wlh[:, 2]], -1) * (scale / 2) + offset).numpy()
        for b, f in enumerate(step):
            if f < 0:                                                  # an idle slot is untouched
                assert torch.equal(hist[b], before[0][b]) and torch.equal(keep[b], before[1][b]) and cnt[b] == before[2][b]
                continue
            want[b].append(_np_crop(scans[f].numpy(), int(count[f]), box.center[b].numpy(), box.rot[b].numpy(), half[b]))
    for b in range(B):
        w = np.concatenate(want[b]) if want[b] else np.zeros((0, 3))
        n = int(cnt[b])
        assert n == len(w) and n <= H
        assert np.abs(hist[b, :n].numpy() - w).max(initial=0) < 1e-12         # frames in order, points in scan order
        assert bool(keep[b, :n].all()) and not bool(keep[b, n:].any()) and bool((hist[b, n:] == -9.0).all())


def test_crop_append_overflow_reports_the_true_count_and_writes_nothing_past_h():
    rng = np.random.default_rng(1)
    scans = torch.tensor(rng.uniform(-1, 1, (2, 300, 3)), dtype=torch.float32)
    box = bx.Box(torch.zeros(1, 3), torch.full((1, 3), 4.0), torch.eye(3)[None])     # every point inside
    H = 450
    base = torch.full((1, H + 50, 3), 7.0)
    hist = base[:, :H]                                                                # a view: the tail must stay 7
    keep = torch.zeros(1, H, dtype=torch.bool)
    cnt = torch.zeros(1, dtype=torch.int64)
    for f in (0, 1, 0):
        bx.crop_append(scans, box, 1.0, 0.0, torch.tensor([f]), None, hist, keep, cnt)
    assert int(cnt[0]) == 900                                                         # 3 x 300, of which 450 fit
    assert torch.equal(hist[0, :300], scans[0]) and torch.equal(hist[0, 300:], scans[1, :150]) and bool(keep.all())
    assert bool(base[0, H:].eq(7.0).all())


def _track(cfg, n_frames=6, seed=7, history=dtm.HISTORY_POINTS):
    seq = synthetic_sequence(n_frames=n_frames, n_points=3000, seed=seed)
    m = _Echo(_cfg(**cfg))
    trk = DeviceTracker(m, max_points=3000, use_graph=False, history=history)
    pts = [torch.tensor(f["pc"].points.T.copy()) for f in seq]
    return seq, m, trk, pts


def test_device_tracker_all_history_is_the_concatenation_of_past_crops():
    seq, m, trk, pts = _track({"shape_aggregation": "all"}, history=3000)
    assert trk.mode == "all"
    b = trk.reset(pts[0], seq[0]["3d_bbox"].to_tensor())
    results = [bx.Box(b.center.clone(), b.wlh.clone(), b.rot.clone())]
    cfg = m.config
    for f in range(1, len(seq)):
        b = trk.step(pts[f])
        n = int(trk.hist_count[0])
        parts = []
        for t in range(f):                                             # frames 0 .. f-1, each in its own result box
            r = results[t]
            local, keep = bx.crop_in_box_frame(pts[t][None], bx.Box(r.center[None], r.wlh[None], r.rot[None]),
                                               cfg.model_bb_scale, cfg.model_bb_offset)
            parts.append(local[0][keep[0]])
        want = torch.cat(parts)
        assert n == want.shape[0] and torch.equal(trk.hist[0, :n], want), f
        assert bool(trk.hist_keep[0, :n].all()) and not bool(trk.hist_keep[0, n:].any())
        host, _ = m.generate_template(seq, f, [dc.Box.from_tensor(r) for r in results])
        assert host.shape[0] == n, (f, host.shape[0], n)
        results.append(bx.Box(b.center.clone(), b.wlh.clone(), b.rot.clone()))
    assert trk.H > 3000                                                # five frames of ~700 points outgrew the start


@pytest.mark.parametrize("ref", ["previous_gt", "current_gt"])
def test_device_tracker_search_area_uses_the_ground_truth_box(ref, monkeypatch):
    seq, m, trk, pts = _track({"reference_BB": ref})
    seen = []
    real = dtm.resample

    def spy(points, keep, size, **kw):
        seen.append((size, points[keep].clone()))
        return real(points, keep, size, **kw)
    monkeypatch.setattr(dtm, "resample", spy)
    trk.reset(pts[0], seq[0]["3d_bbox"].to_tensor())
    results = [seq[0]["3d_bbox"]]
    for f in range(1, len(seq)):
        seen.clear()
        gt = seq[f - 1 if ref == "previous_gt" else f]["3d_bbox"]
        b = trk.step(pts[f], ref_box=gt.to_tensor())
        search = [p for size, p in seen if size == m.config.search_size]
        assert len(search) == 1
        host, ref_bb = m.generate_search_area(seq, f, results)
        assert ref_bb is gt and torch.equal(search[0], host), f
        assert torch.equal(b.wlh, gt.to_tensor().wlh)                 # the result takes the reference box's size
        results.append(dc.Box.from_tensor(b))


def test_device_tracker_ground_truth_modes_need_a_reference_box():
    seq, m, trk, pts = _track({"reference_BB": "current_gt"})
    trk.reset(pts[0], seq[0]["3d_bbox"].to_tensor())
    with pytest.raises(ValueError, match="ref_box"):
        trk.step(pts[1])


@pytest.mark.parametrize("key,value", [("shape_aggregation", "everything"), ("reference_BB", "next_gt")])
def test_unknown_modes_are_rejected_at_construction(key, value):
    m = _Echo(_cfg(**{key: value}))
    with pytest.raises(ValueError, match=key):
        DeviceTracker(m, max_points=100, use_graph=False)
    with pytest.raises(ValueError, match=key):
        BatchedDeviceTracker(m, [], slots=4)


def test_mode_strings_are_matched_like_the_host_loop():
    cfg = _cfg(shape_aggregation="FirstAndPrevious_v2", reference_BB="Previous_GT")
    assert dtm.template_mode(cfg) == "firstandprevious" and dtm.reference_mode(cfg) == "previous_gt"
    assert dtm.template_mode(_cfg(shape_aggregation="all")) == "all"
    assert dtm.template_mode(_cfg(shape_aggregation="first")) == "first"


def test_chunk_plan_counts_the_history():
    lengths = [4, 6, 3, 9, 1, 2]
    assert history_bytes(8, 1000) == 8 * 1000 * 21
    fixed = 40
    chunks = plan_chunks(lengths, 10, 140, fixed)
    assert [j for c in chunks for j in c] == list(range(len(lengths)))
    assert all(sum(lengths[j] for j in c) * 10 + fixed <= 140 for c in chunks)
    assert len(chunks) > len(plan_chunks(lengths, 10, 140))
    with pytest.raises(ValueError, match="max_resident_bytes"):
        plan_chunks([9], 10, 100, fixed_bytes=20)


def test_crop_append_argument_errors_return_status():
    L = _lib.lib()
    p = [16] * 6
    assert L.o3d_crop_append(*p, 2, 8, 4, 16, 16, None, None) < 0
    assert b"null" in L.o3d_last_error()
    assert L.o3d_crop_append(16, None, None, 16, 16, 16, 2, 8, 4, 16, 16, 16, None) < 0      # frame is required
    assert L.o3d_crop_append(*p, 70000, 8, 4, 16, 16, 16, None) < 0                        # B > 65535
    assert b"B=" in L.o3d_last_error()
    assert L.o3d_crop_append(*p, 2, 8, -1, 16, 16, 16, None) < 0                           # H < 0
    assert b"H=" in L.o3d_last_error()
    assert L.o3d_crop_append(*p, 0, 8, 4, 16, 16, 16, None) == 0                           # nothing to do: no launch
