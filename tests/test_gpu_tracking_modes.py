"""shape_aggregation 'all' and reference_BB 'previous_gt' / 'current_gt' on the GPU: the history append kernel against the
box-frame crop kernel and the tensor formulation, one slot of the batched step against the B=1 DeviceTracker, and
`evaluate_batched` / the trackers across slot counts, graph / eager and history capacities."""
import numpy as np
import pytest
import torch

from open3dsot_b200 import ops
from open3dsot_b200.tracking import boxes as bx
from open3dsot_b200.tracking.batched_tracker import BatchedDeviceTracker
from open3dsot_b200.tracking.device_tracker import DeviceTracker
from open3dsot_b200.tracking.evaluate import evaluate_batched
from test_gpu_batched_tracking import _boxes, _model, _tracklets

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("H", [100000, 700])
def test_crop_append_kernel_matches_crop_kernel_and_tensor_formulation(H):
    """Three appends over random scans (5000 points: a partial second tile), with an empty scan, partial counts, an idle slot;
    H = 700 overflows."""
    g = torch.Generator().manual_seed(H)
    F, N, B, scale, offset = 6, 5000, 5, 1.25, 0.2
    scans = (torch.randn(F, N, 3, generator=g) * 2.5).cuda()
    count = torch.tensor([5000, 0, 4097, 1234, 5000, 3], device="cuda")
    hist = torch.full((B, H, 3), -9.0, device="cuda")
    keep = torch.zeros(B, H, dtype=torch.bool, device="cuda")
    cnt = torch.zeros(B, dtype=torch.int64, device="cuda")
    ref_h, ref_k, ref_c = hist.cpu().double(), keep.cpu(), cnt.cpu()
    want = [[] for _ in range(B)]
    for step in ([0, 2, -1, 4, 1], [3, 5, -1, 0, 2], [4, 0, -1, 2, 2]):
        yaw = torch.rand(B, generator=g) * 6.28
        c, s, z, o = torch.cos(yaw), torch.sin(yaw), torch.zeros(B), torch.ones(B)
        rot = torch.stack([torch.stack([c, -s, z], -1), torch.stack([s, c, z], -1), torch.stack([z, z, o], -1)], -2)
        box = bx.Box(torch.randn(B, 3, generator=g) * 0.5, torch.rand(B, 3, generator=g) * 3 + 1.5, rot)
        frame = torch.tensor(step)
        bx.crop_append(scans, box.to("cuda"), scale, offset, frame.cuda(), count, hist, keep, cnt)
        bx.crop_append(scans.cpu().double(), bx.Box(*(t.double() for t in box)), scale, offset, frame, count.cpu(), ref_h, ref_k,
                       ref_c)
        # the crop kernel on the same boxes: the appended points are its kept local coordinates, bit for bit
        local, kk = bx.crop_in_box_frame(scans, box.to("cuda"), scale, offset, frame.clamp(min=0).cuda(), count)
        for b, f in enumerate(step):
            if f >= 0:
                want[b].append(local[b][kk[b]])
    cnt_h, ref_cn = cnt.cpu(), ref_c
    assert not bool(keep[2].any()) and int(cnt_h[2]) == 0                     # the idle slot is untouched
    for b in range(B):
        w = torch.cat(want[b]) if want[b] else torch.zeros(0, 3, device="cuda")
        n = int(cnt_h[b])
        assert n == w.shape[0], b                                               # the true count, also past H
        m = min(n, H)
        assert torch.equal(hist[b, :m], w[:m]) and bool(keep[b, :m].all()) and not bool(keep[b, m:].any())
        assert bool((hist[b, m:] == -9.0).all())                               # nothing written past the kept points / H
        # against the fp64 tensor formulation: equal up to points within rounding of the box boundary
        assert abs(n - int(ref_cn[b])) <= 2, (b, n, int(ref_cn[b]))
        if n == int(ref_cn[b]) and m:
            assert float((hist[b, :m].cpu().double() - ref_h[b, :m]).abs().max()) < 1e-5
    if H < 1000:
        assert int(cnt_h.max()) > H                                            # the small history did overflow


def _ref_box(trk_mode, seq, i):
    return seq[i - 1 if trk_mode == "previous_gt" else i]["3d_bbox"].to_tensor("cuda")


@pytest.mark.parametrize("cfg_name", ["BAT_Car.yaml", "P2B_Car.yaml"])
@pytest.mark.parametrize("mode", ["all", "previous_gt", "current_gt"])
def test_slot_matches_device_tracker(cfg_name, mode):
    """Slot k of the batched step against the B=1 DeviceTracker fed slot k's keyed draws, eager, limit_box off, 6 frames."""
    over = {"shape_aggregation": "all"} if mode == "all" else {"reference_BB": mode}
    cfg, net = _model(cfg_name, limit_box=False, **over)
    n_points, seed = 6000, 11
    tracks = _tracklets([7, 7, 7], n_points=n_points, seed=300)
    trk = BatchedDeviceTracker(net, tracks, slots=3, seed=seed, ids=[4, 9, 2], max_points=n_points, use_graph=False)
    _, _, cen, rot = trk.run()
    offsets = trk.plan["offsets"]
    for j, seq in enumerate(tracks):
        tid = trk.ids[j]
        one = DeviceTracker(net, max_points=n_points, use_graph=False, history=1 << 16)
        assert one.mode == ("all" if mode == "all" else "firstandprevious") and one.ref_mode == trk.ref_mode
        pts = [torch.tensor(f["pc"].points.T.copy(), device="cuda") for f in seq]
        one.reset(pts[0], seq[0]["3d_bbox"].to_tensor("cuda"))
        for i in range(1, 7):
            one._load_scan(pts[i])
            if mode != "all":
                one._set_ref(_ref_box(mode, seq, i))
            draws = [ops.keyed_uniform(torch.tensor([tid], device="cuda"), torch.tensor([i], device="cuda"), seed, s, u.shape[0])[0]
                     for s, u in enumerate(one.u_s + one.u_t)]
            for u, d in zip(one.u_s + one.u_t, draws):
                u.copy_(d)
            one._frame()
            o = int(offsets[j]) + i
            dc = float((one.box_c.double().cpu() - torch.from_numpy(cen[o])).abs().max())
            dr = float((one.box_r.double().cpu() - torch.from_numpy(rot[o])).abs().max())
            assert dc < 1e-4 and dr < 1e-5, (cfg_name, mode, j, i, dc, dr)
        if mode == "all":
            assert 0 < int(one.hist_count[0]) <= int(trk.hist_peak.max()) <= trk.H


_LENGTHS = [12, 1, 5, 9, 3, 12, 2, 7, 1, 10]


@pytest.fixture(scope="module")
def all_mode():
    tracks = _tracklets(_LENGTHS, n_points=4000, seed=500)
    cfg, net = _model("P2B_Car.yaml", shape_aggregation="all")
    return tracks, net, {s: evaluate_batched(net, tracks, slots=s, seed=5) for s in (1, 3, 8)}


def test_all_mode_agrees_across_slot_counts(all_mode):
    tracks, net, runs = all_mode
    for s in (1, 3, 8):
        assert [len(x) for x in runs[s]["results"]] == _LENGTHS and [len(x) for x in runs[s]["overlaps"]] == _LENGTHS
    ref = _boxes(runs[1])
    for s in (3, 8):
        assert float(np.abs(_boxes(runs[s]) - ref).max()) < 1e-4, s


def test_all_mode_graph_replay_equals_eager_step(all_mode):
    tracks, net, runs = all_mode
    eager = evaluate_batched(net, tracks, slots=3, seed=5, use_graph=False)
    assert float(np.abs(_boxes(eager) - _boxes(runs[3])).max()) < 1e-5
    assert float(np.abs(np.concatenate(eager["overlaps"]) - np.concatenate(runs[3]["overlaps"])).max()) < 1e-5


def test_all_mode_small_history_runs_the_chunk_again_bitwise(all_mode):
    """A starting capacity far below one tracklet's history forces run() to raise it and track the chunk again; the result is
    bitwise that of a capacity that never overflows."""
    tracks, net, _ = all_mode
    big = BatchedDeviceTracker(net, tracks, slots=3, seed=5, history=1 << 16)
    want = big.run()
    small = BatchedDeviceTracker(net, tracks, slots=3, seed=5, history=256)
    got = small.run()
    assert big.H == 1 << 16 and small.H > 256 and int(small.hist_peak.max()) <= small.H
    for a, b in zip(got, want):
        assert np.array_equal(a, b)


@pytest.mark.parametrize("cfg_name", ["BAT_Car.yaml", "P2B_Car.yaml"])
def test_device_tracker_history_growth_is_bitwise(cfg_name):
    """The graph-captured B=1 tracker in 'all' mode: starting from 512 points, the history grows (copied, graph captured
    again) several times over a 12-frame tracklet and two resets, and every box equals a tracker that never grows.
    limit_box is off: its replacement draw comes from torch's global generator, which the two trackers share."""
    cfg, net = _model(cfg_name, shape_aggregation="all", limit_box=False)
    tracks = _tracklets([12, 9], n_points=5000, seed=700)
    small = DeviceTracker(net, max_points=5000, seed=3, history=512)
    big = DeviceTracker(net, max_points=5000, seed=3, history=1 << 16)
    for seq in tracks:
        pts = [torch.tensor(f["pc"].points.T.copy(), device="cuda") for f in seq]
        for trk in (small, big):
            trk.reset(pts[0], seq[0]["3d_bbox"].to_tensor("cuda"))
        for i in range(1, len(seq)):
            a, b = small.step(pts[i]), big.step(pts[i])
            assert torch.equal(a.center, b.center) and torch.equal(a.rot, b.rot), (i, small.H)
        assert int(small.hist_count[0]) == int(big.hist_count[0]) <= small.H
    assert small.H > 2048 and big.H == 1 << 16
