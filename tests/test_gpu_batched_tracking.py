"""Split evaluation with many tracklets in flight, on the GPU: the keyed draws against their numpy restatement, the on-device
overlap / distance against utils/metrics.py, one slot of the batched step against the B=1 DeviceTracker, and
`evaluate_batched` across slot counts, runs, graph / eager and against the host metric classes."""
import os

import numpy as np
import pytest
import torch

from _philox import keyed_uniform
from open3dsot_b200 import ops
from open3dsot_b200.config import load_config
from open3dsot_b200.datasets.data_classes import Box
from open3dsot_b200.datasets.synthetic import synthetic_sequence
from open3dsot_b200.models import get_model
from open3dsot_b200.tracking.batched_tracker import BatchedDeviceTracker
from open3dsot_b200.tracking.device_tracker import DeviceTracker
from open3dsot_b200.tracking.evaluate import evaluate_batched
from open3dsot_b200.utils.metrics import Precision, Success, estimateAccuracy, estimateOverlap

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _model(cfg_name, **over):
    cfg = load_config(os.path.join(ROOT, "cfgs", cfg_name), {"up_axis": [0, 0, 1], **over})   # the synthetic tracklets are z-up
    torch.manual_seed(0)
    return cfg, get_model(cfg.net_model)(cfg).cuda().eval()


def _tracklets(lengths, n_points=4000, seed=100):
    return [synthetic_sequence(n_frames=n, n_points=n_points, seed=seed + i, speed=0.4 + 0.05 * i, yaw_rate=1.0 + i)
            for i, n in enumerate(lengths)]


def test_keyed_uniform_matches_restatement_and_ignores_slot_and_k():
    seed, n = 20261016, 1030                                                   # n % 4 != 0: a partial last block
    ids, frames = [7, 0, 123456, 3], [1, 5, 2, 40]
    dev = "cuda"
    for stream in (0, 4):
        out = ops.keyed_uniform(torch.tensor(ids, device=dev), torch.tensor(frames, device=dev), seed, stream, n).cpu().numpy()
        for k, (t, f) in enumerate(zip(ids, frames)):
            assert np.array_equal(out[k], keyed_uniform(seed, t, f, stream, n)), (stream, k)
    # the same (tracklet, frame) in another slot and beside another number of slots
    a = ops.keyed_uniform(torch.tensor([7], device=dev), torch.tensor([1], device=dev), seed, 2, n)
    b = ops.keyed_uniform(torch.tensor([9, 11, 7, 2, 5], device=dev), torch.tensor([3, 1, 1, 8, 1], device=dev), seed, 2, n)
    assert torch.equal(a[0], b[2])


def _rot_up(yaw, y_up):
    c, s = np.cos(yaw), np.sin(yaw)
    if not y_up:
        return np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])
    roty = np.array([[c, 0.0, s], [0.0, 1.0, 0.0], [-s, 0.0, c]])
    rotx = np.array([[1.0, 0.0, 0.0], [0.0, 0.0, 1.0], [0.0, -1.0, 0.0]])     # box height (local z) along world -y: KITTI camera frame
    return roty @ rotx


def _pairs(y_up, rng):
    """(gt fp64, result fp32) box pairs: random, disjoint, nested, identical, edge-touching."""
    pairs = []
    up = 1 if y_up else 2
    for _ in range(40):
        c = rng.normal(0, 3, 3)
        wlh = rng.uniform(0.5, 4.5, 3)
        gt = Box(c, wlh, _rot_up(rng.uniform(-np.pi, np.pi), y_up))
        d = rng.normal(0, 0.8, 3)
        res = (c + d, wlh * rng.uniform(0.8, 1.2, 3), _rot_up(rng.uniform(-np.pi, np.pi), y_up))
        pairs.append((gt, res))
    g = Box(np.zeros(3), np.array([2.0, 4.0, 1.5]), _rot_up(0.3, y_up))
    far = np.zeros(3); far[0] = 50.0
    pairs.append((g, (far, g.wlh, g.rotation_matrix)))                                        # disjoint
    pairs.append((g, (np.zeros(3), g.wlh * 0.5, g.rotation_matrix)))                          # nested
    exact = Box(np.array([1.5, -2.25, 0.75]), np.array([1.5, 3.75, 1.5]), np.eye(3) if not y_up else _rot_up(0.0, True))
    pairs.append((exact, (exact.center, exact.wlh, exact.rotation_matrix)))                   # identical, fp32-exact
    side = exact.center.copy(); side[0] += exact.wlh[1]
    pairs.append((exact, (side, exact.wlh, exact.rotation_matrix)))                           # sharing an edge
    shift = exact.center.copy(); shift[up] += 0.5
    pairs.append((exact, (shift, exact.wlh, exact.rotation_matrix)))                          # same footprint, shifted up
    return pairs


@pytest.mark.parametrize("y_up", [False, True])
@pytest.mark.parametrize("dim", [2, 3])
def test_track_metrics_match_host_functions(y_up, dim):
    rng = np.random.default_rng(3 + 2 * dim + int(y_up))
    up_axis = [0, -1, 0] if y_up else [0, 0, 1]
    pairs = _pairs(y_up, rng)
    K = len(pairs)
    f32 = lambda i: torch.tensor(np.stack([p[1][i] for p in pairs]), dtype=torch.float32, device="cuda").contiguous()
    center, wlh, rot = f32(0), f32(1), f32(2)
    f64 = lambda a: torch.tensor(np.stack(a), dtype=torch.float64, device="cuda").contiguous()
    gt_c, gt_s, gt_r = f64([p[0].center for p in pairs]), f64([p[0].wlh for p in pairs]), f64([p[0].rotation_matrix for p in pairs])
    frame = torch.arange(K, device="cuda").flip(0).contiguous()                # slot k scores pool frame K-1-k
    gt_c, gt_s, gt_r = gt_c.flip(0).contiguous(), gt_s.flip(0).contiguous(), gt_r.flip(0).contiguous()
    frame[1] = -1                                                              # an idle slot writes nothing
    ov = torch.full((K,), -7.0, dtype=torch.float64, device="cuda")
    di = torch.full((K,), -7.0, dtype=torch.float64, device="cuda")
    ops.track_metrics(center, rot, wlh, gt_c, gt_r, gt_s, frame, dim, up_axis, ov, di)
    ov, di = ov.cpu().numpy(), di.cpu().numpy()
    for k, (gt, _) in enumerate(pairs):
        f = K - 1 - k
        if k == 1:
            assert ov[f] == -7.0 and di[f] == -7.0
            continue
        res = Box(center[k].cpu().double().numpy(), wlh[k].cpu().double().numpy(), rot[k].cpu().double().numpy())
        want_o = estimateOverlap(gt, res, dim=dim, up_axis=up_axis)
        want_d = estimateAccuracy(gt, res, dim=dim, up_axis=up_axis)
        assert abs(ov[f] - want_o) < 1e-12, (k, ov[f], want_o)
        assert abs(di[f] - want_d) < 1e-12, (k, di[f], want_d)
    # the five special pairs land at frames 4 (disjoint) .. 0 (shifted up)
    assert ov[4] == 0.0 and abs(ov[2] - 1.0) < 1e-12 and abs(ov[1]) < 1e-12 and di[2] == 0.0


@pytest.mark.parametrize("cfg_name", ["BAT_Car.yaml", "P2B_Car.yaml", "M2_track_kitti.yaml"])
def test_slot_matches_device_tracker(cfg_name):
    """Slot k of the batched step against the B=1 DeviceTracker fed slot k's keyed draws, eager, limit_box off, 6 frames."""
    cfg, net = _model(cfg_name, limit_box=False)
    n_points, seed = 6000, 11
    tracks = _tracklets([7, 7, 7], n_points=n_points, seed=300)
    trk = BatchedDeviceTracker(net, tracks, slots=3, seed=seed, ids=[4, 9, 2], max_points=n_points, use_graph=False)
    _, _, cen, rot = trk.run()
    offsets = trk.plan["offsets"]
    for j, seq in enumerate(tracks):
        tid = trk.ids[j]
        one = DeviceTracker(net, max_points=n_points, use_graph=False)
        pts = [torch.tensor(f["pc"].points.T.copy(), device="cuda") for f in seq]
        one.reset(pts[0], seq[0]["3d_bbox"].to_tensor("cuda"))
        for i in range(1, 7):
            one._load_scan(pts[i])
            draws = [ops.keyed_uniform(torch.tensor([tid], device="cuda"), torch.tensor([i], device="cuda"), seed, s, u.shape[0])[0]
                     for s, u in enumerate(one.u_s + one.u_t)]
            for u, d in zip(one.u_s + one.u_t, draws):
                u.copy_(d)
            one._frame()
            o = int(offsets[j]) + i
            dc = float((one.box_c.double().cpu() - torch.from_numpy(cen[o])).abs().max())
            dr = float((one.box_r.double().cpu() - torch.from_numpy(rot[o])).abs().max())
            assert dc < 1e-4 and dr < 1e-5, (cfg_name, j, i, dc, dr)


_LENGTHS = [12, 1, 5, 9, 3, 12, 2, 7, 1, 10]


def _boxes(res):
    return np.array([np.concatenate([b.center, b.rotation_matrix.ravel()]) for seq in res["results"] for b in seq])


@pytest.fixture(scope="module")
def limited():
    """P2B-Car (limit_box on in its config) and BAT-Car with limit_box switched on, over ~10 tracklets of 1-12 frames."""
    tracks = _tracklets(_LENGTHS, n_points=4000, seed=500)
    out = {}
    for name, over in (("P2B_Car.yaml", {}), ("BAT_Car.yaml", {"limit_box": True})):
        cfg, net = _model(name, **over)
        assert cfg.limit_box
        out[name] = (net, {s: evaluate_batched(net, tracks, slots=s, seed=5) for s in (1, 3, 8)})
    return tracks, out


@pytest.mark.parametrize("name", ["P2B_Car.yaml", "BAT_Car.yaml"])
def test_results_agree_across_slot_counts(limited, name):
    tracks, out = limited
    runs = out[name][1]
    for s in (1, 3, 8):
        r = runs[s]
        assert r["frames"] == sum(_LENGTHS) and [len(x) for x in r["results"]] == _LENGTHS
        assert [len(x) for x in r["overlaps"]] == _LENGTHS and [len(x) for x in r["distances"]] == _LENGTHS
    ref = _boxes(runs[1])
    for s in (3, 8):
        assert float(np.abs(_boxes(runs[s]) - ref).max()) < 1e-4, s


@pytest.mark.parametrize("name", ["P2B_Car.yaml", "BAT_Car.yaml"])
def test_same_slots_runs_are_bitwise_identical(limited, name):
    tracks, out = limited
    net, runs = out[name]
    again = evaluate_batched(net, tracks, slots=3, seed=5)
    assert np.array_equal(_boxes(again), _boxes(runs[3]))
    assert again["overlaps"] == runs[3]["overlaps"] and again["distances"] == runs[3]["distances"]


def test_graph_replay_equals_eager_step(limited):
    tracks, out = limited
    net, runs = out["P2B_Car.yaml"]
    eager = evaluate_batched(net, tracks, slots=3, seed=5, use_graph=False)
    assert float(np.abs(_boxes(eager) - _boxes(runs[3])).max()) < 1e-5
    assert float(np.abs(np.concatenate(eager["overlaps"]) - np.concatenate(runs[3]["overlaps"])).max()) < 1e-5


@pytest.mark.parametrize("name", ["P2B_Car.yaml", "BAT_Car.yaml"])
def test_success_precision_match_host_classes(limited, name):
    tracks, out = limited
    net, runs = out[name]
    cfg = net.config
    for s in (1, 8):
        r = runs[s]
        succ, prec = Success(), Precision()
        for seq, boxes, ov, di in zip(tracks, r["results"], r["overlaps"], r["distances"]):
            host_o = [estimateOverlap(f["3d_bbox"], b, dim=cfg.IoU_space, up_axis=cfg.up_axis) for f, b in zip(seq, boxes)]
            host_d = [estimateAccuracy(f["3d_bbox"], b, dim=cfg.IoU_space, up_axis=cfg.up_axis) for f, b in zip(seq, boxes)]
            assert np.abs(np.array(ov) - host_o).max() < 1e-12 and np.abs(np.array(di) - host_d).max() < 1e-12
            succ(host_o)
            prec(host_d)
        assert abs(r["success"] - succ.compute()) < 1e-9 and abs(r["precision"] - prec.compute()) < 1e-9


def test_multiple_chunks_equal_one_chunk(limited):
    """A budget that splits the split into several chunks gives the per-tracklet results of a single chunk."""
    tracks, out = limited
    net, runs = out["P2B_Car.yaml"]
    from open3dsot_b200.tracking.batched_tracker import pool_frame_bytes
    small = evaluate_batched(net, tracks, slots=3, seed=5, max_resident_bytes=15 * pool_frame_bytes(4000))
    assert float(np.abs(_boxes(small) - _boxes(runs[3])).max()) < 1e-4
