"""Live multi-target tracking on the GPU: `o3d_crop_resample` bitwise against crop_box_frame -> keyed_uniform -> resample, a slot
against the B=1 DeviceTracker, the stream against BatchedDeviceTracker on the same scans, independence from the other targets
and from max_targets, reproducibility, graph replay against the eager step, no host sync, the kernel that runs, and the
command line against evaluate_batched."""
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from open3dsot_b200 import ops, track
from open3dsot_b200.config import load_config
from open3dsot_b200.datasets.data_classes import Box, PointCloud
from open3dsot_b200.datasets.kitti import kittiDataset
from open3dsot_b200.datasets.synthetic import synthetic_scene, synthetic_sequence
from open3dsot_b200.models import get_model
from open3dsot_b200.tracking.batched_tracker import BatchedDeviceTracker
from open3dsot_b200.tracking.device_tracker import DeviceTracker
from open3dsot_b200.tracking.evaluate import evaluate_batched
from open3dsot_b200.tracking.multi_tracker import MultiTargetTracker, track_stream
from test_kitti_reader import _write_scene

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODELS = ["BAT_Car.yaml", "P2B_Car.yaml", "M2_track_kitti.yaml"]


def _model(cfg_name, **over):
    cfg = load_config(os.path.join(ROOT, "cfgs", cfg_name), {"up_axis": [0, 0, 1], **over})   # the synthetic scenes are z-up
    torch.manual_seed(0)
    return cfg, get_model(cfg.net_model)(cfg).cuda().eval()


# ------------------------------------------------------------------ the kernel
def _rotz(yaw):
    c, s = np.cos(yaw), np.sin(yaw)
    return np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])


def _unfused(scans, count, frame, center, rot, half, size, seed, key, kf, perm, pick, prefix=None, pkeep=None):
    local, keep = ops.crop_box_frame(scans, center, rot, half, frame, count)
    if prefix is not None:
        local, keep = torch.cat([prefix, local], 1), torch.cat([pkeep, keep], 1)
    u_perm = ops.keyed_uniform(key, kf, seed, perm, local.shape[1])
    u_pick = ops.keyed_uniform(key, kf, seed, pick, size)
    out, _, n = ops.resample(local.contiguous(), keep.contiguous(), size, u_perm, u_pick)
    return out, n


def _check(scans, count, frame, center, rot, half, size, key, kf, prefix=None, pkeep=None, seed=20261017, perm=2, pick=3):
    got, n = ops.crop_resample(scans, count, frame, center, rot, half, size, seed, key, kf, perm, pick, prefix, pkeep)
    want, wn = _unfused(scans, count, frame, center, rot, half, size, seed, key, kf, perm, pick, prefix, pkeep)
    assert torch.equal(n, wn), (n.tolist(), wn.tolist())
    assert torch.equal(got, want), float((got - want).abs().max())
    return n.cpu().numpy()


def _inputs(K, S, N, seed, halves):
    g = torch.Generator().manual_seed(seed)
    scans = (torch.rand(S, N, 3, generator=g) * 20 - 10).cuda()
    count = torch.tensor([N, N - N // 5][:S], device="cuda")                  # the second scan: count < N
    frame = torch.tensor([k % S for k in range(K)], device="cuda")
    center = (torch.rand(K, 3, generator=g) * 4 - 2).cuda()
    rot = torch.tensor(np.stack([_rotz(y) for y in np.random.default_rng(seed).uniform(-np.pi, np.pi, K)]), dtype=torch.float32,
                       device="cuda")
    half = torch.tensor([[h, h * 1.3, h * 0.8] for h in (halves[k % len(halves)] for k in range(K))], dtype=torch.float32,
                        device="cuda")
    key = torch.randint(0, 1 << 20, (K,), generator=g).cuda()
    kf = torch.randint(0, 400, (K,), generator=g).cuda()
    return scans, count, frame, center, rot, half, key, kf


# box sizes from empty (n = 0) through a few points, 2 < n < size and n >= size to the whole cube (every point kept)
HALVES = [0.0, 0.35, 1.0, 3.0, 5.0, 7.0, 40.0]


@pytest.mark.parametrize("K", [1, 7, 64])
@pytest.mark.parametrize("size", [512, 1024, 2048])
@pytest.mark.parametrize("prefix", [False, True])
@pytest.mark.parametrize("scans", [1, 2])
def test_crop_resample_is_bitwise_the_three_kernel_path(K, size, prefix, scans):
    N = 6000
    halves = HALVES if K > 1 else [5.0]
    s, count, frame, center, rot, half, key, kf = _inputs(K, scans, N, 7 * K + size + scans, halves)
    pre = pk = None
    if prefix:
        g = torch.Generator().manual_seed(K + size)
        pre = (torch.rand(K, N, 3, generator=g) * 2 - 1).cuda()
        pk = (torch.rand(K, N, generator=g) < 0.05).cuda()
    n = _check(s, count, frame, center, rot, half, size, key, kf, pre, pk)
    if K == 64 and not prefix:
        assert (n == 0).any() and (n >= size).any() and ((n > 2) & (n < size)).any() and (n == count.cpu().numpy()[frame.cpu()]).any()


def test_crop_resample_edge_cases():
    """n >= size, 2 < n < size, n <= 2 (1 and 2 points), n = 0, count < N, a box that keeps every point; the prefix-only form."""
    N, size = 3000, 512
    g = torch.Generator().manual_seed(5)
    scan = (torch.rand(2, N, 3, generator=g) * 10 - 5).cuda()
    scan[0, 10] = torch.tensor([20.0, 20.0, 20.0])                             # isolated points, for n = 1 and n = 2
    scan[0, 11] = torch.tensor([20.1, 20.0, 20.0])
    count = torch.tensor([N, 1700], device="cuda")
    cases = [((0, 0, 0), 4.0, 0), ((0, 0, 0), 1.5, 0), ((20, 20, 20), 0.05, 0), ((20.05, 20, 20), 0.2, 0),
             ((0, 0, 0), 0.0, 0), ((0, 0, 0), 50.0, 1), ((0, 0, 0), 50.0, 0), ((100, 0, 0), 1.0, 1)]
    K = len(cases)
    center = torch.tensor([c for c, _, _ in cases], dtype=torch.float32, device="cuda")
    half = torch.tensor([[h] * 3 for _, h, _ in cases], dtype=torch.float32, device="cuda")
    frame = torch.tensor([f for _, _, f in cases], device="cuda")
    rot = torch.eye(3, device="cuda").repeat(K, 1, 1)
    key, kf = torch.arange(K, device="cuda") * 3 + 1, torch.arange(K, device="cuda") + 1
    n = _check(scan, count, frame, center, rot, half, size, key, kf)
    assert n[0] >= size and 2 < n[1] < size and n[2] == 1 and n[3] == 2 and n[4] == 0 and n[5] == 1700 and n[6] == N and n[7] == 0
    # prefix only (N = 0): the resampling of the prefix alone, with the same draws
    pre = (torch.rand(K, 900, 3, generator=g)).cuda()
    pk = (torch.rand(K, 900, generator=g) < torch.linspace(0, 1, K)[:, None]).cuda()
    got, gn = ops.crop_resample(scan[:, :0], count, frame, center, rot, half, size, 9, key, kf, 0, 1, pre, pk)
    want, _, wn = ops.resample(pre, pk, size, ops.keyed_uniform(key, kf, 9, 0, 900), ops.keyed_uniform(key, kf, 9, 1, size))
    assert torch.equal(gn, wn) and torch.equal(got, want)


# ------------------------------------------------------------------ a slot against the B=1 tracker
@pytest.mark.parametrize("cfg_name", MODELS)
def test_slot_matches_device_tracker(cfg_name):
    """Target j of the stream against the B=1 DeviceTracker fed target j's keyed draws, eager, limit_box off, 6 frames."""
    cfg, net = _model(cfg_name, limit_box=False)
    n_points, seed, ids = 6000, 11, [4, 9, 2]
    scene = synthetic_scene(n_frames=7, n_points=n_points, n_objects=3, seed=300, extent=12.0)
    pts = [torch.tensor(s, device="cuda") for s in scene["scans"]]
    trk = MultiTargetTracker(net, n_points, max_targets=4, seed=seed, use_graph=False)
    trk.step(pts[0])
    for j, tid in enumerate(ids):
        trk.add(tid, scene["boxes"][j][0])
    states = []
    for i in range(1, 7):
        trk.step(pts[i])
        states.append((trk.box_c.clone(), trk.box_r.clone()))
    for j, tid in enumerate(ids):
        k = trk.targets()[tid]
        one = DeviceTracker(net, max_points=n_points, use_graph=False)
        one.reset(pts[0], scene["boxes"][j][0].to_tensor("cuda"))
        for i in range(1, 7):
            one._load_scan(pts[i])
            draws = [ops.keyed_uniform(torch.tensor([tid], device="cuda"), torch.tensor([i], device="cuda"), seed, s, u.shape[0])[0]
                     for s, u in enumerate(one.u_s + one.u_t)]
            for u, d in zip(one.u_s + one.u_t, draws):
                u.copy_(d)
            one._frame()
            c, r = states[i - 1]
            dc = float((one.box_c - c[k]).abs().max())
            dr = float((one.box_r - r[k]).abs().max())
            assert dc < 1e-4 and dr < 1e-5, (cfg_name, j, i, dc, dr)


# ------------------------------------------------------------------ the stream against the batched tracker
STARTS, ENDS = [0, 0, 2, 4, 5], [4, 3, 9, 8, 9]           # at most 3 targets at once; the slots of targets 0 / 1 are reused
IDS = [12, 3, 40, 7, 25]


def _scene():
    return synthetic_scene(n_frames=10, n_points=6000, n_objects=5, seed=900, extent=15.0)


def _stream(net, scene, which=range(5), max_targets=3, seed=5, use_graph=True):
    starts = {}
    for j in which:
        starts.setdefault(STARTS[j], []).append((IDS[j], scene["boxes"][j][STARTS[j]]))
    ends = {IDS[j]: ENDS[j] for j in which}
    scans = [torch.tensor(s, device="cuda") for s in scene["scans"]]
    return track_stream(net, scans, starts, ends, max_targets, seed=seed, max_points=6000, use_graph=use_graph)


def _flat(res, tid):
    return np.array([np.concatenate([b.center, b.rotation_matrix.ravel()]) for _, b in sorted(res[tid].items())])


@pytest.fixture(scope="module", params=MODELS)
def streamed(request):
    cfg, net = _model(request.param)
    scene = _scene()
    return request.param, net, scene, _stream(net, scene)


def test_stream_matches_batched_tracker(streamed):
    name, net, scene, res = streamed
    tracks = [[{"pc": PointCloud(scene["scans"][t].T.copy()), "3d_bbox": scene["boxes"][j][t]} for t in range(STARTS[j], ENDS[j] + 1)]
              for j in range(5)]
    trk = BatchedDeviceTracker(net, tracks, slots=3, seed=5, ids=IDS, max_points=6000)
    _, _, cen, rot = trk.run()
    offsets = trk.plan["offsets"]
    for j, tid in enumerate(IDS):
        assert sorted(res[tid]) == list(range(STARTS[j], ENDS[j] + 1))
        for t in range(1, ENDS[j] - STARTS[j] + 1):
            b = res[tid][STARTS[j] + t]
            o = int(offsets[j]) + t
            dc, dr = float(np.abs(b.center - cen[o]).max()), float(np.abs(b.rotation_matrix - rot[o]).max())
            assert dc < 1e-4 and dr < 1e-4, (name, tid, t, dc, dr)


def test_targets_do_not_depend_on_the_others_or_on_max_targets(streamed):
    name, net, scene, res = streamed
    alone = _stream(net, scene, which=[2, 3], max_targets=8)
    for j in (2, 3):
        tid = IDS[j]
        assert float(np.abs(_flat(alone, tid) - _flat(res, tid)).max()) < 1e-4, (name, tid)


def test_runs_are_reproducible_and_replay_equals_eager(streamed):
    name, net, scene, res = streamed
    again = _stream(net, scene)
    eager = _stream(net, scene, use_graph=False)
    for tid in IDS:
        assert np.array_equal(_flat(again, tid), _flat(res, tid)), (name, tid)
        assert np.array_equal(_flat(eager, tid), _flat(res, tid)), (name, tid)


# ------------------------------------------------------------------ no host sync, and the kernel that runs
def _norm(name):
    return re.sub(r"\s*([<>,])\s*", r"\1", name.replace("(anonymous namespace)::", ""))


def _ran(names, kernel):
    rx = re.compile(r"(?:^|[\s:])" + re.escape(kernel) + r"(?=\(|$)")
    return any(rx.search(n) for n in names)


def test_step_add_drop_do_not_sync_and_one_kernel_crops():
    cfg, net = _model("BAT_Car.yaml")
    scene = _scene()
    scans = [torch.tensor(s, device="cuda") for s in scene["scans"]]
    trk = MultiTargetTracker(net, 6000, 4, seed=2)
    trk.step(scans[0])                                                          # capture (synchronises once)
    trk.add(1, scene["boxes"][0][0])
    trk.step(scans[1])
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        trk.add(2, scene["boxes"][1][1])
        trk.step(scans[2])
        trk.drop(1)
        trk.add(3, scene["boxes"][2][2])
        out = trk.step(scans[3])
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert out["ids"].tolist() == [3, 2, -1, -1]

    names = {_norm(n) for n in json.loads(_profile_one_replay())}
    assert _ran(names, "crop_resample_kernel"), sorted(names)
    assert not _ran(names, "crop_box_frame_kernel") and not _ran(names, "resample_kernel"), sorted(names)


# One replay of a running tracker's step under torch.profiler, in a child process: a CUPTI session around a graph replay in the
# suite's process leaves later sessions (the kernel-path tests of other files) with missing kernel records.
_PROFILE_CHILD = r"""
import json, os, sys
import torch
sys.path.insert(0, sys.argv[1])
from open3dsot_b200.config import load_config
from open3dsot_b200.datasets.synthetic import synthetic_scene
from open3dsot_b200.models import get_model
from open3dsot_b200.tracking.multi_tracker import MultiTargetTracker
cfg = load_config(os.path.join(sys.argv[1], "cfgs", "BAT_Car.yaml"), {"up_axis": [0, 0, 1]})
torch.manual_seed(0)
net = get_model(cfg.net_model)(cfg).cuda().eval()
scene = synthetic_scene(n_frames=4, n_points=6000, n_objects=2, seed=900, extent=15.0)
scans = [torch.tensor(s, device="cuda") for s in scene["scans"]]
trk = MultiTargetTracker(net, 6000, 4, seed=2)
trk.step(scans[0])
trk.add(1, scene["boxes"][0][0])
trk.step(scans[1])
torch.cuda.synchronize()
def profiled(i):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        trk.step(scans[i])
        torch.cuda.synchronize()
    return sorted({e.name for e in prof.events()})
names = profiled(2)
if not any("kernel" in n for n in names):
    names = profiled(3)   # CUPTI now and then delivers no records for a short session: observe one more replay
print(json.dumps(names))
"""


def _profile_one_replay():
    r = subprocess.run([sys.executable, "-c", _PROFILE_CHILD, ROOT], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    return r.stdout.strip().splitlines()[-1]


# ------------------------------------------------------------------ the command line
def test_command_line_matches_evaluate_batched(tmp_path, capsys):
    root = str(tmp_path / "kitti")
    seqs = [synthetic_sequence(n_frames=n, n_points=1500, seed=40 + i, n_object=300, speed=0.3 + 0.1 * i, yaw_rate=1.0 + i)
            for i, n in enumerate([6, 4, 5, 3])]
    for s in (seqs[1], seqs[3]):                                # the second car of each scene drives 12 m to the left
        for f in s:
            f["pc"] = PointCloud(f["pc"].points + np.array([[0.0], [12.0], [0.0]], np.float32))
            b = f["3d_bbox"]
            f["3d_bbox"] = Box(b.center + np.array([0.0, 12.0, 0.0]), b.wlh, b.rotation_matrix)
    _write_scene(root, "0019", [((5, "Car"), seqs[0]), ((8, "Car"), seqs[1])], extra_dontcare=False)
    _write_scene(root, "0020", [((2, "Car"), seqs[2]), ((6, "Car"), seqs[3])], extra_dontcare=False)
    ds = kittiDataset(root, "test", "Car", preloading=False, preload_offset=-1)
    tracklets = ds.tracklets()
    npts = max(f["pc"].points.shape[1] for t in tracklets for f in t)
    out = str(tmp_path / "results.jsonl")
    cfg_path = os.path.join(ROOT, "cfgs", "BAT_Car.yaml")
    got = track.main(["--cfg", cfg_path, "--path", root, "--split", "test", "--out", out, "--max_targets", "3",
                      "--max_points", str(npts)])
    printed = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert printed["success"] == got["success"] and printed["precision"] == got["precision"]
    lines = [json.loads(l) for l in open(out)]
    assert [(l["scene"], l["frame"]) for l in lines] == [("0019", f) for f in range(6)] + [("0020", f) for f in range(5)]
    want_ids = {("0019", f): [5, 8] if f < 4 else [5] for f in range(6)}
    want_ids.update({("0020", f): [2, 6] if f < 3 else [2] for f in range(5)})
    for l in lines:
        assert sorted(t["id"] for t in l["targets"]) == want_ids[(l["scene"], l["frame"])]
    cfg = load_config(cfg_path)
    torch.manual_seed(0)
    net = get_model(cfg.net_model)(cfg).cuda()
    ref = evaluate_batched(net, tracklets, slots=3, seed=0)
    assert got["frames"] == ref["frames"] == 6 + 4 + 5 + 3
    assert abs(got["success"] - ref["success"]) < 1e-4 and abs(got["precision"] - ref["precision"]) < 1e-4, (got, ref)
