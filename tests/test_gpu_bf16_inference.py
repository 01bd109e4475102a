"""BF16 inference precision (runtime.inference_precision_scope("bf16"), o3d_stack_t.precision = 1) on the GPU:

  - the fused SA layer and the pw_tc forward (plain and lifted loaders) against a float64 composition that rounds the weights and
    every GEMM input to bf16 at the points the kernels do (what is left is fp32 accumulation order), and against the unrounded
    float64 composition (the real precision loss);
  - whole models in eval mode, bf16 against fp32, with the discrete choices of the fp32 pass injected;
  - fp32 and bf16 blocks of the same weights side by side, fp32 results bitwise unchanged;
  - the trackers in bf16: graph replay against eager, repeat runs, a slot of the batched step against the B=1 tracker, and a live
    target against K and the other targets;
  - one profiled bf16 replay runs the bf16 kernel instantiations and no 3xTF32 forward.
Measured values are printed (pytest -s) and recorded in DESIGN.md section 8."""
import copy
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from open3dsot_b200 import fused, ops, runtime
from open3dsot_b200.config import load_config
from open3dsot_b200.datasets.synthetic import synthetic_motion_batch, synthetic_scene, synthetic_sequence, synthetic_siamese_batch
from open3dsot_b200.models import get_model
from open3dsot_b200.tracking.batched_tracker import BatchedDeviceTracker
from open3dsot_b200.tracking.device_tracker import DeviceTracker
from open3dsot_b200.tracking.evaluate import evaluate_batched
from open3dsot_b200.tracking.multi_tracker import track_stream
from _params import det_state_dict
from test_gpu_sa_fused import CASES as SA_CASES, _cloud, _module

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODELS = ["BAT_Car.yaml", "P2B_Car.yaml", "M2_track_kitti.yaml"]

EMULATED_BAR = 1e-3      # kernel vs the bf16-rounding float64 composition: fp32 accumulation order (+ rare rounding-boundary flips)
UNROUNDED_BAR = 3e-2     # kernel vs the plain float64 composition: bf16 operand rounding (8-bit significand) through the stack
MODEL_BAR = 5e-2         # whole model, bf16 vs fp32, per output tensor


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def bf(t):
    """round to bf16 (nearest even) and back: what cvt.rn.bf16x2.f32 does to an fp32 value"""
    return t.float().to(torch.bfloat16).double()


def _bn64(cur, bn, dim):
    shape = [1, -1] + [1] * (dim - 2)
    istd = 1.0 / torch.sqrt(bn.running_var.double() + bn.eps)
    return (cur - bn.running_mean.double().view(shape)) * (bn.weight.double() * istd).view(shape) + bn.bias.double().view(shape)


# ------------------------------------------------------------------ the fused SA layer
def _sa_reference(sa, xyz, feats, npoint, rounded):
    """float64 SA layer on the kernel's ball-query indices.  rounded: the gathered features, the tiled weight columns (all but W0's
    coordinate columns) and every hidden layer's output are rounded to bf16, as sa_fused_kernel<true> does; the coordinate term
    W0[:, 0:3] . (dx, dy, dz), BatchNorm, ReLU and the max-pool stay exact."""
    r = bf if rounded else (lambda t: t.double())
    grouper = sa.groupers[0]
    new_xyz = xyz[:, :npoint].contiguous()
    idx = ops.ball_query(new_xyz, xyz, grouper.radius, grouper.nsample).long()
    B, M, S = idx.shape
    rel_xyz = (xyz.unsqueeze(1).expand(-1, M, -1, -1).gather(2, idx.unsqueeze(-1).expand(-1, -1, -1, 3)) - new_xyz.unsqueeze(2))
    if grouper.normalize_xyz:
        rel_xyz = rel_xyz / grouper.radius
    rel_xyz = rel_xyz.double().permute(0, 3, 1, 2)                                       # (B, 3, M, S)
    units = list(sa.mlps[0].children())
    cur = None
    for l, unit in enumerate(units):
        W = unit.conv.weight.double()[:, :, 0, 0]
        if l == 0:
            y = torch.einsum("oc,bcms->boms", W[:, :3], rel_xyz)
            if feats is not None:
                C = feats.shape[1]
                g_f = torch.gather(feats.unsqueeze(2).expand(-1, -1, M, -1), 3, idx.unsqueeze(1).expand(-1, C, -1, -1))
                y = y + torch.einsum("oc,bcms->boms", r(unit.conv.weight[:, 3:, 0, 0]), r(g_f))
        else:
            y = torch.einsum("oc,bcms->boms", r(unit.conv.weight[:, :, 0, 0]), r(cur) if rounded else cur)
        if unit.conv.bias is not None:
            y = y + unit.conv.bias.double().view(1, -1, 1, 1)
        cur = F.relu(_bn64(y, unit.bn[0], 4))
    return cur.max(dim=3).values, idx


@pytest.mark.parametrize("case", SA_CASES, ids=[c[0] for c in SA_CASES])
def test_fused_sa_layer_bf16_against_emulated_and_float64(case):
    name, B, N, C, mlp, npoint, radius, S, normalize = case
    xyz, g = _cloud(B, N, seed=7 + len(name))
    xyz = xyz.cuda()
    feats = (torch.randn(B, C, N, generator=g) * 0.7).cuda() if C else None
    sa = _module(mlp, radius, S, seed=3 + len(name), normalize=normalize)
    with torch.no_grad():
        with runtime.inference_precision_scope("bf16"):
            _, got, _ = sa(xyz, feats, npoint, True)
        emu, idx = _sa_reference(sa, xyz, feats, npoint, rounded=True)
        exact, _ = _sa_reference(sa, xyz, feats, npoint, rounded=False)
    e_emu, e_exact = rel(got, emu), rel(got, exact)
    print(f"\n[sa_fused bf16 {name}] vs emulated {e_emu:.2e}, vs float64 {e_exact:.2e}")
    assert e_emu < EMULATED_BAR, (name, e_emu)
    assert e_exact < UNROUNDED_BAR, (name, e_exact)


def test_fused_sa_layer_bf16_ball_query_indices_are_the_plain_kernels():
    """o3d_sa_fused_forward's idx output in bf16 mode against o3d_ball_query (the MLP precision cannot touch the query)"""
    import ctypes
    from open3dsot_b200 import _lib
    name, B, N, C, mlp, npoint, radius, S, normalize = SA_CASES[1]
    xyz, g = _cloud(B, N, seed=7 + len(name))
    xyz = xyz.cuda()
    feats = (torch.randn(B, C, N, generator=g) * 0.7).cuda()
    sa = _module(mlp, radius, S, seed=3)
    specs = fused.parse_stack(sa.mlps[0])
    meta = fused._Meta(specs, S, False, xyz_first=True, c0=C)
    d = fused._describe(meta, B * npoint * S, fused._r4(C) + 4, meta.params)
    d.precision = _lib.PRECISION_BF16
    block = fused._sa_fused_prepare(d, xyz.device)
    feat_cl = fused.to_channels_last(feats)
    new_xyz = xyz[:, :npoint].contiguous()
    out = torch.empty(B, npoint, fused._r4(mlp[-1]), device="cuda")
    idx = torch.empty(B, npoint, S, dtype=torch.int32, device="cuda")
    _lib.check(_lib.lib().o3d_sa_fused_forward(ctypes.byref(d), block.data_ptr(), xyz.data_ptr(), new_xyz.data_ptr(),
                                               feat_cl.data_ptr(), feat_cl.shape[2], B, N, npoint, float(radius), S, 0,
                                               out.data_ptr(), out.shape[2], idx.data_ptr(), None), "o3d_sa_fused_forward")
    assert torch.equal(idx, ops.ball_query(new_xyz, xyz, radius, S))


# ------------------------------------------------------------------ the pw_tc forward: plain (TcAct) and lifted (TcLift) loaders
def _stack_modules(widths, seed):
    torch.manual_seed(seed)
    layers = []
    for cin, cout in zip(widths[:-1], widths[1:]):
        conv, bn = torch.nn.Conv1d(cin, cout, 1), torch.nn.BatchNorm1d(cout)
        with torch.no_grad():
            conv.weight.mul_(2.0)
            bn.running_mean.normal_(0, 0.3)
            bn.running_var.uniform_(0.25, 1.75)
            bn.weight.uniform_(0.5, 1.5)
            bn.bias.normal_(0, 0.2)
        layers += [conv, bn, torch.nn.ReLU()]
    return torch.nn.Sequential(*layers).cuda().eval()


def _stack_reference(seq, x, S, rounded):
    r = bf if rounded else (lambda t: t.double())
    cur = x.double()
    mods = list(seq)
    for i in range(0, len(mods), 3):
        conv, bn = mods[i], mods[i + 1]
        y = (r(cur) if rounded else cur) @ r(conv.weight[:, :, 0]).t() + conv.bias.double()
        cur = F.relu(_bn64(y, bn, 2))
    if S:
        cur = cur.view(-1, S, cur.shape[1]).max(dim=1).values
    return cur


# M2-Track's SegPointNet / MiniPointNet inference layers (64 -> 64 -> 128 -> 1024 pooled; 1088 -> 512 -> 256 -> 128), at the
# 2 x 1024 points per target of a tracking step, and a 3-layer 256-channel stack
PW_CASES = [("seg_pooled", [64, 64, 128, 1024], 4 * 2048, 64), ("seg_head", [1088, 512, 256, 128], 4 * 2048, 0),
            ("mini_pooled", [64, 128, 256], 2 * 1024, 32), ("wide_ragged", [256, 256, 200], 1000, 0)]


@pytest.mark.parametrize("case", PW_CASES, ids=[c[0] for c in PW_CASES])
def test_pw_tc_forward_bf16_against_emulated_and_float64(case):
    name, widths, P, S = case
    seq = _stack_modules(widths, seed=len(name))
    g = torch.Generator().manual_seed(11)
    x = torch.randn(P, widths[0], generator=g).cuda()
    with torch.no_grad(), runtime.inference_precision_scope("bf16"):
        got = fused.mlp_stack(x, fused.parse_stack(seq), S, False)
    emu, exact = _stack_reference(seq, x, S, True), _stack_reference(seq, x, S, False)
    e_emu, e_exact = rel(got, emu), rel(got, exact)
    print(f"\n[pw_tc bf16 {name}] vs emulated {e_emu:.2e}, vs float64 {e_exact:.2e}")
    assert e_emu < EMULATED_BAR and e_exact < UNROUNDED_BAR, (name, e_emu, e_exact)


@pytest.mark.parametrize("case", [c for c in SA_CASES if c[0] in ("sa1_search", "sa2_search", "sa3_template_batch")],
                         ids=lambda c: c[0])
def test_lifted_loader_bf16_against_emulated_and_float64(case):
    """The multi-kernel SA path (fused SA layer off): z = W0_f . f on the pw_tc forward, then the lifted stack whose layer-1 loader
    (TcLift) evaluates Y0 = z[idx] + rel . u, BN and ReLU in fp32 and rounds only the result."""
    name, B, N, C, mlp, npoint, radius, S, normalize = case
    xyz, g = _cloud(B, N, seed=7 + len(name))
    xyz = xyz.cuda()
    feats = (torch.randn(B, C, N, generator=g) * 0.7).cuda() if C else None
    sa = _module(mlp, radius, S, seed=3 + len(name), normalize=normalize)
    runtime.set_sa_fused(False)
    try:
        with torch.no_grad(), runtime.inference_precision_scope("bf16"):
            _, got, _ = sa(xyz, feats, npoint, True)
    finally:
        runtime.set_sa_fused(True)
    with torch.no_grad():
        emu = _lifted_reference(sa, xyz, feats, npoint)
        exact, _ = _sa_reference(sa, xyz, feats, npoint, rounded=False)
    e_emu, e_exact = rel(got, emu), rel(got, exact)
    print(f"\n[pw_tc lifted bf16 {name}] vs emulated {e_emu:.2e}, vs float64 {e_exact:.2e}")
    assert e_emu < EMULATED_BAR and e_exact < UNROUNDED_BAR, (name, e_emu, e_exact)


def _lifted_reference(sa, xyz, feats, npoint):
    """the lifted path's rounding points: z from bf16 features and weights (fp32 out), Y0 = z[idx] + rel . u exact, every GEMM input
    after it rounded"""
    grouper = sa.groupers[0]
    new_xyz = xyz[:, :npoint].contiguous()
    idx = ops.ball_query(new_xyz, xyz, grouper.radius, grouper.nsample).long()
    B, M, S = idx.shape
    rel_xyz = (xyz.unsqueeze(1).expand(-1, M, -1, -1).gather(2, idx.unsqueeze(-1).expand(-1, -1, -1, 3)) - new_xyz.unsqueeze(2))
    if grouper.normalize_xyz:
        rel_xyz = rel_xyz / grouper.radius
    units = list(sa.mlps[0].children())
    W0 = units[0].conv.weight[:, :, 0, 0]
    y = torch.einsum("oc,bmsc->bmso", W0[:, :3].double(), rel_xyz.double())
    if feats is not None:
        f_cl = feats.transpose(1, 2)                                                     # (B, N, C)
        z = (bf(f_cl) @ bf(W0[:, 3:]).t()).float().double()                                # z is stored in fp32
        y = y + torch.gather(z.unsqueeze(1).expand(-1, M, -1, -1), 2, idx.unsqueeze(-1).expand(-1, -1, -1, z.shape[-1]))
    if units[0].conv.bias is not None:
        y = y + units[0].conv.bias.double()
    bn0 = units[0].bn[0]
    cur = F.relu((y - bn0.running_mean.double()) / torch.sqrt(bn0.running_var.double() + bn0.eps) * bn0.weight.double()
                 + bn0.bias.double())
    for unit in units[1:]:
        bn = unit.bn[0]
        yy = bf(cur.float()) @ bf(unit.conv.weight[:, :, 0, 0]).t()
        if unit.conv.bias is not None:
            yy = yy + unit.conv.bias.double()
        cur = F.relu((yy - bn.running_mean.double()) / torch.sqrt(bn.running_var.double() + bn.eps) * bn.weight.double()
                     + bn.bias.double())
    return cur.max(dim=2).values.permute(0, 2, 1)


# ------------------------------------------------------------------ whole models, bf16 against fp32
class Choices:
    """CHOICE_HOOK: records the discrete choices in call order; with `inject`, substitutes the recorded ones"""

    def __init__(self, inject=None):
        self.inject, self.seen = inject, {}

    def __call__(self, kind, info, compute):
        own = compute()
        n = len(self.seen.setdefault(kind, []))
        self.seen[kind].append(own)
        if self.inject is None:
            return own
        return self.inject[kind][n].view_as(own).contiguous()


def _model_inputs(cfg_file):
    cfg = load_config(os.path.join(ROOT, "cfgs", cfg_file))
    net = get_model(cfg.net_model)(cfg)
    net.load_state_dict(det_state_dict(net.state_dict(), seed=41))
    if "M2" in cfg_file:
        batch = synthetic_motion_batch(16, 1024, seed=77)
    else:
        batch = synthetic_siamese_batch(16, 512, 1024, seed=20260924, box_aware="BAT" in cfg_file)
    return net.cuda().eval(), {k: v.cuda() for k, v in batch.items()}


@pytest.mark.parametrize("cfg_file", MODELS)
def test_whole_model_bf16_against_fp32(cfg_file):
    net, batch = _model_inputs(cfg_file)
    rec = Choices()
    runtime.CHOICE_HOOK = rec
    try:
        with torch.no_grad(), runtime.static_weights_scope():
            ref = net({k: v.clone() for k, v in batch.items()})
        runtime.CHOICE_HOOK = Choices(rec.seen)
        with torch.no_grad(), runtime.inference_precision_scope("bf16"):
            got = net({k: v.clone() for k, v in batch.items()})
    finally:
        runtime.CHOICE_HOOK = None
    # M2-Track's estimation_boxes picks, per sample, the refined or the auxiliary box by an arg-max over the motion-state logits:
    # a discrete choice the hook does not cover, so it is compared through its inputs (aux_estimation_boxes, motion_pred, ...)
    skip = {"estimation_boxes"} if "M2" in cfg_file else set()
    errs = {k: rel(got[k], ref[k]) for k, v in ref.items()
            if k not in skip and torch.is_tensor(v) and v.is_floating_point() and v.numel() > 1}
    assert errs
    print(f"\n[model bf16 vs fp32 {cfg_file}] " + ", ".join(f"{k} {e:.2e}" for k, e in sorted(errs.items())))
    assert max(errs.values()) < MODEL_BAR, errs


def test_bf16_and_fp32_blocks_coexist_and_fp32_is_unchanged():
    net, batch = _model_inputs("BAT_Car.yaml")
    fresh = copy.deepcopy(net)                   # own parameter tensors: no cached block of `net` can reach it

    def run(model, precision):
        with torch.no_grad(), runtime.static_weights_scope(), runtime.inference_precision_scope(precision):
            out = model({k: v.clone() for k, v in batch.items()})
        return {k: v.clone() for k, v in out.items() if torch.is_tensor(v)}

    ref = run(fresh, "fp32")
    b1 = run(net, "bf16")
    f1 = run(net, "fp32")
    b2 = run(net, "bf16")
    f2 = run(net, "fp32")
    for k in ref:
        assert torch.equal(f1[k], ref[k]) and torch.equal(f2[k], ref[k]), k
        assert torch.equal(b1[k], b2[k]), k
    assert any(not torch.equal(b1[k], ref[k]) for k in ref if ref[k].is_floating_point())


def test_bf16_refuses_training_and_autograd():
    net, batch = _model_inputs("P2B_Car.yaml")
    with runtime.inference_precision_scope("bf16"):
        with pytest.raises(RuntimeError, match="bf16"):
            net({k: v.clone() for k, v in batch.items()})                      # grad enabled: the parameters need gradients
        net.train()
        with torch.no_grad(), pytest.raises(RuntimeError, match="bf16"):
            net({k: v.clone() for k, v in batch.items()})
    net.eval()


# ------------------------------------------------------------------ trackers in bf16
def _tmodel(cfg_name, **over):
    cfg = load_config(os.path.join(ROOT, "cfgs", cfg_name), {"up_axis": [0, 0, 1], **over})
    torch.manual_seed(0)
    return cfg, get_model(cfg.net_model)(cfg).cuda().eval()


def _tracklets(lengths, n_points=4000, seed=500):
    return [synthetic_sequence(n_frames=n, n_points=n_points, seed=seed + i, speed=0.4 + 0.05 * i, yaw_rate=1.0 + i)
            for i, n in enumerate(lengths)]


def _boxes(res):
    return np.array([np.concatenate([b.center, b.rotation_matrix.ravel()]) for seq in res["results"] for b in seq])


@pytest.mark.parametrize("cfg_name", MODELS)
def test_batched_bf16_graph_equals_eager_and_repeats(cfg_name):
    _, net = _tmodel(cfg_name)
    tracks = _tracklets([8, 3, 6, 1, 5])
    a = evaluate_batched(net, tracks, slots=3, seed=5, precision="bf16")
    b = evaluate_batched(net, tracks, slots=3, seed=5, precision="bf16")
    e = evaluate_batched(net, tracks, slots=3, seed=5, precision="bf16", use_graph=False)
    f = evaluate_batched(net, tracks, slots=3, seed=5)
    assert np.array_equal(_boxes(a), _boxes(b)) and a["overlaps"] == b["overlaps"]
    assert np.array_equal(_boxes(a), _boxes(e)) and a["overlaps"] == e["overlaps"]
    d = float(np.abs(_boxes(a) - _boxes(f)).max())
    print(f"\n[evaluate_batched {cfg_name}] bf16 vs fp32 max box difference {d:.2e}; success {a['success']:.2f} / {f['success']:.2f}")


@pytest.mark.parametrize("cfg_name", MODELS)
def test_bf16_slot_matches_device_tracker(cfg_name):
    """slot k of the batched step against the B=1 DeviceTracker fed slot k's keyed draws, both bf16, eager"""
    cfg, net = _tmodel(cfg_name, limit_box=False)
    n_points, seed = 6000, 11
    tracks = _tracklets([6, 6, 6], n_points=n_points, seed=300)
    trk = BatchedDeviceTracker(net, tracks, slots=3, seed=seed, ids=[4, 9, 2], max_points=n_points, use_graph=False,
                               precision="bf16")
    _, _, cen, rot = trk.run()
    offsets = trk.plan["offsets"]
    worst = 0.0
    for j, seq in enumerate(tracks):
        tid = trk.ids[j]
        one = DeviceTracker(net, max_points=n_points, use_graph=False, precision="bf16")
        pts = [torch.tensor(f["pc"].points.T.copy(), device="cuda") for f in seq]
        one.reset(pts[0], seq[0]["3d_bbox"].to_tensor("cuda"))
        for i in range(1, 6):
            one._load_scan(pts[i])
            draws = [ops.keyed_uniform(torch.tensor([tid], device="cuda"), torch.tensor([i], device="cuda"), seed, s, u.shape[0])[0]
                     for s, u in enumerate(one.u_s + one.u_t)]
            for u, d in zip(one.u_s + one.u_t, draws):
                u.copy_(d)
            one._frame()
            o = int(offsets[j]) + i
            dc = float((one.box_c.double().cpu() - torch.from_numpy(cen[o])).abs().max())
            dr = float((one.box_r.double().cpu() - torch.from_numpy(rot[o])).abs().max())
            worst = max(worst, dc, dr)
            assert dc < 1e-3 and dr < 1e-3, (cfg_name, j, i, dc, dr)
    print(f"\n[bf16 slot vs B=1 {cfg_name}] max difference {worst:.2e}")


IDS, STARTS, ENDS = [12, 3, 40, 7, 25], [0, 0, 2, 4, 5], [4, 3, 9, 8, 9]     # at most 3 targets at once


def _stream(net, scene, which, max_targets, use_graph=True):
    starts = {}
    for j in which:
        starts.setdefault(STARTS[j], []).append((IDS[j], scene["boxes"][j][STARTS[j]]))
    ends = {IDS[j]: ENDS[j] for j in which}
    scans = [torch.tensor(s, device="cuda") for s in scene["scans"]]
    return track_stream(net, scans, starts, ends, max_targets, seed=5, max_points=6000, use_graph=use_graph, precision="bf16")


def _flat(res, tid):
    return np.array([np.concatenate([b.center, b.rotation_matrix.ravel()]) for _, b in sorted(res[tid].items())])


@pytest.mark.parametrize("cfg_name", MODELS)
def test_bf16_live_target_ignores_k_and_the_others(cfg_name):
    _, net = _tmodel(cfg_name)
    scene = synthetic_scene(n_frames=10, n_points=6000, n_objects=5, seed=900, extent=15.0)
    full = _stream(net, scene, range(5), 3)
    alone = _stream(net, scene, [2, 3], 8)
    eager = _stream(net, scene, range(5), 3, use_graph=False)
    worst = 0.0
    for j in (2, 3):
        d = float(np.abs(_flat(alone, IDS[j]) - _flat(full, IDS[j])).max())
        worst = max(worst, d)
        assert d < 1e-3, (cfg_name, IDS[j], d)
    for tid in IDS:
        assert np.array_equal(_flat(eager, tid), _flat(full, tid)), (cfg_name, tid)
    print(f"\n[bf16 live target {cfg_name}] alone vs among others, K 8 vs 3: max difference {worst:.2e}")


# ------------------------------------------------------------------ the kernels one bf16 replay runs
_PROFILE_CHILD = r"""
import json, os, sys
import torch
sys.path.insert(0, sys.argv[1])
from open3dsot_b200.config import load_config
from open3dsot_b200.datasets.synthetic import synthetic_scene
from open3dsot_b200.models import get_model
from open3dsot_b200.tracking.multi_tracker import MultiTargetTracker
names = set()
for cfg_file in ("BAT_Car.yaml", "M2_track_kitti.yaml"):
    cfg = load_config(os.path.join(sys.argv[1], "cfgs", cfg_file), {"up_axis": [0, 0, 1]})
    torch.manual_seed(0)
    net = get_model(cfg.net_model)(cfg).cuda().eval()
    scene = synthetic_scene(n_frames=5, n_points=6000, n_objects=2, seed=900, extent=15.0)
    scans = [torch.tensor(s, device="cuda") for s in scene["scans"]]
    trk = MultiTargetTracker(net, 6000, 4, seed=2, precision="bf16")
    trk.step(scans[0])
    trk.add(1, scene["boxes"][0][0])
    trk.step(scans[1])
    torch.cuda.synchronize()
    for i in (2, 3, 4):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            trk.step(scans[i])
            torch.cuda.synchronize()
        got = {e.name for e in prof.events()}
        if any("kernel" in n for n in got):
            names |= got
            break
print(json.dumps(sorted(names)))
"""


def _norm(name):
    return re.sub(r"\s*([<>,])\s*", r"\1", name.replace("(anonymous namespace)::", ""))


def test_profiled_bf16_replay_runs_bf16_kernels_only():
    r = subprocess.run([sys.executable, "-c", _PROFILE_CHILD, ROOT], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    names = {_norm(n) for n in json.loads(r.stdout.strip().splitlines()[-1])}
    assert any("sa_fused_kernel<true>" in n for n in names), sorted(names)
    assert any("pw_tc_kernel<Bf16<TcAct>," in n for n in names), sorted(names)
    assert not any("sa_fused_kernel<false>" in n for n in names), sorted(names)
    assert not any(re.search(r"pw_tc_kernel<(TcAct|TcLift),TcFwdEpi", n) for n in names), sorted(names)
