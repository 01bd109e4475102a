"""The single-kernel inference set-abstraction layer (csrc/sa_fused.cu, `o3d_sa_fused_forward`) against

  (a) a float64 torch composition of the reference's module body (pointnet2_modules.py:58-76: QueryAndGroup, SharedMLP with
      running-statistics BatchNorm, max-pool) on the bit-exact ball-query indices,
  (b) the multi-kernel path the training step uses (O3D_SA_FUSED=0),

at the three backbone shapes of BAT / P2B (template and search), on ragged / padded shapes (channel counts that are not
multiples of 4 / 32 / 128, empty balls, duplicated points, normalize_xyz) and through the C ABI's index output."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from open3dsot_b200 import _lib, fused, ops, runtime
from open3dsot_b200.pointnet2.utils.pointnet2_modules import PointnetSAModule
from _params import det_state_dict

pytestmark = pytest.mark.gpu
RTOL = 1e-4


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _cloud(B, N, seed, spread=1.2):
    g = torch.Generator().manual_seed(seed)
    xyz = torch.rand(B, N, 3, generator=g) * spread
    xyz[:, N // 8: N // 4] = xyz[:, : N // 4 - N // 8]          # exact duplicates
    return xyz, g


def _module(mlp, radius, nsample, seed, normalize=False, device="cuda"):
    sa = PointnetSAModule(mlp=list(mlp), radius=radius, nsample=nsample, use_fps=False, normalize_xyz=normalize)
    sa.load_state_dict(det_state_dict(sa.state_dict(), seed=seed))
    g = torch.Generator().manual_seed(seed + 100)
    for n, b in sa.named_buffers():                         # running statistics away from (0, 1)
        if n.endswith("running_mean"):
            b.copy_(torch.randn(b.shape, generator=g) * 0.3)
        elif n.endswith("running_var"):
            b.copy_(torch.rand(b.shape, generator=g) * 1.5 + 0.25)
    return sa.to(device).eval()


def _reference64(sa, xyz, feats, npoint, idx=None):
    """float64 composition on the kernel-exact neighbour indices (`idx`: indices from elsewhere — tests/test_oracle_sa_eval.py
    feeds the CPU oracle's to show that this yardstick and the pinned oracle are the same function)"""
    grouper = sa.groupers[0]
    new_xyz = xyz[:, :npoint].contiguous()
    if idx is None:
        idx = ops.ball_query(new_xyz, xyz, grouper.radius, grouper.nsample)
    idx = idx.long()                                                                     # (B, npoint, S)
    B, M, S = idx.shape
    g_xyz = (xyz.unsqueeze(1).expand(-1, M, -1, -1).gather(2, idx.unsqueeze(-1).expand(-1, -1, -1, 3))
             - new_xyz.unsqueeze(2)).double()               # the fp32 difference, as the reference forms it
    if grouper.normalize_xyz:
        g_xyz = (g_xyz.float() / grouper.radius).double()
    cur = g_xyz.permute(0, 3, 1, 2)                          # (B, 3, M, S)
    if feats is not None:
        f64 = feats.double()                                 # (B, C, N)
        C = f64.shape[1]
        g_f = torch.gather(f64.unsqueeze(2).expand(-1, -1, M, -1), 3, idx.unsqueeze(1).expand(-1, C, -1, -1))
        cur = torch.cat([cur, g_f], dim=1)
    for unit in sa.mlps[0].children():
        conv, bn = unit.conv, unit.bn[0]
        cur = F.conv2d(cur, conv.weight.double(), None if conv.bias is None else conv.bias.double())
        cur = F.batch_norm(cur, bn.running_mean.double(), bn.running_var.double(), bn.weight.double(), bn.bias.double(), False, 0.0,
                           bn.eps)
        cur = F.relu(cur)
    return cur.max(dim=3).values, idx


CASES = [
    # name, B, N, C, mlp, npoint, radius, nsample, normalize
    ("sa1_search", 1, 1024, 0, [0, 64, 64, 128], 512, 0.3, 32, False),
    ("sa2_search", 1, 512, 128, [128, 128, 128, 256], 256, 0.5, 32, False),
    ("sa3_search", 1, 256, 256, [256, 256, 256, 256], 128, 0.7, 32, False),
    ("sa1_template", 1, 512, 0, [0, 64, 64, 128], 256, 0.3, 32, False),
    ("sa3_template_batch", 5, 128, 256, [256, 256, 256, 256], 64, 0.7, 32, False),
    ("ragged_channels", 3, 100, 5, [5, 7, 130], 8, 0.4, 16, True),           # C % 4 != 0, cout 7 / 130, two channel tiles
    ("empty_balls", 2, 64, 12, [12, 33, 20, 9], 32, 0.01, 8, False),         # most balls hold only the centre itself / nothing
    ("one_layer_wide", 2, 80, 40, [40, 200], 16, 0.5, 64, False),            # nsample 64: one centre per CTA, single layer
    ("nsample_4", 2, 70, 0, [0, 24, 48], 32, 0.3, 4, False),
    ("vote_aggregation", 2, 128, 257, [257, 256, 256, 256], 64, 0.3, 16, True),   # the RPN's cluster layer: 9 input k-blocks
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_fused_sa_layer_matches_float64_and_the_multi_kernel_path(case):
    name, B, N, C, mlp, npoint, radius, S, normalize = case
    xyz, g = _cloud(B, N, seed=7 + len(name))
    xyz = xyz.cuda()
    feats = (torch.randn(B, C, N, generator=g) * 0.7).cuda() if C else None
    sa = _module(mlp, radius, S, seed=3, normalize=normalize)
    assert fused._sa_fused_ok(fused.parse_stack(sa.mlps[0]), S, npoint, N, C), "case outside the fused kernel's range"
    with torch.no_grad():
        _, nf_fused, _ = sa(xyz, feats, npoint, True)
        runtime.set_sa_fused(False)
        try:
            _, nf_multi, _ = sa(xyz, feats, npoint, True)
        finally:
            runtime.set_sa_fused(True)
        want, _ = _reference64(sa, xyz, feats, npoint)
    assert nf_fused.shape == want.shape
    e_f, e_m = rel(nf_fused, want), rel(nf_multi, want)
    assert e_f < 1e-5, f"{name}: fused vs float64 {e_f:.2e} (multi-kernel path: {e_m:.2e})"
    assert rel(nf_fused, nf_multi) < RTOL


def test_fused_sa_layer_index_output_is_the_ball_query():
    B, N, C, npoint, S, radius = 3, 200, 16, 48, 16, 0.35
    xyz, g = _cloud(B, N, seed=21)
    xyz = xyz.cuda()
    feats = torch.randn(B, C, N, generator=g).cuda()
    sa = _module([C, 32, 64], radius, S, seed=5)
    specs = fused.parse_stack(sa.mlps[0])
    meta = fused._Meta(specs, S, False, xyz_first=True, c0=C)
    d = fused._describe(meta, B * npoint * S, C + 4, meta.params)
    L = _lib.lib()
    block = torch.empty(int(L.o3d_sa_fused_prepared_bytes(ctypes.byref(d))), dtype=torch.uint8, device="cuda")
    _lib.check(L.o3d_sa_fused_prepare(ctypes.byref(d), block.data_ptr(), None), "prepare")
    new_xyz = xyz[:, :npoint].contiguous()
    feat_cl = feats.transpose(1, 2).contiguous()
    out = torch.empty(B, npoint, 64, device="cuda")
    idx = torch.full((B, npoint, S), -1, dtype=torch.int32, device="cuda")
    _lib.check(L.o3d_sa_fused_forward(ctypes.byref(d), block.data_ptr(), xyz.data_ptr(), new_xyz.data_ptr(), feat_cl.data_ptr(), C, B, N,
                                      npoint, radius, S, 0, out.data_ptr(), 64, idx.data_ptr(), None), "forward")
    torch.cuda.synchronize()
    assert torch.equal(idx, ops.ball_query(new_xyz, xyz, radius, S))
    want, _ = _reference64(sa, xyz, feats, npoint)
    assert rel(out.transpose(1, 2), want) < 1e-5


def test_fused_sa_layer_rejects_shapes_outside_its_range():
    sa = _module([8, 16, 300], 0.3, 16, seed=1)                       # 300 output channels
    assert not fused._sa_fused_ok(fused.parse_stack(sa.mlps[0]), 16, 32, 64, 8)
    sa = _module([8, 16, 32], 0.3, 24, seed=1)                        # nsample 24 does not divide 64
    assert not fused._sa_fused_ok(fused.parse_stack(sa.mlps[0]), 24, 32, 64, 8)
    sa = _module([8, 16, 300], 0.3, 16, seed=1)
    xyz, g = _cloud(2, 64, seed=2)
    with torch.no_grad():                                             # ... and such a layer still runs (multi-kernel path)
        _, nf, _ = sa(xyz.cuda(), torch.randn(2, 8, 64, generator=g).cuda(), 32, True)
    assert nf.shape == (2, 300, 32)
