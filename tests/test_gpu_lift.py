"""Lifted first layer (include/o3d_b200.h `o3d_lift_t`): the set-abstraction layer, BoxAwareXCorr and P2B_XCorr with the
first 1x1 convolution applied to the source points (no grouped tensor) against

  (a) the oracle composition on the CPU (oracle/modules.py — itself pinned to the reference, tests/test_oracle_golden.py),
  (b) the materialising path of round 1 (O3D_LIFT=0: ball-query+group kernel, then a GEMM over the grouped rows),

forward and every gradient, on shapes that take the CUDA-core fallback (Y0 stored) and on shapes that take the tensor-core
path (Y0 virtual: gathered inside the wgmma operand loaders / dgrad epilogue)."""
import pytest
import torch

from open3dsot_b200 import runtime
from open3dsot_b200.models.head.xcorr import BoxAwareXCorr, P2B_XCorr
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
    xyz[:, N // 8: N // 4] = xyz[:, : N // 4 - N // 8]          # exact duplicates: ties, heavy first-hit padding
    return xyz, g


def _run_sa(lift, xyz, feats, mlp, npoint, radius, nsample, use_fps, xyz_grad, train, seed):
    runtime.set_lift(lift)
    try:
        sa = PointnetSAModule(mlp=list(mlp), radius=radius, nsample=nsample, use_fps=use_fps)
        sa.load_state_dict(det_state_dict(sa.state_dict(), seed=seed))
        sa = sa.cuda().train(train)
        x = xyz.clone().cuda().requires_grad_(xyz_grad)
        f = None if feats is None else feats.clone().cuda().requires_grad_(True)
        nx, nf, _ = sa(x, f, npoint, True)
        # a loss with structure in both the channel and the point dimension
        w = torch.linspace(0.5, 1.5, nf.shape[1], device="cuda")[None, :, None]
        loss = (nf * w).square().sum() + (nx.sum() if xyz_grad else 0.0)
        params = list(sa.parameters())
        ins = ([x] if xyz_grad else []) + ([f] if f is not None else [])
        gr = torch.autograd.grad(loss, ins + params)
        stats = [b.clone() for n, b in sa.named_buffers() if "running" in n]
        return nf, gr, stats
    finally:
        runtime.set_lift(True)


SA_CASES = [
    # name, B, N, C, mlp, npoint, radius, nsample, use_fps, xyz_grad, train
    ("small_fps", 2, 96, 8, [8, 16, 16, 32], 24, 0.35, 16, True, False, True),            # CUDA-core fallback: Y0 materialised
    ("small_xyzgrad", 2, 96, 8, [8, 16, 16, 32], 24, 0.35, 16, False, True, True),
    ("sa1_nofeat", 8, 512, 0, [0, 64, 64, 128], 256, 0.3, 32, True, False, True),         # tensor-core path, K1 = 64
    ("sa2", 8, 256, 128, [128, 128, 128, 256], 128, 0.5, 32, False, False, True),        # K1 = 128
    ("sa3", 8, 128, 256, [256, 256, 256, 256], 64, 0.7, 32, False, False, True),         # K1 = 256, two channel tiles
    ("rpn_vote", 12, 128, 257, [257, 256, 256, 256], 64, 0.3, 16, False, True, True),    # nsample 16, ragged channels, d/d xyz
    # eval mode keeps Y0 virtual below the wgrad's P >= 4096 floor (P = 2048): layer 1's weight gradient on the tensor cores
    ("sa2_eval", 1, 256, 128, [128, 128, 128, 256], 64, 0.5, 32, False, False, False),
]


@pytest.mark.parametrize("case", SA_CASES, ids=[c[0] for c in SA_CASES])
def test_lifted_sa_matches_materialised_path(case):
    name, B, N, C, mlp, npoint, radius, nsample, use_fps, xyz_grad, train = case
    xyz, g = _cloud(B, N, seed=3)
    feats = torch.randn(B, C, N, generator=g) if C else None
    o_l, g_l, s_l = _run_sa(True, xyz, feats, mlp, npoint, radius, nsample, use_fps, xyz_grad, train, seed=5)
    o_m, g_m, s_m = _run_sa(False, xyz, feats, mlp, npoint, radius, nsample, use_fps, xyz_grad, train, seed=5)
    assert rel(o_l, o_m) < RTOL
    for a, b in zip(s_l, s_m):
        assert rel(a, b) < RTOL
    scale = max(float(t.norm()) for t in g_m)
    for a, b in zip(g_l, g_m):
        err = float((a.double() - b.double()).norm())
        assert err < 3e-4 * max(float(b.norm()), 1e-2 * scale), (name, tuple(b.shape), err, float(b.norm()))


def test_lifted_sa_matches_oracle_small():
    """Against the CPU oracle composition (which the reference-generated golden vectors pin): forward + gradients."""
    from oracle import modules as om
    B, N, C, M = 2, 96, 8, 24
    xyz, g = _cloud(B, N, seed=11)
    feats = torch.randn(B, C, N, generator=g)
    sa = PointnetSAModule(mlp=[C, 16, 16, 32], radius=0.35, nsample=16, use_fps=True)
    base = det_state_dict(sa.state_dict(), seed=1)
    sa.load_state_dict(base)
    sa = sa.cuda().train()
    f = feats.clone().cuda().requires_grad_(True)
    nx, nf, _ = sa(xyz.cuda(), f, M, True)
    nf.square().sum().backward()
    sd = {"sa." + k: v.clone() for k, v in base.items()}
    for k in sd:
        if sd[k].is_floating_point() and "running" not in k:
            sd[k].requires_grad_(True)
    fo = feats.clone().requires_grad_(True)
    _, wf, _ = om.sa_module(sd, "sa", xyz, fo, M, 0.35, 16, True, True)
    wf.square().sum().backward()
    assert rel(nf, wf) < RTOL
    assert rel(f.grad, fo.grad) < 3e-4
    for k, p in sa.named_parameters():
        assert rel(p.grad, sd["sa." + k].grad) < 1e-3, k


def _run_head(kind, lift, B, f, Mt, Ns, hidden, seed):
    runtime.set_lift(lift)
    try:
        g = torch.Generator().manual_seed(seed)
        tf = torch.randn(B, f, Mt, generator=g).cuda().requires_grad_(True)
        sf = torch.randn(B, f, Ns, generator=g).cuda().requires_grad_(True)
        txyz, sxyz = torch.rand(B, Mt, 3, generator=g).cuda(), torch.rand(B, Ns, 3, generator=g).cuda()
        tbc = torch.rand(B, Mt, 9, generator=g).cuda().requires_grad_(True)
        sbc = torch.rand(B, Ns, 9, generator=g).cuda()
        m = P2B_XCorr(f, hidden, f) if kind == "p2b" else BoxAwareXCorr(f, hidden, f, k=4, bc_channel=9)
        m.load_state_dict(det_state_dict(m.state_dict(), seed=9))
        m = m.cuda().train()
        out = m(tf, sf, txyz) if kind == "p2b" else m(tf, sf, txyz, sxyz, tbc, sbc)
        w = torch.linspace(0.5, 1.5, out.shape[1], device="cuda")[None, :, None]
        loss = (out * w).square().sum()
        ins = [tf, sf] if kind == "p2b" else [tf, tbc]
        gr = torch.autograd.grad(loss, ins + list(m.parameters()), allow_unused=True)
        return out, gr
    finally:
        runtime.set_lift(True)


HEAD_CASES = [("p2b", 2, 16, 16, 20, 16), ("bat", 2, 16, 12, 20, 16),               # CUDA-core fallback
              ("p2b", 8, 256, 64, 128, 256), ("bat", 16, 256, 64, 128, 256)]        # tensor-core path at the models' widths


@pytest.mark.parametrize("case", HEAD_CASES, ids=[f"{c[0]}_{c[2]}" for c in HEAD_CASES])
def test_lifted_xcorr_heads_match_materialised_path(case):
    kind, B, f, Mt, Ns, hidden = case
    o_l, g_l = _run_head(kind, True, B, f, Mt, Ns, hidden, seed=2)
    o_m, g_m = _run_head(kind, False, B, f, Mt, Ns, hidden, seed=2)
    assert rel(o_l, o_m) < RTOL
    scale = max(float(t.norm()) for t in g_m if t is not None)
    for a, b in zip(g_l, g_m):
        if b is None:
            assert a is None
            continue
        err = float((a.double() - b.double()).norm())
        assert err < 3e-4 * max(float(b.norm()), 1e-2 * scale), (kind, tuple(b.shape), err, float(b.norm()))
