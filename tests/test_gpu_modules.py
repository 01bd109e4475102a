"""GPU parity of the modules and whole models against (a) the golden vectors produced by the reference's own
Python and (b) the oracle, in both execution modes (fused = product default, composed = op-by-op cross-check)."""
import os

import numpy as np
import pytest
import torch

from _params import det_state_dict
from open3dsot_b200 import runtime
from open3dsot_b200.config import load_config
from open3dsot_b200.datasets.synthetic import synthetic_siamese_batch
from open3dsot_b200.models import get_model
from open3dsot_b200.models.head.rpn import P2BVoteNetRPN
from open3dsot_b200.models.head.xcorr import BoxAwareXCorr, P2B_XCorr
from open3dsot_b200.pointnet2.utils import pointnet2_modules as pm
from open3dsot_b200.pointnet2.utils import pointnet2_utils as pu

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RTOL = 1e-4
MODES = ["composed"] + (["fused"] if os.path.exists(os.path.join(ROOT, "open3dsot_b200", "fused.py")) else [])


def rel(a, b):
    a = torch.as_tensor(a).detach().double().cpu()
    b = torch.as_tensor(b).detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


@pytest.fixture(scope="module")
def gm(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "ref_modules.npz")))


@pytest.fixture(scope="module")
def gmod(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "ref_models.npz")))


@pytest.fixture(params=MODES)
def mode(request):
    old = runtime.fused_enabled()
    runtime.set_fused(request.param == "fused")
    yield request.param
    runtime.set_fused(old)


def _c(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def test_query_and_group_module(gm):
    xyz, feats = _c(gm["qg_xyz"]), _c(gm["qg_feats"])
    new_xyz = xyz[:, :24].contiguous()
    for norm in (0, 1):
        qg = pu.QueryAndGroup(0.35, 16, use_xyz=True, return_idx=True, normalize_xyz=bool(norm))
        nf, idx = qg(xyz, new_xyz, feats)
        assert np.array_equal(idx.cpu().numpy(), gm[f"qg_idx_norm{norm}"])
        assert rel(nf, gm[f"qg_out_norm{norm}"]) < 1e-6


@pytest.mark.parametrize("tag,use_fps", [("fps", True), ("arange", False)])
def test_sa_module(gm, mode, tag, use_fps):
    xyz, feats = _c(gm["qg_xyz"]), _c(gm["qg_feats"])
    sa = pm.PointnetSAModule(mlp=[8, 16, 16, 32], radius=0.35, nsample=16, use_fps=use_fps)
    sa.load_state_dict(det_state_dict(sa.state_dict(), seed=1))
    sa = sa.cuda().train()
    f_in = feats.clone().requires_grad_(True)
    nx, nf, sidx = sa(xyz, f_in, 24, True)
    assert np.array_equal(sidx.cpu().numpy(), gm[f"sa_{tag}_idx"])
    assert rel(nx, gm[f"sa_{tag}_newxyz"]) == 0
    assert rel(nf, gm[f"sa_{tag}_train_out"]) < RTOL
    nf.square().sum().backward()
    assert rel(f_in.grad, gm[f"sa_{tag}_train_gfeat"]) < RTOL
    assert rel(sa.mlps[0].layer0.conv.weight.grad, gm[f"sa_{tag}_train_gw0"]) < RTOL
    assert rel(sa.mlps[0].layer2.conv.weight.grad, gm[f"sa_{tag}_train_gw2"]) < RTOL
    assert rel(sa.mlps[0].layer1.bn.bn.weight.grad, gm[f"sa_{tag}_train_ggamma1"]) < RTOL
    assert rel(sa.mlps[0].layer2.bn.bn.running_mean, gm[f"sa_{tag}_rm2"]) < 1e-5
    assert rel(sa.mlps[0].layer2.bn.bn.running_var, gm[f"sa_{tag}_rv2"]) < 1e-5
    assert int(sa.mlps[0].layer2.bn.bn.num_batches_tracked) == 1
    sa.load_state_dict(det_state_dict(sa.state_dict(), seed=1))
    sa.eval()
    with torch.no_grad():
        _, nf_e, _ = sa(xyz, feats, 24, True)
    assert rel(nf_e, gm[f"sa_{tag}_eval_out"]) < RTOL


def test_fp_module(gm, mode):
    fp = pm.PointnetFPModule(mlp=[12, 16, 12])
    fp.load_state_dict(det_state_dict(fp.state_dict(), seed=2))
    fp = fp.cuda().train()
    kf = _c(gm["fp_kf"]).requires_grad_(True)
    y = fp(_c(gm["fp_unknown"]), _c(gm["fp_known"]), _c(gm["fp_uf"]), kf)
    assert rel(y, gm["fp_out"]) < RTOL
    y.square().sum().backward()
    assert rel(kf.grad, gm["fp_gkf"]) < RTOL


def test_xcorr_and_rpn(gm, mode):
    tf, sf, txyz, sxyz, tbc, sbc = (_c(gm[k]) for k in ("xc_tf", "xc_sf", "xc_txyz", "xc_sxyz", "xc_tbc", "xc_sbc"))
    px = P2B_XCorr(16, 16, 16); px.load_state_dict(det_state_dict(px.state_dict(), seed=3)); px = px.cuda().train()
    assert rel(px(tf, sf, txyz), gm["p2bx_out"]) < RTOL
    bx = BoxAwareXCorr(16, 16, 16, k=4, bc_channel=9); bx.load_state_dict(det_state_dict(bx.state_dict(), seed=4))
    bx = bx.cuda().train()
    assert rel(bx(tf, sf, txyz, sxyz, tbc, sbc), gm["bax_out"]) < RTOL
    rp = P2BVoteNetRPN(16, vote_channel=16, num_proposal=8); rp.load_state_dict(det_state_dict(rp.state_dict(), seed=5))
    rp = rp.cuda().train()
    boxes, cla, vxyz, cen = rp(sxyz, sf)
    assert rel(boxes, gm["rpn_boxes"]) < RTOL and rel(cla, gm["rpn_cla"]) < RTOL
    assert rel(vxyz, gm["rpn_vote_xyz"]) < RTOL and rel(cen, gm["rpn_centers"]) < RTOL


def _run_head(kind, fused_flag, grads=True):
    """Build a head with deterministic parameters and inputs, run it in one mode, return output and gradients."""
    g = torch.Generator().manual_seed(77)
    B, f, Mt, Ns = 3, 32, 16, 40
    tf = torch.randn(B, f, Mt, generator=g).cuda().requires_grad_(True)
    sf = torch.randn(B, f, Ns, generator=g).cuda().requires_grad_(True)
    txyz, sxyz = torch.rand(B, Mt, 3, generator=g).cuda(), torch.rand(B, Ns, 3, generator=g).cuda()
    tbc, sbc = torch.rand(B, Mt, 9, generator=g).cuda(), torch.rand(B, Ns, 9, generator=g).cuda().requires_grad_(True)
    if kind == "p2b":
        m = P2B_XCorr(f, 32, f)
    elif kind == "bat":
        m = BoxAwareXCorr(f, 32, f, k=4, bc_channel=9)
    else:
        m = P2BVoteNetRPN(f, vote_channel=32, num_proposal=16)
    m.load_state_dict(det_state_dict(m.state_dict(), seed=9))
    m = m.cuda().train()
    old = runtime.fused_enabled()
    runtime.set_fused(fused_flag)
    try:
        if kind == "p2b":
            outs = [m(tf, sf, txyz)]
        elif kind == "bat":
            outs = [m(tf, sf, txyz, sxyz, tbc, sbc)]
        else:
            outs = list(m(sxyz, sf))[:3]      # boxes depend on a ball query of computed votes: compared separately
        loss = sum(o.square().sum() for o in outs)
        params = [p for p in m.parameters()]
        inputs = [t for t in (tf, sf) if t.requires_grad]
        gr = torch.autograd.grad(loss, inputs + params, allow_unused=True)
    finally:
        runtime.set_fused(old)
    return outs, gr


@pytest.mark.parametrize("kind", ["p2b", "bat", "rpn"])
def test_fused_heads_match_composed_on_device(kind):
    """Fused xcorr heads / RPN against the op-by-op composition (torch fp32 convs, TF32 off) on identical inputs."""
    o_f, g_f = _run_head(kind, True)
    o_c, g_c = _run_head(kind, False)
    for a, b in zip(o_f, o_c):
        assert rel(a, b) < RTOL
    scale = max(float(g.norm()) for g in g_c if g is not None)
    bad = []
    for i, (a, b) in enumerate(zip(g_f, g_c)):
        if b is None:
            continue
        err, nb = float((a.double() - b.double()).norm()), float(b.norm())
        # BN shifts of a layer that feeds another conv+BN have an analytically (almost) vanishing gradient: what is
        # left is a cancellation residue of O(1e-5) of the summed magnitudes, so only its absolute size is checked
        tiny = nb < 2e-2 * scale
        if not (err < 3e-4 * max(nb, 1e-3 * scale) or (tiny and err < 2e-2 * scale)):
            bad.append((i, tuple(b.shape), err, nb, scale))
    assert not bad, f"gradient mismatches (index, shape, abs err, norm): {bad}"


@pytest.mark.parametrize("name,cfg_file,B,seed", [("bat", "BAT_Car.yaml", 2, 21), ("p2b", "P2B_Car.yaml", 2, 22)])
def test_whole_model_against_reference_golden(gmod, mode, name, cfg_file, B, seed):
    cfg = load_config(os.path.join(ROOT, "cfgs", cfg_file))
    net = get_model(cfg.net_model)(cfg)
    base = det_state_dict(net.state_dict(), seed=seed)
    net.load_state_dict(base)
    net = net.cuda().train()
    batch = synthetic_siamese_batch(B, 256, 512, seed=1234 + seed, box_aware=(name == "bat"), device="cuda")
    batch["box_label"] = torch.tensor(gmod[f"{name}_box_label"], device="cuda")
    # P2B (2 pairs of 256 / 512 points): BatchNorm over few positions amplifies round-off — the reference's own composition on
    # torch CUDA ops deviates from its CPU run by 3e-4 here — hence its wider bars below
    # The bounds below leave headroom for such flips; the full-size, flip-free comparison is tests/test_gpu_parity_full.py.
    with torch.no_grad():
        ep = net(batch)
    assert np.array_equal(ep["sample_idxs"].cpu().numpy(), gmod[f"{name}_sample_idxs"])
    tight = 2e-4 if name == "bat" else 1e-2
    print(f"\n[golden {name} {mode}] train fwd: " + ", ".join(f"{k} {rel(ep[k], gmod[f'{name}_{k}']):.1e}" for k in
                                                            ("estimation_cla", "vote_xyz", "center_xyz", "estimation_boxes")))
    for k in ("estimation_cla", "vote_xyz", "center_xyz"):
        assert rel(ep[k], gmod[f"{name}_{k}"]) < tight, k
    assert rel(ep["estimation_boxes"], gmod[f"{name}_estimation_boxes"]) < tight
    net.load_state_dict(base)
    net.eval()
    with torch.no_grad():
        ep = net(batch)
    print(f"[golden {name} {mode}] eval boxes {rel(ep['estimation_boxes'], gmod[f'{name}_eval_boxes']):.1e}")
    assert rel(ep["estimation_boxes"], gmod[f"{name}_eval_boxes"]) < 2e-4
    net.load_state_dict(base)
    net.train()
    loss = net.training_step({k: v.clone() for k, v in batch.items()}, 0)
    print(f"[golden {name} {mode}] loss {rel(loss, gmod[f'{name}_loss']):.1e}")
    assert rel(loss, gmod[f"{name}_loss"]) < (1e-4 if name == "bat" else 1e-3)
    loss.backward()
    sd = dict(net.named_parameters())
    norms = np.array([float(sd[k].grad.norm()) for k in sorted(sd)])
    assert np.all(np.isfinite(norms))
    ref = gmod[f"{name}_gradnorms"]
    big = ref > 1e-3 * ref.max()
    # layer-wise gradient norms track the reference (P2B at B=1 is the round-off-amplifying case, see above)
    assert np.median(np.abs(norms[big] - ref[big]) / ref[big]) < (2e-2 if name == "bat" else 2e-1)


def test_m2track_fused_matches_reference_golden(gmod):
    """M2-Track (BASELINE.json configs[2]) on the fused kernels.  Its forward contains two arg-max decisions (point
    mask, motion state), so: (a) every dense net is held to 2e-4 against the composed (plain torch) mirror on identical
    inputs; (b) the segmentation logits — upstream of any discrete decision — are held to 2e-4 against the REFERENCE's
    own CPU run; (c) the final boxes / loss, downstream of the arg-maxes, to 2e-2."""
    from open3dsot_b200.datasets.synthetic import synthetic_motion_batch
    cfg = load_config(os.path.join(ROOT, "cfgs", "M2_track_kitti.yaml"))
    net = get_model(cfg.net_model)(cfg)
    base = det_state_dict(net.state_dict(), seed=31)
    batch = synthetic_motion_batch(4, 256, seed=77, device="cuda")
    net.load_state_dict(base)
    net = net.cuda().train()
    x = torch.cat([batch["points"].transpose(1, 2), batch["candidate_bc"].transpose(1, 2)], dim=1).contiguous()
    mp_in = torch.randn(4, 13, 512, generator=torch.Generator().manual_seed(1)).cuda()
    outs = {}
    for mode in (False, True):
        runtime.set_fused(mode)
        try:
            net.load_state_dict(base)
            xin, min_ = x.clone().requires_grad_(True), mp_in.clone().requires_grad_(True)
            seg = net.seg_pointnet(xin)
            mini = net.mini_pointnet(min_)
            head = net._mlp(net.motion_mlp, mini)
            loss = seg.square().sum() + head.square().sum()
            params = list(net.seg_pointnet.parameters()) + list(net.mini_pointnet.parameters()) + list(net.motion_mlp.parameters())
            gr = torch.autograd.grad(loss, [xin, min_] + params)
            outs[mode] = ((seg, mini, head), gr)
        finally:
            runtime.set_fused(True)
    for a, b in zip(outs[True][0], outs[False][0]):
        assert rel(a, b) < 2e-4
    scale = max(float(g.norm()) for g in outs[False][1])
    for a, b in zip(outs[True][1], outs[False][1]):
        # nine BN/ReLU layers and two global max-pools deep: a handful of arg-max / ReLU-mask decisions within round-off
        # of their threshold differ between the two fp32 evaluations -> O(1e-3) relative on the gradients
        assert float((a.double() - b.double()).norm()) < 5e-3 * max(float(b.norm()), 2e-2 * scale)
    # whole model against the reference's CPU run
    net.load_state_dict(base)
    net.train()
    with torch.no_grad():
        ep = net({k: v.clone() for k, v in batch.items()})
    assert rel(ep["seg_logits"], gmod["m2_seg_logits"]) < 2e-4
    assert rel(ep["pred_bc"], gmod["m2_pred_bc"]) < 2e-4
    assert rel(ep["estimation_boxes"], gmod["m2_estimation_boxes"]) < 2e-2
    net.load_state_dict(base)
    loss = net.training_step({k: v.clone() for k, v in batch.items()}, 0)
    assert rel(loss, gmod["m2_loss"]) < 2e-2
    loss.backward()
    assert all(torch.isfinite(p.grad).all() for p in net.parameters() if p.grad is not None)
