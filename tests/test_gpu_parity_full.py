"""Full-size, flip-free parity of the CUDA path against the CPU oracle (oracle/modules.py, itself pinned to the reference's
own Python through tests/golden/*) at BASELINE.json's shapes:

  configs[1]  BAT_Car   48 pairs x 512 / 1024 points  (forward, loss, every parameter gradient)
  configs[3]  P2B_Car   8 pairs x 512 / 1024 points   (B >= 2: B = 1 is a degenerate BatchNorm case)
  configs[4]  BAT_PEDESTRIAN_NUSCENES at 256 / 512 points, 16 pairs
  configs[2]  M2_track_kitti 64 x 2048 points: the dense nets upstream of its arg-max decisions, against the host mirror in
              composed mode on the CPU (which tests/test_oracle_golden.py holds to the reference's own CPU run)

Method.  Index tensors (FPS, every backbone ball query) must be bit-exact.  The forward then takes two kinds of discrete
decisions on COMPUTED values — the RPN's ball query over voted coordinates and BoxAwareXCorr's top-k over predicted box
clouds — where a candidate within fp32 round-off of the threshold may legitimately fall the other way on the GPU.  The
product's own choices are recorded and their agreement with the oracle's is reported; then the oracle's choices are INJECTED
(runtime.CHOICE_HOOK) so that every float tensor — each SA layer's output, the xcorr output, seeds, votes, proposals, the
loss terms and every parameter gradient — is compared with identical discrete choices.  Tolerances are the measured ones,
stated next to each assert."""
import os

import numpy as np
import pytest
import torch

from open3dsot_b200 import runtime
from open3dsot_b200.config import load_config
from open3dsot_b200.datasets.synthetic import synthetic_siamese_batch
from open3dsot_b200.models import get_model
from oracle import modules as om
from _params import det_state_dict

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


class Choices:
    """CHOICE_HOOK: records the product's discrete choices in call order; substitutes the oracle's where asked."""

    def __init__(self, inject):
        self.inject = inject          # {(kind, call_number): tensor}
        self.seen = {}                # kind -> [product's own tensors, call order]

    def __call__(self, kind, info, compute):
        own = compute()
        n = len(self.seen.setdefault(kind, []))
        self.seen[kind].append(own)
        sub = self.inject.get((kind, n))
        return own if sub is None else sub.to(own.device).view_as(own).contiguous()


def _oracle_run(name, cfg, base, pnames, batch, dtype=torch.float32, force=None):
    cast = lambda v: v.clone().to(dtype) if v.is_floating_point() else v.clone()   # noqa: E731
    sd = {k: cast(v) for k, v in base.items()}
    for k in pnames:
        sd[k].requires_grad_(True)
    om.TAPS = {}
    om.set_force(force)
    try:
        trn = om.bat_training_loss if name == "bat" else om.p2b_training_loss
        loss, ld, out = trn(sd, cfg, {k: cast(v) for k, v in batch.items()})
        loss.backward()
        taps = om.TAPS
    finally:
        om.TAPS = None
        om.set_force(None)
    return loss.detach(), {k: v.detach() for k, v in ld.items()}, out, taps, {k: sd[k].grad for k in pnames}


CASES = [("bat", "BAT_Car.yaml", 48, 512, 1024), ("p2b", "P2B_Car.yaml", 8, 512, 1024),
         ("bat", "BAT_PEDESTRIAN_NUSCENES.yaml", 16, 256, 512)]


@pytest.mark.parametrize("name,cfg_file,B,M,N", CASES, ids=["bat_car_48x512x1024", "p2b_car_8x512x1024", "bat_ped_16x256x512"])
def test_full_size_parity_with_injected_choices(name, cfg_file, B, M, N):
    torch.set_num_threads(min(os.cpu_count() or 1, 32))
    cfg = load_config(os.path.join(ROOT, "cfgs", cfg_file))
    net = get_model(cfg.net_model)(cfg)
    base = det_state_dict(net.state_dict(), seed=41)
    pnames = [k for k, _ in net.named_parameters()]
    batch = synthetic_siamese_batch(B, M, N, seed=20260924, box_aware=(name == "bat"))
    o_loss, o_ld, o_out, taps, o_grads = _oracle_run(name, cfg, base, pnames, batch)

    net.load_state_dict(base)
    net = net.cuda().train()
    dev_batch = {k: v.cuda() for k, v in batch.items()}
    # ---- pass 1: the product's own discrete choices (nothing injected)
    hook = Choices({})
    runtime.CHOICE_HOOK = hook
    try:
        with torch.no_grad():
            ep = net({k: v.clone() for k, v in dev_batch.items()})
    finally:
        runtime.CHOICE_HOOK = None
    assert np.array_equal(ep["sample_idxs"].cpu().numpy(), o_out["sample_idxs"].numpy())        # FPS: bit-exact
    bq = hook.seen["ball_query"]                       # call order: template SA1-3, search SA1-3, RPN vote clustering
    assert len(bq) == 7
    for i in range(3):
        for br in range(2):                            # backbone ball queries run on INPUT coordinates: bit-exact
            assert torch.equal(bq[3 * br + i].cpu(), taps[f"backbone.SA_modules.{i}:bq_idx"][br]), (i, br)
    vote_agree = float((bq[6].cpu() == taps["rpn.vote_aggregation:bq_idx"][0]).float().mean())
    assert vote_agree > 0.99                           # computed coordinates: a few on-the-radius neighbours may differ
    inject = {("ball_query", 6): taps["rpn.vote_aggregation:bq_idx"][0]}
    if name == "bat":
        tk = hook.seen["boxaware_topk"][0].cpu()
        topk_agree = float((tk == taps["xcorr:topk"][0]).float().mean())
        assert topk_agree > 0.98                       # cdist's matmul formulation vs direct differences near ties
        inject[("boxaware_topk", 0)] = taps["xcorr:topk"][0]

    # ---- pass 2: oracle's choices injected; every float tensor, the loss terms and all gradients
    net.load_state_dict(base)
    outs = {}
    hs = []
    for i in range(3):
        hs.append(net.backbone.SA_modules[i].register_forward_hook(
            lambda m, a, o, i=i: outs.setdefault(f"sa{i}", []).append(o[1].detach())))
    hs.append(net.xcorr.register_forward_hook(lambda m, a, o: outs.setdefault("xcorr", []).append(o.detach())))
    hs.append(net.rpn.vote_aggregation.register_forward_hook(lambda m, a, o: outs.setdefault("vote_sa", []).append(o[1].detach())))
    ld = {}
    ref_compute = net.compute_loss

    def spy(data, output):
        d = ref_compute(data, output)
        ld.update({k: v.detach() for k, v in d.items()})
        outs["end_points"] = {k: v.detach() for k, v in output.items() if torch.is_tensor(v)}
        return d
    net.compute_loss = spy
    runtime.CHOICE_HOOK = Choices(inject)
    try:
        loss = net.training_step({k: v.clone() for k, v in dev_batch.items()}, 0)
        loss.backward()
    finally:
        runtime.CHOICE_HOOK = None
        for h in hs:
            h.remove()
    # the same oracle in float64 with the same discrete choices = the exact answer (yardstick for both forward and gradients)
    bq_forced = [taps[f"backbone.SA_modules.{i}:bq_idx"][br] for br in range(2) for i in range(3)] + [taps["rpn.vote_aggregation:bq_idx"][0]]
    force = {"ball_query": bq_forced, "topk": [taps["xcorr:topk"][0]] if name == "bat" else []}
    x_loss, x_ld, x_out, x_taps, x_grads = _oracle_run(name, cfg, base, pnames, batch, dtype=torch.float64, force=force)

    errs = {}      # name -> (CUDA vs float32 oracle, CUDA vs float64 oracle, float32 oracle vs float64 oracle)

    def cmp(key, ours, o32, o64):
        errs[key] = (rel(ours, o32), rel(ours, o64), rel(o32, o64))
    for i in range(3):
        for br in range(2):
            cmp(f"sa{i}[{br}]", outs[f"sa{i}"][br], taps[f"backbone.SA_modules.{i}:out"][br], x_taps[f"backbone.SA_modules.{i}:out"][br])
    cmp("xcorr", outs["xcorr"][0], taps["xcorr:out"][0], x_taps["xcorr:out"][0])
    cmp("vote_sa", outs["vote_sa"][0], taps["rpn.vote_aggregation:out"][0], x_taps["rpn.vote_aggregation:out"][0])
    ep = outs["end_points"]
    for k in ("estimation_cla", "vote_xyz", "center_xyz", "estimation_boxes") + (("pred_search_bc",) if name == "bat" else ()):
        cmp(k, ep[k], o_out[k], x_out[k])
    for k in o_ld:
        cmp(k, ld[k], o_ld[k], x_ld[k])
    cmp("loss", loss, o_loss, x_loss)
    print(f"\n[{name} {B}x{M}/{N}] vote ball-query agreement {vote_agree:.5f}"
          + (f", box-cloud top-k agreement {topk_agree:.5f}" if name == "bat" else "")
          + "; forward errors with injected choices (vs oracle32 / vs oracle64 / oracle32 vs oracle64): "
          + ", ".join(f"{k} {a:.1e}/{b:.1e}/{c:.1e}" for k, (a, b, c) in errs.items()))
    for k, (a, b, c) in errs.items():
        # north_star: 1e-4 relative on float features / votes.  Where the float32 oracle is itself further than 5e-5 from the exact
        # answer (deep head tensors at small batch), the CUDA path is required to be at least as close to exact as that.
        assert a < 1e-4 or b < max(1e-4, 1.5 * c), (k, a, b, c)

    # ---- gradients.  A gradient passes through ~40 ReLU masks and 8 max-pool selections; any two fp32 evaluations of the
    # network (different summation order is enough) put a few of the ~10^8 pre-activations on different sides of zero, and each
    # such flip adds or removes a FULL-SIZE gradient contribution: the relative difference between two correct fp32 gradients is
    # O(sqrt(flip fraction)) ~ 1e-3, not 1e-6.  So the yardstick is the oracle itself: the same oracle run in float64 with the
    # same discrete index choices is the exact answer, and the CUDA path must be as close to it as the oracle's own float32 run.
    params = dict(net.named_parameters())

    def total(ga):
        num = sum(float((ga[k].double().cpu() - x_grads[k]).norm()) ** 2 for k in pnames) ** 0.5
        return num / sum(float(x_grads[k].norm()) ** 2 for k in pnames) ** 0.5
    e_cuda = total({k: params[k].grad.detach() for k in pnames})
    e_o32 = total(o_grads)
    scale = max(float(x_grads[k].norm()) for k in pnames)
    relg = {k: float((params[k].grad.detach().cpu().double() - x_grads[k]).norm()) / max(float(x_grads[k].norm()), 1e-3 * scale)
            for k in pnames}
    relo = {k: float((o_grads[k].double() - x_grads[k]).norm()) / max(float(x_grads[k].norm()), 1e-3 * scale) for k in pnames}
    worst = sorted(relg.items(), key=lambda kv: -kv[1])[:3]
    print(f"[{name}] gradient error vs the float64 oracle over all {len(pnames)} parameters: CUDA path {e_cuda:.1e}, "
          f"float32 oracle {e_o32:.1e}; worst CUDA tensors: " + ", ".join(f"{k} {v:.1e} (oracle32 {relo[k]:.1e})" for k, v in worst))
    # A single marginal unit (e.g. in the 1,024-position proposal head of the pedestrian case) that any 1e-7 perturbation tips
    # moves the whole-model gradient error by ~1e-2 at once, whatever computed it.  Flip noise has a heavy tail, so the whole-model bound is a coarse one; the sharp gradient checks are the per-module ones
    # below (test_module_gradients_against_float64_oracle), where no chain of forty masks sits between the kernel and the number.
    assert e_cuda < max(4 * e_o32, 3e-2), (e_cuda, e_o32)


def test_m2track_dense_nets_full_size_against_cpu_mirror():
    """configs[2] shape (64 x 2048 points): the segmentation net and BoxCloud head — upstream of M2-Track's arg-max decisions
    — against the host mirror in composed mode (plain torch) on the CPU."""
    from open3dsot_b200.datasets.synthetic import synthetic_motion_batch
    cfg = load_config(os.path.join(ROOT, "cfgs", "M2_track_kitti.yaml"))
    net = get_model(cfg.net_model)(cfg)
    base = det_state_dict(net.state_dict(), seed=31)
    batch = synthetic_motion_batch(64, 1024, seed=77)
    torch.set_num_threads(min(os.cpu_count() or 1, 32))
    with runtime.composed_mode():
        net.load_state_dict(base)
        net.train()
        with torch.no_grad():
            ref = net({k: v.clone() for k, v in batch.items()})
    net.load_state_dict(base)
    net = net.cuda().train()
    with torch.no_grad():
        ep = net({k: v.cuda() for k, v in batch.items()})
    assert tuple(ep["seg_logits"].shape) == tuple(ref["seg_logits"].shape) and ep["seg_logits"].shape[-1] == 2048
    e_seg, e_bc = rel(ep["seg_logits"], ref["seg_logits"]), rel(ep["pred_bc"], ref["pred_bc"])
    print(f"\n[m2track 64x2048] seg_logits {e_seg:.1e}, pred_bc {e_bc:.1e}")
    assert e_seg < 1e-4 and e_bc < 1e-4


# ---- per-module gradients against the float64 oracle, at the shapes of BASELINE.json's configs ---------------------------------
SA_SHAPES = [  # B, N, C, mlp, npoint, nsample, radius   (SA1 / SA2 / SA3 of the search and template branches, car and pedestrian)
    (48, 1024, 0, [0, 64, 64, 128], 512, 32, 0.3), (48, 512, 128, [128, 128, 128, 256], 256, 32, 0.5),
    (48, 256, 256, [256, 256, 256, 256], 128, 32, 0.7), (16, 64, 256, [256, 256, 256, 256], 32, 32, 0.7),
    (16, 256, 0, [0, 64, 64, 128], 128, 32, 0.3)]


@pytest.mark.parametrize("shape", SA_SHAPES, ids=[f"B{s[0]}_N{s[1]}_C{s[2]}" for s in SA_SHAPES])
def test_sa_layer_gradients_against_float64_oracle(shape):
    """One set-abstraction layer (ball query + lifted first layer + wgmma GEMMs + max-pool), forward and EVERY gradient, against
    the oracle composition evaluated in float64.  Without a flipped ReLU / arg-max decision the error is at fp32 round-off; every
    decision at its threshold adds ~1e-4, and the 48-cloud shapes (up to 1.6e6 positions x 3 layers of units) collect a handful.
    The bar is 2e-3; a wrong kernel shows as O(1e-1)."""
    from open3dsot_b200.pointnet2.utils.pointnet2_modules import PointnetSAModule
    B, N, C, mlp, npoint, S, r = shape
    g = torch.Generator().manual_seed(N + C)
    xyz = synthetic_siamese_batch(B, 512, 1024, seed=3)["search_points"][:, :N].contiguous()      # resampled points: exact duplicates
    feats = torch.randn(B, max(C, 1), N, generator=g)
    sa = PointnetSAModule(mlp=list(mlp), radius=r, nsample=S, use_fps=False)
    base = det_state_dict(sa.state_dict(), seed=1)
    pn = [k for k, _ in sa.named_parameters()]
    sd = {"sa." + k: (v.clone().double() if v.is_floating_point() else v.clone()) for k, v in base.items()}
    for k in pn:
        sd["sa." + k].requires_grad_(True)
    f64 = feats.double().requires_grad_(True)
    _, y64, _ = om.sa_module(sd, "sa", xyz.double(), f64 if C else None, npoint, r, S, False, True)
    w = torch.linspace(0.5, 1.5, y64.shape[1], dtype=torch.float64)[None, :, None]
    (y64 * w).square().sum().backward()
    sa.load_state_dict(base)
    sa = sa.cuda().train()
    f = feats.cuda().requires_grad_(True)
    _, y = sa(xyz.cuda(), f if C else None, npoint)
    (y * w.float().cuda()).square().sum().backward()
    assert rel(y, y64) < 1e-5
    den = sum(float(sd["sa." + k].grad.norm()) ** 2 for k in pn) ** 0.5
    num = sum(float((p.grad.double().cpu() - sd["sa." + k].grad).norm()) ** 2 for k, p in sa.named_parameters()) ** 0.5
    print(f"\n[SA {shape[:3]}] forward {rel(y, y64):.1e}, parameter gradients {num / den:.1e}"
          + (f", feature gradient {rel(f.grad, f64.grad):.1e}" if C else ""))
    assert num / den < 2e-3
    if C:
        assert rel(f.grad, f64.grad) < 2e-3
