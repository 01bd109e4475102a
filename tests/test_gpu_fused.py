"""The fused point-wise MLP kernels (csrc/pwmlp.cu through open3dsot_b200.fused.mlp_stack) against a plain
fp64 PyTorch statement of the same stack (1x1 conv -> BatchNorm(train|eval) -> ReLU -> max over groups), forward
and backward, including ragged P, Cout not a multiple of 4, negative BN gammas and every group size in use."""
import zlib

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from open3dsot_b200 import fused
from open3dsot_b200.pointnet2.utils import pytorch_utils as pt

pytestmark = pytest.mark.gpu
RTOL = 1e-4


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def reference_stack(x, specs, S, training, batch_stats=None):
    """fp64 statement of the stack on a (P, K) matrix; returns output and leaves grads to autograd.  The max over a pooling
    group sends its gradient to the FIRST position holding the maximum (as F.max_pool2d does), whatever max(dim) would pick
    among exact ties.  `batch_stats`, a list, receives (mean, unbiased variance) of every training-mode BatchNorm."""
    h = x.double()
    for s in specs:
        W = s.weight.reshape(s.weight.shape[0], -1).double()
        h = h[:, :W.shape[1]] @ W.t()
        if s.bias is not None:
            h = h + s.bias.double()
        if s.bn is not None:
            if training:
                mu, var = h.mean(0), h.var(0, unbiased=False)
                if batch_stats is not None:
                    batch_stats.append((mu.detach(), h.var(0, unbiased=True).detach()))
            else:
                mu, var = s.bn.running_mean.double(), s.bn.running_var.double()
            h = (h - mu) / torch.sqrt(var + s.bn.eps) * s.bn.weight.double() + s.bn.bias.double()
        if s.relu:
            h = F.relu(h)
    if S > 0:
        g = h.view(-1, S, h.shape[1])
        mx = g.detach().max(dim=1, keepdim=True)[0]
        first = (g.detach() == mx).to(torch.uint8).argmax(dim=1, keepdim=True)   # argmax returns the first maximal index
        h = g.gather(1, first).squeeze(1)
    return h


def check_grads(g_out, g_ref, S, xshape, max_flips=3):
    """Gradients must agree to 2e-4 relative.  One bounded exception: a discrete decision that sits within fp32
    round-off of its threshold — two positions of a pooling group with (almost) equal values, or a pre-activation within
    ~1e-6 of zero — can fall the other way in the fp32 kernels than in the fp64 reference.  That moves ONE element's
    gradient, i.e. it shows up as an error confined to a few rows of the input gradient (and an O(1e-3) ripple in the
    parameter gradients).  At most `max_flips` such rows / pooling groups are accepted (0 where the inputs hold exact ties,
    which both sides must break the same way)."""
    scale = max(float(g.double().norm()) for g in g_ref if g is not None)
    tol = 2e-4
    if g_ref[0] is not None:
        rows = S if S > 0 else 1
        e = (g_out[0].double() - g_ref[0].double()).reshape(-1, rows, xshape[1]).norm(dim=(1, 2))
        thr = 2e-4 * float(g_ref[0].double().norm()) / max(e.numel(), 1) ** 0.5
        flipped = int((e > 50 * thr).sum())
        assert flipped <= max_flips, f"{flipped} rows / pooling groups disagree with the reference"
        if flipped:
            tol = 1e-2
    for gn, gr in zip(g_out, g_ref):
        if gr is None:
            continue
        err = float((gn.double() - gr.double()).norm())
        assert err < tol * max(float(gr.double().norm()), 1e-3 * scale), (tuple(gr.shape), err, float(gr.norm()))


def randomise(module, seed):
    g = torch.Generator().manual_seed(seed)
    for name, p in module.named_parameters():
        if p.dim() == 1 and "bn" in name and name.endswith("weight"):
            p.data = (0.5 + torch.rand(p.shape, generator=g)) * torch.where(torch.rand(p.shape, generator=g) < 0.2, -1.0, 1.0)
        elif p.dim() == 1:
            p.data = 0.2 * torch.randn(p.shape, generator=g)
    for name, b in module.named_buffers():
        if name.endswith("running_mean"):
            b.data = 0.1 * torch.randn(b.shape, generator=g)
        elif name.endswith("running_var"):
            b.data = 0.5 + torch.rand(b.shape, generator=g)


CASES = [
    # (channels, P, S, builder)
    ("sa1", [4, 64, 64, 128], 32 * 70, 32, "shared"),
    ("sa2", [132, 128, 128, 256], 32 * 37, 32, "shared"),
    ("rpn", [264, 256, 256, 256], 16 * 24, 16, "shared"),
    ("bax", [268, 256, 256, 256], 4 * 100, 4, "shared"),
    ("p2b", [260, 64, 64], 64 * 12, 64, "shared"),
    ("dense_bn_relu", [12, 16, 12], 333, 0, "shared"),
    ("seq_cla", [256, 256, 256, 1], 2 * 128 + 5, 0, "seq"),
    ("seq_prop", [256, 256, 5], 130, 0, "seq"),
    ("seq_vote", [260, 256, 259], 257, 0, "seq"),
]


@pytest.mark.parametrize("name,chans,P,S,kind", CASES)
@pytest.mark.parametrize("training", [True, False])
def test_mlp_stack_matches_fp64_reference(name, chans, P, S, kind, training):
    torch.manual_seed(zlib.crc32(name.encode()) % 1000)   # fixed per case (hash() is randomised per process)
    if kind == "shared":
        mod = pt.SharedMLP(list(chans), bn=True)
    else:
        mod = pt.Seq(chans[0])
        for c in chans[1:-1]:
            mod.conv1d(c, bn=True)
        mod.conv1d(chans[-1], activation=None)
    randomise(mod, 7)
    mod = mod.cuda()
    mod.train(training)
    specs = fused.parse_stack(mod)
    x = torch.randn(P, chans[0], device="cuda")
    x[:, -1] = 0  # the kernels see zero-padded channels; keep the same convention here
    x1 = x.clone().requires_grad_(True)
    rm_before = [s.bn.running_mean.clone() for s in specs if s.bn is not None]
    out = fused.mlp_stack(x1, specs, S, training)
    x2 = x.clone().requires_grad_(True)
    want = reference_stack(x2, specs, S, training)
    assert out.shape == want.shape
    assert rel(out, want) < RTOL
    if training:
        for s, before in zip([s for s in specs if s.bn is not None], rm_before):
            assert not torch.equal(s.bn.running_mean, before)      # running statistics were updated in place
    go = torch.randn_like(want)
    params = [p for p in mod.parameters()]
    g_ref = torch.autograd.grad(want, [x2] + params, go, allow_unused=True)
    g_out = torch.autograd.grad(out, [x1] + params, go.float(), allow_unused=True)
    check_grads(g_out, g_ref, S, x1.shape)


def test_running_stats_follow_torch_batchnorm():
    torch.manual_seed(0)
    mod = pt.SharedMLP([8, 16], bn=True).cuda().train()
    ref = nn.BatchNorm1d(16).cuda().train()
    x = torch.randn(640, 8, device="cuda")
    specs = fused.parse_stack(mod)
    fused.mlp_stack(x, specs, 0, True)
    y = x @ specs[0].weight.reshape(16, 8).t()
    ref(y)
    assert rel(specs[0].bn.running_mean, ref.running_mean) < 1e-5
    assert rel(specs[0].bn.running_var, ref.running_var) < 1e-5
    assert int(specs[0].bn.num_batches_tracked) == 1


# ---------------------------------------------------------------------------------------------- wgmma core
TC_CASES = [
    ("tc_sa2", [132, 128, 128, 256], 32 * 64, 32),
    ("tc_sa3", [260, 256, 256, 256], 32 * 37, 32),      # ragged P (1184 = 9.25 tiles), K = 260 (9 k-blocks, tail)
    ("tc_bax", [268, 256, 256, 256], 4 * 160, 4),
    ("tc_dense", [64, 128, 256], 300, 0),
    ("tc_sa1", [4, 64, 64, 128], 32 * 150, 32),         # 64-channel layers: one partial 128-row tile
]


@pytest.mark.parametrize("level", [1, 3])
@pytest.mark.parametrize("name,chans,P,S", TC_CASES + [("tc_wgrad_big", [260, 256, 256, 256], 32 * 160, 32)])
def test_tensor_core_stack_matches_fp64_reference(name, chans, P, S, level):
    """wgmma 3xTF32 forward + dgrad against the fp64 statement: same 1e-4 bar as the exact-fp32 kernels."""
    from open3dsot_b200 import runtime
    torch.manual_seed(3)
    mod = pt.SharedMLP(list(chans), bn=True)
    randomise(mod, 11)
    mod = mod.cuda().train()
    specs = fused.parse_stack(mod)
    x = torch.randn(P, chans[0], device="cuda")
    x[:, -1] = 0
    x1 = x.clone().requires_grad_(True)
    old = runtime.tc_level()
    runtime.set_tc(level)
    try:
        out = fused.mlp_stack(x1, specs, S, True)
        x2 = x.clone().requires_grad_(True)
        want = reference_stack(x2, specs, S, True)
        assert rel(out, want) < RTOL
        go = torch.randn_like(want)
        params = [p for p in mod.parameters()]
        g_ref = torch.autograd.grad(want, [x2] + params, go, allow_unused=True)
        g_out = torch.autograd.grad(out, [x1] + params, go.float(), allow_unused=True)
    finally:
        runtime.set_tc(old)
    check_grads(g_out, g_ref, S, x1.shape)
