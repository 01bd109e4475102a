"""Whole-model inference (eval mode, no autograd) through the execution variants the tracking loop uses — all on identical
weights and inputs:

  * template / search branches on two streams (fused.run_ahead) vs one stream: the SAME kernels on the same data -> bitwise equal;
  * every SA layer as one kernel (csrc/sa_fused.cu) vs the multi-kernel path: 1e-4;
  * the forward captured in a CUDA graph and replayed (two parallel graph branches) vs eager: bitwise equal, replay after replay;
  * the same capture with every static-weight block built privately during the capture (nothing cached beforehand);
  * static-weight caches (prepared parameter blocks): invalidated by an in-place update of the weights or of the running
    BatchNorm statistics.
BAT (box-aware fusion) and P2B (cosine fusion), B = 1 (the tracker's shape) and B = 3."""
import os

import pytest
import torch

from _params import det_state_dict
from open3dsot_b200 import runtime
from open3dsot_b200.config import load_config
from open3dsot_b200.datasets.synthetic import synthetic_siamese_batch
from open3dsot_b200.models import get_model

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEYS = ("estimation_boxes", "estimation_cla", "vote_xyz", "center_xyz")


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _model(cfg_file, seed):
    cfg = load_config(os.path.join(ROOT, "cfgs", cfg_file))
    net = get_model(cfg.net_model)(cfg)
    net.load_state_dict(det_state_dict(net.state_dict(), seed=seed))
    g = torch.Generator().manual_seed(seed + 1)
    for n, b in net.named_buffers():                         # running statistics as after training, not (0, 1)
        if n.endswith("running_mean"):
            b.copy_(torch.randn(b.shape, generator=g) * 0.1)
        elif n.endswith("running_var"):
            b.copy_(torch.rand(b.shape, generator=g) * 0.5 + 0.75)
    return net.cuda().eval()


def _forward(net, batch, overlap=True, sa_fused=True):
    runtime.set_branch_overlap(overlap)
    runtime.set_sa_fused(sa_fused)
    try:
        with torch.no_grad():
            out = net(batch)
        torch.cuda.synchronize()
        return {k: out[k].clone() for k in KEYS}
    finally:
        runtime.set_branch_overlap(True)
        runtime.set_sa_fused(True)


@pytest.mark.parametrize("cfg_file,B", [("BAT_Car.yaml", 1), ("BAT_Car.yaml", 3), ("P2B_Car.yaml", 1), ("P2B_Car.yaml", 3)])
def test_branch_overlap_is_bitwise_and_fused_sa_within_tolerance(cfg_file, B):
    net = _model(cfg_file, seed=31)
    batch = synthetic_siamese_batch(B, 512, 1024, seed=5, device="cuda")
    a = _forward(net, batch, overlap=True)
    b = _forward(net, batch, overlap=False)
    for k in KEYS:
        assert torch.equal(a[k], b[k]), f"{k}: two-stream execution changed the result"
    c = _forward(net, batch, overlap=False, sa_fused=False)
    for k in ("estimation_cla", "vote_xyz"):
        assert rel(a[k], c[k]) < 1e-4, f"{k}: single-kernel SA layers vs multi-kernel path {rel(a[k], c[k]):.2e}"
    # proposals are selected by a ball query of computed votes: compare only when both paths picked the same neighbours
    if torch.equal(a["center_xyz"], c["center_xyz"]):
        assert rel(a["estimation_boxes"], c["estimation_boxes"]) < 1e-3


@pytest.mark.parametrize("cfg_file,warm_caches", [("BAT_Car.yaml", True), ("P2B_Car.yaml", True), ("BAT_Car.yaml", False),
                                                   ("P2B_Car.yaml", False)],
                         ids=["BAT_Car.yaml", "P2B_Car.yaml", "BAT_Car.yaml-cold_caches", "P2B_Car.yaml-cold_caches"])
def test_graph_capture_with_two_branches_replays_bitwise(cfg_file, warm_caches):
    net = _model(cfg_file, seed=33)
    b1 = synthetic_siamese_batch(1, 512, 1024, seed=6, device="cuda")
    b2 = synthetic_siamese_batch(1, 512, 1024, seed=7, device="cuda")
    static = {k: v.clone() for k, v in b1.items() if torch.is_tensor(v)}
    with torch.no_grad():
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            if warm_caches:
                with runtime.static_weights_scope():
                    net(static)                              # warm-up: caches filled outside the capture
            else:
                net(static)                                  # warm-up without the scope: kernels load, nothing is cached
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with runtime.static_weights_scope(), torch.cuda.graph(g):
            out = net(static)                                # cold caches: every static-weight block is built in the graph
        for batch in (b1, b2, b1):
            for k in static:
                static[k].copy_(batch[k])
            g.replay()
            torch.cuda.synchronize()
            got = {k: out[k].clone() for k in KEYS}
            want = _forward(net, batch)
            for k in KEYS:
                assert torch.equal(got[k], want[k]), f"{k}: graph replay differs from the eager forward"


def _check_static_weight_caches_follow(update, what):
    net = _model("BAT_Car.yaml", seed=35)
    batch = synthetic_siamese_batch(1, 512, 1024, seed=8, device="cuda")
    with torch.no_grad(), runtime.static_weights_scope():
        a = {k: net(batch)[k].clone() for k in KEYS}
        a2 = {k: net(batch)[k].clone() for k in KEYS}       # second call: served from the cached blocks
        for k in KEYS:
            assert torch.equal(a[k], a2[k])
        update(net)
        b = {k: net(batch)[k].clone() for k in KEYS}
    fresh = _forward(net, batch)                             # no cache involved
    for k in KEYS:
        assert torch.equal(b[k], fresh[k]), f"{k}: a stale prepared block was used after the {what} changed"
    assert not torch.equal(a["estimation_cla"], b["estimation_cla"])


def _scale_parameters(net):
    for p in net.parameters():
        p.mul_(1.01)                                         # bumps every parameter's version counter


def _shift_running_statistics(net):
    for n, b in net.named_buffers():                         # parameters untouched: only the folded statistics move
        if n.endswith("running_mean"):
            b.add_(0.05)
        elif n.endswith("running_var"):
            b.mul_(1.1)


def test_static_weight_caches_follow_in_place_updates():
    _check_static_weight_caches_follow(_scale_parameters, "weights")


def test_static_weight_caches_follow_in_place_running_statistics_updates():
    _check_static_weight_caches_follow(_shift_running_statistics, "running statistics")
