"""Diagnostic: gradient agreement of the CUDA path with the float64 oracle under different execution modes."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import torch
from open3dsot_b200 import runtime
from open3dsot_b200.config import load_config
from open3dsot_b200.datasets.synthetic import synthetic_siamese_batch
from open3dsot_b200.models import get_model
from oracle import modules as om
from _params import det_state_dict
from test_gpu_parity_full import _oracle_run, Choices

torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False
name, cfg_file, B, M, N = sys.argv[1], sys.argv[2], int(sys.argv[3]), int(sys.argv[4]), int(sys.argv[5])
cfg = load_config(os.path.join("cfgs", cfg_file))
net = get_model(cfg.net_model)(cfg)
base = det_state_dict(net.state_dict(), seed=41)
pn = [k for k, _ in net.named_parameters()]
batch = synthetic_siamese_batch(B, M, N, seed=20260924, box_aware=(name == "bat"))
_, _, _, taps, g32 = _oracle_run(name, cfg, base, pn, batch)
bq = [taps[f"backbone.SA_modules.{i}:bq_idx"][br] for br in range(2) for i in range(3)] + [taps["rpn.vote_aggregation:bq_idx"][0]]
force = {"ball_query": bq, "topk": [taps["xcorr:topk"][0]] if name == "bat" else []}
_, _, _, _, g64 = _oracle_run(name, cfg, base, pn, batch, dtype=torch.float64, force=force)
den = sum(float(g64[k].norm()) ** 2 for k in pn) ** 0.5


def report(tag, g):
    num = sum(float((g[k].double().cpu() - g64[k]).norm()) ** 2 for k in pn) ** 0.5
    dot = sum(float((g[k].double().cpu() * g64[k]).sum()) for k in pn)
    print(f"{tag:28s} total rel err {num / den:.2e}   scale <g,g64>/<g64,g64> = {dot / den ** 2:.6f}")


report("oracle32", g32)
net = net.cuda().train()
dev = {k: v.cuda() for k, v in batch.items()}
inject = {("ball_query", 6): taps["rpn.vote_aggregation:bq_idx"][0]}
if name == "bat":
    inject[("boxaware_topk", 0)] = taps["xcorr:topk"][0]
MODES = [("fused lift tc3", True, True, 3), ("fused lift tc0", True, True, 0), ("fused nolift tc3", True, False, 3),
         ("fused nolift tc0", True, False, 0), ("composed (torch ops)", False, False, 0)]
for tag, fused_on, lift, tc in MODES:
    net.load_state_dict(base)
    net.zero_grad(set_to_none=True)
    runtime.set_fused(fused_on); runtime.set_lift(lift); runtime.set_tc(tc)
    runtime.CHOICE_HOOK = Choices(inject) if (fused_on and lift) else None
    try:
        loss = net.training_step({k: v.clone() for k, v in dev.items()}, 0)
        loss.backward()
    finally:
        runtime.CHOICE_HOOK = None
    report(tag, {k: p.grad.detach() for k, p in net.named_parameters()})
