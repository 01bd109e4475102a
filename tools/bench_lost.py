"""Cost of the live tracker's evidence: the in-box point count kernel alone, and the step it runs in.

  python tools/bench_lost.py [--steps 20] [--warmup 3] [--launches 200] [--out results.json]

For K = 1, 32 and 128 rows and N = 60,000 and 120,000-point scans:
  * "kernel": `o3d_box_points` alone, K rows over one shared scan (synthetic_scene, a box per row around one of its objects),
    --launches launches captured in one CUDA graph and timed with CUDA events over several replays after a warm-up replay;
    reported as microseconds per launch and point tests (K * N) per second;
  * "step": a MultiTargetTracker of K slots with every slot active, BAT-Car and M2-Track, one feed of device scans, --steps
    CUDA-event-timed `step()` calls after --warmup untimed ones; reported as milliseconds per step, and the kernel's time at
    the same (K, N) as a share of it.
Weights are untrained (the timing does not depend on them).  The card's name and power limit are printed with the numbers."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_multi_target import gpu_info, timed  # noqa: E402
from open3dsot_b200 import ops  # noqa: E402
from open3dsot_b200.config import load_config  # noqa: E402
from open3dsot_b200.datasets.synthetic import synthetic_scene  # noqa: E402
from open3dsot_b200.models import get_model  # noqa: E402
from open3dsot_b200.tracking import boxes as bx  # noqa: E402
from open3dsot_b200.tracking.multi_tracker import EVIDENCE_WLH_FACTOR, MultiTargetTracker  # noqa: E402

MODELS = {"bat_car": "BAT_Car.yaml", "m2track": "M2_track_kitti.yaml"}
SLOTS = (1, 32, 128)
POINTS = (60_000, 120_000)


def scene(N, K, frames):
    sc = synthetic_scene(n_frames=frames, n_points=N, n_objects=min(K, 32), seed=11, extent=60.0)
    return [torch.from_numpy(s).cuda() for s in sc["scans"]], sc["boxes"]


def kernel_us(scan, boxes, K, launches, reps=5):
    """Microseconds per `o3d_box_points` launch over K rows of one scan: `launches` launches in one graph, `reps` replays."""
    rows = [boxes[k % len(boxes)][0] for k in range(K)]
    center = torch.tensor([b.center for b in rows], dtype=torch.float32, device="cuda")
    rot = torch.tensor([b.rotation_matrix for b in rows], dtype=torch.float32, device="cuda")
    half = bx.inclusive_half(torch.tensor([b.wlh for b in rows], dtype=torch.float32, device="cuda"), EVIDENCE_WLH_FACTOR)
    scans = scan[None].contiguous()
    count = torch.tensor([scan.shape[0]], device="cuda")
    frame = torch.zeros(K, dtype=torch.int64, device="cuda")
    out = torch.empty(K, dtype=torch.int32, device="cuda")
    ops.box_points(scans, count, frame, center, rot, half, out=out)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(launches):
            ops.box_points(scans, count, frame, center, rot, half, out=out)
    g.replay()
    torch.cuda.synchronize()
    ms = timed(lambda i: g.replay(), reps)
    return ms * 1e3 / (reps * launches), int(out.sum())


def step_ms(net, scans, boxes, K, warmup, steps):
    trk = MultiTargetTracker(net, scans[0].shape[0], K, seed=0)
    trk.step(scans[0])
    for j in range(K):
        trk.add(j, boxes[j % len(boxes)][0])
    n = len(scans) - 1
    for i in range(warmup):
        trk.step(scans[1 + i % n])
    torch.cuda.synchronize()
    return timed(lambda i: trk.step(scans[1 + (warmup + i) % n]), steps) / steps


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--launches", type=int, default=200)
    p.add_argument("--out", default=None)
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lost: needs a CUDA device")
    gpu = gpu_info()
    print(f"GPU: {gpu}", flush=True)
    nets = {name: None for name in MODELS}
    for name, cfg_name in MODELS.items():
        cfg = load_config(os.path.join(ROOT, "cfgs", cfg_name), {"up_axis": [0, 0, 1], "degrees": True})
        torch.manual_seed(0)
        nets[name] = get_model(cfg.net_model)(cfg).cuda().eval()
    rows = []
    for N in POINTS:
        for K in SLOTS:
            scans, boxes = scene(N, K, 8)
            us, inside = kernel_us(scans[1], boxes, K, a.launches)
            row = {"N": N, "K": K, "kernel_us": us, "point_tests_per_s": K * N / (us * 1e-6), "points_in_boxes": inside}
            for name, net in nets.items():
                ms = step_ms(net, scans, boxes, K, a.warmup, a.steps)
                row[f"{name}_step_ms"] = ms
                row[f"{name}_kernel_share"] = us * 1e-3 / ms
            rows.append(row)
            print(json.dumps(row), flush=True)
            del scans
            torch.cuda.empty_cache()
    res = {"gpu": gpu, "rows": rows}
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
