"""fp32 (3xTF32) against bf16 (BF16 operands, FP32 accumulation) inference, in one process so that the two alternate on the same card.

  kernel   sa_fused_kernel on BAT-Car's three search-branch SA layers at K = 1, 32, 128 clouds, and the pw_tc forward on M2-Track's
           SegPointNet / MiniPointNet stacks at 2 x 1024 points per target for K = 1, 32, 128: CUDA events over a captured graph of
           `--reps` launches; achieved FLOP/s (2 * positions * sum cin * cout of the tensor-core layers) and its share of the
           H100 SXM data-sheet dense BF16 rate (989 TFLOP/s);
  e2e      evaluate_batched frames/s at 32 slots (BAT-Car, M2-Track) and MultiTargetTracker target-frames/s at K = 8, 32, 128 on
           60,000-point scans, fp32 and bf16 alternated;
  accuracy BAT-Car trained with Trainer for `--epochs` seeded epochs on synthetic tracklets (as tools/bench_train_loop.py sets
           them up), then the held-out synthetic split evaluated in fp32 and in bf16: Success / Precision, the per-frame box
           difference and the frame at which the two tracks first part; the untrained model's fp32 numbers are printed beside
           them, so whether the training produced a model that tracks is visible.

The card's name and power limit are printed with the numbers; the JSON goes to stdout and to --out.

    python tools/bench_precision.py [--reps 50] [--epochs 40] [--out results/bench_precision.json]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from open3dsot_b200 import _lib, fused, runtime  # noqa: E402
from open3dsot_b200.config import load_config  # noqa: E402
from open3dsot_b200.datasets.synthetic import synthetic_scene, synthetic_sequence  # noqa: E402
from open3dsot_b200.models import get_model  # noqa: E402
from open3dsot_b200.pointnet2.utils.pointnet2_modules import PointnetSAModule  # noqa: E402
from open3dsot_b200.tracking.evaluate import evaluate_batched  # noqa: E402
from open3dsot_b200.tracking.multi_tracker import MultiTargetTracker  # noqa: E402

BF16_PEAK = 989e12
PRECISIONS = ("fp32", "bf16")


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def graph_ms(fn, reps, windows=3):
    """per-call device milliseconds of fn() captured `reps` times in one CUDA graph (warm-up first); min and max over windows"""
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            fn()
    g.replay()
    torch.cuda.synchronize()
    out = []
    for _ in range(windows):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        g.replay()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b) / reps)
    return min(out), max(out)


# BAT-Car search branch: (N, C, mlp, npoint, radius, nsample)
SA_LAYERS = [("sa1", 1024, 0, [0, 64, 64, 128], 512, 0.3, 32), ("sa2", 512, 128, [128, 128, 128, 256], 256, 0.5, 32),
             ("sa3", 256, 256, [256, 256, 256, 256], 128, 0.7, 32)]


def bench_sa(reps):
    rows = []
    for name, N, C, mlp, npoint, radius, S in SA_LAYERS:
        torch.manual_seed(0)
        sa = PointnetSAModule(mlp=list(mlp), radius=radius, nsample=S, use_fps=False).cuda().eval()
        specs = fused.parse_stack(sa.mlps[0])
        flops_pos = sum(2 * (s.weight.shape[1] - (3 if l == 0 else 0)) * s.weight.shape[0] for l, s in enumerate(specs))
        for K in (1, 32, 128):
            g = torch.Generator().manual_seed(K)
            xyz = (torch.rand(K, N, 3, generator=g) * 1.2).cuda()
            feat_cl = fused.to_channels_last(torch.randn(K, C, N, generator=g).cuda()) if C else None
            new_xyz = xyz[:, :npoint].contiguous()
            meta = fused._Meta(specs, S, False, xyz_first=True, c0=C)
            ldo = fused._r4(mlp[-1])
            out = torch.empty(K, npoint, ldo, device="cuda")
            row = {"layer": name, "K": K, "positions": K * npoint * S}
            for prec in PRECISIONS:
                d = fused._describe(meta, K * npoint * S, fused._r4(C) + 4, meta.params)
                d.precision = _lib.PRECISION_BF16 if prec == "bf16" else _lib.PRECISION_TF32X3
                block = fused._sa_fused_prepare(d, xyz.device)
                L = _lib.lib()

                def call(d=d, block=block):
                    _lib.check(L.o3d_sa_fused_forward(ctypes.byref(d), block.data_ptr(), xyz.data_ptr(), new_xyz.data_ptr(),
                                                      None if feat_cl is None else feat_cl.data_ptr(),
                                                      0 if feat_cl is None else feat_cl.shape[2], K, N, npoint, float(radius), S, 0,
                                                      out.data_ptr(), ldo, None, torch.cuda.current_stream().cuda_stream),
                               "o3d_sa_fused_forward")
                lo, hi = graph_ms(call, reps)
                tflops = flops_pos * row["positions"] / (lo * 1e-3) / 1e12
                row[prec] = {"us": lo * 1e3, "us_max": hi * 1e3, "tflops": tflops, "bf16_roof_share": tflops * 1e12 / BF16_PEAK}
            row["speedup"] = row["fp32"]["us"] / row["bf16"]["us"]
            rows.append(row)
            print(json.dumps(row), flush=True)
    return rows


def _seq(widths):
    layers = []
    for cin, cout in zip(widths[:-1], widths[1:]):
        layers += [torch.nn.Conv1d(cin, cout, 1), torch.nn.BatchNorm1d(cout), torch.nn.ReLU()]
    return torch.nn.Sequential(*layers).cuda().eval()


# M2-Track (cfgs/M2_track_kitti.yaml): SegPointNet's per-point stack up to the pooled 1024-channel layer and its per-point head,
# MiniPointNet's per-point stack; 2 x 1024 points per target
PW_STACKS = [("seg_pooled", [64, 64, 128, 1024], 64), ("seg_head", [1088, 512, 256, 128], 0), ("mini", [64, 128, 256], 64)]


def bench_pw(reps):
    rows = []
    for name, widths, S in PW_STACKS:
        torch.manual_seed(0)
        seq = _seq(widths)
        specs = fused.parse_stack(seq)
        for K in (1, 32, 128):
            P = K * 2048
            x = torch.randn(P, widths[0], device="cuda")
            flops = 2.0 * P * sum(a * b for a, b in zip(widths[:-1], widths[1:]))
            row = {"stack": name, "K": K, "positions": P}
            for prec in PRECISIONS:
                with torch.no_grad(), runtime.static_weights_scope(), runtime.inference_precision_scope(prec):
                    lo, hi = graph_ms(lambda: fused.mlp_stack(x, specs, S, False), reps)
                tflops = flops / (lo * 1e-3) / 1e12
                row[prec] = {"us": lo * 1e3, "us_max": hi * 1e3, "tflops": tflops, "bf16_roof_share": tflops * 1e12 / BF16_PEAK}
            row["speedup"] = row["fp32"]["us"] / row["bf16"]["us"]
            rows.append(row)
            print(json.dumps(row), flush=True)
    return rows


def _model(cfg_name, **over):
    cfg = load_config(os.path.join(ROOT, "cfgs", cfg_name), {"up_axis": [0, 0, 1], **over})
    torch.manual_seed(0)
    return get_model(cfg.net_model)(cfg).cuda().eval()


def bench_e2e(rounds):
    out = {"evaluate_batched": {}, "multi_target": {}}
    tracks = [synthetic_sequence(n_frames=40, n_points=20000, seed=700 + i, speed=0.4, yaw_rate=1.0) for i in range(64)]
    frames = sum(len(t) for t in tracks)
    for cfg_name in ("BAT_Car.yaml", "M2_track_kitti.yaml"):
        net = _model(cfg_name)
        res = {p: [] for p in PRECISIONS}
        for p in PRECISIONS:
            evaluate_batched(net, tracks[:8], slots=32, seed=0, precision=p)       # warm-up: graphs and blocks
        for _ in range(rounds):
            for p in PRECISIONS:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                evaluate_batched(net, tracks, slots=32, seed=0, precision=p)
                res[p].append(frames / (time.perf_counter() - t0))
        out["evaluate_batched"][cfg_name] = {"frames_per_s": res, "frames": frames, "slots": 32,
                                             "speedup": max(res["bf16"]) / max(res["fp32"])}
        print(json.dumps({cfg_name: out["evaluate_batched"][cfg_name]}), flush=True)
    net = _model("BAT_Car.yaml")
    warm, timed = 3, 10
    scene = synthetic_scene(n_frames=2 + warm + timed, n_points=60000, n_objects=128, seed=7, extent=70.0)
    scans = [torch.tensor(s, device="cuda") for s in scene["scans"]]
    for K in (8, 32, 128):
        res = {p: [] for p in PRECISIONS}
        for _ in range(rounds):
            for p in PRECISIONS:
                trk = MultiTargetTracker(net, 60000, K, seed=0, precision=p)
                trk.step(scans[0])
                for j in range(K):
                    trk.add(j, scene["boxes"][j][0])
                for i in range(warm):
                    trk.step(scans[1 + i])
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for i in range(timed):
                    trk.step(scans[1 + warm + i])
                b.record()
                b.synchronize()
                res[p].append(K * timed / (a.elapsed_time(b) / 1e3))
                del trk
        out["multi_target"][K] = {"target_frames_per_s": res, "speedup": max(res["bf16"]) / max(res["fp32"])}
        print(json.dumps({"multi_target_K": K, **out["multi_target"][K]}), flush=True)
    return out


def bench_accuracy(epochs, seconds):
    from open3dsot_b200.trainer import Trainer
    cfg = load_config(os.path.join(ROOT, "cfgs", "BAT_Car.yaml"), {"up_axis": [0, 0, 1], "batch_size": 48, "epoch": 10 ** 6})
    train = [synthetic_sequence(n_frames=20, n_points=20000, seed=20260924 + i) for i in range(48)]
    rng = np.random.default_rng(20261016)
    val = [synthetic_sequence(n_frames=int(n), n_points=20000, seed=1000 + i, speed=0.3 + 0.4 * rng.random(),
                              yaw_rate=4 * rng.random() - 2) for i, n in enumerate(rng.integers(20, 80, 32))]
    torch.manual_seed(0)
    net = get_model(cfg.net_model)(cfg).cuda()
    untrained = evaluate_batched(net.eval(), val, slots=32, seed=0)
    tr = Trainer(net.train(), cfg, train, val, log_dir=None, slots=32)
    t0, done = time.perf_counter(), 0
    while done < epochs and time.perf_counter() - t0 < seconds:
        tr.train_epoch()
        done += 1
    net.eval()
    res = {p: evaluate_batched(net, val, slots=32, seed=0, precision=p) for p in PRECISIONS}
    diffs, first_any, first_far = [], [], []
    for a, b in zip(res["fp32"]["results"], res["bf16"]["results"]):
        d = np.array([np.abs(np.asarray(x.center) - np.asarray(y.center)).max() for x, y in zip(a, b)])
        diffs.append(d)
        first_any.append(int(np.argmax(d > 0)) if (d > 0).any() else None)
        first_far.append(int(np.argmax(d > 0.1)) if (d > 0.1).any() else None)
    allf = np.concatenate(diffs)
    out = {"epochs": done, "train_seconds": time.perf_counter() - t0,
           "untrained_fp32": {"success": untrained["success"], "precision": untrained["precision"]},
           "fp32": {"success": res["fp32"]["success"], "precision": res["fp32"]["precision"]},
           "bf16": {"success": res["bf16"]["success"], "precision": res["bf16"]["precision"]},
           "center_diff_m": {"median": float(np.median(allf)), "p99": float(np.quantile(allf, 0.99)), "max": float(allf.max())},
           "first_frame_differs": first_any, "first_frame_over_0.1m": first_far,
           "val": {"tracklets": len(val), "frames": res["fp32"]["frames"]}}
    print(json.dumps({"accuracy": out}), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=2, help="fp32 / bf16 alternations of every end-to-end measurement")
    ap.add_argument("--epochs", type=int, default=40)
    ap.add_argument("--train-seconds", type=float, default=420.0, help="stop training after this long (epochs done are reported)")
    ap.add_argument("--skip", default="", help="comma list of sections to skip: kernel, e2e, accuracy")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_precision.py needs a CUDA device")
    skip = set(filter(None, a.skip.split(",")))
    res = {"gpu": card()}
    print(json.dumps(res), flush=True)
    if "kernel" not in skip:
        res["sa_fused"] = bench_sa(a.reps)
        res["pw_tc"] = bench_pw(a.reps)
    if "e2e" not in skip:
        res["e2e"] = bench_e2e(a.rounds)
    if "accuracy" not in skip:
        res["accuracy"] = bench_accuracy(a.epochs, a.train_seconds)
    res["gpu_after"] = card()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
