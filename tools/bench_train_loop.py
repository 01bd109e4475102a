"""What the training loop costs beside the training step, on seeded synthetic tracklets (BAT-Car, bench.py's batch of 48).

Three per-step times, each over several windows so their spread is visible:
  step      `TrainStep.step` alone, replaying on one fixed batch (CUDA events);
  sampler   the device sampler's replay plus `TrainStep.step`, as bench.py's sampler mode pairs them (CUDA events);
  epoch     `Trainer.train_epoch()`: epoch-order indices, sampler replay, step and the on-device loss sums, with its one
            read-back per epoch (host clock around the epoch, which ends in that synchronising read-back).
And the validation seconds per epoch: `Trainer.test` over 144 synthetic tracklets of 10-200 frames at 32 slots.
The card's name and power limit are printed with the numbers.

    python tools/bench_train_loop.py [--batch 48] [--epochs 3] [--val-tracklets 144] [--val-points 20000]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from open3dsot_b200.config import load_config  # noqa: E402
from open3dsot_b200.datasets.synthetic import synthetic_sequence  # noqa: E402
from open3dsot_b200.models import get_model  # noqa: E402
from open3dsot_b200.trainer import Trainer  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        name, power = (s.strip() for s in out[0].split(","))
        return name, power
    except Exception as e:                                     # the numbers stay usable without the label
        return f"unknown ({e.__class__.__name__})", "unknown"


def timed(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=48)
    ap.add_argument("--epochs", type=int, default=3, help="timed epochs (after one warm-up epoch)")
    ap.add_argument("--train-tracklets", type=int, default=24)
    ap.add_argument("--train-frames", type=int, default=20)
    ap.add_argument("--train-points", type=int, default=20000)
    ap.add_argument("--val-tracklets", type=int, default=144)
    ap.add_argument("--val-points", type=int, default=20000)
    ap.add_argument("--slots", type=int, default=32)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train_loop.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    cfg = load_config(os.path.join(ROOT, "cfgs", "BAT_Car.yaml"), {"up_axis": [0, 0, 1], "batch_size": args.batch,
                                                                    "epoch": 10 ** 6})
    train = [synthetic_sequence(n_frames=args.train_frames, n_points=args.train_points, seed=20260924 + i)
             for i in range(args.train_tracklets)]
    rng = np.random.default_rng(20261016)
    lengths = np.exp(rng.uniform(np.log(10), np.log(200), args.val_tracklets)).round().astype(int)
    lengths[:2] = (10, 200)
    val = [synthetic_sequence(n_frames=int(n), n_points=args.val_points, seed=1000 + i, speed=0.3 + 0.4 * rng.random(),
                              yaw_rate=4 * rng.random() - 2) for i, n in enumerate(lengths)]
    torch.manual_seed(0)
    tr = Trainer(get_model(cfg.net_model)(cfg).to(dev), cfg, train, val, log_dir=None,
                 slots=args.slots)             # fit() is not called: nothing is written
    steps = len(tr.epoch_order(0)) // args.batch

    tr.train_epoch()                                            # warm-up: sampler graph, step warm-up and capture
    epoch_ms = []
    for _ in range(args.epochs):
        _, seconds, n = tr.train_epoch()
        epoch_ms.append(seconds / n * 1e3)
    fixed = tr.sampler.next_batch(args.batch)[0]
    fixed = {k: v.clone() for k, v in fixed.items()}
    step_ms = [timed(lambda: tr.step.step(fixed), steps) for _ in range(args.epochs)]
    sampler_ms = [timed(lambda: tr.step.step(tr.sampler.next_batch(args.batch)[0]), steps) for _ in range(args.epochs)]
    tr.test(val)                                                # warm-up: tracker graphs and static-weight blocks
    val_s = []
    for _ in range(2):
        tr.step.step(fixed)                                     # a training step in between, as in fit()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = tr.test(val)
        val_s.append(time.perf_counter() - t0)
    name, power = card()
    print(json.dumps({
        "workload": f"BAT_Car.yaml, batch {args.batch}, {args.train_tracklets} synthetic tracklets x {args.train_frames} scans of "
                    f"{args.train_points} points ({steps} steps per epoch); validation over {args.val_tracklets} tracklets of "
                    f"{int(lengths.min())}-{int(lengths.max())} frames, {args.val_points} points per scan, {args.slots} slots",
        "ms_per_step": {"step": step_ms, "sampler_and_step": sampler_ms, "trainer_epoch": epoch_ms},
        "loop_overhead_ms": float(np.mean(epoch_ms) - np.mean(sampler_ms)),
        "val_seconds": val_s, "val_frames": res["frames"], "val_frames_per_s": res["frames"] / min(val_s),
        "gpu": name, "power_limit": power}))


if __name__ == "__main__":
    main()
