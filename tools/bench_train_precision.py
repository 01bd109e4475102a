"""fp32 (3xTF32) against bf16 (BF16 operands, FP32 accumulation) training, in one process so that the two alternate on the same card.

  step         the training step as bench.py times it: graph-captured engine.TrainStep, the same starting state for every timed
               step, a 256 MiB L2 flush between steps (not timed), CUDA events over `--steps` steps after `--warmup`; fp32 and
               bf16 alternated for `--rounds` rounds each, for BAT-Car, P2B-Car and M2-Track at batch `--batch`;
  kernels      the per-kernel device time of 3 steps of BAT-Car in each precision from torch.profiler (warm caches, no flush),
               the kernels whose time changed most and the ones that dominate;
  convergence  BAT-Car trained with Trainer for `--epochs` seeded epochs on the synthetic split of tools/bench_precision.py, in
               fp32 and in bf16 with each of `--seeds`: the per-epoch loss terms, then every model evaluated in fp32 on the
               held-out tracklets (Success / Precision).

The card's name, power limit and max SM clock are printed with the numbers; the JSON goes to stdout and to --out.

    python tools/bench_train_precision.py [--skip kernels,convergence] [--epochs 40] [--seeds 0,1] [--precisions fp32,bf16]
                                          [--out FILE]
"""
import argparse
import json
import os
import sys
import time
from collections import defaultdict

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_precision import PRECISIONS, card  # noqa: E402
from open3dsot_b200.config import load_config  # noqa: E402
from open3dsot_b200.datasets.synthetic import synthetic_motion_batch, synthetic_sequence, synthetic_siamese_batch  # noqa: E402
from open3dsot_b200.engine import TrainStep  # noqa: E402
from open3dsot_b200.models import get_model  # noqa: E402
from open3dsot_b200.tracking.evaluate import evaluate_batched  # noqa: E402

MODELS = ("BAT_Car.yaml", "P2B_Car.yaml", "M2_track_kitti.yaml")


def _setup(cfg_name, batch, precision):
    cfg = load_config(os.path.join(ROOT, "cfgs", cfg_name), {"batch_size": batch})
    torch.manual_seed(0)
    net = get_model(cfg.net_model)(cfg).cuda().train()
    eng = TrainStep(net, lr=cfg.lr, weight_decay=cfg.wd, use_graph=True, warmup=2, precision=precision)
    if cfg.net_model.lower() == "m2track":
        batches = [{k: v.cuda() for k, v in synthetic_motion_batch(batch, cfg.point_sample_size, seed=20260924 + i).items()}
                   for i in range(4)]
    else:
        batches = [{k: v.cuda() for k, v in synthetic_siamese_batch(batch, cfg.template_size, cfg.search_size, seed=20260924 + i,
                                                                    box_aware=getattr(cfg, "box_aware", False)).items()}
                   for i in range(4)]
    state = [eng.flat.flat, eng.opt.exp_avg, eng.opt.exp_avg_sq, eng.opt.state, *net.buffers()]
    return eng, batches, state, [t.clone() for t in state]


def time_steps(eng, batches, state, initial, steps, warmup, flush):
    for i in range(max(warmup, 3) + 3):                          # includes the graph capture
        eng.step(batches[i % len(batches)])
    torch.cuda.synchronize()
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
    for i in range(steps):
        with torch.no_grad():
            for t, t0 in zip(state, initial):
                t.copy_(t0)
        flush.fill_(float(i))
        evs[i][0].record()
        eng.step(batches[i % len(batches)])
        evs[i][1].record()
    torch.cuda.synchronize()
    return sum(a.elapsed_time(b) for a, b in evs) / steps


def bench_step(batch, steps, warmup, rounds):
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device="cuda")
    out = {}
    for cfg_name in MODELS:
        runs = {p: _setup(cfg_name, batch, p) for p in PRECISIONS}
        ms = {p: [] for p in PRECISIONS}
        for _ in range(rounds):
            for p in PRECISIONS:
                ms[p].append(time_steps(*runs[p], steps, warmup, flush))
        best = {p: min(v) for p, v in ms.items()}
        out[cfg_name] = {"ms_per_step": ms, "pairs_per_s": {p: batch * 1e3 / best[p] for p in PRECISIONS},
                         "speedup": best["fp32"] / best["bf16"], "batch": batch}
        print(json.dumps({"step": cfg_name, **out[cfg_name]}), flush=True)
        del runs
        torch.cuda.empty_cache()
    return out


def bench_kernels(batch, top):
    per = {}
    for p in PRECISIONS:
        eng, batches, _, _ = _setup("BAT_Car.yaml", batch, p)
        for i in range(6):
            eng.step(batches[i % 4])
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for i in range(3):
                eng.step(batches[i % 4])
            torch.cuda.synchronize()
        t = defaultdict(float)
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA:
                name = e.name.replace("(anonymous namespace)::", "").split("(")[0]
                t[name] += e.device_time_total / 3e3              # ms per step
        per[p] = dict(t)
        del eng
    names = set(per["fp32"]) | set(per["bf16"])
    rows = sorted(({"kernel": n, "fp32_ms": per["fp32"].get(n, 0.0), "bf16_ms": per["bf16"].get(n, 0.0)} for n in names),
                  key=lambda r: -max(r["fp32_ms"], r["bf16_ms"]))
    out = {"total_ms": {p: sum(per[p].values()) for p in PRECISIONS}, "top": rows[:top]}
    print(json.dumps({"kernels": out}), flush=True)
    return out


def bench_convergence(epochs, seeds, seconds, precisions=PRECISIONS):
    from open3dsot_b200.trainer import Trainer
    train = [synthetic_sequence(n_frames=20, n_points=20000, seed=20260924 + i) for i in range(48)]
    rng = np.random.default_rng(20261016)
    val = [synthetic_sequence(n_frames=int(n), n_points=20000, seed=1000 + i, speed=0.3 + 0.4 * rng.random(),
                              yaw_rate=4 * rng.random() - 2) for i, n in enumerate(rng.integers(20, 80, 32))]
    out = []
    for seed in seeds:
        for p in precisions:
            cfg = load_config(os.path.join(ROOT, "cfgs", "BAT_Car.yaml"),
                              {"up_axis": [0, 0, 1], "batch_size": 48, "epoch": 10 ** 6, "train_precision": p})
            torch.manual_seed(seed)
            net = get_model(cfg.net_model)(cfg).cuda()
            tr = Trainer(net.train(), cfg, train, val, log_dir=None, seed=seed, slots=32)
            t0, losses = time.perf_counter(), []
            while len(losses) < epochs and time.perf_counter() - t0 < seconds:
                losses.append(tr.train_epoch()[0])
            res = evaluate_batched(net.eval(), val, slots=32, seed=0)
            row = {"seed": seed, "train_precision": p, "epochs": len(losses), "train_seconds": time.perf_counter() - t0,
                   "losses": losses, "success": res["success"], "precision": res["precision"]}
            print(json.dumps({"convergence": {k: v for k, v in row.items() if k != "losses"}, "last_losses": losses[-1]}),
                  flush=True)
            out.append(row)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=48)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3, help="fp32 / bf16 alternations of every step measurement")
    ap.add_argument("--top", type=int, default=25, help="rows of the kernel table")
    ap.add_argument("--epochs", type=int, default=40)
    ap.add_argument("--seeds", default="0,1")
    ap.add_argument("--precisions", default="fp32,bf16", help="training precisions of the convergence runs")
    ap.add_argument("--train-seconds", type=float, default=1800.0, help="stop each training run after this long")
    ap.add_argument("--skip", default="", help="comma list of sections to skip: step, kernels, convergence")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train_precision.py needs a CUDA device")
    skip = set(filter(None, a.skip.split(",")))
    res = {"gpu": card()}
    print(json.dumps(res), flush=True)
    if "step" not in skip:
        res["step"] = bench_step(a.batch, a.steps, a.warmup, a.rounds)
    if "kernels" not in skip:
        res["kernels"] = bench_kernels(a.batch, a.top)
    if "convergence" not in skip:
        res["convergence"] = bench_convergence(a.epochs, [int(s) for s in a.seeds.split(",")], a.train_seconds,
                                             a.precisions.split(","))
    res["gpu_after"] = card()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
