"""Live multi-target tracking throughput on a synthetic scene of moving boxes (datasets/synthetic.py: synthetic_scene).

  python tools/bench_multi_target.py [--cfg cfgs/BAT_Car.yaml] [--points 60000 120000] [--targets 1 8 32 64 128]

Reports, per scan size:
  * MultiTargetTracker (one captured step for all slots): scans/s and target-frames/s at each K, every slot active;
  * the same stream tracked by K B=1 DeviceTrackers (one graph replay per target and scan), at --b1-targets;
  * kernel level at --kernel-targets: o3d_crop_resample against crop_box_frame -> keyed_uniform x 2 -> resample on identical inputs
    (a firstandprevious template crop: a first-frame prefix of N candidates + the scan), time per call and peak memory above the
    inputs, after checking that both give the same bits.
  * feeds (--feeds, --per-feed targets each): scans/s and target-frames/s of one tracker advancing F feeds per step, with every
    scan given as raw nuScenes-like rows ((n, 5) float32 and two affine transforms), prepared either by the host (numpy float64
    transforms, then `put`) or by the device (`put_raw`, one `o3d_scan_ingest` launch per step); host seconds per step spent
    preparing the scans are reported for both, timed in the same run.
Times are CUDA-event times over --frames steps (--reps calls for the kernels) after --warmup untimed ones per shape.  Weights
are untrained (the timing does not depend on them).  The card's name and power limit are printed with the numbers."""
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

from open3dsot_b200 import ops  # noqa: E402
from open3dsot_b200.config import load_config  # noqa: E402
from open3dsot_b200.datasets.synthetic import synthetic_scene  # noqa: E402
from open3dsot_b200.models import get_model  # noqa: E402
from open3dsot_b200.tracking import boxes as bx  # noqa: E402
from open3dsot_b200.tracking.batched_tracker import STREAM_TEMPLATE_PERM, STREAM_TEMPLATE_PICK  # noqa: E402
from open3dsot_b200.tracking.device_tracker import DeviceTracker  # noqa: E402
from open3dsot_b200.tracking.multi_tracker import MultiTargetTracker  # noqa: E402


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()
        return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def timed(fn, n):
    """CUDA-event milliseconds of n calls of fn()."""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for i in range(n):
        fn(i)
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def bench_multi(net, scans, boxes, K, warmup, frames):
    trk = MultiTargetTracker(net, scans[0].shape[0], K, seed=0)
    trk.step(scans[0])
    for j in range(K):
        trk.add(j, boxes[j][0])
    for i in range(warmup):
        trk.step(scans[1 + i])
    ms = timed(lambda i: trk.step(scans[1 + warmup + i]), frames)
    return frames / (ms / 1e3)


def bench_b1(net, scans, boxes, K, warmup, frames):
    trks = [DeviceTracker(net, max_points=scans[0].shape[0], seed=j) for j in range(K)]
    for j, t in enumerate(trks):
        t.reset(scans[0], boxes[j][0].to_tensor("cuda"))

    def one(i):
        for t in trks:
            t.step(scans[i])

    for i in range(warmup):
        one(1 + i)
    ms = timed(lambda i: one(1 + warmup + i), frames)
    return frames / (ms / 1e3)


def _xf(yaw, t):
    c, s = np.cos(yaw), np.sin(yaw)
    return np.array([[c, -s, 0.0, t[0]], [s, c, 0.0, t[1]], [0.0, 0.0, 1.0, t[2]]])


def _inverse(m):
    r = m[:, :3].T
    return np.hstack([r, -(r @ m[:, 3])[:, None]])


def bench_feeds(net, scans_np, boxes, F, per_feed, warmup, frames, device_ingest):
    """F feeds of `per_feed` targets; every feed replays the scene's scans as sensor rows (n, 5) + (sensor -> ego, ego -> global)."""
    to_ego, to_global = _xf(0.3, (1.0, 0.0, 1.8)), _xf(-1.1, (400.0, 1100.0, 0.0))
    to_sensor = _inverse(to_ego) @ np.vstack([_inverse(to_global), [0, 0, 0, 1]])
    rows = []
    for s in scans_np:
        r = np.zeros((s.shape[0], 5), np.float32)
        r[:, :3] = (s.astype(np.float64) @ to_sensor[:, :3].T + to_sensor[:, 3]).astype(np.float32)
        rows.append(r)
    trk = MultiTargetTracker(net, scans_np[0].shape[0], F * per_feed, seed=0, feeds=F)
    host_s = [0.0]

    def one(t):
        t0 = time.perf_counter()
        for f in range(F):
            if device_ingest:
                trk.put_raw(f, rows[t], (to_ego, to_global))
            else:
                p = rows[t][:, :3].T.astype(np.float64)
                p = to_ego[:, :3] @ p + to_ego[:, 3][:, None]
                p = to_global[:, :3] @ p + to_global[:, 3][:, None]
                trk.put(f, np.ascontiguousarray(p.T, dtype=np.float32))
        trk.advance()
        host_s[0] += time.perf_counter() - t0

    one(0)
    for f in range(F):
        for j in range(per_feed):
            trk.add(f * per_feed + j, boxes[j][0], feed=f)
    for i in range(warmup):
        one(1 + i)
    torch.cuda.synchronize()
    host_s[0] = 0.0
    ms = timed(lambda i: one(1 + warmup + i), frames)
    return frames / (ms / 1e3), host_s[0] / frames


def bench_kernel(cfg, scans, boxes, K, reps):
    """A firstandprevious template crop of K targets on a (2, N, 3) scan pair: fused against the three-kernel sequence."""
    dev = "cuda"
    N = scans[0].shape[0]
    pair = torch.stack([scans[0], scans[1]]).contiguous()
    count = torch.tensor([N, N], device=dev)
    frame = torch.zeros(K, dtype=torch.int64, device=dev)
    box = bx.Box(*(torch.tensor(np.stack(v), dtype=torch.float32, device=dev) for v in
                   ([b[1].center for b in boxes[:K]], [b[1].wlh for b in boxes[:K]], [b[1].rotation_matrix for b in boxes[:K]])))
    half = torch.stack([box.wlh[:, 1], box.wlh[:, 0], box.wlh[:, 2]], -1) * (cfg.model_bb_scale / 2) + cfg.model_bb_offset
    box0 = bx.Box(*(torch.tensor(np.stack(v), dtype=torch.float32, device=dev) for v in
                    ([b[0].center for b in boxes[:K]], [b[0].wlh for b in boxes[:K]], [b[0].rotation_matrix for b in boxes[:K]])))
    prefix, pkeep = bx.crop_in_box_frame(pair, box0, cfg.model_bb_scale, cfg.model_bb_offset, frame, count)
    prefix, pkeep = prefix.contiguous(), pkeep.contiguous()
    key, kf = torch.arange(K, device=dev), torch.ones(K, dtype=torch.int64, device=dev)
    size, seed = cfg.template_size, 0
    frame1 = torch.ones(K, dtype=torch.int64, device=dev)

    def fused(_=0):
        return ops.crop_resample(pair, count, frame1, box.center, box.rot, half, size, seed, key, kf, STREAM_TEMPLATE_PERM,
                                 STREAM_TEMPLATE_PICK, prefix, pkeep)

    def unfused(_=0):
        local, keep = ops.crop_box_frame(pair, box.center, box.rot, half, frame1, count)
        cand, ck = torch.cat([prefix, local], 1), torch.cat([pkeep, keep], 1)
        up = ops.keyed_uniform(key, kf, seed, STREAM_TEMPLATE_PERM, cand.shape[1])
        uk = ops.keyed_uniform(key, kf, seed, STREAM_TEMPLATE_PICK, size)
        out, _, n = ops.resample(cand, ck, size, up, uk)
        return out, n

    a, b = fused(), unfused()
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]), "fused and three-kernel outputs differ"
    res = {"survivors_mean": float(a[1].double().mean())}
    for name, fn in (("fused", fused), ("unfused", unfused)):
        for _ in range(5):
            fn()
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        fn()
        torch.cuda.synchronize()
        res[name + "_peak_mb"] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
        res[name + "_ms"] = timed(fn, reps) / reps
    return res


def main(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--cfg", default=os.path.join(ROOT, "cfgs", "BAT_Car.yaml"))
    p.add_argument("--points", type=int, nargs="+", default=[60000, 120000])
    p.add_argument("--targets", type=int, nargs="+", default=[1, 8, 32, 64, 128])
    p.add_argument("--b1-targets", type=int, nargs="+", default=[1, 8, 32])
    p.add_argument("--kernel-targets", type=int, nargs="+", default=[64, 128])
    p.add_argument("--feeds", type=int, nargs="+", default=[1, 4, 16])
    p.add_argument("--per-feed", type=int, default=8)
    p.add_argument("--frames", type=int, default=20)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--reps", type=int, default=50)
    p.add_argument("--out", default=None, help="also write the results as JSON here")
    a = p.parse_args(argv)
    torch.cuda.set_device(0)
    cfg = load_config(a.cfg)
    torch.manual_seed(0)
    net = get_model(cfg.net_model)(cfg).cuda().eval()
    info = gpu_info()
    print(f"# {info}; {os.path.basename(a.cfg)}; {a.frames} timed steps after {a.warmup} warm-up steps per shape", flush=True)
    kmax = max(a.targets + a.b1_targets + a.kernel_targets + [a.per_feed])
    results = {"gpu": info, "cfg": os.path.basename(a.cfg), "rows": []}
    for n in a.points:
        scene = synthetic_scene(n_frames=2 + a.warmup + a.frames, n_points=n, n_objects=kmax, seed=7, extent=70.0)
        scans = [torch.tensor(s, device="cuda") for s in scene["scans"]]
        for K in a.targets:
            sps = bench_multi(net, scans, scene["boxes"], K, a.warmup, a.frames)
            row = {"points": n, "K": K, "tracker": "multi", "scans_per_s": sps, "target_frames_per_s": sps * K}
            results["rows"].append(row)
            print(f"multi   N={n:6d} K={K:3d}: {sps:8.1f} scans/s  {sps * K:9.1f} target-frames/s", flush=True)
        for K in a.b1_targets:
            sps = bench_b1(net, scans, scene["boxes"], K, a.warmup, a.frames)
            row = {"points": n, "K": K, "tracker": "b1", "scans_per_s": sps, "target_frames_per_s": sps * K}
            results["rows"].append(row)
            print(f"B=1 x K N={n:6d} K={K:3d}: {sps:8.1f} scans/s  {sps * K:9.1f} target-frames/s", flush=True)
            torch.cuda.empty_cache()
        for K in a.kernel_targets:
            r = bench_kernel(cfg, scans, scene["boxes"], K, a.reps)
            results["rows"].append({"points": n, "K": K, "tracker": "kernel", **r})
            print(f"kernel  N={n:6d} K={K:3d}: fused {r['fused_ms']:.3f} ms / {r['fused_peak_mb']:.0f} MB, three kernels "
                  f"{r['unfused_ms']:.3f} ms / {r['unfused_peak_mb']:.0f} MB (mean survivors {r['survivors_mean']:.0f})", flush=True)
        for F in a.feeds:
            for dev_ingest in (False, True):
                sps, host = bench_feeds(net, scene["scans"], scene["boxes"], F, a.per_feed, a.warmup, a.frames, dev_ingest)
                how = "device" if dev_ingest else "host"
                results["rows"].append({"points": n, "feeds": F, "K": F * a.per_feed, "tracker": "feeds", "scan_prep": how,
                                        "steps_per_s": sps, "scans_per_s": sps * F, "target_frames_per_s": sps * F * a.per_feed,
                                        "host_s_per_step": host})
                print(f"feeds   N={n:6d} F={F:3d} K={F * a.per_feed:3d} {how:6s} transforms: {sps * F:8.1f} scans/s  "
                      f"{sps * F * a.per_feed:9.1f} target-frames/s  host {host * 1e3:7.2f} ms/step", flush=True)
                torch.cuda.empty_cache()
        del scans
        torch.cuda.empty_cache()
    print(json.dumps(results))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
