"""Cost of multi-object tracking scores on the device (tracking/mot.py, `o3d_mot_clear`) against the host reference, and what
the scores show for three ways of running the live tracker.

  python tools/bench_mot.py [--reps 5] [--steps 30] [--out results.json]

  * "eval": synthetic runs of two sizes, hypotheses = ground truth moved by N(0, 0.4 m) in the plane, each missed with
    probability 0.15, 1 false positive per frame (Poisson), 3% of tracks changing id per frame and a swap of two tracks' ids in
    10% of frames; objects present with probability 0.9 per frame.  nuScenes-val-like: 150 sequences x 40 frames x 50 objects;
    KITTI-like: 21 sequences x 300 frames x 10 objects.  IoU >= 0.5 in 3-D, z up.  "kernel_ms": CUDA events around the
    `o3d_mot_clear` launch (inputs already on the device), best of --reps after a warm-up; "call_ms": host clock around the
    whole `mot_metrics` call (checks, packing, upload, kernel, read-back, per-sequence IDF1), best of --reps;
    "reference_s_per_sequence": `mot_reference` over the first sequences of the run (their number is printed), whose integer
    outputs must equal the kernel's.
  * "table": MOTA / IDF1 / IDSW / FP of the synthetic detection-driven scenes of tools/bench_births.py (4 feeds of 60,000-point
    scenes with 6 objects each, detections from the ground truth with N(0, 0.2 m) centre noise, dropped with probability 0.2,
    and 2 false positives per scan), --steps frames, BAT-Car with untrained weights (the network's boxes are not meaningful;
    the table shows what the scores separate), scored by centre distance <= 2 m in 3-D: "gt_starts" (every object added from
    its first ground-truth box), "lost_coast" (the same with lost=(5, 3), coast=0.5, lost targets dropped) and "births"
    (no target added: detections=(16, 2.0), births=(0.5, 2), lost=(5, 3), lost targets dropped).
The card's name and power limit are printed with the numbers."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_births import _loop_data  # noqa: E402
from bench_coast import _model  # noqa: E402
from bench_multi_target import gpu_info  # noqa: E402
from open3dsot_b200 import ops  # noqa: E402
from open3dsot_b200.datasets.data_classes import Box  # noqa: E402
from open3dsot_b200.datasets.synthetic import synthetic_scene  # noqa: E402
from open3dsot_b200.tracking import mot  # noqa: E402
from open3dsot_b200.tracking.multi_tracker import MultiTargetTracker  # noqa: E402

UP = (0, 0, 1)


def synthetic_run(S, T, n, seed=0, extent=40.0):
    """A MotRun of S sequences x T frames x about n objects (module docstring)."""
    rng = np.random.default_rng(seed)
    seq_frame, frame_gt, frame_hyp = [0], [0], [0]
    gid, hid_all, gbox, hbox = [], [], [], []
    for _ in range(S):
        pos = np.concatenate([rng.uniform(-extent, extent, (n, 2)), np.zeros((n, 1))], 1)
        vel = np.concatenate([rng.normal(0, 0.5, (n, 2)), np.zeros((n, 1))], 1)
        wlh = np.stack([rng.uniform(1.5, 2.2, n), rng.uniform(3.5, 5.0, n), rng.uniform(1.4, 1.8, n)], 1)
        yaw = rng.uniform(-np.pi, np.pi, n)
        hid, nxt = np.arange(n), 10_000
        for _t in range(T):
            pos += vel
            if rng.random() < 0.1:
                a, b = rng.choice(n, 2, replace=False)
                hid[a], hid[b] = hid[b], hid[a]
            ch = rng.random(n) < 0.03
            hid[ch] = nxt + np.arange(ch.sum())
            nxt += int(ch.sum())
            present = np.nonzero(rng.random(n) < 0.9)[0]
            det = present[rng.random(len(present)) >= 0.15]
            n_fp = rng.poisson(1.0)
            gc, hc = pos[present], pos[det].copy()
            hc[:, :2] += rng.normal(0, 0.4, (len(det), 2))
            hc = np.concatenate([hc, np.concatenate([rng.uniform(-extent, extent, (n_fp, 2)), np.zeros((n_fp, 1))], 1)])
            hw = np.concatenate([wlh[det] * rng.uniform(0.9, 1.1, (len(det), 3)), np.tile(wlh[:1], (n_fp, 1))])
            hy = np.concatenate([yaw[det] + rng.normal(0, 0.1, len(det)), rng.uniform(-np.pi, np.pi, n_fp)])
            gid.append(present)
            hid_all.append(np.concatenate([hid[det], nxt + np.arange(n_fp)]))
            nxt += n_fp
            gbox.append(_boxes(gc, wlh[present], yaw[present]))
            hbox.append(_boxes(hc, hw, hy))
            frame_gt.append(frame_gt[-1] + len(present))
            frame_hyp.append(frame_hyp[-1] + len(hc))
        seq_frame.append(len(frame_gt) - 1)
    a = lambda v: np.asarray(v, np.int64)
    return mot.MotRun(a(seq_frame), a(frame_gt), a(frame_hyp), np.concatenate(gid).astype(np.int64),
                      np.concatenate(hid_all).astype(np.int64), np.concatenate(gbox), np.concatenate(hbox))


def _boxes(c, wlh, yaw):
    R = np.zeros((len(c), 3, 3))
    R[:, 0, 0], R[:, 0, 1], R[:, 1, 0], R[:, 1, 1], R[:, 2, 2] = np.cos(yaw), -np.sin(yaw), np.sin(yaw), np.cos(yaw), 1.0
    return np.concatenate([c, wlh, R.reshape(-1, 9)], 1)


def _subset(run, k):
    f1 = run.seq_frame[k]
    return mot.MotRun(run.seq_frame[:k + 1], run.frame_gt[:f1 + 1], run.frame_hyp[:f1 + 1], run.gt_id[:run.frame_gt[f1]],
                      run.hyp_id[:run.frame_hyp[f1]], run.gt_box[:run.frame_gt[f1]], run.hyp_box[:run.frame_hyp[f1]])


def bench_eval(reps):
    out = []
    for name, (S, T, n, k_ref) in (("nuscenes_val_like", (150, 40, 50, 2)), ("kitti_like", (21, 300, 10, 1))):
        run = synthetic_run(S, T, n, seed=len(out))
        checked, dense = mot.check_run(run)
        args = mot.upload_run(checked, dense)
        launch = lambda: ops.mot_clear(*args, "iou", 0.5, 3, UP, dense.max_gt, dense.max_hyp, mot.work_rows(S))
        launch()
        torch.cuda.synchronize()
        kernel = []
        for _ in range(reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            launch()
            e1.record()
            torch.cuda.synchronize()
            kernel.append(e0.elapsed_time(e1))
        call = []
        for _ in range(reps):
            t0 = time.perf_counter()
            res = mot.mot_metrics(run, "iou", 0.5, 3, UP)
            call.append((time.perf_counter() - t0) * 1e3)
        sub = _subset(run, k_ref)
        t0 = time.perf_counter()
        want = mot.reference_counts(sub, "iou", 0.5, 3, UP)
        ref_s = (time.perf_counter() - t0) / k_ref
        got = mot.device_counts(sub, "iou", 0.5, 3, UP)
        same = all(np.array_equal(g.counts, w.counts) and np.array_equal(g.cooc, w.cooc) for g, w in zip(got, want))
        pairs = int(np.sum(np.diff(run.frame_gt) * np.diff(run.frame_hyp)))
        row = {"run": name, "sequences": S, "frames": int(len(run.frame_gt) - 1), "gt_boxes": int(len(run.gt_id)),
               "hyp_boxes": int(len(run.hyp_id)), "pairs": pairs, "kernel_ms": min(kernel), "kernel_ms_all": kernel,
               "call_ms": min(call), "reference_sequences": k_ref, "reference_s_per_sequence": ref_s,
               "reference_equal": bool(same), "mota": res["total"]["mota"], "idf1": res["total"]["idf1"]}
        out.append(row)
        print(json.dumps({"eval": row}), flush=True)
    return out


def _scores_of(net, data, boxes, mode, steps):
    F = len(data)
    kw = {"gt_starts": {}, "lost_coast": {"lost": (5, 3), "coast": 0.5},
          "births": {"lost": (5, 3), "detections": (16, 2.0), "births": (0.5, 2)}}[mode]
    trk = MultiTargetTracker(net, 60_000, 8 * F, seed=0, feeds=F, **kw)
    seqs = [[] for _ in range(F)]
    for t in range(steps):
        for f, (scans, dets) in enumerate(data):
            trk.put_raw(f, scans[t], **({"detections": dets[t]} if mode == "births" else {}))
        trk.advance()
        if t == 0 and mode != "births":              # targets start on the first scan from its ground truth
            for f in range(F):
                for o in range(len(boxes[f])):
                    trk.add(100 * f + o, boxes[f][o][0], feed=f)
        st = {k: v.cpu().numpy() for k, v in trk.boxes().items()}
        feed_of = {tid: trk._feed_of[k] for tid, k in trk.targets().items()}
        for f in range(F):
            hyp = [(int(i), Box(st["center"][k].astype(np.float64), st["wlh"][k].astype(np.float64),
                                st["rot"][k].astype(np.float64))) for k, i in enumerate(st["ids"]) if i >= 0 and feed_of.get(int(i)) == f]
            seqs[f].append(([(o, boxes[f][o][t]) for o in range(len(boxes[f]))], hyp))
        if mode != "gt_starts":
            trk.drop_lost()
    r = mot.mot_metrics(seqs, "distance", 2.0, 3, UP)["total"]
    return {k: r[k] for k in ("mota", "idf1", "num_switches", "num_false_positives", "num_misses", "num_objects")}


def bench_table(steps):
    net = _model("BAT_Car.yaml").eval()
    F = 4
    data = _loop_data(F, steps)
    boxes = [synthetic_scene(n_frames=steps, n_points=60_000, n_objects=6, seed=3000 + f, extent=40.0)["boxes"] for f in range(F)]
    rows = []
    for mode in ("gt_starts", "lost_coast", "births"):
        row = {"mode": mode, **_scores_of(net, data, boxes, mode, steps)}
        rows.append(row)
        print(json.dumps({"table": row}), flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mot: needs a CUDA device")
    gpu = gpu_info()
    print(json.dumps({"gpu": gpu}), flush=True)
    res = {"gpu": gpu, "eval": bench_eval(args.reps), "table": bench_table(args.steps)}
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
