"""Multi-object tracking scores on the GPU: `o3d_mot_clear` (csrc/mot_eval.cu) against the host reference (tracking/mot.py
reference_counts) on random runs, its independence of the launch, `--mot` on the command line and a detection-driven
MultiTargetTracker run with births."""
import json
import os

import numpy as np
import pytest
import torch

from open3dsot_b200 import track
from open3dsot_b200.datasets.data_classes import Box, PointCloud
from open3dsot_b200.datasets.synthetic import synthetic_scene, synthetic_sequence
from open3dsot_b200.tracking import mot
from open3dsot_b200.tracking.multi_tracker import BIRTH_ID_BASE, MultiTargetTracker, detection_rows
from test_kitti_reader import _write_scene

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
Z_UP, Y_UP = (0, 0, 1), (0, -1, 0)


def _rot(yaw, up):
    """A box's rotation with its height along the up axis: about z (z up), or a KITTI camera box (y down: the box's z axis to
    -y, its y axis to z) turned about y."""
    c, s = np.cos(yaw), np.sin(yaw)
    if up == Z_UP:
        return np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])
    return np.array([[c, 0.0, s], [0.0, 1.0, 0.0], [-s, 0.0, c]]) @ np.array([[1.0, 0.0, 0.0], [0.0, 0.0, -1.0], [0.0, 1.0, 0.0]])


def random_run(rng, n_seq, frames, n_obj, up, extent=30.0, noise=0.4, p_present=0.9, p_detect=0.85, n_fp=1.0):
    """Objects moving through a square, each frame a random subset of them (dropouts); hypotheses are perturbed ground truth
    with missed detections, id changes and swaps between two objects' hypotheses, and false positives with new ids.  Continuous
    positions: no two assignments tie."""
    plane = (0, 1) if up == Z_UP else (0, 2)
    seqs = []
    for _ in range(n_seq):
        T, n = int(rng.integers(frames[0], frames[1] + 1)), int(rng.integers(n_obj[0], n_obj[1] + 1))
        pos = np.zeros((n, 3))
        pos[:, plane] = rng.uniform(-extent, extent, (n, 2))
        vel = np.zeros((n, 3))
        vel[:, plane] = rng.normal(0, 0.5, (n, 2))
        wlh = np.stack([rng.uniform(1.5, 2.2, n), rng.uniform(3.5, 5.0, n), rng.uniform(1.4, 1.8, n)], 1)
        yaw = rng.uniform(-np.pi, np.pi, n)
        hid = np.arange(n) + 1000
        nxt = 5000
        seq = []
        for _t in range(T):
            pos += vel
            if rng.random() < 0.1 and n >= 2:                                    # two hypotheses swap objects
                a, b = rng.choice(n, 2, replace=False)
                hid[a], hid[b] = hid[b], hid[a]
            change = rng.random(n) < 0.03                                        # an id change (a fragmented track)
            hid[change] = nxt + np.arange(change.sum())
            nxt += int(change.sum())
            present = np.nonzero(rng.random(n) < p_present)[0]
            gt = [(int(o), Box(pos[o], wlh[o], _rot(yaw[o], up))) for o in rng.permutation(present)]
            hyp = []
            for o in present:
                if rng.random() < p_detect:
                    c = pos[o].copy()
                    c[list(plane)] += rng.normal(0, noise, 2)
                    c[2 if up == Z_UP else 1] += rng.normal(0, 0.1)
                    hyp.append((int(hid[o]), Box(c, wlh[o] * rng.uniform(0.9, 1.1, 3), _rot(yaw[o] + rng.normal(0, 0.1), up))))
            for _ in range(rng.poisson(n_fp)):
                c = np.zeros(3)
                c[list(plane)] = rng.uniform(-extent, extent, 2)
                hyp.append((nxt, Box(c, (1.8, 4.2, 1.6), _rot(rng.uniform(-np.pi, np.pi), up))))
                nxt += 1
            seq.append((gt, [hyp[i] for i in rng.permutation(len(hyp))]))
        seqs.append(seq)
    return seqs


def _check(got, want):
    assert len(got) == len(want)
    for s, (g, w) in enumerate(zip(got, want)):
        assert np.array_equal(g.counts, w.counts), (s, g.counts, w.counts)
        assert np.array_equal(g.present, w.present) and np.array_equal(g.tracked, w.tracked), s
        assert np.array_equal(g.cooc, w.cooc), s
        assert abs(g.total_cost - w.total_cost) <= 1e-9 * max(abs(w.total_cost), 1e-300), (s, g.total_cost, w.total_cost)


def _bits(raw):
    return [(r.counts.tobytes(), np.float64(r.total_cost).tobytes(), r.present.tobytes(), r.tracked.tobytes(), r.cooc.tobytes())
            for r in raw]


CASES = [("iou", 0.3, 2, Z_UP), ("iou", 0.5, 3, Z_UP), ("iou", 0.3, 2, Y_UP), ("iou", 0.2, 3, Y_UP),
         ("distance", 2.0, 3, Z_UP), ("distance", 1.5, 2, Y_UP), ("distance", 2.5, 2, Z_UP)]


@pytest.mark.parametrize("metric,thr,dim,up", CASES)
def test_kernel_equals_the_reference_on_random_runs(metric, thr, dim, up):
    rng = np.random.default_rng(100 + CASES.index((metric, thr, dim, up)))
    seqs = random_run(rng, 5, (1, 40), (0, 25), up, extent=12.0)
    seqs.append([([], [])] * 3)                                              # frames with no box
    got = mot.device_counts(seqs, metric, thr, dim, up)
    want = mot.reference_counts(seqs, metric, thr, dim, up)
    _check(got, want)
    assert sum(int(r.counts[3]) for r in want) > 0 and sum(int(r.counts[2]) for r in want) > 0     # switches and matches


def test_long_sequences_and_frames_at_the_limit():
    rng = np.random.default_rng(7)
    long = random_run(rng, 1, (300, 300), (6, 10), Z_UP, extent=10.0)
    # 256 objects and 256 hypotheses on a tight grid: every object has several valid partners (the general assignment)
    g = np.stack(np.meshgrid(np.arange(16), np.arange(16)), -1).reshape(-1, 2) * 2.2
    frames = []
    for t in range(2):
        gt = [(i, Box([g[i, 0], g[i, 1], 0.0], (2.0, 2.0, 1.5), _rot(0.0, Z_UP))) for i in range(256)]
        jit = rng.normal(0, 0.6, (256, 2))
        hyp = [(i + 1000 * t, Box([g[i, 0] + jit[i, 0], g[i, 1] + jit[i, 1], 0.0], (2.0, 2.0, 1.5), _rot(rng.normal(0, 0.2), Z_UP)))
               for i in range(256)]
        frames.append((gt, hyp))
    seqs = long + [frames]
    for metric, thr in (("iou", 0.1), ("distance", 2.0)):
        want = mot.reference_counts(seqs, metric, thr, 2, Z_UP)
        _check(mot.device_counts(seqs, metric, thr, 2, Z_UP), want)
        assert want[1].counts[3] > 0                                          # the second frame switches


def test_results_do_not_depend_on_the_launch():
    rng = np.random.default_rng(11)
    seqs = random_run(rng, 9, (1, 50), (0, 30), Z_UP, extent=12.0)
    batch = mot.device_counts(seqs, "iou", 0.3, 3, Z_UP)
    assert _bits(mot.device_counts(seqs, "iou", 0.3, 3, Z_UP)) == _bits(batch)               # repeated launches
    for s in (0, 4, 8):
        assert _bits(mot.device_counts([seqs[s]], "iou", 0.3, 3, Z_UP)) == _bits([batch[s]])  # alone
    order = rng.permutation(len(seqs))
    again = mot.device_counts([seqs[i] for i in order], "iou", 0.3, 3, Z_UP)
    assert _bits(again) == _bits([batch[i] for i in order])                                 # reordered


def test_command_line_scores_the_run(tmp_path, capsys, monkeypatch):
    root = str(tmp_path / "kitti")
    seqs = [synthetic_sequence(n_frames=n, n_points=1500, seed=40 + i, n_object=300, speed=0.3 + 0.1 * i, yaw_rate=1.0 + i)
            for i, n in enumerate([8, 6])]
    for f in seqs[1]:
        f["pc"] = PointCloud(f["pc"].points + np.array([[0.0], [12.0], [0.0]], np.float32))
        b = f["3d_bbox"]
        f["3d_bbox"] = Box(b.center + np.array([0.0, 12.0, 0.0]), b.wlh, b.rotation_matrix)
    _write_scene(root, "0019", [((5, "Pedestrian"), seqs[0]), ((8, "Pedestrian"), seqs[1])], extra_dontcare=False)
    from open3dsot_b200.datasets.kitti import kittiDataset
    ds = kittiDataset(root, "test", "Pedestrian", preloading=False, preload_offset=-1)
    npts = max(f["pc"].points.shape[1] for t in ds.tracklets() for f in t)
    lines = []
    for t in range(8):
        rows = []
        for annos in ds.tracklet_anno_list:
            for a in annos:
                if a["frame"] == t:
                    b = ds.box_from_anno(a)
                    w = np.sqrt(max(1e-12, 1 + np.trace(b.rotation_matrix))) / 2
                    R = b.rotation_matrix
                    rows.append(list(b.center) + list(b.wlh) + [w, (R[2, 1] - R[1, 2]) / (4 * w), (R[0, 2] - R[2, 0]) / (4 * w),
                                                                  (R[1, 0] - R[0, 1]) / (4 * w), 0.9])
        lines.append({"scene": "0019", "frame": t, "class": "Pedestrian", "boxes": rows})
    (tmp_path / "d.jsonl").write_text("\n".join(json.dumps(l) for l in lines) + "\n")
    captured = []                      # the boxes the run scored: track_feeds' results
    from open3dsot_b200.tracking import multi_tracker
    real = multi_tracker.track_feeds

    def spy(*a, **k):
        out = real(*a, **k)
        captured.append(out[0])
        return out
    monkeypatch.setattr(multi_tracker, "track_feeds", spy)
    base = ["--cfg", os.path.join(ROOT, "cfgs", "M2_track_kitti.yaml"), "--path", root, "--split", "test", "--max_targets", "3",
            "--max_points", str(npts), "--lost", "1", "3", "--coast", "0.5", "--detections", str(tmp_path / "d.jsonl"),
            "--detection_gate", "2.0", "--max_detections", "8"]
    plain = track.main(base + ["--out", str(tmp_path / "plain.jsonl")])
    got = track.main(base + ["--out", str(tmp_path / "mot.jsonl"), "--mot", "iou", "0.5"])
    printed = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert json.dumps(printed["mot"]) == json.dumps(got["mot"])
    assert {k: v for k, v in got.items() if k not in ("mot", "out")} == {k: v for k, v in plain.items() if k != "out"}
    assert (tmp_path / "plain.jsonl").read_text() == (tmp_path / "mot.jsonl").read_text()
    want = mot.mot_reference(track.mot_sequences(track.scene_plan(ds), captured[-1], ds), "iou", 0.5, *_space(base[1]))
    assert json.dumps(_ints(got["mot"])) == json.dumps(_ints(want))
    assert abs(got["mot"]["total"]["total_cost"] - want["total"]["total_cost"]) <= 1e-9 * max(1.0, want["total"]["total_cost"])
    assert got["mot"]["total"]["num_objects"] == 14 and got["mot"]["total"]["num_matches"] > 0


def _space(cfg_path):
    from open3dsot_b200.config import load_config
    cfg = load_config(cfg_path)
    return cfg.IoU_space, cfg.up_axis


def _ints(r):
    keep = lambda d: {k: v for k, v in d.items() if isinstance(v, int)}
    return {"total": keep(r["total"]), "sequences": [keep(s) for s in r["sequences"]]}


def test_born_targets_are_scored_as_hypotheses():
    from test_gpu_multi_target import _model
    _, net = _model("M2_track_kitti.yaml")
    sc = synthetic_scene(n_frames=10, n_points=3000, n_objects=3, seed=90, extent=14.0)
    rng = np.random.default_rng(5)
    trk = MultiTargetTracker(net, 3000, 6, seed=7, detections=(16, 2.0), births=(0.2, 4))
    frames = []
    for t in range(10):
        boxes = [sc["boxes"][j][t] for j in range(3)]
        rows = detection_rows(boxes, rng.uniform(0.5, 1.0, 3))
        trk.put(0, sc["scans"][t], detections=rows)
        trk.advance()
        st = trk.boxes()
        ids, c, s, r = (st[k].cpu().numpy() for k in ("ids", "center", "wlh", "rot"))
        hyp = [(int(i), Box(c[k].astype(np.float64), s[k].astype(np.float64), r[k].astype(np.float64)))
               for k, i in enumerate(ids) if i >= 0]
        frames.append(([(j, boxes[j]) for j in range(3)], hyp))
    assert all(i >= BIRTH_ID_BASE for _, hyp in frames for i, _ in hyp) and any(hyp for _, hyp in frames)
    got = mot.mot_metrics([frames], "distance", 2.0, 3, Z_UP)["total"]
    want = mot.mot_reference([frames], "distance", 2.0, 3, Z_UP)["total"]
    assert json.dumps(_ints({"total": got, "sequences": []})) == json.dumps(_ints({"total": want, "sequences": []}))
    assert got["num_predictions"] == sum(len(h) for _, h in frames) and got["num_matches"] > 0
