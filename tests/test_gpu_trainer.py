"""The training loop on the GPU: static-weight caches after training steps, `Trainer.fit` end to end for BAT, P2B and
M2-Track over synthetic tracklets, resuming, the captured sampler following the epoch's indices, the command line over a
small KITTI tree, and evaluation split across two processes, with and without diverged BatchNorm statistics."""
import glob
import json
import math
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

from open3dsot_b200.config import load_config
from open3dsot_b200.datasets.device_sampler import DeviceMotionSampler, DeviceSiameseSampler
from open3dsot_b200.datasets.synthetic import synthetic_sequence
from open3dsot_b200.engine import TrainStep
from open3dsot_b200.models import get_model
from open3dsot_b200.tracking.evaluate import evaluate_batched

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SMALL = {"up_axis": [0, 0, 1], "batch_size": 8, "epoch": 2}      # the synthetic tracklets are z-up


def _cfg(name, **over):
    return load_config(os.path.join(ROOT, "cfgs", name), {**SMALL, **over})


def _model(cfg):
    torch.manual_seed(0)
    return get_model(cfg.net_model)(cfg).cuda()


def _tracklets(lengths, n_points=3000, seed=100):
    return [synthetic_sequence(n_frames=n, n_points=n_points, seed=seed + i, speed=0.4 + 0.05 * i, yaw_rate=1.0 + i,
                               n_object=400) for i, n in enumerate(lengths)]


def _boxes(res):
    return np.array([np.concatenate([b.center, b.rotation_matrix.ravel()]) for seq in res["results"] for b in seq])


def _same(a, b):
    assert np.array_equal(_boxes(a), _boxes(b))
    assert a["overlaps"] == b["overlaps"] and a["distances"] == b["distances"]
    assert a["success"] == b["success"] and a["precision"] == b["precision"]


@pytest.mark.parametrize("name", ["BAT_Car.yaml", "M2_track_kitti.yaml"])
def test_evaluation_after_training_steps_uses_the_new_weights(name):
    """validate -> train (graph replays) -> validate: the second validation scores the trained model, bit for bit what a
    fresh model loaded with the trained state_dict scores."""
    cfg = _cfg(name)
    net = _model(cfg).train()
    val = _tracklets([6, 4, 5], seed=300)
    cls = DeviceMotionSampler if cfg.train_type == "train_motion" else DeviceSiameseSampler
    smp = cls(_tracklets([8, 8], seed=200), cfg, "cuda", seed=1)
    ts = TrainStep(net, lr=cfg.lr, weight_decay=cfg.wd, warmup=1)
    for _ in range(3):                                  # eager, capture, replay
        ts.step(smp.next_batch(8)[0])
    before = evaluate_batched(net, val, slots=4, seed=1)
    net.train()
    for _ in range(3):                                  # replays only: no tensor version changes
        ts.step(smp.next_batch(8)[0])
    after = evaluate_batched(net, val, slots=4, seed=1)
    fresh = get_model(cfg.net_model)(cfg).cuda()
    fresh.load_state_dict(net.state_dict())
    want = evaluate_batched(fresh, val, slots=4, seed=1)
    assert not np.array_equal(_boxes(before), _boxes(want))          # training moved the result
    _same(after, want)


def _ckpts(log_dir):
    return sorted(glob.glob(os.path.join(log_dir, "lightning_logs", "version_0", "checkpoints", "*.ckpt")))


@pytest.mark.parametrize("name", ["BAT_Car.yaml", "P2B_Car.yaml", "M2_track_kitti.yaml"])
def test_fit_end_to_end(tmp_path, name):
    from open3dsot_b200.trainer import Trainer, TopK
    cfg = _cfg(name)
    train, val = _tracklets([8, 6, 7], seed=400), _tracklets([6, 3, 5, 4], seed=500)
    log = str(tmp_path / "run")
    tr = Trainer(_model(cfg), cfg, train, val, log, slots=4)
    tr.fit()
    rows = [json.loads(l) for l in open(os.path.join(log, "metrics.jsonl"))]
    assert [r["epoch"] for r in rows] == [0, 1]
    spe = tr.global_step // 2
    assert spe == (21 * cfg.num_candidates) // 8 and [r["global_step"] for r in rows] == [spe, 2 * spe]
    for r in rows:
        losses = {k: v for k, v in r.items() if k.endswith("/train")}
        assert losses and all(math.isfinite(v) for v in losses.values()), r
        assert r["pairs_per_second"] > 0 and r["val_seconds"] > 0 and 0 <= r["precision"] <= 100
    d = os.path.join(log, "lightning_logs", "version_0", "checkpoints")
    want = sorted([os.path.join(d, TopK.filename(e, (e + 1) * spe)) for e in (0, 1)] + [os.path.join(d, "last.ckpt")])
    assert _ckpts(log) == want
    for e in (0, 1):
        t2 = Trainer(get_model(cfg.net_model)(cfg).cuda(), cfg, [], [], str(tmp_path / f"test{e}"), slots=4)
        t2.resume(os.path.join(d, TopK.filename(e, (e + 1) * spe)))
        assert (t2.epoch, t2.global_step) == (e + 1, (e + 1) * spe)
        res = t2.test(val)
        assert (res["success"], res["precision"]) == (rows[e]["success"], rows[e]["precision"]), e


def test_resume_restores_the_state_and_continues(tmp_path):
    """Resume from the best file of a save_top_k=1 run into the same log directory: the state comes back bit for bit, the
    epoch order continues, and the new run writes its own top-k file without deleting the one it resumed from."""
    from open3dsot_b200.trainer import Trainer, TopK
    cfg = _cfg("BAT_Car.yaml", epoch=1, save_top_k=1)
    train, val = _tracklets([8, 6, 7], seed=400), _tracklets([5, 4], seed=500)
    log = str(tmp_path / "run")
    a = Trainer(_model(cfg), cfg, train, val, log, slots=4)
    a.fit()
    saved = (a.step.flat.flat.clone(), a.step.opt.exp_avg.clone(), a.step.opt.exp_avg_sq.clone(), a.step.opt.state.clone(),
             {k: v.clone() for k, v in a.model.named_buffers()})
    best = a.top_k.best_path
    assert best == os.path.join(log, "lightning_logs", "version_0", "checkpoints", TopK.filename(0, a.global_step))
    cfg2 = _cfg("BAT_Car.yaml", epoch=2, save_top_k=1)
    torch.manual_seed(123)
    b = Trainer(get_model(cfg2.net_model)(cfg2).cuda(), cfg2, train, val, log, slots=4)
    b.resume(best)
    assert torch.equal(b.step.flat.flat, saved[0]) and torch.equal(b.step.opt.exp_avg, saved[1])
    assert torch.equal(b.step.opt.exp_avg_sq, saved[2]) and torch.equal(b.step.opt.state, saved[3])
    assert all(torch.equal(v, saved[4][k]) for k, v in b.model.named_buffers())
    assert (b.epoch, b.global_step, b.lr) == (a.epoch, a.global_step, a.lr)
    assert b.epoch_order(1) == a.epoch_order(1) and b.epoch_order(1) != a.epoch_order(0)
    assert b.top_k.best_path == best and b.top_k.best_score == a.top_k.best_score
    row = b.fit()
    assert row["epoch"] == 1 and row["global_step"] == 2 * a.global_step
    assert all(math.isfinite(v) for k, v in row.items() if k.endswith("/train"))
    assert os.path.isfile(best)
    mine = os.path.join(log, "lightning_logs", "version_1", "checkpoints", TopK.filename(1, b.global_step))
    assert os.path.isfile(mine) and b.top_k.best_path == mine


def test_captured_sampler_follows_the_given_indices():
    from test_trainer import check_batch_follows, one_frame_tracklets
    cfg = _cfg("BAT_Car.yaml")
    smp = DeviceSiameseSampler(one_frame_tracklets(8), cfg, "cuda", seed=3)
    assert smp.use_graph
    outs = []
    for indices in ([31, 0, 5, 18, 7, 26, 12, 3], [1, 2, 4, 8, 16, 30, 9, 20]):
        indices = torch.tensor(indices, device="cuda")
        batch, valid = smp.next_batch(8, indices=indices)
        assert bool(valid.all())
        check_batch_follows(batch, smp, indices)
        outs.append({k: v.clone() for k, v in batch.items()})
    assert len(smp._graphs) == 1                                   # one capture, replayed with each index set
    assert not torch.equal(outs[0]["bbox_size"], outs[1]["bbox_size"])


def test_command_line_trains_then_tests(tmp_path):
    import yaml
    from test_kitti_reader import _write_scene
    data = str(tmp_path / "kitti")
    _write_scene(data, "0000", [((1, "Car"), synthetic_sequence(n_frames=8, n_points=3000, seed=4, n_object=400)),
                                ((2, "Car"), synthetic_sequence(n_frames=6, n_points=3000, seed=5, n_object=400))])
    _write_scene(data, "0019", [((1, "Car"), synthetic_sequence(n_frames=6, n_points=3000, seed=6, n_object=400)),
                                ((3, "Car"), synthetic_sequence(n_frames=4, n_points=3000, seed=7, n_object=400))])
    with open(os.path.join(ROOT, "cfgs", "BAT_Car.yaml")) as f:
        cfg = yaml.safe_load(f)
    cfg.update(path=data, train_split="train_tiny", val_split="test_tiny", test_split="test_tiny")
    cfg_file = str(tmp_path / "bat.yaml")
    with open(cfg_file, "w") as f:
        yaml.safe_dump(cfg, f)
    log = str(tmp_path / "log")
    env = dict(os.environ, PYTHONPATH=ROOT)
    run = lambda *a: subprocess.run([sys.executable, "-m", "open3dsot_b200.main", "--cfg", cfg_file, "--log_dir", log, *a],
                                    cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    p = run("--batch_size", "8", "--epoch", "2")
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-4000:]
    rows = [json.loads(l) for l in open(os.path.join(log, "metrics.jsonl"))]
    assert len(rows) == 2
    from open3dsot_b200.checkpoint import load_lightning_checkpoint, model_checkpoint_state
    d = os.path.join(log, "lightning_logs", "version_0", "checkpoints")
    best = model_checkpoint_state(load_lightning_checkpoint(os.path.join(d, "last.ckpt")))["best_model_path"]
    assert os.path.isfile(best)
    epoch = int(os.path.basename(best).split("-")[0].split("=")[1])
    p = run("--test", "--checkpoint", best)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-4000:]
    out = json.load(open(os.path.join(log, "test.json")))
    assert (out["success"], out["precision"]) == (rows[epoch]["success"], rows[epoch]["precision"])
    assert json.loads(p.stdout.strip().splitlines()[-1]) == out


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


_SHARD_LENGTHS = [12, 1, 5, 9, 3, 12, 2, 7]


def _shard_worker(rank, world, port, out_dir):
    import torch.distributed as dist
    from open3dsot_b200 import ddp
    from open3dsot_b200.tracking.evaluate import evaluate_sharded
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK="0")
    ddp.init_distributed(backend="gloo")
    torch.cuda.set_device(0)
    res = evaluate_sharded(_model(_cfg("BAT_Car.yaml")).eval(), _tracklets(_SHARD_LENGTHS, seed=600), slots=3, seed=5)
    if rank == 0:
        torch.save({k: res[k] for k in ("overlaps", "distances", "success", "precision", "frames")} | {"boxes": _boxes(res)},
                   os.path.join(out_dir, "sharded.pt"))
    dist.destroy_process_group()


def test_sharded_evaluation_matches_one_process(tmp_path):
    import torch.multiprocessing as mp
    mp.spawn(_shard_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    got = torch.load(os.path.join(str(tmp_path), "sharded.pt"), weights_only=False)
    one = evaluate_batched(_model(_cfg("BAT_Car.yaml")).eval(), _tracklets(_SHARD_LENGTHS, seed=600), slots=3, seed=5)
    assert [len(o) for o in got["overlaps"]] == _SHARD_LENGTHS and got["frames"] == sum(_SHARD_LENGTHS)
    assert float(np.abs(got["boxes"] - _boxes(one)).max()) < 1e-4
    assert float(np.abs(np.concatenate(got["overlaps"]) - np.concatenate(one["overlaps"])).max()) < 1e-3


def _buffer_worker(rank, world, port, out_dir):
    """Two ranks whose BatchNorm running statistics have drifted apart, as per-rank training leaves them."""
    import torch.distributed as dist
    from open3dsot_b200 import ddp
    from open3dsot_b200.trainer import Trainer
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK="0")
    torch.cuda.set_device(0)
    ddp.init_distributed(backend="gloo")
    cfg = _cfg("BAT_Car.yaml")
    tr = Trainer(_model(cfg), cfg, [], [], out_dir, slots=3)
    if rank == 1:
        with torch.no_grad():
            for m in tr.model.modules():
                if isinstance(m, torch.nn.modules.batchnorm._BatchNorm) and m.track_running_stats:
                    m.running_mean.add_(0.5)
                    m.running_var.mul_(4.0)
    res = tr.test(_tracklets(_SHARD_LENGTHS, seed=600))
    torch.save({"boxes": _boxes(res), "overlaps": res["overlaps"],
                "buffers": {k: v.cpu() for k, v in tr.model.named_buffers()}}, os.path.join(out_dir, f"rank{rank}.pt"))
    dist.destroy_process_group()


def test_sharded_validation_scores_rank_0_s_model(tmp_path):
    """Validation under DDP scores the model rank 0 saves: rank 0's BatchNorm buffers are everyone's before the split."""
    import torch.multiprocessing as mp
    mp.spawn(_buffer_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    r0, r1 = (torch.load(os.path.join(str(tmp_path), f"rank{r}.pt"), weights_only=False) for r in range(2))
    assert all(torch.equal(v, r1["buffers"][k]) for k, v in r0["buffers"].items())
    assert np.array_equal(r0["boxes"], r1["boxes"]) and r0["overlaps"] == r1["overlaps"]
    one = evaluate_batched(_model(_cfg("BAT_Car.yaml")).eval(), _tracklets(_SHARD_LENGTHS, seed=600), slots=3, seed=0)
    assert float(np.abs(r0["boxes"] - _boxes(one)).max()) < 1e-4       # the slot-count tolerance of the batched tracker
