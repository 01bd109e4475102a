"""The training loop's host logic without a GPU: the reference's epoch order under 1-3 ranks, StepLR, Adam state in
torch.optim.Adam's layout and the shipped checkpoints' optimizer / scheduler / callback state, ModelCheckpoint's top-k
bookkeeping (also after a resume), the command line, the device sampler following given sample indices, and the split of
an evaluation across ranks (2 gloo ranks)."""
import glob
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from open3dsot_b200.checkpoint import load_lightning_checkpoint, model_checkpoint_state
from open3dsot_b200.config import load_config
from open3dsot_b200.engine import FlatAdam
from open3dsot_b200.ddp import FlatParams
from open3dsot_b200.main import parse_args, parse_config
from open3dsot_b200.models import get_model
from open3dsot_b200.tracking.evaluate import gather_shards, shard_plan
from open3dsot_b200.trainer import TopK, Trainer, check_supported, epoch_indices, step_lr, steps_per_epoch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CKPT_DIR = os.path.join(ROOT, "tests", "golden", "ckpt")
CFGS = sorted(glob.glob(os.path.join(ROOT, "cfgs", "*.yaml")))


@pytest.mark.parametrize("n,world", [(97, 1), (97, 2), (97, 3), (96, 2), (96, 3), (5, 3)])
def test_epoch_order_is_distributed_samplers(n, world):
    for epoch in (0, 1, 7):
        parts = [epoch_indices(n, epoch, seed=3, rank=r, world=world) for r in range(world)]
        for r in range(world):
            ds = torch.utils.data.DistributedSampler(range(n), num_replicas=world, rank=r, shuffle=True, seed=3)
            ds.set_epoch(epoch)
            assert parts[r] == list(ds)
        assert epoch_indices(n, epoch, seed=3, rank=0, world=world) == parts[0]        # a function of (seed, epoch) only
        flat = [i for p in parts for i in p]
        assert set(flat) == set(range(n)) and len(flat) == -(-n // world) * world      # covers; only the padding repeats
        if n % world == 0:
            assert len(set(flat)) == len(flat)                                          # disjoint
    assert epoch_indices(n, 1, seed=3) != epoch_indices(n, 2, seed=3)
    assert epoch_indices(n, 1, seed=3) != epoch_indices(n, 1, seed=4)


@pytest.mark.parametrize("n,batch,world", [(1000, 64, 1), (1000, 64, 2), (1000, 64, 3), (63, 64, 1), (130, 64, 2)])
def test_steps_per_epoch(n, batch, world):
    data = range(n)
    want = len(torch.utils.data.DataLoader(
        data, sampler=torch.utils.data.DistributedSampler(data, num_replicas=world, rank=world - 1, shuffle=True),
        batch_size=batch, drop_last=True))
    assert steps_per_epoch(n, batch, world) == want == (-(-n // world)) // batch


@pytest.mark.parametrize("cfg_file", [os.path.basename(c) for c in CFGS])
def test_learning_rate_is_steplr(cfg_file):
    cfg = load_config(os.path.join(ROOT, "cfgs", cfg_file))
    p = torch.nn.Parameter(torch.zeros(1))
    opt = torch.optim.Adam([p], lr=cfg.lr)
    sched = torch.optim.lr_scheduler.StepLR(opt, step_size=cfg.lr_decay_step, gamma=cfg.lr_decay_rate)
    for epoch in range(3 * cfg.lr_decay_step):
        assert step_lr(cfg.lr, cfg.lr_decay_rate, cfg.lr_decay_step, epoch) == opt.param_groups[0]["lr"], epoch
        opt.step()
        sched.step()


def _net():
    torch.manual_seed(0)
    return torch.nn.Sequential(torch.nn.Linear(4, 8), torch.nn.BatchNorm1d(8), torch.nn.Linear(8, 3))


def test_adam_state_round_trip_and_torch_layout():
    net = _net()
    flat = FlatParams(net)
    opt = FlatAdam(flat, lr=3e-4, weight_decay=0.5)
    assert opt.state_dict()["state"] == {}                                               # before the first step: empty
    g = torch.Generator().manual_seed(1)
    opt.exp_avg.copy_(torch.randn(flat.numel, generator=g))
    opt.exp_avg_sq.copy_(torch.rand(flat.numel, generator=g))
    opt.state[0] = 7.0
    sd = opt.state_dict(initial_lr=1e-3)
    assert sorted(sd["state"]) == list(range(len(list(net.parameters()))))
    grp = sd["param_groups"][0]
    assert grp["betas"] == (0.5, 0.999) and grp["eps"] == 1e-6 and grp["weight_decay"] == 0.5 and grp["initial_lr"] == 1e-3
    assert abs(grp["lr"] - 3e-4) < 1e-10 and grp["amsgrad"] is False
    other = FlatAdam(FlatParams(_net()))
    other.load_state_dict(sd)
    assert torch.equal(other.exp_avg, opt.exp_avg) and torch.equal(other.exp_avg_sq, opt.exp_avg_sq)
    assert torch.equal(other.state[:1], opt.state[:1])
    ref = torch.optim.Adam(net.parameters(), lr=3e-4, betas=(0.5, 0.999), eps=1e-6)
    ref.load_state_dict(sd)
    for i, p in enumerate(net.parameters()):
        st = ref.state[p]
        assert float(st["step"]) == 7.0
        assert torch.equal(st["exp_avg"], sd["state"][i]["exp_avg"]) and st["exp_avg"].shape == p.shape
        assert torch.equal(st["exp_avg_sq"], sd["state"][i]["exp_avg_sq"])
    back = FlatAdam(FlatParams(_net()))
    back.load_state_dict(ref.state_dict())                                               # torch's own dict reads back
    assert torch.equal(back.exp_avg, opt.exp_avg) and float(back.state[0]) == 7.0


def test_adam_state_mismatches_raise():
    opt = FlatAdam(FlatParams(_net()))
    sd = opt.state_dict()
    sd["param_groups"][0]["params"] = sd["param_groups"][0]["params"][:-1]
    with pytest.raises(ValueError, match="parameters"):
        opt.load_state_dict(sd)
    opt.state[0] = 2.0
    sd = opt.state_dict()
    sd["state"][1]["step"] = torch.tensor(3.0)
    with pytest.raises(ValueError, match="steps differ"):
        FlatAdam(FlatParams(_net())).load_state_dict(sd)
    sd = opt.state_dict()
    sd["state"][0]["exp_avg"] = torch.zeros(3, 3)
    with pytest.raises(ValueError, match="shape"):
        FlatAdam(FlatParams(_net())).load_state_dict(sd)


@pytest.mark.parametrize("ckpt,cfg_file,epoch,step,lr", [("bat_kitti_car.ckpt", "BAT_Car.yaml", 25, 19525, 4e-05),
                                                          ("mmtrack_kitti_car.ckpt", "M2_track_kitti.yaml", 92, 22448, 1.6e-06)])
def test_resume_from_shipped_checkpoints(tmp_path, ckpt, cfg_file, epoch, step, lr):
    cfg = load_config(os.path.join(ROOT, "cfgs", cfg_file))
    net = get_model(cfg.net_model)(cfg)
    tr = Trainer(net, cfg, [], [], str(tmp_path))
    ck = tr.resume(os.path.join(CKPT_DIR, ckpt))
    assert (tr.epoch, tr.global_step) == (epoch, step)
    assert abs(tr.lr - lr) < 1e-15 and float(tr.step.opt.state[1]) == float(torch.tensor(lr, dtype=torch.float32))
    assert float(tr.step.opt.state[0]) == 0.0 and float(tr.step.opt.exp_avg.abs().max()) == 0.0   # the fixtures' empty state
    assert tr.gamma == 0.2                                                            # M2_track_kitti.yaml says 0.1
    cb = model_checkpoint_state(ck)
    assert tr.top_k.best_path == cb["best_model_path"] and tr.top_k.best_score == float(cb["best_model_score"])
    w = net.state_dict()
    k = next(k for k in w if k.endswith("weight") and w[k].dim() >= 2)
    assert torch.equal(w[k], ck["state_dict"][k])
    # what we save reads back with the same state, and in the fixtures' layout
    out = tr.save(os.path.join(str(tmp_path), "x.ckpt"))
    ours = load_lightning_checkpoint(out)
    assert (ours["epoch"], ours["global_step"]) == (epoch, step)
    ref_sched = ck["lr_schedulers"][0]
    for key in ("step_size", "gamma", "base_lrs", "last_epoch", "_step_count"):
        assert ours["lr_schedulers"][0][key] == ref_sched[key], key
    assert abs(ours["lr_schedulers"][0]["_last_lr"][0] - ref_sched["_last_lr"][0]) < 1e-18
    assert set(model_checkpoint_state(ours)) == set(cb)
    assert len(ours["optimizer_states"][0]["param_groups"][0]["params"]) == len(ck["optimizer_states"][0]["param_groups"][0]["params"])


def test_resume_refuses_a_mismatched_checkpoint(tmp_path):
    cfg = load_config(os.path.join(ROOT, "cfgs", "P2B_Car.yaml"))
    tr = Trainer(get_model(cfg.net_model)(cfg), cfg, [], [], str(tmp_path))
    with pytest.raises(ValueError, match="parameters"):
        tr.resume(os.path.join(CKPT_DIR, "bat_kitti_car.ckpt"))


def test_top_k_bookkeeping(tmp_path):
    d = str(tmp_path)
    scores = [50.0, 70.0, 60.0, 60.0, 80.0]
    steps = [10, 20, 30, 40, 50]
    assert TopK.filename(24, 19525) == "epoch=24-step=19524.ckpt"
    f = lambda e: os.path.join(d, TopK.filename(e, steps[e]))
    # -1: every file, the best is the highest score (the first of a tie)
    t = TopK(-1, d)
    assert [t.update(s, e, steps[e]) for e, s in enumerate(scores)] == [(f(e), []) for e in range(5)]
    assert t.best_path == f(4) and t.best_score == 80.0 and len(t.best_k) == 5
    # 0: no file
    t = TopK(0, d)
    assert [t.update(s, e, steps[e]) for e, s in enumerate(scores)] == [(None, [])] * 5 and t.best_path == ""
    # 2: the best two; a tie with the second best does not replace it
    t = TopK(2, d)
    got = [t.update(s, e, steps[e]) for e, s in enumerate(scores)]
    assert got == [(f(0), []), (f(1), []), (f(2), [f(0)]), (None, []), (f(4), [f(2)])]
    assert set(t.best_k) == {f(1), f(4)} and t.best_path == f(4)
    sd = t.state_dict()
    assert sd["monitor"] == "precision/test" and float(sd["best_model_score"]) == 80.0 and sd["dirpath"] == d
    assert float(sd["current_score"]) == 80.0


def test_cli_defaults_and_override_rule(tmp_path):
    a = parse_args(["--cfg", "x.yaml"])
    assert (a.batch_size, a.epoch, a.save_top_k, a.check_val_every_n_epoch, a.workers) == (100, 60, -1, 1, 10)
    assert (a.checkpoint, a.log_dir, a.test, a.preloading) == (None, None, False, False)
    cfg = parse_config(["--cfg", os.path.join(ROOT, "cfgs", "BAT_Car.yaml"), "--epoch", "3"])
    yaml_cfg = load_config(os.path.join(ROOT, "cfgs", "BAT_Car.yaml"))
    assert yaml_cfg.batch_size != 100 and cfg.batch_size == 100             # defaults overwrite the file, as in the reference
    assert cfg.epoch == 3 and cfg.preloading is False and cfg.net_model == yaml_cfg.net_model


@pytest.mark.parametrize("key,value", [("optimizer", "SGD"), ("gradient_clip_val", 0.5), ("random_sample", True)])
def test_unsupported_settings_raise(key, value):
    cfg = load_config(os.path.join(ROOT, "cfgs", "BAT_Car.yaml"))
    check_supported(cfg)
    cfg[key] = value
    with pytest.raises(ValueError, match=key):
        check_supported(cfg)


def test_shard_plan_covers_once_and_balances_frames():
    lengths = [120, 3, 40, 40, 77, 1, 9, 200, 15, 15, 60]
    assert shard_plan(lengths, 1) == [list(range(len(lengths)))]
    for world in (2, 3, 4):
        shards = shard_plan(lengths, world)
        flat = sorted(j for s in shards for j in s)
        assert flat == list(range(len(lengths)))
        loads = [sum(lengths[j] for j in s) for s in shards]
        assert max(loads) - min(loads) <= max(lengths), loads
    assert shard_plan([5, 5, 5, 5], 2) == [[0, 2], [1, 3]]
    assert shard_plan([1], 3) == [[0], [], []]


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _fake(j):
    """a tracklet's per-frame results, distinct per tracklet"""
    n = 2 + j % 4
    return [1.0 - 0.01 * j - 0.001 * t for t in range(n)], [0.1 * j + 0.01 * t for t in range(n)], [(j, t) for t in range(n)]


def _gather_worker(rank, world, port, n, out_dir):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    mine = shard_plan([len(_fake(j)[0]) for j in range(n)], world)[rank]
    local = {"overlaps": [_fake(j)[0] for j in mine], "distances": [_fake(j)[1] for j in mine],
             "results": [_fake(j)[2] for j in mine]}
    torch.save(gather_shards(n, mine, local), os.path.join(out_dir, f"rank{rank}.pt"))
    dist.destroy_process_group()


def test_gather_reassembles_global_order(tmp_path):
    from open3dsot_b200.utils.metrics import Precision, Success
    n = 9
    mp.spawn(_gather_worker, args=(2, _free_port(), n, str(tmp_path)), nprocs=2, join=True)
    r0, r1 = (torch.load(os.path.join(tmp_path, f"rank{r}.pt"), weights_only=False) for r in range(2))
    assert r0 == r1
    assert r0["overlaps"] == [_fake(j)[0] for j in range(n)] and r0["results"] == [_fake(j)[2] for j in range(n)]
    succ, prec = Success(), Precision()
    for j in range(n):
        succ(_fake(j)[0])
        prec(_fake(j)[1])
    assert r0["success"] == succ.compute() and r0["precision"] == prec.compute()
    assert r0["frames"] == sum(len(_fake(j)[0]) for j in range(n))


def test_resumed_top_k_starts_empty_and_keeps_the_old_run_s_files(tmp_path):
    """Lightning 1.3.8 restores only the best score and path: the resumed run writes its own first k files and deletes
    nothing of the run it resumed from, even when its scores are worse."""
    old = os.path.join(str(tmp_path), "version_0", "epoch=3-step=39.ckpt")
    new = os.path.join(str(tmp_path), "version_1")
    t = TopK(1, new)
    t.load_state_dict({"monitor": "precision/test", "best_model_score": torch.tensor(90.0), "best_model_path": old,
                       "current_score": torch.tensor(90.0), "dirpath": os.path.dirname(old)})
    assert (t.best_path, t.best_score, t.best_k) == (old, 90.0, {})
    f = lambda e: os.path.join(new, TopK.filename(e, 10 * (e + 1)))
    assert t.update(50.0, 4, 50) == (f(4), [])
    assert t.update(60.0, 5, 60) == (f(5), [f(4)])
    assert t.best_path == f(5)


def test_trainer_refuses_frozen_parameters(tmp_path):
    cfg = load_config(os.path.join(ROOT, "cfgs", "P2B_Car.yaml"))
    net = get_model(cfg.net_model)(cfg)
    next(net.parameters()).requires_grad_(False)
    with pytest.raises(ValueError, match="frozen"):
        Trainer(net, cfg, [], [], str(tmp_path))


def one_frame_tracklets(n, n_points=2000):
    """n one-frame tracklets, each with its own box size: a sample's `bbox_size` names its frame, and a candidate-0 sample
    (no search offset) is the only one whose `box_label` centre is exactly zero."""
    from open3dsot_b200.datasets.synthetic import synthetic_sequence
    return [synthetic_sequence(n_frames=1, n_points=n_points, seed=700 + k, n_object=400,
                               wlh=(1.5 + 0.1 * k, 3.6 + 0.15 * k, 1.4 + 0.05 * k)) for k in range(n)]


def check_batch_follows(batch, smp, indices):
    """sample i of `batch` was built from sample index indices[i] (frame indices[i] // C, candidate indices[i] % C)"""
    idx = indices.cpu()
    nc = smp.num_candidates
    assert torch.equal(batch["bbox_size"].cpu(), smp.data.wlh.cpu()[idx // nc])
    assert torch.equal((batch["box_label"][:, :3] == 0).all(1).cpu(), idx % nc == 0)


def test_sampler_batch_follows_the_given_indices():
    from open3dsot_b200.datasets.device_sampler import DeviceSiameseSampler
    cfg = load_config(os.path.join(ROOT, "cfgs", "BAT_Car.yaml"), {"up_axis": [0, 0, 1]})
    smp = DeviceSiameseSampler(one_frame_tracklets(8), cfg, "cpu", seed=3)
    assert not smp.use_graph and len(smp) == 8 * cfg.num_candidates == 32
    assert len(torch.unique(smp.data.wlh, dim=0)) == 8
    for indices in (torch.tensor([31, 0, 5, 18, 7, 26, 12, 3]), torch.tensor([1, 2, 4, 8, 16, 30, 9, 20])):
        batch, valid = smp.next_batch(8, indices=indices)
        assert bool(valid.all())
        check_batch_follows(batch, smp, indices)
    with pytest.raises(ValueError, match="indices"):
        smp.next_batch(8, indices=torch.arange(4))
