"""Training and testing from a config, as the reference's `main.py` drives Lightning (main.py:66-93): epochs over the
training split, a validation every `check_val_every_n_epoch` epochs, the best checkpoints by `precision/test`, resumable
runs.  The pieces are the project's own: the device sampler, the graph-captured `engine.TrainStep`, split evaluation with
many tracklets in flight, sharded across ranks under DDP, and checkpoints in Lightning 1.3.8's layout.

    Trainer(model, cfg, train_tracklets, val_tracklets, log_dir).fit()

Lightning itself, TensorBoard and the sanity-validation steps are not reproduced; nor are SGD, gradient clipping and the
`random_sample` sampler, which no shipped config uses."""
import json
import math
import os
import time

import torch

from . import ddp
from .checkpoint import ModelCheckpoint, load_lightning_checkpoint, model_checkpoint_state, save_lightning_checkpoint
from .tracking.evaluate import evaluate_sharded

MONITOR = "precision/test"
# main.py:34-38: the reference's command-line defaults, which override the config's keys of the same name
DEFAULTS = {"batch_size": 100, "epoch": 60, "save_top_k": -1, "check_val_every_n_epoch": 1}


def check_supported(cfg):
    """A ValueError naming the first setting the trainer does not implement."""
    if str(cfg.get("optimizer", "Adam")).lower() != "adam":
        raise ValueError(f"optimizer: {cfg.optimizer!r} is not supported; only Adam is")
    if float(cfg.get("gradient_clip_val", 0) or 0) != 0:
        raise ValueError(f"gradient_clip_val: {cfg.gradient_clip_val} is not supported; only 0 (no clipping) is")
    if cfg.get("random_sample", False):
        raise ValueError("random_sample: True is not supported; epochs pass over every frame (random_sample: False)")
    if str(cfg.get("precision", "fp32")) != "fp32":
        raise ValueError(f"precision: {cfg.precision!r} is for inference only (--test); training and its validation run in fp32")
    if cfg.get("train_precision", "fp32") not in ("fp32", "bf16"):
        raise ValueError(f"train_precision: {cfg.train_precision!r} is not supported; only 'fp32' and 'bf16' are")


def epoch_indices(n, epoch, seed=0, rank=0, world=1):
    """The samples rank `rank` of `world` trains on in `epoch`: `DistributedSampler(shuffle=True)` over `n` samples, with
    `set_epoch(epoch)` and `seed`.  One permutation seeded by seed + epoch, padded by repeating its head to a multiple of
    `world`, of which the rank takes every `world`-th entry from `rank` on."""
    g = torch.Generator()
    g.manual_seed(seed + epoch)
    perm = torch.randperm(n, generator=g).tolist()
    total = -(-n // world) * world
    pad = total - n
    perm += (perm * math.ceil(pad / n))[:pad] if pad else []
    return perm[rank:total:world]


def steps_per_epoch(n, batch_size, world=1):
    """Full batches per rank and epoch (the reference's DataLoader drops the last partial one)."""
    return -(-n // world) // batch_size


def step_lr(base_lr, gamma, step_size, epoch):
    """`StepLR`'s learning rate in `epoch`: base_lr * gamma ** (epoch // step_size), multiplied out step by step as StepLR
    does, so the value is the same float."""
    lr = base_lr
    for _ in range(epoch // step_size):
        lr *= gamma
    return lr


class TopK:
    """ModelCheckpoint(monitor='precision/test', mode='max', save_top_k=k, save_last=True) of Lightning 1.3: which epoch files
    to write and delete, and the state it stores in a checkpoint's `callbacks`.  k = -1 keeps every file, 0 none, k > 0 the
    best k; a score that only ties the k-th best does not replace it."""

    def __init__(self, k, dirpath):
        self.k, self.dirpath = int(k), dirpath
        self.best_k = {}                      # path -> score
        self.best_score, self.best_path, self.current = None, "", None

    @staticmethod
    def filename(epoch, global_step):
        """Lightning 1.3 names the file of 0-based epoch e by the steps done minus one."""
        return f"epoch={epoch}-step={global_step - 1}.ckpt"

    def update(self, score, epoch, global_step):
        """Returns (path to write or None, paths to delete).  Only files this run wrote are ever deleted."""
        score = float(torch.tensor(float(score)))     # Lightning keeps the monitored score as a float32 tensor, and stores it so
        self.current = score
        if self.k == 0 or not math.isfinite(score):
            return None, []
        path = os.path.join(self.dirpath, self.filename(epoch, global_step))
        drop = []
        if 0 < self.k <= len(self.best_k):
            worst = min(self.best_k, key=self.best_k.get)
            if not score > self.best_k[worst]:
                return None, []
            del self.best_k[worst]
            drop.append(worst)
        self.best_k[path] = score
        self.best_path = max(self.best_k, key=self.best_k.get)
        self.best_score = self.best_k[self.best_path]
        return path, drop

    def state_dict(self):
        t = lambda v: None if v is None else torch.tensor(float(v))
        return {"monitor": MONITOR, "best_model_score": t(self.best_score), "best_model_path": self.best_path,
                "current_score": t(self.current), "dirpath": self.dirpath}

    def load_state_dict(self, sd):
        """As Lightning 1.3.8's `on_load_checkpoint`: the best score and path are restored; the top-k set starts empty, so a
        resumed run writes its own first k files and never deletes a file of the run it resumed from."""
        score = sd.get("best_model_score")
        self.best_score = None if score is None else float(score)
        self.best_path = sd.get("best_model_path") or ""
        self.current = None if sd.get("current_score") is None else float(sd["current_score"])
        self.best_k = {}


def load_weights(model, state_dict):
    """`model.load_state_dict` that also accepts the reference's extra metric-module buffers (`prec.*`, `success.*`, ...:
    torchmetrics state, no weights) and refuses a file that lacks any of the model's entries."""
    missing, unexpected = model.load_state_dict(state_dict, strict=False)
    unexpected = [k for k in unexpected if k.split(".")[0] not in ("prec", "success", "seg_acc", "motion_acc")]
    if missing or unexpected:
        raise ValueError(f"checkpoint weights do not fit the model: missing {missing[:5]}, unexpected {unexpected[:5]}")


def _next_version(log_dir):
    root = os.path.join(log_dir, "lightning_logs")
    used = [int(d[8:]) for d in (os.listdir(root) if os.path.isdir(root) else []) if d.startswith("version_") and d[8:].isdigit()]
    return max(used, default=-1) + 1


class Trainer:
    """`fit()` trains `model` for `cfg.epoch` epochs on `train_tracklets` (the readers' `tracklets()` lists) with the
    reference's Adam(betas=(0.5, 0.999), eps=1e-6) and StepLR, validating on `val_tracklets` every
    `cfg.check_val_every_n_epoch` epochs with `slots` tracklets in flight; `test(tracklets)` evaluates; `save` / `resume`
    write and read checkpoints in the layout of the reference's.  Under torch.distributed every rank runs one, on its own GPU."""

    def __init__(self, model, cfg, train_tracklets, val_tracklets, log_dir, seed=0, slots=32):
        from .engine import TrainStep
        check_supported(cfg)
        frozen = [n for n, p in model.named_parameters() if not p.requires_grad]
        if frozen:      # the flat Adam covers trainable parameters only; the reference's covers all of model.parameters()
            raise ValueError(f"Trainer: frozen parameters {frozen[:5]} would shift the checkpoint's Adam state indices")
        self.model, self.cfg, self.seed, self.slots = model, cfg, int(seed), int(slots)
        self.val_tracklets = list(val_tracklets)
        self.log_dir = log_dir
        get = lambda k: cfg.get(k, DEFAULTS[k])
        self.batch_size, self.max_epochs = int(get("batch_size")), int(get("epoch"))
        self.val_every = int(get("check_val_every_n_epoch"))
        self.rank, self.world = (torch.distributed.get_rank(), torch.distributed.get_world_size()) if ddp.is_distributed() else (0, 1)
        self.base_lr, self.gamma, self.step_size = float(cfg.lr), float(cfg.lr_decay_rate), int(cfg.lr_decay_step)
        self.epoch, self.global_step = 0, 0
        self.dirpath = None
        self.top_k = TopK(get("save_top_k"), "")
        self.sampler = None
        from .datasets.device_sampler import DeviceMotionSampler, DeviceSiameseSampler, DeviceTracklets
        if not isinstance(train_tracklets, DeviceTracklets):      # (or the tracklets already on the device)
            train_tracklets = [t for t in train_tracklets if len(t)] or None
        if train_tracklets is not None:
            cls = DeviceMotionSampler if str(cfg.get("train_type", "")).lower() == "train_motion" else DeviceSiameseSampler
            self.sampler = cls(train_tracklets, cfg, next(model.parameters()).device, seed=self.seed + self.rank)
        self.model.train()
        # the training steps' GEMM precision; validation and test() run in fp32 whatever it is (eval-mode stacks ignore it)
        self.train_precision = str(cfg.get("train_precision", "fp32"))
        self.step = TrainStep(model, lr=self.base_lr, weight_decay=cfg.wd, precision=self.train_precision)
        self.step.opt.set_lr(self.lr)
        self._keys = None

    @property
    def lr(self):
        return step_lr(self.base_lr, self.gamma, self.step_size, self.epoch)

    def epoch_order(self, epoch):
        """This rank's sample indices in `epoch`, cut to whole batches."""
        n = len(self.sampler)
        idx = epoch_indices(n, epoch, self.seed, self.rank, self.world)
        return idx[: steps_per_epoch(n, self.batch_size, self.world) * self.batch_size]

    # ---- training ---------------------------------------------------------------------------------------------------
    def train_epoch(self):
        """One epoch; returns the mean of every loss term the model logs and the epoch's host-clock seconds.  The terms are
        summed on the device and read back once."""
        if self.sampler is None:
            raise ValueError("Trainer: no training tracklets")
        dev = self.step.flat.flat.device
        B = self.batch_size
        order = torch.tensor(self.epoch_order(self.epoch), dtype=torch.int64, device=dev)
        steps = order.numel() // B
        if steps == 0:
            raise ValueError(f"Trainer: {len(self.sampler)} samples over {self.world} rank(s) make no batch of {B}")
        self.step.opt.set_lr(self.lr)
        self.model.train()
        acc = None
        t0 = time.perf_counter()
        for s in range(steps):
            batch, _ = self.sampler.next_batch(B, indices=order[s * B:(s + 1) * B])
            self.step.step(batch)
            logged = self.model.logged
            if acc is None:
                self._keys = list(logged)
                acc = torch.zeros(len(self._keys), dtype=torch.float64, device=dev)
            acc += torch.stack([logged[k].reshape(()) for k in self._keys])
        if self.world > 1:
            torch.distributed.all_reduce(acc)
            acc /= self.world
        means = (acc / steps).tolist()
        seconds = time.perf_counter() - t0
        self.global_step += steps
        self.epoch += 1
        return dict(zip(self._keys, means)), seconds, steps

    def fit(self):
        """Train until `cfg.epoch` epochs are done, from where `resume` left off.  Returns the metrics of the last epoch."""
        if self.dirpath is None:
            version = _next_version(self.log_dir) if self.rank == 0 else None
            if self.world > 1:
                box = [version]
                torch.distributed.broadcast_object_list(box, src=0)
                version = box[0]
            self.dirpath = os.path.join(self.log_dir, "lightning_logs", f"version_{version}", "checkpoints")
            self.top_k.dirpath = self.dirpath
            if self.rank == 0:
                os.makedirs(self.dirpath, exist_ok=True)
        row = None
        while self.epoch < self.max_epochs:
            epoch, lr = self.epoch, self.lr
            losses, train_s, steps = self.train_epoch()
            row = {"epoch": epoch, "global_step": self.global_step, "lr": lr, **losses, "success": None, "precision": None,
                   "train_seconds": train_s, "pairs_per_second": steps * self.batch_size * self.world / train_s,
                   "val_seconds": None, "train_precision": self.train_precision}
            if (epoch + 1) % self.val_every == 0 and self.val_tracklets:
                t0 = time.perf_counter()
                res = self.test(self.val_tracklets)
                row.update(success=res["success"], precision=res["precision"], val_seconds=time.perf_counter() - t0)
                path, drop = self.top_k.update(res["precision"], epoch, self.global_step)
                if path is not None:
                    self.save(path)
                if self.rank == 0:
                    for p in drop:
                        if os.path.exists(p):
                            os.remove(p)
            self.save(os.path.join(self.dirpath, "last.ckpt"))
            if self.rank == 0:
                line = json.dumps(row)
                print(line, flush=True)
                with open(os.path.join(self.log_dir, "metrics.jsonl"), "a") as f:
                    f.write(line + "\n")
        return row

    def test(self, tracklets):
        """Success / Precision of the model on `tracklets` (split across the ranks under DDP); the model is left in
        training mode.  Under DDP, rank 0's buffers (the BatchNorm running statistics, which each rank updates from its own
        batches) are broadcast first, as the reference's DDP wrapper does on the first forward after training: every rank
        scores the model `save()` writes."""
        ddp.broadcast_buffers(self.model)
        try:
            return evaluate_sharded(self.model, tracklets, slots=self.slots, seed=self.seed)
        finally:
            self.model.train()

    # ---- checkpoints --------------------------------------------------------------------------------------------------
    def scheduler_state(self):
        """StepLR.state_dict() after `self.epoch` scheduler steps, with the fields Lightning 1.3.8's checkpoints hold."""
        return {"step_size": self.step_size, "gamma": self.gamma, "base_lrs": [self.base_lr], "last_epoch": self.epoch,
                "_step_count": self.epoch + 1, "verbose": False, "_get_lr_called_within_step": False, "_last_lr": [self.lr]}

    def save(self, path):
        """The model, Adam state, epoch / step counters, scheduler and checkpoint bookkeeping, as Lightning 1.3.8 lays them
        out.  Only rank 0 writes."""
        if self.rank != 0:
            return None
        os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
        return save_lightning_checkpoint(self.model, path, epoch=self.epoch, global_step=self.global_step,
                                         optimizer_states=[self.step.opt.state_dict(initial_lr=self.base_lr)],
                                         lr_schedulers=[self.scheduler_state()],
                                         callbacks={ModelCheckpoint: self.top_k.state_dict()})

    def resume(self, path):
        """Continue from a checkpoint of ours or of the reference's: weights and BatchNorm buffers, Adam moments and step,
        epoch and global step, the scheduler (its step_size and gamma take precedence over the config's, as in Lightning)
        and the best-score bookkeeping.  The epoch order continues as an uninterrupted run's."""
        ckpt = load_lightning_checkpoint(path)
        opt_states = ckpt.get("optimizer_states") or []
        if len(opt_states) > 1:
            raise ValueError(f"resume: {len(opt_states)} optimizer states; the trainer has one Adam")
        snap = (self.step.opt.exp_avg.clone(), self.step.opt.exp_avg_sq.clone(), self.step.opt.state.clone())
        if opt_states:
            self.step.opt.load_state_dict(opt_states[0])        # validated before the weights change
        try:
            load_weights(self.model, ckpt["state_dict"])
        except Exception:
            self.step.opt.exp_avg.copy_(snap[0]); self.step.opt.exp_avg_sq.copy_(snap[1]); self.step.opt.state.copy_(snap[2])
            raise
        self.epoch, self.global_step = int(ckpt["epoch"]), int(ckpt["global_step"])
        sched = (ckpt.get("lr_schedulers") or [{}])[0]
        self.gamma = float(sched.get("gamma", self.gamma))
        self.step_size = int(sched.get("step_size", self.step_size))
        self.base_lr = float((sched.get("base_lrs") or [self.base_lr])[0])
        state = model_checkpoint_state(ckpt)
        if state is not None:
            self.top_k.load_state_dict(state)
        self.step.opt.set_lr(self.lr)
        return ckpt
