"""Training-step engine: flat parameter bucket + one-launch Adam + optional whole-step CUDA graph.

The reference trains through Lightning (`main.py:82-86`): per step DDP-wrapped `training_step`, backward, bucketed
all-reduce, `Adam(betas=(0.5, 0.999), eps=1e-6)` (`models/base_model.py:28-36`).  A BAT step is a few milliseconds of GPU
work spread over ~10^3 kernel launches, so the step is launch-bound unless it is captured: `TrainStep` records
zero-grad -> training_step -> backward -> gradient all-reduce -> Adam into ONE CUDA graph over static batch buffers
and replays it; the loss stays on the device (the reference's twelve `.item()` syncs per step, `bat.py:146-163`, are
not reproduced).
"""
import torch

from . import _lib, ddp, ops, runtime


class BatchSlab:
    """A batch dict laid out in ONE contiguous byte buffer (every tensor a 256-byte-aligned view of it): a step's inputs
    move host -> device (pinned slab -> device slab) and device -> static graph inputs with one copy each instead of one
    per tensor — at a few milliseconds per step seven small copies per hop are visible, and under DDP eight processes
    issuing them skew the ranks."""

    def __init__(self, spec, device, pin=False):
        self.spec = spec                                          # [(key, shape, dtype, offset, nbytes)]
        total = spec[-1][3] + spec[-1][4] if spec else 0
        self.buf = torch.empty(total, dtype=torch.uint8, device=device)
        if pin and self.buf.device.type == "cpu":
            self.buf = self.buf.pin_memory()
        self.tensors = {k: self.buf[off:off + nb].view(dt).view(shape) for k, shape, dt, off, nb in spec}
        self.nbytes = total

    @classmethod
    def like(cls, batch, device, pin=False):
        spec, off = [], 0
        for k, v in batch.items():
            nb = v.numel() * v.element_size()
            spec.append((k, tuple(v.shape), v.dtype, off, nb))
            off += (nb + 255) & ~255
        return cls(spec, device, pin)

    def load(self, batch):
        for k, v in batch.items():
            self.tensors[k].copy_(v, non_blocking=True)
        return self

    def sibling(self, device, pin=False):
        return BatchSlab(self.spec, device, pin)


class FlatAdam:
    """Adam over `FlatParams` with the step counter and learning rate in device memory (graph-replayable)."""

    def __init__(self, flat, lr=1e-3, betas=(0.5, 0.999), eps=1e-6, weight_decay=0.0):
        self.flat = flat
        self.betas, self.eps, self.wd = betas, eps, weight_decay
        self.exp_avg = torch.zeros_like(flat.flat)
        self.exp_avg_sq = torch.zeros_like(flat.flat)
        self.state = torch.tensor([0.0, lr], dtype=torch.float32, device=flat.flat.device)

    def set_lr(self, lr):
        self.state[1] = lr

    def step(self):
        ops._call("o3d_adam_step", self.flat.flat.data_ptr(), self.flat.grad.data_ptr(), self.exp_avg.data_ptr(),
                  self.exp_avg_sq.data_ptr(), self.flat.numel, self.state.data_ptr(), self.betas[0], self.betas[1],
                  self.eps, self.wd, ops._stream())
        runtime.advance_weights_generation()

    def _slices(self):
        off = 0
        for p in self.flat.params:
            yield off, p
            off += p.numel()

    def state_dict(self, initial_lr=None):
        """`torch.optim.Adam.state_dict()` of one param group over `flat.params` (the model's trainable parameters, in order;
        the indices match an Adam over all of `model.parameters()`, the reference's, only when none is frozen, which
        `trainer.Trainer` requires): `state`
        keyed by parameter index with `step`, `exp_avg` and `exp_avg_sq` (CPU copies of slices of the flat buffers), or empty
        before the first step, as Adam's is."""
        step, lr = (float(v) for v in self.state.cpu())
        state = {}
        if step > 0:
            for i, (off, p) in enumerate(self._slices()):
                n = p.numel()
                state[i] = {"step": torch.tensor(step), "exp_avg": self.exp_avg[off:off + n].view_as(p).cpu().clone(),
                            "exp_avg_sq": self.exp_avg_sq[off:off + n].view_as(p).cpu().clone()}
        group = {"lr": lr, "betas": tuple(self.betas), "eps": self.eps, "weight_decay": self.wd, "amsgrad": False,
                 "initial_lr": lr if initial_lr is None else initial_lr, "params": list(range(len(self.flat.params)))}
        return {"state": state, "param_groups": [group]}

    def load_state_dict(self, sd):
        """Moments and step from an Adam state dict (ours or a Lightning checkpoint's `optimizer_states[0]`).  An empty `state`
        means zero moments and step 0.  The learning rate is left to the caller's schedule."""
        params = self.flat.params
        groups = sd["param_groups"]
        n = sum(len(g["params"]) for g in groups)
        if len(groups) != 1 or n != len(params):
            raise ValueError(f"Adam state: {len(groups)} param group(s) over {n} parameters; the model has one group of "
                             f"{len(params)}")
        state = sd["state"]
        exp_avg, exp_avg_sq = torch.zeros_like(self.exp_avg), torch.zeros_like(self.exp_avg_sq)
        steps = set()
        for i, (off, p) in enumerate(self._slices()):
            s = state.get(groups[0]["params"][i])
            if s is None:
                if state:
                    raise ValueError(f"Adam state: parameter {i} has no state while others have")
                continue
            for key, dst in (("exp_avg", exp_avg), ("exp_avg_sq", exp_avg_sq)):
                if tuple(s[key].shape) != tuple(p.shape):
                    raise ValueError(f"Adam state: parameter {i} {key} has shape {tuple(s[key].shape)}, the model's is "
                                     f"{tuple(p.shape)}")
                dst[off:off + p.numel()].copy_(s[key].reshape(-1))
            steps.add(float(s["step"]))
        if len(steps) > 1:
            raise ValueError(f"Adam state: the parameters' steps differ ({sorted(steps)}); the flat optimizer keeps one")
        self.exp_avg.copy_(exp_avg)
        self.exp_avg_sq.copy_(exp_avg_sq)
        self.state[0] = steps.pop() if steps else 0.0


class TrainStep:
    """`step(batch) -> loss` for a model exposing `training_step(batch, idx)`; `batch` is a dict of device tensors.
    `precision`: "fp32" (3xTF32 GEMMs, default) or "bf16" (BF16 operands with FP32 accumulation in the tensor-core GEMMs of the
    MLP stacks, runtime.training_precision_scope); the eager steps and the captured one both run in it."""

    def __init__(self, model, lr=1e-3, weight_decay=0.0, use_graph=True, warmup=3, capture_collective=True, precision="fp32"):
        self.precision = runtime.check_precision(precision)
        self.model = model
        self.capture_collective = capture_collective
        self.flat = ddp.FlatParams(model)
        ddp.broadcast_parameters(self.flat, model)
        self.opt = FlatAdam(self.flat, lr=lr, weight_decay=weight_decay)
        self.use_graph = use_graph
        self.warmup = warmup
        self.graph = None
        self.static_batch = None
        self.static_loss = None
        self.calls = 0

    def _fwd_bwd(self, batch):
        self.flat.zero_grad()
        loss = self.model.training_step(dict(batch), 0)
        from . import runtime
        with runtime.grad_inplace_scope():       # parameter gradients are added straight into the flat bucket's views
            loss.backward()
        return loss.detach()

    def _finish(self):
        ddp.allreduce_gradients(self.flat)      # one NCCL all-reduce of the flat bucket (no-op on a single rank)
        self.opt.step()

    def _eager(self, batch):
        if isinstance(batch, BatchSlab):
            batch = batch.tensors
        loss = self._fwd_bwd(batch)
        self._finish()
        return loss

    def _capture(self, batch):
        # static inputs live in ONE slab, so a step's batch arrives with a single copy (BatchSlab) instead of one per tensor
        if isinstance(batch, BatchSlab):
            batch = batch.tensors
        self.static_slab = BatchSlab.like(batch, device=self.flat.flat.device)
        self.static_slab.load(batch)
        self.static_batch = self.static_slab.tensors
        # settle allocator / lazy initialisation on a side stream, WITHOUT advancing training: parameters, optimizer
        # state and BatchNorm buffers are snapshotted and restored around the two throw-away steps
        buffers = list(self.model.buffers())
        snap = (self.flat.flat.clone(), self.opt.exp_avg.clone(), self.opt.exp_avg_sq.clone(), self.opt.state.clone(),
                [b.clone() for b in buffers])
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(2):
                self._eager(self.static_batch)
        torch.cuda.current_stream().wait_stream(s)
        with torch.no_grad():
            self.flat.flat.copy_(snap[0]); self.opt.exp_avg.copy_(snap[1]); self.opt.exp_avg_sq.copy_(snap[2])
            self.opt.state.copy_(snap[3])
            for b, old in zip(buffers, snap[4]):
                b.copy_(old)
        # The whole step — zero-grad, forward, backward, the NCCL all-reduce of the flat bucket and Adam — is ONE graph, also
        # under DDP: nothing trails the replay.  NCCL collectives are capturable; the capture runs in thread-local error mode so
        # that the process group's watchdog thread (which polls CUDA events) cannot invalidate it.  Should a NCCL / torch build
        # refuse the capture, the collective and Adam fall back to being enqueued right behind the replay.
        self.graph_has_update = True
        if ddp.is_distributed() and not self.capture_collective:
            self.graph_has_update = False
        try:
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph, capture_error_mode="thread_local"):
                self.static_loss = self._fwd_bwd(self.static_batch)
                if self.graph_has_update:
                    self._finish()
        except Exception:
            if not (ddp.is_distributed() and self.graph_has_update):
                raise
            torch.cuda.synchronize()
            self.graph_has_update = False
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph, capture_error_mode="thread_local"):
                self.static_loss = self._fwd_bwd(self.static_batch)

    def step(self, batch):
        with runtime.training_precision_scope(self.precision):
            return self._step(batch)

    def _step(self, batch):
        self.calls += 1
        if not self.use_graph or self.calls <= self.warmup:
            return self._eager(batch)
        if self.graph is None:
            self._capture(batch)
        if isinstance(batch, BatchSlab):
            self.static_slab.buf.copy_(batch.buf, non_blocking=True)      # ONE device copy for the whole batch
        else:
            for k, v in batch.items():
                self.static_batch[k].copy_(v, non_blocking=True)
        self.graph.replay()
        if not self.graph_has_update:
            self._finish()
        runtime.advance_weights_generation()        # the replayed Adam and BatchNorm writes bump no tensor version
        return self.static_loss
