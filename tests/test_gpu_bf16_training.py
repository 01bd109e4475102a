"""BF16 training precision (runtime.training_precision_scope("bf16"), engine.TrainStep(precision="bf16"), o3d_stack_t.precision
= 2) on the GPU:

  - every bf16 training instantiation (forward, dgrad with each epilogue stride, plain and lifted; the split-K weight gradient,
    plain and lifted; the fused narrow-layer backward) on dense, pooled and lifted stacks, against a float64 composition that
    rounds to bf16 where the kernels do (the weights, each GEMM input row, dY after the BN-backward / ReLU coefficients, the
    weight gradient's layer input) and against the unrounded float64 composition, with the kernels that ran read from a CUDA
    profile and no 3xTF32 GEMM among them;
  - whole models: one training step of BAT-Car and P2B-Car against the float64 oracle, and of M2-Track against its float64 host
    mirror and a float64 emulation of the bf16 rounding, with every discrete decision on computed values held fixed;
  - the training step: graph replay against the eager step from one state, repeat runs, and no leakage of a bf16 step into a
    later fp32 one;
  - the trainer end to end in bf16: checkpoints hold fp32 tensors, score as logged, and a resumed run continues in bf16.
Measured values are printed (pytest -s) and recorded in DESIGN.md section 4.5."""
import functools
import glob
import json
import math
import os
import re
import subprocess
import sys
import tempfile
import zlib

import pytest
import torch
import torch.nn.functional as F

from open3dsot_b200 import fused, runtime
from open3dsot_b200.datasets.synthetic import synthetic_siamese_batch
from open3dsot_b200.engine import TrainStep
from test_gpu_engine import _bat, _restore, _snapshot
from test_gpu_lift_paths import Case as LiftCase, make_inputs
from test_gpu_stack_paths import _ran, build_stack
from test_gpu_trainer import _cfg, _model, _tracklets

pytestmark = pytest.mark.gpu
EMULATED_BAR = 1e-3      # against the float64 composition that rounds to bf16 where the kernels do: fp32 accumulation order
# Gradients against that composition: 1e-3 (EMULATED_BAR), or the case's own `grad_bar` where it is measured higher.  The
# composition's activations are float64 where the kernels' are fp32, so about 1 in 4e4 of them rounds to the other bf16
# neighbour; that moves the forward by ~3e-5 per element, and every ReLU mask or pooling arg-max decided within that distance
# flips and moves one gradient element by its whole value.  Eight of the eleven cases measure <= 6e-4 and keep 1e-3 (2e-3 for the
# one at 5.6e-4), which an operand left unrounded (about one bf16 ulp, 1e-3 relative, on a GEMM) still crosses.  The two pooled
# cases at P = 65,536 (hundreds of thousands of pooling groups) measure 5e-3 and 7e-3, the 384-wide dense case 1.6e-3; their
# bars are set at twice to three times those values.
UNROUNDED_BAR = 3e-2     # forward output against the plain float64 composition: bf16 operand rounding through the stack
# Gradients against the plain float64 composition.  The bf16 forward moves each pre-activation by ~1e-3 of its scale, which flips
# the ReLU mask (and the pooling arg-max) of the elements that close to the threshold; each flip changes that element's gradient by
# its whole value, so the relative L2 error grows as the square root of the flipped fraction: 4e-2 to 1.3e-1 on these random
# stacks.  Rounding only the backward's operands (dY, the weights, the layer input) costs 3e-3 to 4e-3 on the same stacks, and
# the rounding-aware composition still agrees to EMULATED_BAR, so the kernels are not the cause (DESIGN.md section 4.5).
GRAD_UNROUNDED_BAR = 1.5e-1

TF = {ld: f"pw_tc_kernel<Bf16<TcAct>,TcFwdEpi<{ld}>>" for ld in (64, 128, 256, 0)}
LF = {ld: f"pw_tc_kernel<Bf16<TcLift>,TcFwdEpi<{ld}>>" for ld in (128, 256)}
TD = {ld: f"pw_tc_kernel<Bf16<TcDy>,TcDgradEpi<{ld},false>>" for ld in (64, 128, 256, 0)}
LD = {ld: f"pw_tc_kernel<Bf16<TcDy>,TcDgradEpi<{ld},true>>" for ld in (64, 128, 256, 0)}
TW, LW = "pw_wgrad_tc_kernel<Bf16<TcAct>>", "pw_wgrad_tc_kernel<Bf16<TcLift>>"
FA = {n: f"pw_bwd_tc_kernel<Bf16<TcAct>,{n}>" for n in (64, 128)}
FL = {n: f"pw_bwd_tc_kernel<Bf16<TcLift>,{n}>" for n in (64, 128)}
TAIL_DG, RED = "pw_dgrad_kernel<64>", "wgrad_reduce_kernel"
KERNELS = [*TF.values(), *LF.values(), *TD.values(), *LD.values(), TW, LW, *FA.values(), *FL.values()]
# every 3xTF32 tensor-core GEMM: none may run inside the bf16 scope
FP32_GEMMS = ["pw_tc_kernel<TcAct,", "pw_tc_kernel<TcLift,", "pw_tc_kernel<TcDy,", "pw_wgrad_tc_kernel<TcAct>",
              "pw_wgrad_tc_kernel<TcLift>", "pw_bwd_tc_kernel<TcAct,", "pw_bwd_tc_kernel<TcLift,"]


class Case:
    """chans (lifted: chans[0] = C0, the lifted layer's width), layer kinds as in test_gpu_stack_paths, P, pooling group S; lift:
    None or (grp, clouds, rows) of the lifted first layer; want: the kernels the case exists to reach."""

    def __init__(self, name, chans, kinds, P, S=0, lift=None, want=(), grad_bar=EMULATED_BAR):
        self.name, self.chans, self.kinds, self.P, self.S, self.lift, self.want = name, chans, kinds, P, S, lift, tuple(want)
        self.grad_bar = grad_bar


CASES = [
    # dense: forward epilogues 128 / 256, dgrad strides 64 / 128 / 256, the split-K weight gradient
    Case("dense_64_128_256_128", [64, 128, 256, 128], "BR BR BR", 5000,
         want=[TF[128], TF[256], TD[64], TD[128], TD[256], TW, RED]),
    # a first layer with a ragged tail (K0 = 132): tensor cores on 128 input channels, runtime-stride dgrad, the tail's dgrad and
    # weight gradient on the fp32 CUDA-core kernels; pooled last layer
    Case("ktail_pooled", [132, 128, 256], "BR BR", 32 * 140, S=32, want=[TF[128], TF[256], TD[0], TD[128], TW, TAIL_DG]),
    # runtime-stride forward (Nw = 384) and dgrad (K = 384), a 64-wide forward
    Case("wide384", [64, 384, 64], "BR B", 2048, want=[TF[0], TF[64], TD[64], TD[0]], grad_bar=4e-3),
    # the fused narrow-layer backward at P = 65,536, dense layers and a pooled dY
    Case("fused_pooled", [64, 128, 64, 128], "BR BR BR", 65536, S=16, want=[FA[64], FA[128], RED], grad_bar=1.5e-2),
    Case("fused_dense_bias", [128, 128, 64], "bR B", 65536, want=[FA[128]]),
    # lifted first layer: the lifted loader in the forward, the lifted dgrad epilogue with each stride, the lifted weight gradient
    Case("lift_c64", [64, 256, 128], "BR BR BR", 4096, S=32, lift=(32, 2, 300), want=[LF[256], LD[64], LW, TF[128], TD[256]]),
    Case("lift_c128", [128, 256, 128], "BR BR BR", 4096, S=32, lift=(32, 2, 200), want=[LF[256], LD[128], LW]),
    Case("lift_c256", [256, 256, 256], "BR BR BR", 4096, S=32, lift=(32, 4, 256), want=[LF[256], LD[256], LW]),
    Case("lift_c96", [96, 128, 128], "BR BR BR", 16 * 260, S=16, lift=(16, 2, 500), want=[LF[128], LD[0], LW], grad_bar=2e-3),
    # the fused backward with a lifted input, both widths
    Case("lift_fused_c64", [64, 128, 128], "BR BR BR", 65536, S=32, lift=(32, 2, 1000), want=[FL[64], FA[128]]),
    Case("lift_fused_c128", [128, 64, 128], "BR BR BR", 65536, S=64, lift=(64, 2, 1000), want=[FL[128], FA[64]],
         grad_bar=2e-2),
]


def test_every_bf16_training_kernel_is_a_declared_target():
    declared = {k for c in CASES for k in c.want}
    assert set(KERNELS) <= declared, sorted(set(KERNELS) - declared)
    assert len({c.name for c in CASES}) == len(CASES)


def _r4(c):
    return (c + 3) & ~3


def _tc_main(c):
    return (c // 128) * 128 if c >= 128 else (c if c >= 64 else 0)


def _plan(case):
    """per GEMM layer: (forward rounded, input channels of the rounded dgrad, input channels of the rounded weight gradient), as
    csrc/stack.cu make_plan assigns the tensor-core kernels in training"""
    P, S, n = case.P, case.S, len(case.chans) - 1
    plan = []
    for l in range(n):
        K, Nw = _r4(case.chans[l]), _r4(case.chans[l + 1])
        last = l == n - 1
        if case.lift is not None and l == 0:       # layer 1 of a lifted stack: Y0 virtual, all three GEMMs on the tensor cores
            plan.append((True, K, K))
            continue
        f = (Nw % 128 == 0 or Nw == 64) and K >= 32 and P >= 128 and not (last and S > 0 and 64 % S != 0)
        b = K >= 64 and Nw >= 32 and P >= 128
        w = Nw >= 64 and K >= 64 and P >= 4096
        plan.append((f, _tc_main(K) if b else 0, _tc_main(K) if w else 0))
    return plan


def bf(t):
    """round to bf16 (nearest even) through fp32, as cvt.rn.bf16x2.f32 does to the kernels' fp32 values"""
    return t.float().to(torch.bfloat16).double()


class _Gemm(torch.autograd.Function):
    """y = x . W^T in float64 with the bf16 training rounding points: the forward rounds x and W; the dgrad rounds dy and the first
    kd input channels' weights; the weight gradient rounds dy and the first kw input channels of x (the rest is the fp32 tail)"""

    @staticmethod
    def forward(ctx, x, W, fwd, kd, kw):
        ctx.save_for_backward(x, W)
        ctx.kd, ctx.kw = kd, kw
        return bf(x) @ bf(W).t() if fwd else x @ W.t()

    @staticmethod
    def backward(ctx, gy):
        x, W = ctx.saved_tensors
        kd, kw = ctx.kd, ctx.kw
        dx = torch.cat([bf(gy) @ bf(W[:, :kd]), gy @ W[:, kd:]], 1)
        dW = torch.cat([bf(gy).t() @ bf(x[:, :kw]), gy.t() @ x[:, kw:]], 1)
        return dx, dW, None, None, None


def reference(specs, h, S, plan, rounded):
    """float64 training stack over the GEMM layers `specs` from the input rows h; rounded: the bf16 rounding points of `plan`"""
    for s, (f, kd, kw) in zip(specs, plan):
        W = s.weight.reshape(s.weight.shape[0], -1).double()
        h = _Gemm.apply(h[:, :W.shape[1]], W, f and rounded, kd if rounded else 0, kw if rounded else 0)
        if s.bias is not None:
            h = h + s.bias.double()
        if s.bn is not None:
            mu, var = h.mean(0), h.var(0, unbiased=False)
            h = (h - mu) / torch.sqrt(var + s.bn.eps) * s.bn.weight.double() + s.bn.bias.double()
        if s.relu:
            h = F.relu(h)
    if S > 0:
        g = h.view(-1, S, h.shape[1])
        first = (g.detach() == g.detach().max(dim=1, keepdim=True)[0]).to(torch.uint8).argmax(dim=1, keepdim=True)
        h = g.gather(1, first).squeeze(1)
    return h


def _lift_rows(lf, z, s, u, grow, P):
    """the lifted layer's Y0 = z[grow] + s . u in float64, then its BatchNorm (batch statistics) and ReLU"""
    y = torch.zeros(P, (z if z is not None else u).shape[1], dtype=torch.float64, device=grow.device)
    if z is not None:
        y = y + z.double()[grow]
    if s is not None:
        y = y + s.double() @ u.double()
    mu, var = y.mean(0), y.var(0, unbiased=False)
    y = (y - mu) / torch.sqrt(var + lf.bn.eps) * lf.bn.weight.double() + lf.bn.bias.double()
    return F.relu(y) if lf.relu else y


# Which kernels ran is observed in a child process that runs this file's path cases under the CUDA profiler; the pytest process
# itself never starts CUPTI, as in the suite's other profiling tests.
PROFILE_OUT = "O3D_BF16_TRAIN_PROFILE_OUT"


def _norm(name):
    return re.sub(r"\s*([<>,])\s*", r"\1", name.replace("(anonymous namespace)::", ""))


def _profiled(name, want, fn):
    out = os.environ.get(PROFILE_OUT)
    if out is None:
        return fn()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        res = fn()
    names = {_norm(e.name) for e in prof.events()}
    # CUPTI now and then delivers no records, or only part of them, for a short session.  The kernel choice depends on the shapes
    # only, so identical calls are observed again (up to three more) while a wanted kernel is missing, and the records are joined.
    for _ in range(3):
        if all(_ran(names, k) for k in want):
            break
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            fn()
        names |= {_norm(e.name) for e in prof.events()}
    with open(out, "a") as f:
        f.write(json.dumps({"id": name, "names": sorted(names)}) + "\n")
    return res


@functools.lru_cache(maxsize=1)
def _child_profiles():
    with tempfile.TemporaryDirectory() as tmp:
        out = os.path.join(tmp, "kernels.jsonl")
        here = os.path.abspath(__file__)
        r = subprocess.run([sys.executable, "-m", "pytest", here, "-q", "-m", "gpu", "-p", "no:cacheprovider", "-k",
                            "test_bf16_training_path"], cwd=os.path.dirname(os.path.dirname(here)),
                           env={**os.environ, PROFILE_OUT: out}, capture_output=True, text=True, timeout=1800)
        rec = {}
        if os.path.exists(out):
            with open(out) as f:
                for line in f:
                    e = json.loads(line)
                    rec[e["id"]] = set(e["names"])
    return rec, r.stdout[-3000:]


def _errors(names, got, want):
    """per tensor: |error| / max(|reference|, 1e-3 * the largest reference norm) (the floor covers the gradients that vanish
    exactly, e.g. a bias before a training-mode BatchNorm)"""
    scale = max(float(b.double().norm()) for b in want)
    return {n: float((a.double() - b.double()).norm()) / max(float(b.double().norm()), 1e-3 * scale)
            for n, a, b in zip(names, got, want)}


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_bf16_training_path_against_emulated_and_float64(case):
    seed = zlib.crc32(case.name.encode()) % 1000
    torch.manual_seed(seed)
    kinds = case.kinds
    chans = ([4] + case.chans) if case.lift else case.chans
    mod = build_stack(chans, kinds.split(), 7).cuda().train()
    specs = fused.parse_stack(mod)
    plan = _plan(case)
    rows_out = case.P // case.S if case.S else case.P
    go = torch.randn(rows_out, case.chans[-1], generator=torch.Generator().manual_seed(1)).cuda()
    if case.lift:
        grp, clouds, rows = case.lift
        lc = LiftCase(case.name, case.chans, kinds, case.P, grp, case.S, clouds=clouds, rows=rows, pattern="pad")
        z, ridx, s, u, grow, geom = make_inputs(lc, seed)
        ins = {n: t for n, t in (("dz", z), ("ds", s), ("du", u)) if t is not None}
        params = [p for n, p in mod.named_parameters() if not n.startswith("conv0.")]
        pnames = ["d" + n for n, _ in mod.named_parameters() if not n.startswith("conv0.")]
    else:
        ins = {"dx": torch.randn(case.P, case.chans[0], generator=torch.Generator().manual_seed(2)).cuda()}
        params, pnames = list(mod.parameters()), ["d" + n for n, _ in mod.named_parameters()]
    leaves = {n: t.clone().requires_grad_(True) for n, t in ins.items()}

    def step():
        with runtime.training_precision_scope("bf16"):
            if case.lift:
                out = fused.lifted_stack(specs, geom, z=leaves.get("dz"), ridx=ridx, s=leaves.get("ds"), u=leaves.get("du"),
                                         S=case.S, training=True)
            else:
                out = fused.mlp_stack(leaves["dx"], specs, case.S, True)
            grads = torch.autograd.grad(out, list(leaves.values()) + params, go)
        torch.cuda.synchronize()
        return out, grads

    out, grads = _profiled(case.name, case.want, step)
    if os.environ.get(PROFILE_OUT) is not None:
        return                           # the child only records the kernels; the parent checks the numbers and the record
    # run to run: a second call from the same inputs.  Only the order of the fp64 BatchNorm sums and of the lifted scatter's fp32
    # atomics may differ; a race on a shared-memory stage would show as a difference of order one
    out2, grads2 = step()
    rr = max([float((out2.double() - out.double()).norm() / out.double().norm())]
             + list(_errors(list(ins) + pnames, grads2, grads).values()))
    print(f"\n[bf16 train {case.name}] run to run {rr:.1e}")
    assert rr < 1e-4, (case.name, rr)
    refs = {n: t.double().requires_grad_(True) for n, t in ins.items()}
    results = {}
    for rounded in (True, False):
        if case.lift:
            h = _lift_rows(specs[0], refs.get("dz"), refs.get("ds"), refs.get("du"), grow, case.P)
            want = reference(specs[1:], h, case.S, plan, rounded)
        else:
            want = reference(specs, refs["dx"], case.S, plan, rounded)
        g_ref = torch.autograd.grad(want, list(refs.values()) + params, go.double())
        e_out = float((out.double() - want.detach()).norm() / want.detach().norm())
        results[rounded] = ({"out": e_out}, _errors(list(ins) + pnames, grads, g_ref))
    for rounded, bar, gbar in ((True, EMULATED_BAR, case.grad_bar), (False, UNROUNDED_BAR, GRAD_UNROUNDED_BAR)):
        e_out, e_g = results[rounded]
        worst = max(e_g, key=e_g.get)
        print(f"\n[bf16 train {case.name} {'emulated' if rounded else 'float64'}] output {e_out['out']:.1e}, inputs "
              + ", ".join(f"{n} {e_g[n]:.1e}" for n in ins) + f", worst parameter {worst} {e_g[worst]:.1e}")
        assert e_out["out"] < bar, (case.name, rounded, e_out)
        bad = {n: e for n, e in e_g.items() if not e < gbar}
        assert not bad, (case.name, "emulated" if rounded else "float64", bad)
    rec, log = _child_profiles()
    assert case.name in rec, ("no kernel record for this case", log)
    names = rec[case.name]
    kernels = sorted(n for n in names if "kernel" in n)
    missing = [k for k in case.want if not _ran(names, k)]
    assert not missing, (missing, kernels)
    fp32 = [k for k in FP32_GEMMS if _ran(names, k)]
    assert not fp32, (fp32, kernels)


# ------------------------------------------------------------------------------------------------ the training step
def test_bf16_graph_replay_equals_eager_step_and_repeats():
    """From one state, the captured bf16 step and the eager bf16 step give a bitwise equal loss, and two eager runs from one
    state give a bitwise equal loss.  Their gradients differ by the order of the BatchNorm / scatter atomics as in fp32, but by
    up to 6e-3 here instead of 2e-6: bf16 rounding turns those last-bit differences into whole-ulp steps of the next GEMM's
    operands (bar 2e-2)."""
    cfg, net = _bat()
    batches = [synthetic_siamese_batch(4, 256, 512, seed=100 + i, device="cuda") for i in range(4)]
    eng = TrainStep(net, lr=cfg.lr, use_graph=True, warmup=1, precision="bf16")
    eng.step(batches[0])
    worst = 0.0
    for b in batches[1:]:
        snap = _snapshot(eng)
        lg = eng.step(b).clone()
        assert eng.graph is not None
        gg = eng.flat.grad.clone()
        _restore(eng, snap)
        with runtime.training_precision_scope("bf16"):
            le = eng._eager(b).clone()
        assert torch.equal(lg, le), (float(lg), float(le))
        rg = float((gg - eng.flat.grad).norm() / eng.flat.grad.norm())
        worst = max(worst, rg)
        assert rg < 2e-2, rg
        _restore(eng, snap)
        with runtime.training_precision_scope("bf16"):
            assert torch.equal(eng._eager(b), le)
    print(f"\n[bf16 graph vs eager, same state] worst gradient difference: {worst:.1e}")


def test_fp32_step_after_bf16_steps_is_unchanged():
    """An fp32 step on a model that took bf16 steps equals, from the same state, an fp32 step of a model that never ran bf16."""
    cfg, net_a = _bat(seed=3)
    _, net_b = _bat(seed=3)
    batches = [synthetic_siamese_batch(4, 256, 512, seed=200 + i, device="cuda") for i in range(3)]
    a16 = TrainStep(net_a, lr=cfg.lr, use_graph=True, warmup=1, precision="bf16")
    for b in batches:
        a16.step(b)
    net_b.load_state_dict(net_a.state_dict())
    a32 = TrainStep(net_a, lr=cfg.lr, use_graph=False)
    b32 = TrainStep(net_b, lr=cfg.lr, use_graph=False)
    b = synthetic_siamese_batch(4, 256, 512, seed=300, device="cuda")
    la, lb = a32.step(b), b32.step(b)
    assert torch.equal(la, lb), (float(la), float(lb))
    rg = float((a32.flat.grad - b32.flat.grad).norm() / b32.flat.grad.norm())
    print(f"\n[fp32 after bf16] loss {float(la):.6f}, gradient difference {rg:.1e}")
    assert rg < 1e-5, rg           # fp32 run to run: the order of the BatchNorm / scatter atomics, measured 6.6e-7


# ------------------------------------------------------------------------------------------------ whole models
MODEL_BAR = 5e-2         # whole model against float64: every tracked output and loss term
# Where the 5e-2 bar does not hold.  These untrained networks amplify a perturbation of their activations strongly in a training
# step: fp32 round-off (~1e-7) already moves the parameter gradient by 2e-3 to 1e-2 from float64.  bf16 rounding (~4e-3) moves
# the deep outputs by 0.05 to 0.5 and the gradient by about its own size.  test_whole_model_training_m2track_bf16_against_float64
# shows that this is the rounding's own effect and not the kernels': a float64 evaluation that only rounds where the kernels do
# is as far from float64 as the bf16 kernels are, tensor by tensor.  For BAT and P2B (no emulation of the lifted layers in the
# oracle) the bars below are twice the measured values (DESIGN.md section 4.5); the set-abstraction outputs and the total loss
# keep MODEL_BAR.
HEAD_BARS = {"xcorr": 0.2, "vote_sa": 0.6, "estimation_cla": 1.0, "vote_xyz": 0.15, "center_xyz": 0.15, "estimation_boxes": 0.4,
             "pred_search_bc": 0.06, "loss_box": 0.35, "gradient": 2.0}
WHOLE = [("bat", "BAT_Car.yaml", 16, 512, 1024), ("p2b", "P2B_Car.yaml", 8, 512, 1024)]


class _Replay:
    """CHOICE_HOOK: records the discrete choices in call order and, with `inject` ({kind: [tensors]} or {(kind, n): tensor}),
    substitutes the given ones"""

    def __init__(self, inject=None):
        self.inject, self.seen = inject or {}, {}

    def __call__(self, kind, info, compute):
        own = compute()
        n = len(self.seen.setdefault(kind, []))
        self.seen[kind].append(own.detach().cpu())
        sub = self.inject.get((kind, n))
        if sub is None and isinstance(self.inject.get(kind), list):
            sub = self.inject[kind][n]
        return own if sub is None else sub.to(own.device).view_as(own).contiguous()


def _grad_error(got, want):
    """relative L2 of the whole parameter-gradient vector"""
    num = sum(float((got[k].double().cpu() - want[k].double().cpu()).norm()) ** 2 for k in want) ** 0.5
    return num / sum(float(want[k].double().norm()) ** 2 for k in want) ** 0.5


def _table(tag, errs):
    print(f"\n[{tag}] relative error against float64 (fp32 / bf16): "
          + ", ".join(f"{k} {a:.1e}/{b:.1e}" for k, (a, b) in errs.items()))


@pytest.mark.parametrize("name,cfg_file,B,M,N", WHOLE, ids=[w[1] for w in WHOLE])
def test_whole_model_training_bf16_against_float64_oracle(name, cfg_file, B, M, N):
    """One training forward and backward of BAT-Car / P2B-Car in fp32 and in bf16 against the oracle (oracle/modules.py) in
    float64, with every discrete decision on computed values held to the float64 oracle's: the RPN's ball query over the votes
    and BoxAwareXCorr's top-k (runtime.CHOICE_HOOK), and the loss's proposal targets (objectness: the distance of each PREDICTED
    proposal centre to the box against 0.3 / 0.6).  Those targets are not differentiated through, so the loss is handed the
    oracle's centres for them only; with the pass's own centres, a proposal centre within bf16 round-off of 0.3 m switches its
    box loss on or off."""
    from _params import det_state_dict
    from open3dsot_b200.config import load_config
    from open3dsot_b200.models import get_model
    from test_gpu_parity_full import _oracle_run
    torch.set_num_threads(min(os.cpu_count() or 1, 32))
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cfg = load_config(os.path.join(root, "cfgs", cfg_file))
    net = get_model(cfg.net_model)(cfg)
    base = det_state_dict(net.state_dict(), seed=41)
    pnames = [k for k, _ in net.named_parameters()]
    batch = synthetic_siamese_batch(B, M, N, seed=20260924, box_aware=(name == "bat"))
    _, _, _, taps, _ = _oracle_run(name, cfg, base, pnames, batch)                    # float32 oracle: the discrete choices
    inject = {("ball_query", 6): taps["rpn.vote_aggregation:bq_idx"][0]}
    force = {"ball_query": [taps[f"backbone.SA_modules.{i}:bq_idx"][br] for br in range(2) for i in range(3)]
             + [taps["rpn.vote_aggregation:bq_idx"][0]], "topk": []}
    if name == "bat":
        inject[("boxaware_topk", 0)] = taps["xcorr:topk"][0]
        force["topk"] = [taps["xcorr:topk"][0]]
    x_loss, x_ld, x_out, x_taps, x_grads = _oracle_run(name, cfg, base, pnames, batch, dtype=torch.float64, force=force)
    centres = x_out["center_xyz"].float().cuda()
    net = net.cuda().train()
    dev_batch = {k: v.cuda() for k, v in batch.items()}
    res = {}
    for prec in ("fp32", "bf16"):
        net.load_state_dict(base)
        net.zero_grad(set_to_none=True)
        outs, ld = {}, {}
        hs = [net.backbone.SA_modules[i].register_forward_hook(
              lambda m, a, o, i=i: outs.setdefault(f"sa{i}", []).append(o[1].detach())) for i in range(3)]
        hs.append(net.xcorr.register_forward_hook(lambda m, a, o: outs.setdefault("xcorr", []).append(o.detach())))
        hs.append(net.rpn.vote_aggregation.register_forward_hook(
            lambda m, a, o: outs.setdefault("vote_sa", []).append(o[1].detach())))
        own = net.compute_loss

        def spy(data, output):
            outs["end_points"] = {k: v.detach() for k, v in output.items() if torch.is_tensor(v)}
            d = own(data, {**output, "center_xyz": centres})
            ld.update({k: v.detach() for k, v in d.items()})
            return d
        net.compute_loss = spy
        runtime.CHOICE_HOOK = _Replay(inject)
        try:
            with runtime.training_precision_scope(prec):
                loss = net.training_step({k: v.clone() for k, v in dev_batch.items()}, 0)
                loss.backward()
        finally:
            runtime.CHOICE_HOOK = None
            del net.compute_loss
            for h in hs:
                h.remove()
        e = {}
        for i in range(3):
            for br in range(2):
                e[f"sa{i}[{br}]"] = rel_t(outs[f"sa{i}"][br], x_taps[f"backbone.SA_modules.{i}:out"][br])
        e["xcorr"] = rel_t(outs["xcorr"][0], x_taps["xcorr:out"][0])
        e["vote_sa"] = rel_t(outs["vote_sa"][0], x_taps["rpn.vote_aggregation:out"][0])
        for k in ("estimation_cla", "vote_xyz", "center_xyz", "estimation_boxes") + (("pred_search_bc",) if name == "bat" else ()):
            e[k] = rel_t(outs["end_points"][k], x_out[k])
        for k in x_ld:
            e[k] = rel_t(ld[k], x_ld[k])
        e["loss"] = rel_t(loss, x_loss)
        params = dict(net.named_parameters())
        e["gradient"] = _grad_error({k: params[k].grad for k in pnames}, x_grads)
        res[prec] = e
    errs = {k: (res["fp32"][k], res["bf16"][k]) for k in res["bf16"]}
    _table(f"{name} {B}x{M}/{N} training step", errs)
    assert max(a for k, (a, _) in errs.items() if k != "gradient") < 1e-4 and errs["gradient"][0] < 3e-2, errs   # the harness
    bad = {k: v for k, (_, v) in errs.items() if not v < HEAD_BARS.get(k, MODEL_BAR)}
    assert not bad, bad


def rel_t(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _emulate_bf16(model):
    """Every 1x1 Conv1d of `model` as the bf16 training kernels compute it: _Gemm with the rounding points of the layer's plan
    (csrc/stack.cu make_plan: P positions, K / Nw padded channel counts).  The Linear heads run on B rows, below the tensor-core
    kernels' P >= 128, and stay exact."""
    for m in model.modules():
        if isinstance(m, torch.nn.Conv1d):
            def forward(x, m=m):
                B, C, N = x.shape
                K, Nw, P = _r4(C), _r4(m.out_channels), B * N
                f = (Nw % 128 == 0 or Nw == 64) and K >= 32 and P >= 128
                kd = _tc_main(K) if K >= 64 and Nw >= 32 and P >= 128 else 0
                kw = _tc_main(K) if Nw >= 64 and K >= 64 and P >= 4096 else 0
                y = _Gemm.apply(x.permute(0, 2, 1).reshape(P, C), m.weight[:, :, 0], f, kd, kw)
                if m.bias is not None:
                    y = y + m.bias
                return y.reshape(B, N, -1).permute(0, 2, 1)
            m.forward = forward
    return model


def test_whole_model_training_m2track_bf16_against_float64():
    """One M2-Track training forward and backward in fp32 and in bf16 against the same model evaluated in float64 on the CPU with
    plain torch operators (runtime.composed_mode: the host mirror that test_gpu_parity_full holds the dense nets to), with the
    float64 pass's arg-max point mask and motion state injected (runtime.CHOICE_HOOK).  A second float64 pass rounds to bf16
    where the kernels do (_emulate_bf16): the bf16 product must agree with it, which tells the kernels' error from the bf16
    rounding's own effect on this network."""
    from _params import det_state_dict
    from open3dsot_b200.config import load_config
    from open3dsot_b200.datasets.synthetic import synthetic_motion_batch
    from open3dsot_b200.models import get_model
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cfg = load_config(os.path.join(root, "cfgs", "M2_track_kitti.yaml"))
    net = get_model(cfg.net_model)(cfg)
    base = det_state_dict(net.state_dict(), seed=41)
    batch = synthetic_motion_batch(16, 1024, seed=77)

    def run(model, b, hook):
        ld, ep = {}, {}
        own = model.compute_loss

        def spy(data, output):
            ep.update({k: v.detach() for k, v in output.items() if torch.is_tensor(v)})
            d = own(data, output)
            ld.update({k: v.detach() for k, v in d.items()})
            return d
        model.compute_loss = spy
        runtime.CHOICE_HOOK = hook
        try:
            loss = model.training_step(b, 0)
            loss.backward()
        finally:
            runtime.CHOICE_HOOK = None
            del model.compute_loss
        return ep, ld, {k: p.grad.detach() for k, p in model.named_parameters() if p.grad is not None}

    ref_net = get_model(cfg.net_model)(cfg)
    ref_net.load_state_dict(base)
    rec = _Replay()
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)        # the loss's own constants follow the model into float64
    try:
        with runtime.composed_mode():
            x_ep, x_ld, x_grads = run(ref_net.double().train(),
                                      {k: (v.double() if v.is_floating_point() else v.clone()) for k, v in batch.items()}, rec)
    finally:
        torch.set_default_dtype(old)
    inject = {k: v for k, v in rec.seen.items()}
    emu_net = get_model(cfg.net_model)(cfg)
    emu_net.load_state_dict(base)
    torch.set_default_dtype(torch.float64)
    try:
        with runtime.composed_mode():
            e_ep, e_ld, e_grads = run(_emulate_bf16(emu_net.double().train()),
                                      {k: (v.double() if v.is_floating_point() else v.clone()) for k, v in batch.items()},
                                      _Replay(inject))
    finally:
        torch.set_default_dtype(old)
    net.load_state_dict(base)
    net = net.cuda().train()
    res = {}
    for prec in ("fp32", "bf16"):
        net.load_state_dict(base)
        net.zero_grad(set_to_none=True)
        with runtime.training_precision_scope(prec):
            ep, ld, grads = run(net, {k: v.cuda() for k, v in batch.items()}, _Replay(inject))
        e = {k: rel_t(ep[k], x_ep[k]) for k in x_ep if x_ep[k].is_floating_point() and x_ep[k].numel() > 1}
        e.update({k: rel_t(ld[k], x_ld[k]) for k in x_ld})
        e["gradient"] = _grad_error(grads, x_grads)
        res[prec] = e
        if prec == "bf16":
            emu = {k: rel_t(ep[k], e_ep[k]) for k in e if k in e_ep}
            emu.update({k: rel_t(ld[k], e_ld[k]) for k in e_ld})
            emu["gradient"] = _grad_error(grads, e_grads)
            res["float64 emulated"] = {k: rel_t(e_ep[k], x_ep[k]) for k in x_ep if k in e}
            res["float64 emulated"].update({k: rel_t(e_ld[k], x_ld[k]) for k in x_ld})
            res["float64 emulated"]["gradient"] = _grad_error(e_grads, x_grads)
    print("\n[m2track 16x1024 training step] relative error (fp32 vs float64 / bf16 vs float64 / emulated vs float64 / bf16 vs "
          "emulated): " + ", ".join(f"{k} {res['fp32'][k]:.1e}/{res['bf16'][k]:.1e}/{res['float64 emulated'][k]:.1e}/{emu[k]:.1e}"
                                     for k in res["bf16"]))
    assert max(res["fp32"].values()) < 2e-2, res["fp32"]
    # the bf16 step is as far from float64 as bf16 rounding itself puts it (within twice the emulation's distance, or 1e-2).
    # bf16 against the emulation is printed too but not bounded: the two differ only where one computes in fp32 and the other in
    # float64 (and in the odd element that rounds to the other bf16 neighbour), and on this network that alone moves the gradient
    # by 0.7 and the final boxes by 0.1
    emu_err = res["float64 emulated"]
    bad = {k: (v, emu_err[k]) for k, v in res["bf16"].items() if not v < 2 * emu_err[k] + 1e-2}
    assert not bad, ("bf16 against float64, beyond the rounding's own effect", bad)


# ------------------------------------------------------------------------------------------------ the trainer
def _ckpts(log_dir):
    return sorted(glob.glob(os.path.join(log_dir, "lightning_logs", "version_*", "checkpoints", "*.ckpt")))


@pytest.mark.parametrize("name", ["BAT_Car.yaml", "P2B_Car.yaml", "M2_track_kitti.yaml"])
def test_fit_end_to_end_in_bf16(tmp_path, name):
    from open3dsot_b200.checkpoint import load_lightning_checkpoint
    from open3dsot_b200.models import get_model
    from open3dsot_b200.trainer import Trainer, TopK
    cfg = _cfg(name, train_precision="bf16")
    train, val = _tracklets([8, 6, 7], seed=400), _tracklets([6, 3, 5, 4], seed=500)
    log = str(tmp_path / "run")
    tr = Trainer(_model(cfg), cfg, train, val, log, slots=4)
    assert tr.step.precision == "bf16"
    tr.fit()
    rows = [json.loads(l) for l in open(os.path.join(log, "metrics.jsonl"))]
    assert [r["epoch"] for r in rows] == [0, 1] and all(r["train_precision"] == "bf16" for r in rows)
    for r in rows:
        assert all(math.isfinite(v) for k, v in r.items() if k.endswith("/train")), r
    spe = tr.global_step // 2
    d = os.path.join(log, "lightning_logs", "version_0", "checkpoints")
    for e in (0, 1):
        path = os.path.join(d, TopK.filename(e, (e + 1) * spe))
        sd = load_lightning_checkpoint(path)["state_dict"]
        assert all(v.dtype == torch.float32 for v in sd.values() if v.is_floating_point()), {k: v.dtype for k, v in sd.items()}
        fresh = get_model(cfg.net_model)(_cfg(name)).cuda()              # an fp32 model
        t2 = Trainer(fresh, _cfg(name), [], [], str(tmp_path / f"test{e}"), slots=4)
        t2.resume(path)
        res = t2.test(val)
        assert (res["success"], res["precision"]) == (rows[e]["success"], rows[e]["precision"]), e


def test_resume_continues_a_bf16_run(tmp_path):
    from open3dsot_b200.models import get_model
    from open3dsot_b200.trainer import Trainer
    cfg = _cfg("BAT_Car.yaml", epoch=1, save_top_k=1, train_precision="bf16")
    train, val = _tracklets([8, 6, 7], seed=400), _tracklets([5, 4], seed=500)
    log = str(tmp_path / "run")
    a = Trainer(_model(cfg), cfg, train, val, log, slots=4)
    a.fit()
    saved = (a.step.flat.flat.clone(), a.step.opt.exp_avg.clone(), a.step.opt.exp_avg_sq.clone(), a.step.opt.state.clone(),
             {k: v.clone() for k, v in a.model.named_buffers()})
    cfg2 = _cfg("BAT_Car.yaml", epoch=2, save_top_k=1, train_precision="bf16")
    torch.manual_seed(123)
    b = Trainer(get_model(cfg2.net_model)(cfg2).cuda(), cfg2, train, val, log, slots=4)
    b.resume(a.top_k.best_path)
    assert torch.equal(b.step.flat.flat, saved[0]) and torch.equal(b.step.opt.exp_avg, saved[1])
    assert torch.equal(b.step.opt.exp_avg_sq, saved[2]) and torch.equal(b.step.opt.state, saved[3])
    assert all(torch.equal(v, saved[4][k]) for k, v in b.model.named_buffers())
    row = b.fit()
    assert row["epoch"] == 1 and row["train_precision"] == "bf16" and b.step.precision == "bf16"
    assert all(math.isfinite(v) for k, v in row.items() if k.endswith("/train"))
