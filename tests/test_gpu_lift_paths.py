"""Every kernel of the lifted first layer (include/o3d_b200.h `o3d_lift_t`: csrc/lift.cu and the lifted variants of the
tensor-core GEMMs in csrc/pwmlp_tc.cu) against a float64 statement, tensor by tensor, with the kernels that ran asserted from a
CUDA profile.

A lifted stack never sees its first layer's input rows:
    Y0[p] = z[cloud(p) * rows_per_cloud + (ridx[p] | p % ridx_mod)] + s[p] . u
and csrc/stack.cu make_plan either stores Y0 (lift_stats_kernel<true>, then layer 1 as an ordinary stack) or keeps it virtual
(the TcLift operand loader, the lifted dgrad epilogue and the lifted weight gradient re-read it through gidx).  Each case names
the kernels it was written to reach and the ones that must not run, so a retuned threshold cannot move it onto the other path
unnoticed, and the output, dz, ds, du, every parameter gradient and the running statistics are compared one at a time: d_s and
d_u are a small part of any combined norm.

The second part runs the three callers (sa_forward, boxaware_xcorr_forward, p2b_xcorr_forward) against oracle/modules.py in
float64 with identical discrete choices, input by input and parameter by parameter."""
import functools
import json
import os
import subprocess
import sys
import tempfile
import zlib

import pytest
import torch

from open3dsot_b200 import fused, runtime
from test_gpu_fused import RTOL, check_grads, reference_stack, rel
from test_gpu_stack_paths import _bns, _norm, _ran, build_stack

# every kernel that exists for the lifted layer (names with the anonymous namespace and blanks removed); the bf16 forward
# loader has its own test (tests/test_gpu_bf16_inference.py)
ST, SF, SC = "lift_stats_kernel<true>", "lift_stats_kernel<false>", "lift_scatter_kernel"
LF = {ld: f"pw_tc_kernel<TcLift,TcFwdEpi<{ld}>>" for ld in (64, 128, 256, 0)}      # LD = layer 1's padded width
LD = {ld: f"pw_tc_kernel<TcDy,TcDgradEpi<{ld},true>>" for ld in (64, 128, 256, 0)}  # LD = C0
LW = "pw_wgrad_tc_kernel<TcLift>"
KERNELS = [ST, SF, SC, *LF.values(), *LD.values(), LW]
ANY_LF, ANY_STATS = "pw_tc_kernel<TcLift,", "lift_stats_kernel<"
NO_LD = list(LD.values())
# the plain stack's tensor-core kernels that a stored Y0 hands layer 1 to
TF128, TW = "pw_tc_kernel<TcAct,TcFwdEpi<128>>", "pw_wgrad_tc_kernel<TcAct>"


class Case:
    """chans = [C0, C1, ...] (C0 = the lifted layer's width); kinds per layer as in test_gpu_stack_paths (layer 0: BR, B or R
    -- its convolution is the lift itself); P positions in `clouds` clouds of `rows` source rows each; grp = the lift group
    (positions walked together by the gather / scatter passes), S = the pooling group of the last layer.  parts: z = gathered
    rows, r = ridx (else ridx_mod = rows), s = per-position scalars with `s_cols` non-zero columns.  pattern = the rows a group
    reads: random, pad ([a, b, c, a, a, ...], ball-query padding), empty (one row per group), revisit (the first row again at
    every third position).  train / grad (False: no autograd, under static_weights_scope); tensor-core level; grid: every
    Y0 exact in fp32; inplace: gradients added to existing .grad under runtime.grad_inplace_scope()."""

    def __init__(self, name, chans, kinds, P, grp, S, parts="zrs", clouds=1, rows=100, pattern="random", s_cols=4, train=True,
                 grad=True, level=3, grid=False, inplace=False, max_flips=3, want=(), avoid=()):
        self.name, self.chans, self.kinds, self.P, self.grp, self.S = name, chans, kinds.split(), P, grp, S
        self.parts, self.clouds, self.rows, self.pattern, self.s_cols = parts, clouds, rows, pattern, s_cols
        self.train, self.grad, self.level, self.grid, self.inplace, self.max_flips = train, grad, level, grid, inplace, max_flips
        self.want, self.avoid = tuple(want), tuple(avoid)
        assert len(self.kinds) == len(chans), name


VIRT = lambda c1, c0: [LF[c1 if c1 in (64, 128, 256) else 0], LD[c0 if c0 in (64, 128, 256) else 0], LW]  # noqa: E731
STORED_AVOID = [SF, ANY_LF, LW, *NO_LD]

CASES = [
    # ---- the four shapes of Y0 at the callers' geometry (rows_per_cloud != pos_per_cloud / S)
    Case("sa_c64_pad", [64, 64, 128], "BR BR BR", 4096, 32, 32, "zrs", clouds=2, rows=300, pattern="pad", s_cols=3,
         want=[SF, SC, *VIRT(64, 64)], avoid=[ST]),
    Case("sa1_s_only_c64", [64, 64, 128], "BR BR BR", 32 * 129, 32, 32, "s", clouds=3, rows=100, pattern="pad",
         want=[SF, SC, *VIRT(64, 64)], avoid=[ST]),
    Case("boxaware_c128_grp64_k4", [128, 128, 128], "BR BR BR", 2 * 512 * 4, 64, 4, "zr", clouds=2, rows=64,
         want=[SF, SC, *VIRT(128, 128)], avoid=[ST]),
    Case("boxaware_c128_grp4_k4", [128, 128, 128], "BR BR BR", 2 * 1025 * 4, 4, 4, "zr", clouds=2, rows=64, pattern="revisit",
         want=[SF, SC, *VIRT(128, 128)], avoid=[ST]),
    Case("p2b_n64_c64", [64, 128, 128], "BR BR BR", 2 * 40 * 64, 64, 64, "zms", clouds=2, rows=64, s_cols=1,
         want=[SF, SC, *VIRT(128, 64)], avoid=[ST]),
    # n1 = 128: layer 1 is the pooled last layer and 64 % 128 != 0 keeps it off the tensor-core forward, so Y0 is stored
    Case("p2b_n128_stored", [64, 128], "BR BR", 2 * 20 * 128, 128, 128, "zms", clouds=2, rows=128,
         want=[ST, SC], avoid=STORED_AVOID),
    # ---- C0 (tpr = C0 / 4 threads per row): shuffle / atomic d_s, block shapes
    Case("c16_grp1_dense", [16, 32, 64], "B BR BR", 1000, 1, 0, clouds=4, rows=50, want=[ST, SC], avoid=STORED_AVOID),
    Case("c20_255_threads", [20, 64, 64], "R BR BR", 4 * 300, 4, 4, clouds=3, rows=77, pattern="pad",
         want=[ST, SC], avoid=STORED_AVOID),
    Case("c20_255_threads_bn", [20, 64, 64], "BR BR BR", 4 * 300, 4, 4, clouds=3, rows=77, pattern="revisit",
         want=[ST, SC], avoid=STORED_AVOID),
    Case("c96_virtual_atomic_ds", [96, 128, 128], "BR BR BR", 16 * 260, 16, 16, clouds=2, rows=500, pattern="revisit",
         want=[SF, SC, *VIRT(128, 96)], avoid=[ST]),
    Case("c192_stored", [192, 128, 256], "BR BR BR", 4096 + 64, 32, 32, clouds=2, rows=200, pattern="pad",
         want=[ST, SC, TF128, TW], avoid=STORED_AVOID),
    Case("c256_two_warp_shuffle", [256, 256, 256], "BR BR BR", 4096, 32, 32, clouds=4, rows=256, pattern="pad",
         want=[SF, SC, *VIRT(256, 256)], avoid=[ST]),
    Case("c384_192_threads_empty_balls", [384, 384, 128], "BR BR BR", 4096, 64, 64, clouds=1, rows=1000, pattern="empty",
         want=[SF, SC, *VIRT(384, 384)], avoid=[ST]),
    # ---- position counts: ragged P (the int4 gidx tail), the 128 / 4096 thresholds
    Case("dense_ragged_4099", [128, 128], "BR BR", 4096 + 3, 1, 0, clouds=1, rows=333, want=[SF, SC, *VIRT(128, 128)],
         avoid=[ST]),
    Case("train_P4064_stored", [64, 128], "BR BR", 4096 - 32, 32, 32, rows=100, pattern="pad", want=[ST, SC, TF128],
         avoid=STORED_AVOID),
    Case("train_P4096_virtual", [64, 128], "BR BR", 4096, 32, 32, rows=100, pattern="pad", want=[SF, SC, *VIRT(128, 64)],
         avoid=[ST]),
    Case("eval_grad_P127_stored", [64, 128, 64], "BR BR BR", 127, 1, 0, rows=40, train=False, want=[ST, SC],
         avoid=STORED_AVOID),
    # eval with a gradient keeps Y0 virtual far below the training wgrad's P >= 4096 floor
    Case("eval_grad_P128_virtual", [64, 128, 64], "BR BR BR", 128, 1, 0, rows=40, train=False, want=[SF, SC, *VIRT(128, 64)],
         avoid=[ST]),
    # ---- eval without a gradient (static weights): gidx only, or no gather launch at all without z
    Case("eval_static_zs", [128, 256, 128], "BR BR BR", 2048, 32, 32, clouds=2, rows=200, pattern="pad", train=False,
         grad=False, want=[SF, LF[256]], avoid=[ST, SC, LW, *NO_LD]),
    Case("eval_static_s_only", [64, 64, 128], "BR BR BR", 2048, 32, 32, "s", clouds=2, rows=200, pattern="pad", train=False,
         grad=False, want=[LF[64]], avoid=[ANY_STATS, SC, LW]),
    Case("eval_static_stored_c20", [20, 64, 64], "BR BR BR", 4 * 64, 4, 4, rows=30, train=False, grad=False, want=[ST],
         avoid=[SF, SC, ANY_LF]),
    # ---- tensor-core levels: 0 none, 1 forward + dgrad (virtual only without the training wgrad), 2 wgrad only
    Case("level0_stored", [64, 128, 128], "BR BR BR", 4096, 32, 32, clouds=2, rows=150, pattern="pad", level=0,
         want=[ST, SC], avoid=[SF, "pw_tc_kernel<", "pw_wgrad_tc_kernel<"]),
    Case("level1_train_stored", [64, 128, 128], "BR BR BR", 4096, 32, 32, clouds=2, rows=150, pattern="pad", level=1,
         want=[ST, SC, TF128], avoid=[*STORED_AVOID, "pw_wgrad_tc_kernel<"]),
    Case("level1_eval_grad_virtual", [64, 128, 128], "BR BR BR", 2048, 32, 32, clouds=2, rows=150, pattern="pad", level=1,
         train=False, want=[SF, SC, *VIRT(128, 64)], avoid=[ST]),
    Case("level2_stored", [64, 128, 128], "BR BR BR", 4096, 32, 32, clouds=2, rows=150, pattern="pad", level=2,
         want=[ST, SC, TW], avoid=[SF, "pw_tc_kernel<", LW]),
    # ---- layer-0 kinds on the virtual path (ReLU only: the statistics pass writes gidx and nothing else)
    Case("l0_bn_only", [128, 128, 128], "B BR BR", 4096, 16, 16, clouds=2, rows=400, pattern="revisit",
         want=[SF, SC, *VIRT(128, 128)], avoid=[ST]),
    Case("l0_relu_only", [128, 128, 128], "R BR BR", 4096, 16, 16, clouds=2, rows=400, pattern="pad",
         want=[SF, SC, *VIRT(128, 128)], avoid=[ST]),
    # ---- gradients added to existing .grad buffers
    Case("inplace_accumulate", [64, 128, 128], "BR BR BR", 4096, 32, 32, clouds=2, rows=300, pattern="pad", inplace=True,
         want=[SF, SC, *VIRT(128, 64)], avoid=[ST]),
    # ---- exact: every Y0 representable in fp32, ReLU-only layer 0, ties of the padding duplicates go to the first position
    Case("grid_exact_ties", [64, 128], "R BR", 4096, 32, 32, clouds=2, rows=300, pattern="pad", grid=True, max_flips=0,
         want=[SF, SC, *VIRT(128, 64)], avoid=[ST]),
]


def test_every_lift_kernel_is_a_declared_target():
    """Adding a lifted kernel variant means adding a case that reaches it."""
    declared = {k for c in CASES for k in c.want if k in KERNELS}
    assert set(KERNELS) <= declared, sorted(set(KERNELS) - declared)
    assert len({c.name for c in CASES}) == len(CASES)
    for c in CASES:
        assert c.P % c.grp == 0 and (c.S == 0 or (c.P % c.S == 0 and 128 % c.S == 0)), c.name
        assert c.P % c.clouds == 0 and c.chans[0] % 4 == 0 and c.kinds[0] in ("BR", "B", "R"), c.name
        assert "m" not in c.parts or (c.rows == c.grp == c.S), c.name          # P2B: one group = one search point's templates
        assert c.train or c.grad or not c.inplace, c.name


# ---------------------------------------------------------------------------------------------- inputs
def _local_rows(P, grp, R, pattern, g):
    """the source row (within its cloud) each position reads; group 0 starts on row 0, the last group on row R - 1"""
    G = P // grp
    first = torch.randint(0, R, (G,), generator=g)
    first[0], first[-1] = 0, R - 1
    rows = torch.randint(0, R, (G, grp), generator=g)
    rows[:, 0] = first
    j = torch.arange(grp)[None, :]
    if pattern == "pad":            # a few neighbours found, the remaining slots repeat the first one
        k = torch.randint(1, max(grp // 4, 1) + 1, (G, 1), generator=g)
        rows = torch.where(j < k, rows, first[:, None])
    elif pattern == "empty":
        rows = first[:, None].expand(G, grp)
    elif pattern == "revisit":      # the first row again at positions 2, 5, 8, ...: never next to itself
        rows = torch.where(j % 3 == 2, first[:, None], rows)
    return rows.reshape(P).contiguous()


def _grid(shape, g, k, den):
    return torch.randint(-k, k + 1, shape, generator=g).double() / den


def make_inputs(case, seed):
    """z (clouds * rows, C0) | None, ridx (P,) int32 | None, s (P, 4) | None, u (4, C0) | None, the global row of every
    position and the _LiftGeom.  s[p] depends on the row and the group only (a relative coordinate), so the padding duplicates
    of a group hold identical Y0 rows."""
    g = torch.Generator().manual_seed(seed)
    P, C0, R, grp = case.P, case.chans[0], case.rows, case.grp
    Q = P // case.clouds
    local = torch.arange(P) % R if "m" in case.parts else _local_rows(P, grp, R, case.pattern, g)
    grow = (torch.arange(P) // Q) * R + local
    z = s = u = ridx = None
    if "z" in case.parts:
        # grid: odd multiples of 2^-13, so that z + s.u (multiples of 2^-12) is never exactly 0
        z = (2 * torch.randint(-4096, 4096, (case.clouds * R, C0), generator=g) + 1).double() / 8192 if case.grid else \
            torch.randn(case.clouds * R, C0, generator=g)
    if "r" in case.parts:
        ridx = local.int()
    if "s" in case.parts:
        mk = (lambda *shape: _grid(shape, g, 32, 64)) if case.grid else (lambda *shape: torch.randn(*shape, generator=g))
        pts, centre = mk(case.clouds * R, 4), mk(P // grp, 4)
        s = pts[grow] - centre.repeat_interleave(grp, 0)
        s[:, case.s_cols:] = 0
        u = _grid((4, C0), g, 64, 64) if case.grid else 0.5 * torch.randn(4, C0, generator=g)
    cuda = lambda t: None if t is None else t.float().cuda().contiguous()      # noqa: E731
    geom = fused._LiftGeom(P, R if "m" in case.parts else 0, R, Q, grp, C0)
    return cuda(z), None if ridx is None else ridx.cuda(), cuda(s), cuda(u), grow.cuda(), geom


def reference_lifted(specs, z, s, u, grow, P, S, training, batch_stats=None):
    """fp64 statement: Y0 = z[grow] + s @ u, layer 0's BatchNorm and ReLU, then reference_stack over the remaining layers"""
    C0 = (z if z is not None else u).shape[1]
    y = torch.zeros(P, C0, dtype=torch.float64, device=grow.device)
    if z is not None:
        y = y + z.double()[grow]
    if s is not None:
        y = y + s.double() @ u.double()
    bn = specs[0].bn
    if bn is not None:
        if training:
            mu, var = y.mean(0), y.var(0, unbiased=False)
            if batch_stats is not None:
                batch_stats.append((mu.detach(), y.var(0, unbiased=True).detach()))
        else:
            mu, var = bn.running_mean.double(), bn.running_var.double()
        y = (y - mu) / torch.sqrt(var + bn.eps) * bn.weight.double() + bn.bias.double()
    if specs[0].relu:
        y = torch.relu(y)
    return reference_stack(y, specs[1:], S, training, batch_stats=batch_stats)


def _lifted_params(mod):
    """the parameters a lifted stack differentiates: everything but layer 0's convolution (the lift replaces it)"""
    return [(n, p) for n, p in mod.named_parameters() if not n.startswith("conv0.")]


# Which kernels ran is observed in a child process that runs this file with PROFILE_OUT set: every test profiles its call there
# and records the kernel names under its own id.  The pytest process itself never starts CUPTI (as in the other profiling
# tests of the suite), so the in-process profiles of later test files see the same process state as without this file.
PROFILE_OUT = "O3D_LIFT_PATHS_PROFILE_OUT"


def _test_id():
    """test name and parameters (the node id without its path, which depends on the rootdir of the run)"""
    return os.environ["PYTEST_CURRENT_TEST"].rsplit(" ", 1)[0].split("::", 1)[1]


def _profiled(fn):
    """fn() -- under the CUDA profiler in the child, whose record gets this test's kernel names"""
    out = os.environ.get(PROFILE_OUT)
    if out is None:
        return fn()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        res = fn()
    names = {_norm(e.name) for e in prof.events()}
    if not any("kernel" in n for n in names):
        # CUPTI now and then delivers no activity records at all for a short session; the kernel choice depends on shapes
        # only, so an identical call is observed instead
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            fn()
        names = {_norm(e.name) for e in prof.events()}
    with open(out, "a") as f:
        f.write(json.dumps({"id": _test_id(), "names": sorted(names)}) + "\n")
    return res


@functools.lru_cache(maxsize=1)
def _child_profiles():
    with tempfile.TemporaryDirectory() as tmp:
        out = os.path.join(tmp, "kernels.jsonl")
        here = os.path.abspath(__file__)
        r = subprocess.run([sys.executable, "-m", "pytest", here, "-q", "-m", "gpu", "-p", "no:cacheprovider"],
                           cwd=os.path.dirname(os.path.dirname(here)), env={**os.environ, PROFILE_OUT: out},
                           capture_output=True, text=True, timeout=1800)
        rec = {}
        if os.path.exists(out):
            with open(out) as f:
                for line in f:
                    e = json.loads(line)
                    rec[e["id"]] = set(e["names"])
    return rec, r.stdout[-3000:]


def _assert_kernels(want, avoid):
    """the kernels this test's call ran (observed in the child) include every `want` and no `avoid`"""
    if os.environ.get(PROFILE_OUT) is not None:
        return                # the child only records; the asserting process is the parent
    rec, log = _child_profiles()
    assert _test_id() in rec, ("no kernel record for this test", log)
    names = rec[_test_id()]
    kernels = sorted(n for n in names if "kernel" in n)
    missing = [k for k in want if not _ran(names, k)]
    assert not missing, (missing, kernels)
    unwanted = [k for k in avoid if _ran(names, k)]
    assert not unwanted, (unwanted, kernels)


def _compare(tag, names, got, want, S, max_flips):
    """every gradient on its own (check_grads: 2e-4 relative, a bounded number of flipped decisions, detected on the first
    tensor, whose rows are positions (S = pooling group) or source rows (S = 0)); the measured errors are printed"""
    for n, a, b in zip(names, got, want):
        assert a.shape == b.shape, n
    # the quantity check_grads bounds: |error| / max(|reference|, 1e-3 * the largest reference norm) (the floor matters for the
    # gradients that vanish exactly, e.g. a bias before a training-mode BatchNorm)
    scale = max(float(b.double().norm()) for b in want)
    errs = {n: float((a.double() - b.double()).norm()) / max(float(b.double().norm()), 1e-3 * scale)
            for n, a, b in zip(names, got, want)}
    print(f"\n[{tag}] " + ", ".join(f"{n} {e:.1e}" for n, e in errs.items()))
    first = got[0].reshape(-1, got[0].shape[-1])
    try:
        check_grads([first] + list(got[1:]), [want[0].reshape(first.shape)] + list(want[1:]), S, first.shape,
                    max_flips=max_flips)
    except AssertionError as e:
        raise AssertionError(f"{tag}: {e}; per-tensor relative errors {errs}") from None


# ---------------------------------------------------------------------------------------------- 1. direct cases
@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_lift_path_matches_fp64_reference(case):
    seed = zlib.crc32(case.name.encode()) % 1000
    torch.manual_seed(seed)
    mod = build_stack([4] + case.chans, case.kinds, 7).cuda().train(case.train)      # conv0: replaced by the lift
    specs = fused.parse_stack(mod)
    z, ridx, s, u, grow, geom = make_inputs(case, seed)
    ins = {n: t for n, t in (("dz", z), ("ds", s), ("du", u)) if t is not None}      # named by their gradients
    named = _lifted_params(mod)
    params = [p for _, p in named]
    before = [(b.running_mean.clone(), b.running_var.clone(), int(b.num_batches_tracked)) for b in _bns(mod)]
    rows_out = case.P // case.S if case.S else case.P
    go = torch.randn(rows_out, case.chans[-1], generator=torch.Generator().manual_seed(1)).cuda()
    leaves = {n: t.clone().requires_grad_(case.grad) for n, t in ins.items()}
    lz, ls, lu = (leaves.get(n) for n in ("dz", "ds", "du"))
    if case.inplace:
        g = torch.Generator().manual_seed(2)
        prior = [torch.randn(p.shape, generator=g).cuda() for p in params]
        for p, v in zip(params, prior):
            p.grad = v.clone()
        ptrs = [p.grad.data_ptr() for p in params]

    def step():
        old = runtime.tc_level()
        runtime.set_tc(case.level)
        try:
            if not case.grad:
                with torch.no_grad(), runtime.static_weights_scope():
                    out = fused.lifted_stack(specs, geom, z=lz, ridx=ridx, s=ls, u=lu, S=case.S, training=False)
                    out = out.clone()
                torch.cuda.synchronize()
                return out, None
            out = fused.lifted_stack(specs, geom, z=lz, ridx=ridx, s=ls, u=lu, S=case.S, training=case.train)
            if case.inplace:
                with runtime.grad_inplace_scope():
                    out.backward(go)
                grads = [t.grad for t in leaves.values()] + [p.grad - v for p, v in zip(params, prior)]
            else:
                grads = list(torch.autograd.grad(out, list(leaves.values()) + params, go))
            torch.cuda.synchronize()
            return out, grads
        finally:
            runtime.set_tc(old)

    out, grads = _profiled(step)
    if case.inplace:
        assert [p.grad.data_ptr() for p in params] == ptrs         # added into the existing buffers

    stats = []
    refs = {n: t.double().requires_grad_(True) for n, t in ins.items()}
    ref_out = reference_lifted(specs, refs.get("dz"), refs.get("ds"), refs.get("du"), grow, case.P, case.S, case.train,
                               batch_stats=stats)
    assert out.shape == ref_out.shape
    e_out = rel(out, ref_out)
    assert e_out < RTOL, (case.name, "output", e_out)
    print(f"\n[{case.name}] output {e_out:.1e}")
    if case.grid:
        # exact ties inside pooling groups (the padding duplicates): both sides must send the gradient to the first of them
        dense = reference_lifted(specs, z, s, u, grow, case.P, 0, case.train).detach()
        tied = (dense.view(-1, case.S, dense.shape[1]) == ref_out.detach()[:, None, :]).sum(1) > 1
        assert int(tied.sum()) > 100, int(tied.sum())
    if not case.grad:
        _assert_kernels(case.want, case.avoid)
        return
    g_ref = torch.autograd.grad(ref_out, list(refs.values()) + params, go.double())
    tnames = list(ins) + ["d" + n for n, _ in named]
    # flipped decisions show as whole positions of d_s (pooling groups when pooled), or else as whole source rows of d_z
    first = tnames.index("ds") if "ds" in ins else 0
    order = [first] + [j for j in range(len(tnames)) if j != first]
    _compare(case.name, [tnames[j] for j in order], [grads[j] for j in order], [g_ref[j] for j in order],
             case.S if "ds" in ins else 0, case.max_flips)
    if case.train:
        assert len(stats) == len(before)
        for bn, (rm0, rv0, n0), (mu, var) in zip(_bns(mod), before, stats):
            m = bn.momentum
            rm = (1 - m) * rm0.double() + m * mu
            rv = (1 - m) * rv0.double() + m * var
            assert rel(bn.running_mean, rm) < 1e-5, ("running_mean", rel(bn.running_mean, rm))
            assert rel(bn.running_var, rv) < 1e-5, ("running_var", rel(bn.running_var, rv))
            assert int(bn.num_batches_tracked) == n0 + 1
    _assert_kernels(case.want, case.avoid)


# ---------------------------------------------------------------------------------------------- 2. the callers vs the oracle
class _Record:
    """runtime.CHOICE_HOOK: keeps the product's own discrete choices (ball query, box-cloud top-k) for the oracle to reuse"""

    def __init__(self):
        self.seen = {}

    def __call__(self, kind, info, compute):
        own = compute()
        self.seen.setdefault(kind, []).append(own.detach().cpu())
        return own


def _oracle_sd(module, prefix):
    sd = {}
    for k, v in module.state_dict().items():
        v = v.detach().cpu().clone()
        sd[f"{prefix}.{k}"] = v.double() if v.is_floating_point() else v
    for k, _ in module.named_parameters():
        sd[f"{prefix}.{k}"].requires_grad_(True)
    return sd


def _run_caller(module, fwd, inputs):
    """the module's training step with its discrete choices recorded: output, output gradient, input grads, parameter grads,
    recorded choices"""
    rec = _Record()
    leaves = [t for t in inputs if t.requires_grad]
    params = list(module.parameters())

    def step():
        runtime.CHOICE_HOOK = rec
        try:
            out = fwd(*inputs)
        finally:
            runtime.CHOICE_HOOK = None
        go = torch.randn(out.shape, generator=torch.Generator().manual_seed(5)).cuda()
        g = torch.autograd.grad(out, leaves + params, go)
        torch.cuda.synchronize()
        return out, go, g

    out, go, g = _profiled(step)
    return out, go, g[:len(leaves)], g[len(leaves):], dict(rec.seen)


def _check_caller(tag, module, prefix, run, o_out, o_in, sd, in_names, rows_first, want):
    """output, each input gradient and each parameter gradient of a caller against the float64 oracle, then the kernels"""
    out, go, g_in, g_par, _ = run
    e = rel(out, o_out)
    assert e < RTOL, (tag, "output", e)
    pn = [k for k, _ in module.named_parameters()]
    o_g = torch.autograd.grad(o_out, o_in + [sd[f"{prefix}.{k}"] for k in pn], go.double().cpu())
    got = [rows_first(g_in[0]).cpu()] + [t.cpu() for t in g_in[1:]] + [t.cpu() for t in g_par]
    ref = [rows_first(o_g[0])] + list(o_g[1:])
    print(f"\n[{tag}] output {e:.1e}")
    _compare(tag, in_names + ["d" + k for k in pn], got, ref, 0, 3)
    _assert_kernels(want, [ST])


def _cloud(B, N, seed):
    g = torch.Generator().manual_seed(seed)
    xyz = torch.rand(B, N, 3, generator=g)
    xyz[:, N // 8: N // 4] = xyz[:, : N // 4 - N // 8]          # exact duplicates: ties, heavy first-hit padding
    return xyz, g


SA_CALLERS = [
    # name, B, N, C, mlp, npoint, radius, nsample, xyz_grad, want
    ("sa_features_c128", 2, 512, 128, [128, 128, 128, 256], 64, 0.25, 32, False, VIRT(128, 128)),
    ("sa_vote_no_features_xyz_grad", 2, 512, 0, [0, 64, 64, 128], 64, 0.25, 32, True, VIRT(64, 64)),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", SA_CALLERS, ids=[c[0] for c in SA_CALLERS])
def test_sa_forward_against_fp64_oracle(case):
    from oracle import modules as om
    from open3dsot_b200.pointnet2.utils.pointnet2_modules import PointnetSAModule
    from _params import det_state_dict
    name, B, N, C, mlp, npoint, radius, S, xyz_grad, want = case
    xyz, g = _cloud(B, N, 3)
    feats = torch.randn(B, C, N, generator=g) if C else None
    sa = PointnetSAModule(mlp=list(mlp), radius=radius, nsample=S, use_fps=False)
    sa.load_state_dict(det_state_dict(sa.state_dict(), seed=5))
    sa = sa.cuda().train()
    sd = _oracle_sd(sa, "sa")
    x = xyz.cuda().requires_grad_(xyz_grad)
    f = None if feats is None else feats.cuda().requires_grad_(True)
    inputs = [x] + ([f] if f is not None else [])
    run = _run_caller(sa, lambda x, f=None: sa(x, f, npoint)[1], inputs)
    seen = run[4]
    x64 = xyz.double().requires_grad_(xyz_grad)
    f64 = None if feats is None else feats.double().requires_grad_(True)
    om.set_force({"ball_query": seen["ball_query"]})
    try:
        _, o_out, _ = om.sa_module(sd, "sa", x64, f64, npoint, radius, S, False, True)
    finally:
        om.set_force(None)
    o_in = ([x64] if xyz_grad else []) + ([f64] if f64 is not None else [])
    in_names = (["dxyz"] if xyz_grad else []) + (["dfeatures"] if f64 is not None else [])
    # rows of the first input gradient = source points: (B, N, 3) as is, (B, C, N) transposed
    first = (lambda t: t.reshape(-1, 3)) if xyz_grad else (lambda t: t.transpose(1, 2).reshape(-1, C))
    _check_caller(name, sa, "sa", run, o_out, o_in, sd, in_names, first, want)


@pytest.mark.gpu
@pytest.mark.parametrize("N,grp", [(513, 4), (512, 64)], ids=["grp4", "grp64"])
def test_boxaware_xcorr_against_fp64_oracle(N, grp):
    from oracle import modules as om
    from open3dsot_b200.models.head.xcorr import BoxAwareXCorr
    from _params import det_state_dict
    B, f, M, k, hidden = 2, 32, 64, 4, 128
    assert fused._pow2_divisor(N * k) == grp and B * N * k >= 4096
    g = torch.Generator().manual_seed(N)
    tf, sf = torch.randn(B, f, M, generator=g), torch.randn(B, f, N, generator=g)
    txyz, sxyz = torch.rand(B, M, 3, generator=g), torch.rand(B, N, 3, generator=g)
    tbc, sbc = torch.rand(B, M, 9, generator=g), torch.rand(B, N, 9, generator=g)
    m = BoxAwareXCorr(f, hidden, f, k=k, bc_channel=9)
    m.load_state_dict(det_state_dict(m.state_dict(), seed=9))
    m = m.cuda().train()
    sd = _oracle_sd(m, "xc")
    ins = [tf.cuda().requires_grad_(True), sf.cuda(), txyz.cuda(), sxyz.cuda(), tbc.cuda().requires_grad_(True), sbc.cuda()]
    run = _run_caller(m, m, ins)
    seen = run[4]
    tf64, tbc64 = tf.double().requires_grad_(True), tbc.double().requires_grad_(True)
    om.set_force({"topk": seen["boxaware_topk"]})
    try:
        o_out, _ = om.boxaware_xcorr(sd, "xc", tf64, sf.double(), txyz.double(), sxyz.double(), tbc64, sbc.double(), k, True)
    finally:
        om.set_force(None)
    _check_caller(f"boxaware_N{N}_grp{grp}", m, "xc", run, o_out, [tf64, tbc64], sd, ["dtemplate_feature", "dtemplate_bc"],
                  lambda t: t.transpose(1, 2).reshape(-1, f), VIRT(hidden, hidden))


@pytest.mark.gpu
def test_p2b_xcorr_against_fp64_oracle():
    from oracle import modules as om
    from open3dsot_b200.models.head.xcorr import P2B_XCorr
    from _params import det_state_dict
    B, f, n1, n2, hidden = 2, 32, 64, 64, 128
    g = torch.Generator().manual_seed(17)
    # Conditioning.  With independent unit-scale features every cosine is near 0 and the template rows dominate Y0, so the max
    # over the templates picks the same row for every search point: the pooled rows barely vary, and fea_layer's training-mode
    # BatchNorm divides by that small spread (measured with unit-scale independent features: gradient norms up to 3e3, every
    # gradient 0.7-1.1e-4 from float64, the output 3.9e-5).  Here every search feature is +-1 times one template feature plus noise (cosines across
    # [-1, 1]) and the template rows are small (cosines do not scale), so the cosine term decides what is pooled.
    tf = 0.05 * torch.randn(B, f, n1, generator=g)
    pick = torch.randint(0, n1, (B, 1, n2), generator=g).expand(B, f, n2)
    sign = torch.where(torch.rand(B, 1, n2, generator=g) < 0.5, -1.0, 1.0)
    sf = sign * tf.gather(2, pick) + 0.025 * torch.randn(B, f, n2, generator=g)
    txyz = 0.05 * torch.rand(B, n1, 3, generator=g)
    m = P2B_XCorr(f, hidden, f)
    m.load_state_dict(det_state_dict(m.state_dict(), seed=9))
    m = m.cuda().train()
    sd = _oracle_sd(m, "xc")
    ins = [tf.cuda().requires_grad_(True), sf.cuda().requires_grad_(True), txyz.cuda()]
    run = _run_caller(m, m, ins)
    tf64, sf64 = tf.double().requires_grad_(True), sf.double().requires_grad_(True)
    o_out = om.p2b_xcorr(sd, "xc", tf64, sf64, txyz.double(), True)
    with torch.no_grad():    # the float32 oracle's own distance from float64, for scale
        o32 = om.p2b_xcorr({k: v.detach().float() if v.is_floating_point() else v for k, v in sd.items()}, "xc", tf, sf, txyz,
                           True)
    print(f"\n[p2b_n64] float32 oracle output {rel(o32, o_out):.1e}")
    _check_caller("p2b_n64", m, "xc", run, o_out, [tf64, sf64], sd, ["dtemplate_feature", "dsearch_feature"],
                  lambda t: t.transpose(1, 2).reshape(-1, f), VIRT(hidden, hidden))
