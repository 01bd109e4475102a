"""The fused backward kernel of a narrow layer (csrc/pwmlp_tc.cu pw_bwd_tc_kernel: dgrad and weight gradient in one pass,
taken by csrc/stack.cu for 64 / 128-channel layers at P >= P_FUSED_BWD = 65536) against the float64 statements of
tests/test_gpu_fused.py and tests/test_gpu_lift_paths.py, with the kernels that ran asserted from a CUDA profile taken in a
child process; and against the two-kernel pair it replaces, called directly through the C ABI on the same inputs."""
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
from test_gpu_fused import RTOL, rel
from test_gpu_lift_paths import Case as LiftCase, _compare, _lifted_params, make_inputs, reference_lifted
from test_gpu_stack_paths import _norm, _ran, build_stack, run_and_compare

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
from bench_fused_backward import Layer  # noqa: E402

pytestmark = pytest.mark.gpu

FA64, FA128 = "pw_bwd_tc_kernel<TcAct,64>", "pw_bwd_tc_kernel<TcAct,128>"        # <X loader, Cin>
FL64, FL128 = "pw_bwd_tc_kernel<TcLift,64>", "pw_bwd_tc_kernel<TcLift,128>"
RED = "wgrad_reduce_kernel"
# the two-kernel pair: the tensor-core weight gradient and the TcDy dgrad
TWO = ["pw_wgrad_tc_kernel<", "pw_tc_kernel<TcDy,"]

# (name, chans, kinds, P, S, want): every tensor-core layer of these stacks qualifies, so no two-kernel backward may run
DENSE = [
    ("sa1_layer2_pooled_s32", [16, 64, 128], "BR BR", 32 * 2100, 32, [FA64, RED]),
    ("pooled_s64", [16, 64, 128], "BR BR", 64 * 1100, 64, [FA64, RED]),
    ("dense_64_64_ragged", [16, 64, 64, 64], "BR BR BR", 65536 + 77, 0, [FA64, RED]),
    ("dense_128_128_ragged", [16, 128, 128], "BR BR", 70000 + 13, 0, [FA128, RED]),
    # layer 1 reads a BN-only layer (BN sums, no ReLU mask), layer 2 a ReLU-only one (mask, no BN)
    ("bn_only_relu_only", [16, 128, 64, 128], "B R BR", 65600, 0, [FA64, FA128, RED]),
    # bias + ReLU, then bias only, then a bare conv: the bias gradients' sums without any BN
    ("bias_layers", [16, 64, 128, 64], "bR b -", 65536, 0, [FA64, FA128, RED]),
]
LIFTED = [
    # BAT-Car SA1 (lifted 64 -> 64, then the pooled 64 -> 128) and SA2's first layer (lifted 128 -> 128)
    LiftCase("sa1_z_and_s", [64, 64, 128], "BR BR BR", 32 * 2048, 32, 32, "zrs", clouds=2, rows=300, pattern="pad", s_cols=3,
             want=[FL64, FA64, RED]),
    LiftCase("s_only", [64, 64, 128], "BR BR BR", 32 * 2050, 32, 32, "s", clouds=2, rows=100, pattern="pad",
             want=[FL64, FA64, RED]),
    LiftCase("sa2_z_only_k4", [128, 128, 128], "BR BR BR", 4 * 16400, 4, 4, "zr", clouds=2, rows=64, pattern="revisit",
             want=[FL128, FA128, RED]),
    LiftCase("inplace_accumulate", [64, 128, 128], "BR BR BR", 32 * 2048, 32, 32, clouds=2, rows=300, pattern="pad",
             inplace=True, want=[FL64, FA128, RED]),
]

# ---------------------------------------------------------------------------------------------- kernels, seen from a child
PROFILE_OUT = "O3D_FUSED_BWD_PROFILE_OUT"


def _test_id():
    return os.environ["PYTEST_CURRENT_TEST"].rsplit(" ", 1)[0].split("::", 1)[1]


def _profiled(fn):
    """fn() -- in the child under the CUDA profiler, recording this test's kernel names"""
    out = os.environ.get(PROFILE_OUT)
    if out is None:
        return fn()
    for _ in range(2):      # CUPTI now and then delivers no records for a short session: the same call is observed again
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            res = fn()
        names = {_norm(e.name) for e in prof.events()}
        if any("kernel" in n for n in names):
            break
    with open(out, "a") as f:
        f.write(json.dumps({"id": _test_id(), "names": sorted(names)}) + "\n")
    return res


@functools.lru_cache(maxsize=1)
def _child_profiles():
    with tempfile.TemporaryDirectory() as tmp:
        out = os.path.join(tmp, "kernels.jsonl")
        here = os.path.abspath(__file__)
        r = subprocess.run([sys.executable, "-m", "pytest", here, "-q", "-m", "gpu", "-p", "no:cacheprovider", "-k",
                            "matches_fp64"], cwd=os.path.dirname(os.path.dirname(here)), env={**os.environ, PROFILE_OUT: out},
                           capture_output=True, text=True, timeout=1800)
        rec = {}
        if os.path.exists(out):
            with open(out) as f:
                for line in f:
                    e = json.loads(line)
                    rec[e["id"]] = set(e["names"])
    return rec, r.stdout[-3000:]


def _assert_kernels(want, avoid):
    if os.environ.get(PROFILE_OUT) is not None:
        return
    rec, log = _child_profiles()
    assert _test_id() in rec, ("no kernel record for this test", log)
    names = rec[_test_id()]
    kernels = sorted(n for n in names if "kernel" in n)
    missing = [k for k in want if not _ran(names, k)]
    assert not missing, (missing, kernels)
    unwanted = [k for k in avoid if _ran(names, k)]
    assert not unwanted, (unwanted, kernels)


# ---------------------------------------------------------------------------------------------- 1. stacks against float64
@pytest.mark.parametrize("name,chans,kinds,P,S,want", DENSE, ids=[c[0] for c in DENSE])
def test_fused_backward_stack_matches_fp64_reference(name, chans, kinds, P, S, want):
    torch.manual_seed(zlib.crc32(name.encode()) % 1000)
    mod = build_stack(chans, kinds, 7).cuda().train()
    x = torch.randn(P, chans[0], device="cuda")
    _profiled(lambda: run_and_compare(mod, x, S, True, 3))
    _assert_kernels(want, TWO)


@pytest.mark.parametrize("case", LIFTED, ids=[c.name for c in LIFTED])
def test_fused_backward_lifted_matches_fp64_reference(case):
    seed = zlib.crc32(case.name.encode()) % 1000
    torch.manual_seed(seed)
    mod = build_stack([4] + case.chans, case.kinds, 7).cuda().train()
    specs = fused.parse_stack(mod)
    z, ridx, s, u, grow, geom = make_inputs(case, seed)
    ins = {n: t for n, t in (("dz", z), ("ds", s), ("du", u)) if t is not None}
    named = _lifted_params(mod)
    params = [p for _, p in named]
    go = torch.randn(case.P // case.S, case.chans[-1], generator=torch.Generator().manual_seed(1)).cuda()
    leaves = {n: t.clone().requires_grad_(True) for n, t in ins.items()}
    if case.inplace:
        g = torch.Generator().manual_seed(2)
        prior = [torch.randn(p.shape, generator=g).cuda() for p in params]
        for p, v in zip(params, prior):
            p.grad = v.clone()

    def step():
        out = fused.lifted_stack(specs, geom, z=leaves.get("dz"), ridx=ridx, s=leaves.get("ds"), u=leaves.get("du"), S=case.S,
                                 training=True)
        if case.inplace:
            with runtime.grad_inplace_scope():
                out.backward(go)
            grads = [t.grad for t in leaves.values()] + [p.grad - v for p, v in zip(params, prior)]
        else:
            grads = list(torch.autograd.grad(out, list(leaves.values()) + params, go))
        torch.cuda.synchronize()
        return out, grads

    out, grads = _profiled(step)
    refs = {n: t.double().requires_grad_(True) for n, t in ins.items()}
    ref_out = reference_lifted(specs, refs.get("dz"), refs.get("ds"), refs.get("du"), grow, case.P, case.S, True)
    assert rel(out, ref_out) < RTOL
    g_ref = torch.autograd.grad(ref_out, list(refs.values()) + params, go.double())
    tnames = list(ins) + ["d" + n for n, _ in named]
    first = tnames.index("ds") if "ds" in ins else 0
    order = [first] + [j for j in range(len(tnames)) if j != first]
    _compare(case.name, [tnames[j] for j in order], [grads[j] for j in order], [g_ref[j] for j in order],
             case.S if "ds" in ins else 0, case.max_flips)
    _assert_kernels(case.want, TWO)


# ---------------------------------------------------------------------------------------------- 2. against the two kernels
def _reference_dw(lay):
    """float64 dW = dY^T X of a tools/bench_fused_backward.Layer"""
    P, S = lay.P, lay.S
    if S:
        p = torch.arange(P, device="cuda")
        g = torch.where(lay.sel.long()[p // S] == (p % S)[:, None], lay.dpool.double()[p // S], 0.0)
    else:
        g = lay.g.double()
    dy = lay.a.double() * g + lay.b.double() + lay.cc.double() * lay.y.double()
    if lay.lifted:
        x = lay.z.double()[lay.gidx.long()] + lay.s.double() @ lay.u.double()
    else:
        x = lay.x.double()
    x = torch.relu(x * lay.scale.double() + lay.shift.double())
    return dy.t() @ x


@pytest.mark.parametrize("P,cout,cin,S,lifted", [
    (48 * 512 * 32, 128, 64, 32, False),        # BAT-Car SA1 layer 2, search branch
    (48 * 512 * 32, 64, 64, 0, True),           # SA1 layer 1
    (48 * 256 * 32, 128, 128, 0, True),         # SA2 layer 1
    (70000 + 13, 128, 128, 0, False),
    (4 * 16400, 128, 128, 4, True),
])
def test_fused_backward_agrees_with_the_two_kernel_pair(P, cout, cin, S, lifted):
    """dX and the BN-backward sums within fp32 round-off of the dgrad kernel's (the same MMA operands, other tile shapes and
    atomic orders); dW as close to the float64 product as the two-kernel pair's (both are fp32 sums of P terms in different
    orders), and bitwise equal from one run to the next"""
    lay = Layer(P, cout, cin, S, lifted, seed=3)
    lay.two_kernel()
    out2, s2, dw2 = lay.out.clone(), lay.s12.clone(), lay.dw.clone()
    runs = []
    for _ in range(2):
        lay.out.zero_()
        lay.s12.zero_()
        lay.dw.zero_()
        lay.fused()
        torch.cuda.synchronize()
        runs.append((lay.out.clone(), lay.s12.clone(), lay.dw.clone()))
    (outf, sf, dwf), (_, _, dw_again) = runs
    assert rel(outf, out2) < 1e-6, rel(outf, out2)
    assert rel(sf[0], s2[0]) < 1e-6 and rel(sf[1], s2[1]) < 1e-6, (rel(sf[0], s2[0]), rel(sf[1], s2[1]))
    ref = _reference_dw(lay)
    e_two, e_fused = rel(dw2, ref), rel(dwf, ref)
    print(f"\n[P={P} {cout}->{cin} S={S} lifted={lifted}] dW vs float64: two-kernel {e_two:.2e}, fused {e_fused:.2e}; "
          f"fused vs two-kernel {rel(dwf, dw2):.2e}")
    assert e_fused < 2 * e_two + 1e-7, (e_fused, e_two)
    assert torch.equal(dwf, dw_again)
