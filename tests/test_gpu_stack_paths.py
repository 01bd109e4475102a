"""Every kernel the fused MLP stack can choose (csrc/stack.cu make_plan and the o3d_pw_* launchers) against the fp64
statement of tests/test_gpu_fused.py, with the kernels that ran asserted from a CUDA profile.

The stack picks one of about twenty GEMM instantiations per layer from P, K, the padded width Nw, the group size S, train or
eval and the tensor-core level.  Each case below names the kernels it exists to reach (and, at a threshold, the ones that must
not run), so a retuned threshold or a new variant cannot silently move a case off the path it was written for."""
import re
import zlib
from collections import OrderedDict

import pytest
import torch
import torch.nn as nn

from open3dsot_b200 import _lib, fused, runtime
from test_gpu_fused import RTOL, check_grads, randomise, reference_stack, rel

MOMENTUM, EPS = 0.05, 1e-3

# every GEMM instantiation of the stack (names with the anonymous namespace and blanks removed)
KERNELS = [
    "pw_fwd_kernel<64>", "pw_fwd_kernel<128>",
    "pw_dgrad_kernel<64>", "pw_dgrad_kernel<128>",
    "pw_wgrad_kernel<64>", "pw_wgrad_kernel<128>",
    "pw_fwd_skinny_kernel<1>", "pw_fwd_skinny_kernel<2>",
    "pw_wgrad_skinny_kernel<1,4>", "pw_wgrad_skinny_kernel<2,2>", "pw_wgrad_skinny_kernel<3,2>",
    "pw_tc_kernel<TcAct,TcFwdEpi<64>>", "pw_tc_kernel<TcAct,TcFwdEpi<128>>", "pw_tc_kernel<TcAct,TcFwdEpi<256>>",
    "pw_tc_kernel<TcAct,TcFwdEpi<0>>",
    "pw_tc_kernel<TcDy,TcDgradEpi<64,false>>", "pw_tc_kernel<TcDy,TcDgradEpi<128,false>>",
    "pw_tc_kernel<TcDy,TcDgradEpi<256,false>>", "pw_tc_kernel<TcDy,TcDgradEpi<0,false>>",
    "pw_wgrad_tc_kernel<TcAct>", "wgrad_reduce_kernel",
    "d2f_kernel",
]
FWD64, FWD128 = "pw_fwd_kernel<64>", "pw_fwd_kernel<128>"
DG64, DG128 = "pw_dgrad_kernel<64>", "pw_dgrad_kernel<128>"
WG64, WG128 = "pw_wgrad_kernel<64>", "pw_wgrad_kernel<128>"
SK1, SK2 = "pw_fwd_skinny_kernel<1>", "pw_fwd_skinny_kernel<2>"
SW1, SW2, SW3 = "pw_wgrad_skinny_kernel<1,4>", "pw_wgrad_skinny_kernel<2,2>", "pw_wgrad_skinny_kernel<3,2>"
TF = {ld: f"pw_tc_kernel<TcAct,TcFwdEpi<{ld}>>" for ld in (64, 128, 256, 0)}
TD = {ld: f"pw_tc_kernel<TcDy,TcDgradEpi<{ld},false>>" for ld in (64, 128, 256, 0)}
TW, RED, D2F = "pw_wgrad_tc_kernel<TcAct>", "wgrad_reduce_kernel", "d2f_kernel"
ANY_TF, ANY_TD = "pw_tc_kernel<TcAct,", "pw_tc_kernel<TcDy,"


def persist_dense(sms):
    """ragged P with more than 3 position tiles per CTA of a <= 128-channel layer (grid = #SMs CTAs)"""
    return 3 * sms * 128 + 77


def persist_pooled(sms):
    return (3 * sms + 1) * 128 + 64


class Case:
    """layer widths; kinds per layer: BR = BN+ReLU, B = BN, bR = bias+ReLU, b = bias, - = bare conv; P (or a function of the
    SM count); S; train / eval; tensor-core level; kernels that must run (`want`) and kernels that must not (`avoid`, name
    prefixes)."""

    def __init__(self, name, chans, kinds, P, S=0, train=True, level=3, want=(), avoid=()):
        self.name, self.chans, self.kinds, self.P, self.S = name, chans, kinds.split(), P, S
        self.train, self.level, self.want, self.avoid = train, level, tuple(want), tuple(avoid)
        assert len(self.kinds) == len(chans) - 1, name

    def positions(self, sms):
        return self.P(sms) if callable(self.P) else self.P


CASES = [
    # ---- skinny forward (K <= 8, dense layer, P >= 4096) and skinny weight gradients (Cin <= 12, P >= 4096)
    Case("skinny1_first", [4, 64, 128], "BR BR", 4096, want=[SK1, SW1, DG64, TF[128], TD[64], TW, RED]),
    Case("skinny1_first_ragged", [4, 64, 128], "BR BR", 4096 + 37, want=[SK1, SW1, TF[128]]),
    Case("skinny2_first", [8, 64, 64], "BR B", 4096, want=[SK2, SW2, TF[64], TD[64], TW]),
    Case("skinny2_first_ragged", [8, 64, 64], "BR BR", 5000, want=[SK2, SW2, TF[64]]),
    Case("skinny1_middle", [16, 4, 64, 32], "BR BR BR", 4096, want=[FWD64, SK1, SW1, TD[64], WG64, DG64]),
    Case("skinny1_middle_pooled_ragged", [16, 4, 64, 32], "BR BR BR", 4100, S=4, want=[SK1, SW1, FWD64, TD[64]]),
    Case("skinny2_middle", [16, 8, 64, 64], "BR BR BR", 4096, want=[SK2, SW2, TF[64]]),
    Case("skinny2_middle_ragged", [16, 8, 64, 64], "BR BR BR", 4096 + 300, want=[SK2, SW2]),
    Case("skinny3_first", [12, 64, 64], "BR BR", 4096, want=[FWD64, SW3], avoid=[SK1, SK2]),
    Case("skinny3_middle_ragged", [16, 12, 64, 64], "BR BR BR", 4096 + 44, want=[SW3, FWD64]),
    # skinny weight gradients of a pooled last layer read the pooled gradient (dpool / sel); CUDA-core pooled forward + dgrad
    Case("skinny3_pooled", [12, 64], "BR", 4096, S=16, want=[FWD64, SW3, DG64], avoid=[SK1, SK2]),
    Case("skinny2_pooled_s2", [8, 64], "BR", 4096, S=2, want=[FWD64, SW2, DG64]),
    Case("skinny1_pooled_s128", [4, 128], "BR", 4096, S=128, want=[FWD128, SW1, DG64], avoid=[ANY_TF]),
    # ---- threshold neighbours
    Case("P4095_no_skinny", [8, 64, 64], "BR BR", 4095, want=[FWD64, WG64, TF[64]], avoid=[SK1, SK2, "pw_wgrad_skinny", TW]),
    Case("K12_tiled_fwd", [12, 64], "BR", 4096, want=[FWD64, SW3], avoid=[SK1, SK2]),
    Case("Cin16_tiled_wgrad", [16, 64], "BR", 4096, want=[FWD64, WG64], avoid=["pw_wgrad_skinny"]),
    Case("P127_cuda_core", [64, 128], "BR", 127, want=[FWD128, DG64, WG64], avoid=[ANY_TF, ANY_TD]),
    Case("P128_tensor_core", [64, 128], "BR", 128, want=[TF[128], TD[64], WG64], avoid=[FWD128, DG64, TW]),
    Case("P4096_tc_wgrad", [64, 128, 128], "BR BR", 4096, want=[TF[128], TD[128], TD[64], TW, RED], avoid=[WG64, WG128]),
    Case("eval_P15", [64, 128, 5], "BR b", 15, train=False, want=[FWD128, FWD64, DG128, DG64, WG128, WG64, D2F],
         avoid=[ANY_TF, ANY_TD]),
    Case("eval_P16", [64, 128, 5], "BR b", 16, train=False, want=[TF[128], TF[0], DG128, D2F], avoid=[FWD64, FWD128]),
    Case("S64_tc_pooled", [64, 128], "BR", 4096, S=64, want=[TF[128], TD[64], TW], avoid=[FWD128]),
    Case("S128_cuda_pooled", [64, 128], "BR", 4096, S=128, want=[FWD128, TD[64], TW], avoid=[ANY_TF]),
    Case("Nw64_tc_train", [64, 64], "BR", 1024, S=16, want=[TF[64], TD[64]], avoid=[FWD64]),
    Case("Nw68_cuda_train", [64, 68, 128], "BR BR", 4096 + 52, want=[FWD128, TF[128], TD[0], TD[64], TW],
         avoid=[DG64, DG128]),
    # ---- tensor-core forward in training with a runtime stride (Nw = 384) and the ragged tensor-core edges
    Case("fwd_tc_nw384", [128, 384], "BR", 1024, S=32, want=[TF[0], TD[128]]),
    Case("k100_kblock_edge", [100, 128, 64], "BR BR", 1000, want=[TF[128], TF[64], TD[128], TD[0], WG128],
         avoid=[DG64, DG128]),
    Case("wgrad_tail4_nw68", [132, 68, 128], "BR BR", 4096 + 52, want=[FWD128, TF[128], TD[0], DG64, TW, RED, SW1]),
    Case("tails64_nw192", [192, 192, 256], "BR BR", 4096 + 100, want=[FWD128, TF[256], TD[0], DG64, TW, WG64]),
    Case("tails72_copy_out", [200, 128, 36], "BR b", 4096 + 12, want=[TF[128], FWD64, TD[128], TD[0], DG128, TW, WG128, D2F]),
    Case("pooled_tail4", [132, 128], "BR", 32 * 130, S=32, want=[TF[128], TD[0], DG64, TW, SW1]),
    Case("pooled_tc_tail64", [192, 256], "BR", 64 * 70, S=64, want=[TF[256], TD[0], DG64, TW, WG64]),
    # ---- layer kinds: bias-only, BN-only and bare layers in the middle, a copy-out last layer
    Case("kinds_mixed", [32, 64, 36, 128, 8], "b B bR -", 2000,
         want=[TF[64], FWD64, TF[128], DG128, DG64, TD[64], WG128, WG64, D2F]),
    Case("kinds_mid_cout37", [64, 37, 128, 128], "BR bR B", 4096, want=[FWD64, TF[128], DG64, TD[128], D2F]),
    Case("pooled_bn_no_relu", [64, 128], "B", 32 * 40, S=32, want=[TF[128], TD[64]]),
    Case("pooled_bias_only", [32, 64, 128], "BR b", 16 * 64, S=16, train=False, want=[TF[64], TF[128], D2F]),
    # ---- group sizes (S = 1, 2, 8 take the element-wise branch of the tensor-core epilogue)
    Case("S1_tc", [32, 64, 128], "BR BR", 2048, S=1, want=[TF[64], TF[128], TD[64], DG64, WG64]),
    Case("S2_eval", [32, 64, 256], "BR BR", 2048, S=2, train=False, want=[TF[64], TF[256]]),
    Case("S4_level0", [64, 128], "BR", 4 * 300, S=4, level=0, want=[FWD128, DG64, WG64], avoid=[ANY_TF, ANY_TD, TW]),
    # ---- tensor-core levels: 0 all CUDA-core, 1 forward + dgrad, 2 weight gradient only
    Case("level0", [64, 128, 256], "BR BR", 32 * 64, S=32, level=0, want=[FWD128, DG128, DG64, WG128, WG64],
         avoid=[ANY_TF, ANY_TD, TW]),
    Case("level1", [64, 128, 256], "BR BR", 4096, S=8, level=1, want=[TF[128], TF[256], TD[128], TD[64], WG128, WG64],
         avoid=[TW]),
    Case("level2", [64, 128, 256], "BR BR", 4096, S=16, level=2, want=[FWD128, DG128, DG64, TW, RED],
         avoid=[ANY_TF, ANY_TD]),
    # ---- persistent tile loop: >= 3 position tiles per CTA, both walk directions (consecutive tensor-core layers alternate)
    Case("persist_dense_ragged", [64, 128, 128, 128], "BR BR BR", persist_dense, want=[TF[128], TD[128], TD[64], TW]),
    Case("persist_m2track_pooled", [16, 64, 128, 256, 512], "BR BR BR BR", persist_pooled, S=64,
         want=[FWD64, TF[128], TF[256], TF[0], TD[256], TD[128], TD[64], TW, RED, DG64, WG64]),
]


def test_every_stack_kernel_is_a_declared_target():
    """Adding a kernel variant means adding a case that reaches it."""
    declared = {k for c in CASES for k in c.want}
    assert set(KERNELS) <= declared, sorted(set(KERNELS) - declared)
    assert declared <= set(KERNELS), sorted(declared - set(KERNELS))
    assert len({c.name for c in CASES}) == len(CASES)
    for c in CASES:
        assert all(k % 4 == 0 for k in c.chans[:1]) and (c.S == 0 or 128 % c.S == 0), c.name
        if not callable(c.P):
            assert c.S == 0 or c.P % c.S == 0, c.name


def _norm(name):
    return re.sub(r"\s*([<>,])\s*", r"\1", name.replace("(anonymous namespace)::", ""))


def _ran(names, pat):
    """`pat` names a kernel (followed by its argument list) or, ending in '<' / ',' or without template arguments, a prefix"""
    tail = "" if pat.endswith(("<", ",")) or pat in ("pw_wgrad_skinny",) else r"(?=\(|$)"
    rx = re.compile(r"(?:^|[\s:])" + re.escape(pat) + tail)
    return any(rx.search(n) for n in names)


def build_stack(chans, kinds, seed):
    layers = OrderedDict()
    for i, (cin, cout, kind) in enumerate(zip(chans[:-1], chans[1:], kinds)):
        layers[f"conv{i}"] = nn.Conv1d(cin, cout, 1, bias=kind != "-")
        if "B" in kind:
            layers[f"bn{i}"] = nn.BatchNorm1d(cout, momentum=MOMENTUM, eps=EPS)
        if "R" in kind:
            layers[f"relu{i}"] = nn.ReLU()
    mod = nn.Sequential(layers)
    randomise(mod, seed)     # BN gammas of both signs, non-zero biases and running statistics
    return mod


def _bns(mod):
    return [m for m in mod if isinstance(m, nn.BatchNorm1d)]


def run_and_compare(mod, x, S, training, level, max_flips=3, profile=False):
    """forward + every gradient through the fused stack (optionally under the profiler) against the fp64 statement, and the
    running statistics of a training call; returns the normalised names of the kernels that ran"""
    specs = fused.parse_stack(mod)
    before = [(b.running_mean.clone(), b.running_var.clone(), int(b.num_batches_tracked)) for b in _bns(mod)]
    x1 = x.clone().requires_grad_(True)
    params = list(mod.parameters())

    def step():
        old = runtime.tc_level()
        runtime.set_tc(level)
        try:
            out = fused.mlp_stack(x1, specs, S, training)
            go = torch.randn(out.shape, generator=torch.Generator().manual_seed(1)).cuda()
            g_out = torch.autograd.grad(out, [x1] + params, go, allow_unused=True)
            torch.cuda.synchronize()
        finally:
            runtime.set_tc(old)
        return out, go, g_out

    def profiled():
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            res = step()
        return res, {_norm(e.name) for e in prof.events()}

    (out, go, g_out), names = profiled() if profile else (step(), set())
    x2 = x.clone().requires_grad_(True)
    stats = []
    want = reference_stack(x2, specs, S, training, batch_stats=stats)
    assert out.shape == want.shape
    assert rel(out, want) < RTOL, rel(out, want)
    g_ref = torch.autograd.grad(want, [x2] + params, go.double(), allow_unused=True)
    check_grads(g_out, g_ref, S, x1.shape, max_flips=max_flips)
    if training:
        assert len(stats) == len(before)
        for bn, (rm0, rv0, n0), (mu, var) in zip(_bns(mod), before, stats):
            m = bn.momentum
            rm = (1 - m) * rm0.double() + m * mu
            rv = (1 - m) * rv0.double() + m * var
            assert rel(bn.running_mean, rm) < 1e-5, ("running_mean", rel(bn.running_mean, rm))
            assert rel(bn.running_var, rv) < 1e-5, ("running_var", rel(bn.running_var, rv))
            assert int(bn.num_batches_tracked) == n0 + 1
    if profile and not any("kernel" in n for n in names):
        # CUPTI now and then delivers no activity records at all for a short session (seen in ~1 of 250 sessions); the
        # kernel choice depends on shapes only, so an identical call is observed instead (its results are not compared)
        names = profiled()[1]
    return names


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_stack_path_matches_fp64_reference(case):
    torch.manual_seed(zlib.crc32(case.name.encode()) % 1000)
    sms = _lib.lib().o3d_device_sms()
    P = case.positions(sms)
    mod = build_stack(case.chans, case.kinds, 7).cuda().train(case.train)
    x = torch.randn(P, case.chans[0], device="cuda")
    names = run_and_compare(mod, x, case.S, case.train, case.level, profile=True)
    kernels = sorted(n for n in names if "kernel" in n)
    missing = [k for k in case.want if not _ran(names, k)]
    assert not missing, (missing, kernels)
    unwanted = [k for k in case.avoid if _ran(names, k)]
    assert not unwanted, (unwanted, kernels)


def test_persistent_cases_walk_three_tiles_per_cta():
    """The persistent-loop cases keep >= 3 position tiles per CTA of their narrowest (<= 128-channel) layers on any SM count."""
    for sms in (114, 132):
        for f in (persist_dense, persist_pooled):
            assert (f(sms) + 127) // 128 >= 3 * sms + 1


# ---------------------------------------------------------------------------------------------- exact ties in a pool group
def _tied_input(P, S, K, seed):
    """groups padded the way the ball query pads them: [a, b, c, a, a, ...]"""
    g = torch.Generator().manual_seed(seed)
    rows = torch.randn(P // S, 3, K, generator=g)
    idx = torch.zeros(S, dtype=torch.long)
    idx[1], idx[2] = 1, 2
    return rows[:, idx].reshape(P, K).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("name,S,level,fast", [
    ("tc_fast_path_s32", 32, 3, TF[128]),           # 16-position blocks merged across the group
    ("tc_elementwise_s8", 8, 3, TF[128]),
    ("cuda_core_s32", 32, 0, FWD128),
])
def test_pooling_ties_go_to_the_first_position(name, S, level, fast):
    torch.manual_seed(zlib.crc32(name.encode()) % 1000)
    mod = build_stack([32, 64, 128], ["BR", "BR"], 5).cuda().train()
    gammas = [b.weight for b in _bns(mod)]
    assert all(bool((g > 0).any()) and bool((g < 0).any()) for g in gammas)   # max / argmax and min / argmin sides
    x = _tied_input(S * 96, S, 32, 11)
    names = run_and_compare(mod, x, S, True, level, max_flips=0, profile=True)
    assert _ran(names, fast), sorted(n for n in names if "kernel" in n)


# ---------------------------------------------------------------------------------------------- prepared blocks per size class
@pytest.mark.gpu
def test_prepared_blocks_follow_the_size_class_of_P():
    torch.manual_seed(4)
    mod = build_stack([64, 128, 128, 5], "BR BR b".split(), 3).cuda().eval()
    specs = fused.parse_stack(mod)
    xs = {P: torch.randn(P, 64, device="cuda") for P in (8, 15, 16, 100, 5000)}
    with torch.no_grad():
        plain = {P: fused.mlp_stack(x, specs, 0, False).clone() for P, x in xs.items()}
        with runtime.static_weights_scope():
            for _ in range(2):              # builds the blocks, then reuses them
                for P, x in xs.items():
                    got = fused.mlp_stack(x, specs, 0, False)
                    assert torch.equal(got, plain[P]), P
    for P, x in xs.items():
        assert rel(plain[P], reference_stack(x, specs, 0, False)) < RTOL, P


# ---------------------------------------------------------------------------------------------- in-place gradient accumulation
@pytest.mark.gpu
def test_inplace_accumulation_adds_to_existing_grads():
    """[8 -> 192 -> 128 -> 36] at P >= 4096: skinny wgrad (K = 8), tensor-core wgrad with a 64-column CUDA-core tail (K = 192),
    CUDA-core wgrad (Nw = 36) and a bias-only last layer (d2f_kernel)."""
    torch.manual_seed(9)
    mod = build_stack([8, 192, 128, 36], "BR BR b".split(), 13).cuda().train()
    specs = fused.parse_stack(mod)
    x = torch.randn(4096 + 20, 8, device="cuda")
    go = torch.randn(x.shape[0], 36, device="cuda")
    params = list(mod.parameters())
    fresh = torch.autograd.grad(fused.mlp_stack(x, specs, 0, True), params, go)
    g = torch.Generator().manual_seed(2)
    prior = [torch.randn(p.shape, generator=g).cuda() for p in params]
    for p, v in zip(params, prior):
        p.grad = v.clone()
    with runtime.grad_inplace_scope():
        fused.mlp_stack(x, specs, 0, True).backward(go)
    torch.cuda.synchronize()
    bn_biases = {id(mod.conv0.bias), id(mod.conv1.bias)}
    for p, v, f in zip(params, prior, fresh):
        if id(p) in bn_biases:
            assert torch.equal(p.grad, v)          # BatchNorm removes the mean: nothing to add
            continue
        err = (p.grad.double() - (v.double() + f.double())).abs()
        bound = 1e-6 * (v.double().abs() + f.double().abs()) + 1e-5 * float(f.double().abs().max())
        assert bool((err <= bound).all()), (tuple(p.shape), float(err.max()))
