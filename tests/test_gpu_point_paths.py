"""Every point-cloud kernel (csrc/fps.cu, ball_query.cu / ball_query.cuh, group_gather.cu, three_nn.cu, xcorr.cu) at the shapes
where its launcher picks another instantiation, staging path, grid shape or loop trip count, with the kernels that ran asserted
from a CUDA profile.

What each output is compared with:
- indices and gathered values: bitwise, against the C oracle (oracle/ops.py) or an exact torch gather;
- sums (scatter gradients, interpolation, cosine map): against a float64 statement, with a bar per tensor (the measured errors
  are printed);
- the fused three-NN weights: bitwise, against a float32 restatement in the kernel's operation order.
Each case names the kernels it was written to reach (`want`) and the ones that must not run (`avoid`), so a retuned threshold
cannot move it onto another path unnoticed."""
import functools
import json
import os
import re
import subprocess
import sys
import tempfile
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from open3dsot_b200 import _lib, fused, ops
from oracle import ops as oops
from test_gpu_ops import dup_cloud
from test_gpu_stack_paths import _norm, _ran

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "open3dsot_b200", "csrc")
SOURCES = ["fps.cu", "ball_query.cu", "ball_query.cuh", "group_gather.cu", "three_nn.cu", "xcorr.cu"]

# every point kernel (names with the anonymous namespace and blanks removed)
FPS = {n: f"fps_kernel<{t},{p}>" for n, (t, p) in {128: (128, 1), 256: (128, 2), 512: (256, 2), 1024: (512, 2),
                                                   2048: (256, 8), 4096: (256, 16), 8192: (512, 16), 16384: (512, 32)}.items()}
BQ, BQG, BQGG = "ball_query_kernel", "ballquery_group_kernel", "ballquery_group_grad_kernel"
ROWS, ROWSG = "group_rows_kernel", "group_rows_grad_kernel"
GRP, GRPG = "group_kernel", "group_grad_kernel"
NN, TI, TIG = "three_nn_kernel", "three_interpolate_kernel", "three_interpolate_grad_kernel"
NNI, NNIG = "three_nn_interpolate_kernel", "three_nn_interpolate_grad_kernel"
TOPK, SIM, SIMG = "boxaware_topk_kernel", "p2b_sim_kernel", "p2b_sim_grad_kernel"
KERNELS = [*FPS.values(), BQ, BQG, BQGG, ROWS, ROWSG, GRP, GRPG, NN, TI, TIG, NNI, NNIG, TOPK, SIM, SIMG]


# bars, each about twice the largest error measured on an H100 over this file's cases (in brackets)
SUM_BAR = 1e-6       # float32 scatter-adds (atomics, any order) against float64: norm-wise relative [4.8e-7]
INTERP_BAR = 2e-7    # three-term interpolation (one product, two FMAs) against float64: norm-wise relative [3.7e-8]
SIM_BAR = 5e-7       # cosine map against float64: max absolute [2.1e-7]
NORM_BAR = 1e-6      # row norms against float64: max relative [4.6e-7]
P2B_GRAD_BAR = 1e-6  # cosine-map gradients against float64, per kind of row: norm-wise relative [3.6e-7]


def fps_kernel_for(N):
    """the instantiation o3d_fps picks for N points (the smallest tier that holds N)"""
    return FPS[min(t for t in FPS if N <= t)]


class Case:
    def __init__(self, name, want, avoid=(), **params):
        self.name, self.want, self.avoid = name, tuple(want), tuple(avoid)
        self.__dict__.update(params)


# ---------------------------------------------------------------------------------------------- case tables
# FPS: both sides of every tier boundary of o3d_fps.  dup: 20 % distinct sites (exact ties from the first round on; npoint > the
# number of sites leaves only zero-distance ties) and two sites with |p|^2 <= 1e-3 that never win; sparse: 40 eligible points,
# all in the upper half of the cloud, the rest never a candidate (npoint > 40 repeats the winners' tie order)
FPS_CASES = [Case(f"fps_N{N}_np{npoint}_{cloud}", [fps_kernel_for(N)], [k for k in FPS.values() if k != fps_kernel_for(N)],
                  B=B, N=N, npoint=npoint, cloud=cloud)
             for B, N, npoint, cloud in [
                 (3, 128, 128, "dup"), (2, 129, 1, "dup"),
                 (2, 256, 100, "dup"), (3, 257, 257, "dup"),
                 (2, 512, 256, "dup"), (2, 513, 64, "dup"),
                 (2, 1024, 1024, "dup"), (2, 1025, 300, "rand"),
                 (2, 2048, 512, "dup"), (2, 2049, 2049, "dup"),
                 (2, 4096, 256, "dup"), (2, 4097, 1, "dup"),
                 (2, 8192, 1024, "rand"), (2, 8193, 8193, "dup"),
                 (2, 16384, 16384, "dup"), (3, 16384, 2048, "rand"),
                 (2, 300, 64, "sparse"), (2, 16384, 100, "sparse")]]

# ball query: name, B, N, M, radius, nsample, cloud (grid: 1/8 grid, every d2 exact, points exactly on the radius 0.25)
BQ_CASES = [Case(n, [BQ], [BQG], B=B, N=N, M=M, r=r, ns=ns, cloud=cloud) for n, B, N, M, r, ns, cloud in [
    ("bq_N4097_smem_attr_ns33", 2, 4097, 1000, 0.25, 33, "grid"),
    ("bq_N17066_smem_cap_ns64", 2, 17066, 517, 0.3, 64, "dup"),
    ("bq_N1023_B3_ns1", 3, 1023, 77, 0.4, 1, "dup"),
    ("bq_ns_over_N", 2, 50, 50, 1.5, 64, "dup"),
    ("bq_N2050_on_radius_ns64", 3, 2050, 333, 0.25, 64, "grid"),
]]

# fused ball query + grouping: C feature channels, nsample > 32 wraps the coordinate loop, C > 128 the feature loop, N % 4 != 0
# (or an odd cloud offset) takes the cooperative staging, ret=False the idx == nullptr branch
BQG_CASES = [Case(n, [BQG], [BQ], B=B, N=N, M=M, C=C, r=r, ns=ns, norm=norm, ret=ret, cloud=cloud)
             for n, B, N, M, C, r, ns, norm, ret, cloud in [
                 ("bqg_c0_N5001_ns64_norm", 2, 5001, 300, 0, 0.3, 64, True, True, "dup"),
                 ("bqg_c4_N1026_ns33", 2, 1026, 100, 4, 0.4, 33, False, True, "dup"),
                 ("bqg_c132_N5000_ns64_no_idx", 2, 5000, 257, 132, 0.3, 64, True, False, "dup"),
                 ("bqg_c260_N999_ns40", 3, 999, 64, 260, 0.5, 40, False, True, "dup"),
                 ("bqg_c132_grid_N4098_ns64", 2, 4098, 200, 132, 0.25, 64, False, True, "grid"),
             ]]

# its gradient: every need_* subset (f = features, x = xyz, n = centres) with rows = M * nsample > 8 warps * 8 * #SMs (132 on an
# H100 SXM), so every CTA of the capped grid loops; pad: radius 0.02, almost every ball holds its centre only (63 padding copies)
BQGG_CASES = [Case(f"bqg_grad_{need}", [BQGG], B=2, N=2000, M=200, C=132, r=0.3, ns=64, norm=need != "x", need=need, pad=False)
              for need in ("fxn", "fx", "fn", "xn", "f", "x", "n")] + [
    Case("bqg_grad_pad_fxn", [BQGG], B=2, N=2000, M=200, C=4, r=0.02, ns=64, norm=True, need="fxn", pad=True)]

# channels-last row gather (BoxAware grouping): L rows from N, C % 4 == 0; L > 8 * 8 * #SMs loops the capped grid
ROWS_CASES = [Case(n, [ROWS, ROWSG], B=B, N=N, L=L, C=C) for n, B, N, L, C in [
    ("rows_c4_L9001", 2, 500, 9001, 4),
    ("rows_c128_N64_L9000", 2, 64, 9000, 128),
    ("rows_c132_L4100", 3, 1000, 4100, 132),
    ("rows_c268_L12000", 2, 300, 12000, 268),
]]

# reference-layout gather / group: L = M (gather) or M * S (group); L % 4 == 0 takes the int4 / float4 path
GROUP_CASES = [Case(n, [GRP, GRPG], op=op, B=B, C=C, N=N, M=M, S=S) for n, op, B, C, N, M, S in [
    ("gather_c1_L2051", "gather", 2, 1, 700, 2051, 1),
    ("gather_c8_L4096", "gather", 2, 8, 300, 4096, 1),
    ("group_c9_L2064", "group", 2, 9, 500, 129, 16),
    ("group_c300_L2051", "group", 2, 300, 257, 293, 7),
    ("group_c8_L1023", "group", 3, 8, 100, 341, 3),
]]

# three_nn: m known points (m < 3 leaves +inf / index 0 slots; m = 5000 needs the shared-memory attribute)
NN_CASES = [Case(f"three_nn_m{m}_n{n}", [NN], [NNI], B=2, n=n, m=m) for n, m in
            [(77, 1), (100, 2), (33, 3), (257, 31), (1001, 32), (95, 33), (1003, 5000)]]

INTERP_CASES = [Case(f"three_interp_c{c}_n{n}", [TI, TIG], B=2, c=c, m=m, n=n) for c, m, n in
                [(1, 50, 300), (3, 7, 1001), (300, 129, 257)]]

# fused three-NN + interpolation (channels-last): c > 128 wraps the float4 loop; every unknown cloud holds copies of known points
FNN_CASES = [Case(f"fnn_m{m}_c{c}", [NNI, NNIG], [NN, TI, TIG], B=2, n=n, m=m, c=c) for n, m, c in
             [(77, 1, 4), (300, 2, 132), (257, 3, 260), (1003, 5000, 128), (2000, 5000, 260)]]

# BoxAware top-k on a 1/64 grid (every d2 exact, ties exact): k = 1..8, D = 1 / 9 / 16, M = k and M at the 48 KB template limit
TOPK_CASES = [Case(f"topk_k{k}_D{D}_M{M}_N{N}", [TOPK], B=B, M=M, N=N, D=D, k=k) for B, M, N, D, k in [
    (2, 1, 130, 1, 1), (3, 2, 129, 16, 2), (2, 1365, 300, 9, 3), (3, 64, 200, 9, 4),
    (2, 12288, 257, 1, 5), (2, 768, 131, 16, 6), (2, 7, 250, 9, 7), (2, 100, 1000, 1, 8), (2, 1365, 129, 9, 8)]]

# P2B cosine: n1 around the 32-lane / 4-slot edges, n2 around the 16-point block, C around the 32-channel chunk; need: the
# gradients taken (C = 1 has a constant cosine map, +-1 or 0: its gradient vanishes and is taken at C = 1 only where every row is
# clamped)
P2B_CASES = [Case(f"p2b_n1_{n1}_n2_{n2}_C{C}_{need or 'fwd'}", [SIM] + ([SIMG] if need else []), B=2, n1=n1, n2=n2, C=C,
                  need=need)
             for n1, n2, C, need in [(1, 1, 1, "ts"), (31, 15, 31, "ts"), (32, 16, 32, "ts"), (33, 17, 33, "ts"),
                                     (127, 256, 257, "ts"), (128, 256, 32, "ts"), (128, 17, 1, ""), (33, 16, 257, "t"),
                                     (32, 15, 31, "s"), (128, 1, 33, "ts")]]

ALL_CASES = (FPS_CASES + BQ_CASES + BQG_CASES + BQGG_CASES + ROWS_CASES + GROUP_CASES + NN_CASES + INTERP_CASES + FNN_CASES +
             TOPK_CASES + P2B_CASES)


# ---------------------------------------------------------------------------------------------- CPU-only checks
def _source_kernels():
    """the __global__ functions of the point sources, fps_kernel replaced by the instantiations o3d_fps launches"""
    names = set()
    for f in SOURCES:
        with open(os.path.join(CSRC, f)) as fh:
            names |= set(re.findall(r"__global__\s+void\s+(?:__launch_bounds__\([^)]*\)\s+)?(\w+)\s*\(", fh.read()))
    with open(os.path.join(CSRC, "fps.cu")) as fh:
        src = fh.read()
    body = src[src.index('extern "C" int o3d_fps('):]
    inst = {f"fps_kernel<{t},{p}>" for t, p in re.findall(r"launch_fps<\s*(\d+)\s*,\s*(\d+)\s*>\s*\(", body)}
    assert "fps_kernel" in names and inst
    return (names - {"fps_kernel"}) | inst


def test_kernel_list_matches_the_sources():
    """A new point kernel or FPS instantiation cannot land without appearing here (and, below, in some case's `want`)."""
    assert len(KERNELS) == len(set(KERNELS))
    assert set(KERNELS) == _source_kernels(), (sorted(set(KERNELS) - _source_kernels()), sorted(_source_kernels() - set(KERNELS)))


def test_every_point_kernel_is_a_declared_target():
    declared = {k for c in ALL_CASES for k in c.want}
    assert set(KERNELS) <= declared, sorted(set(KERNELS) - declared)
    assert declared <= set(KERNELS), sorted(declared - set(KERNELS))
    assert len({c.name for c in ALL_CASES}) == len(ALL_CASES)
    for c in FPS_CASES:
        assert 1 <= c.npoint and c.N <= 16384, c.name
    for t in FPS:          # both neighbours of every tier boundary
        assert any(c.N == t for c in FPS_CASES) and (t == 16384 or any(c.N == t + 1 for c in FPS_CASES)), t
    for c in BQG_CASES + BQGG_CASES + ROWS_CASES + FNN_CASES:
        assert getattr(c, "C", getattr(c, "c", 0)) % 4 == 0, c.name
    for c in TOPK_CASES:
        assert c.k <= c.M and c.M * c.D * 4 <= 48 * 1024, c.name
    assert {c.k for c in TOPK_CASES} == set(range(1, 9)) and {c.D for c in TOPK_CASES} == {1, 9, 16}


def test_point_launchers_refuse_bad_sizes_before_any_launch():
    """Host-side refusals, called with dummy 16-byte-aligned pointers that no kernel may touch: each must return O3D_ERR_ARG
    before any launch."""
    L = _lib.lib()
    P = 16
    # an empty known cloud: the interpolation would read feature row 0 of it for every unknown point
    assert L.o3d_three_nn_interpolate(P, P, P, 1, 8, 0, 4, P, P, P, None) == -1
    assert b"m=0" in L.o3d_last_error()
    assert L.o3d_three_nn_interpolate(P, P, P, 2, 8, -1, 4, P, P, P, None) == -1
    # one point past the ball query's 200 KB shared-memory cloud (N = 17066 is the largest accepted, a GPU case below)
    assert L.o3d_ball_query(P, P, 1, 17067, 1, 0.3, 32, P, None) == -1
    assert b"17067" in L.o3d_last_error()
    assert L.o3d_fps(P, 1, 16385, 8, P, None) == -1
    # template box cloud one row over 48 KB (D = 9: M = 1365 is the largest accepted)
    assert L.o3d_xcorr_boxaware_fwd(P, P, 1, 1366, 8, 9, 4, P, None) == -1


# ---------------------------------------------------------------------------------------------- kernel observation
# Which kernels ran is observed in a child process that runs this file with PROFILE_OUT set: every test profiles its call there
# and records the kernel names under its own id.  The pytest process itself never starts CUPTI (as in the other profiling
# tests of the suite), so the in-process profiles of later test files see the same process state as without this file.
PROFILE_OUT = "O3D_POINT_PATHS_PROFILE_OUT"


def _test_id():
    """test name and parameters (the node id without its path, which depends on the rootdir of the run)"""
    return os.environ["PYTEST_CURRENT_TEST"].rsplit(" ", 1)[0].split("::", 1)[1]


def _profiled(fn):
    """fn() followed by a device synchronisation -- under the CUDA profiler in the child, whose record gets this test's kernels"""
    def run():
        res = fn()
        torch.cuda.synchronize()
        return res

    out = os.environ.get(PROFILE_OUT)
    if out is None:
        return run()
    # A fresh profiling session can miss the records of the short kernels it launches first (on an H100, every call here whose
    # first kernel is short lost that kernel's record; FPS over thousands of points and the 17,066-point ball query did not),
    # and most calls here are one or two short kernels.  The kernel choice depends on shapes only, so the call runs twice in
    # the session and the record is the union.
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        run()
        res = run()
    names = {_norm(e.name) for e in prof.events()}
    if not any("kernel" in n for n in names):
        # CUPTI now and then delivers no activity records at all for a short session: observe another identical session
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            run()
            run()
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


def _assert_kernels(case):
    """the kernels this test's call ran (observed in the child) include every `want` and no `avoid`"""
    if os.environ.get(PROFILE_OUT) is not None:
        return                # the child only records; the asserting process is the parent
    rec, log = _child_profiles()
    assert _test_id() in rec, ("no kernel record for this test", log)
    names = rec[_test_id()]
    kernels = sorted(n for n in names if "kernel" in n)
    missing = [k for k in case.want if not _ran(names, k)]
    assert not missing, (missing, kernels)
    unwanted = [k for k in case.avoid if _ran(names, k)]
    assert not unwanted, (unwanted, kernels)


# ---------------------------------------------------------------------------------------------- helpers
def _gen(case):
    return torch.Generator().manual_seed(zlib.crc32(case.name.encode()))


def _check_sum(tag, got, want, bar):
    """norm-wise relative error of a float32 sum against its float64 statement; printed, then held to `bar`"""
    got, want = got.detach().cpu().double(), want.detach().cpu().double()
    assert got.shape == want.shape, (tag, got.shape, want.shape)
    e = float((got - want).norm() / want.norm().clamp_min(1e-30))
    print(f"[{tag}] {e:.2e} (bar {bar:.0e})")
    assert e < bar, (tag, e, bar)


def _scatter_rows(src, idx, rows):
    """float64 statement of a scatter-add: out[b, idx[b, l]] += src[b, l] (src (B, L, C), idx (B, L))"""
    B, L, C = src.shape
    out = torch.zeros(B, rows, C, dtype=torch.float64)
    for b in range(B):
        out[b].index_add_(0, idx[b].long(), src[b].double())
    return out


def _gather_rows(x, idx):
    """exact gather: x (B, N, C), idx (B, ...) -> (B, ..., C)"""
    return torch.stack([x[b][idx[b].long()] for b in range(x.shape[0])])


def _cloud(kind, B, N, g, seed):
    if kind == "grid":            # 1/8 grid: squared distances exact, and many exactly 1/16 = 0.25^2
        return torch.randint(-6, 7, (B, N, 3), generator=g).float() / 8
    return dup_cloud(B, N, seed, frac_unique=0.5, near_origin=False)


def _centres(kind, xyz, M, g):
    B, N, _ = xyz.shape
    if kind == "grid":
        new = torch.randint(-6, 7, (B, M, 3), generator=g).float() / 8
    else:
        new = xyz[:, torch.randint(0, N, (M,), generator=g)].clone()
    new[:, 3::7] += 50.0          # centres with empty balls
    return new.contiguous()


def _on_radius(xyz, new, r):
    """number of (centre, point) pairs exactly on the radius"""
    d2 = ((new[:, :, None, :].double() - xyz[:, None, :, :].double()) ** 2).sum(-1)
    return int((d2 == r * r).sum())


# ---------------------------------------------------------------------------------------------- FPS
def _fps_cloud(case, g):
    B, N = case.B, case.N
    if case.cloud == "dup":
        return dup_cloud(B, N, seed=N + case.npoint)
    if case.cloud == "rand":
        return torch.randn(B, N, 3, generator=g)
    xyz = (torch.rand(B, N, 3, generator=g) - 0.5) * 0.02            # |p|^2 <= 3e-4: never a candidate
    pick = N // 2 + torch.randperm(N - N // 2, generator=g)[:40]
    xyz[:, pick] = torch.randn(B, 40, 3, generator=g) + 2.0
    return xyz


@pytest.mark.gpu
@pytest.mark.parametrize("case", FPS_CASES, ids=[c.name for c in FPS_CASES])
def test_fps_path(case):
    xyz = _fps_cloud(case, _gen(case))
    x = xyz.cuda()
    got = _profiled(lambda: ops.furthest_point_sampling(x, case.npoint)).cpu()
    assert torch.equal(got, oops.furthest_point_sampling(xyz, case.npoint))
    if case.cloud == "sparse":       # every eligible point is sampled before any repeats
        assert (got[:, 1:41] >= case.N // 2).all() and all(len(set(r[1:41].tolist())) == 40 for r in got)
    _assert_kernels(case)


# ---------------------------------------------------------------------------------------------- ball query
@pytest.mark.gpu
@pytest.mark.parametrize("case", BQ_CASES, ids=[c.name for c in BQ_CASES])
def test_ball_query_path(case):
    g = _gen(case)
    xyz = _cloud(case.cloud, case.B, case.N, g, case.N + case.M)
    new = _centres(case.cloud, xyz, case.M, g)
    if case.cloud == "grid":
        assert _on_radius(xyz, new, case.r) > 100
    x, c = xyz.cuda(), new.cuda()
    got = _profiled(lambda: ops.ball_query(c, x, case.r, case.ns)).cpu()
    want = oops.ball_query(new, xyz, case.r, case.ns)
    assert torch.equal(got, want)
    assert (want[:, 3::7] == 0).all()                               # the empty balls
    _assert_kernels(case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", BQG_CASES, ids=[c.name for c in BQG_CASES])
def test_ballquery_group_path(case):
    g = _gen(case)
    B, N, M, C, r, ns = case.B, case.N, case.M, case.C, case.r, case.ns
    xyz = _cloud(case.cloud, B, N, g, N + M)
    new = _centres(case.cloud, xyz, M, g)
    feat = torch.randn(B, N, C, generator=g) if C else None
    x, c, f = xyz.cuda(), new.cuda(), feat.cuda() if C else None
    grouped, idx = _profiled(lambda: ops.ballquery_group(x, c, f, r, ns, case.norm, case.ret))
    grouped = grouped.cpu()
    widx = oops.ball_query(new, xyz, r, ns)
    if case.ret:
        assert torch.equal(idx.cpu(), widx)
    else:
        assert idx is None
    assert grouped.shape == (B, M, ns, C + 4)
    rel = _gather_rows(xyz, widx) - new[:, :, None, :]               # float32, rounded once as in the kernel
    if case.norm:
        rel = rel / torch.tensor(r, dtype=torch.float32)
    assert torch.equal(grouped[..., C:C + 3], rel)
    assert grouped[..., C + 3].eq(0).all()
    if C:
        assert torch.equal(grouped[..., :C], _gather_rows(feat, widx))
    _assert_kernels(case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", BQGG_CASES, ids=[c.name for c in BQGG_CASES])
def test_ballquery_group_grad_path(case):
    g = _gen(case)
    B, N, M, C, r, ns = case.B, case.N, case.M, case.C, case.r, case.ns
    assert M * ns > 64 * _lib.lib().o3d_device_sms()                 # more rows than the capped grid has warps
    xyz = torch.rand(B, N, 3, generator=g) * 2
    new = xyz[:, :M].contiguous()
    idx = oops.ball_query(new, xyz, r, ns)
    if case.pad:
        assert float((idx == idx[..., :1]).float().mean()) > 0.9    # nearly every row is a padding copy of the first hit
    gg = torch.randn(B, M, ns, C + 4, generator=g)
    need = dict(need_feat="f" in case.need, need_xyz="x" in case.need, need_new_xyz="n" in case.need)
    gd, idd = gg.cuda(), idx.cuda()
    gf, gx, gn = _profiled(lambda: ops.ballquery_group_grad(gd, idd, N, r, case.norm, **need))
    assert (gf is None) != need["need_feat"] and (gx is None) != need["need_xyz"] and (gn is None) != need["need_new_xyz"]
    scale = 1.0 / r if case.norm else 1.0
    gxyz = gg[..., C:C + 3].double() * scale
    if gf is not None:
        _check_sum(f"{case.name} dfeat", gf, _scatter_rows(gg[..., :C].reshape(B, M * ns, C), idx.reshape(B, -1), N), SUM_BAR)
    if gx is not None:
        _check_sum(f"{case.name} dxyz", gx, _scatter_rows(gxyz.reshape(B, M * ns, 3), idx.reshape(B, -1), N), SUM_BAR)
    if gn is not None:
        _check_sum(f"{case.name} dnew_xyz", gn, -gxyz.sum(2), SUM_BAR)
    _assert_kernels(case)


# ---------------------------------------------------------------------------------------------- row gather (BoxAware grouping)
@pytest.mark.gpu
@pytest.mark.parametrize("case", ROWS_CASES, ids=[c.name for c in ROWS_CASES])
def test_group_rows_path(case):
    g = _gen(case)
    B, N, L, C = case.B, case.N, case.L, case.C
    feat = torch.randn(B, N, C, generator=g)
    idx = torch.randint(0, N, (B, L), generator=g, dtype=torch.int32)
    idx[:, 1::3] = idx[:, 0::3][:, :idx[:, 1::3].shape[1]]          # repeated indices, also within one warp's rows
    go = torch.randn(B, L, C, generator=g)
    f, i, gd = feat.cuda().requires_grad_(True), idx.cuda(), go.cuda()

    def step():
        out = fused._GroupRowsCL.apply(f, i)
        return out, torch.autograd.grad(out, f, gd)[0]

    out, gf = _profiled(step)
    assert torch.equal(out.detach().cpu(), _gather_rows(feat, idx))
    _check_sum(f"{case.name} dfeat", gf, _scatter_rows(go, idx, N), SUM_BAR)
    _assert_kernels(case)


# ---------------------------------------------------------------------------------------------- reference-layout gather / group
@pytest.mark.gpu
@pytest.mark.parametrize("case", GROUP_CASES, ids=[c.name for c in GROUP_CASES])
def test_gather_group_path(case):
    g = _gen(case)
    B, C, N, M, S = case.B, case.C, case.N, case.M, case.S
    feat = torch.randn(B, C, N, generator=g)
    shape = (B, M) if case.op == "gather" else (B, M, S)
    idx = torch.randint(0, N, shape, generator=g, dtype=torch.int32)
    idx.view(B, -1)[:, 2::5] = idx.view(B, -1)[:, 0:1]                # repeated indices
    go = torch.randn(B, C, *shape[1:], generator=g)
    f, i, gd = feat.cuda(), idx.cuda(), go.cuda()
    if case.op == "gather":
        out, gf = _profiled(lambda: (ops.gather_points(f, i), ops.gather_points_grad(gd, i, N)))
    else:
        out, gf = _profiled(lambda: (ops.group_points(f, i), ops.group_points_grad(gd, i, N)))
    L = idx[0].numel()
    want = _gather_rows(feat.transpose(1, 2), idx.view(B, L)).transpose(1, 2).reshape(B, C, *shape[1:])
    assert torch.equal(out.cpu(), want)
    ref = _scatter_rows(go.reshape(B, C, L).transpose(1, 2), idx.view(B, L), N).transpose(1, 2)
    _check_sum(f"{case.name} dfeat", gf, ref, SUM_BAR)
    _assert_kernels(case)


# ---------------------------------------------------------------------------------------------- three-NN
def _nn_clouds(case, g):
    """known: 50 % distinct sites (exact distance ties); unknown: every fifth point a copy of a known point (d2 = 0)"""
    known = dup_cloud(case.B, case.m, seed=case.m + 1, frac_unique=0.5, near_origin=False)
    unknown = (torch.rand(case.B, case.n, 3, generator=g) - 0.5) * 4
    pick = torch.randint(0, case.m, (len(range(0, case.n, 5)),), generator=g)
    unknown[:, ::5] = known[:, pick]
    return unknown.contiguous(), known


@pytest.mark.gpu
@pytest.mark.parametrize("case", NN_CASES, ids=[c.name for c in NN_CASES])
def test_three_nn_path(case):
    unknown, known = _nn_clouds(case, _gen(case))
    u, k = unknown.cuda(), known.cuda()
    d2, idx = _profiled(lambda: ops.three_nn(u, k))
    wd2, widx = oops.three_nn(unknown, known)
    assert torch.equal(idx.cpu(), widx)
    assert torch.equal(d2.cpu(), wd2)                                 # bitwise, +inf in the slots m < 3 leaves empty
    assert (wd2[:, ::5, 0] == 0).all()
    _assert_kernels(case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", INTERP_CASES, ids=[c.name for c in INTERP_CASES])
def test_three_interpolate_path(case):
    g = _gen(case)
    B, c, m, n = case.B, case.c, case.m, case.n
    feat = torch.randn(B, c, m, generator=g)
    idx = torch.randint(0, m, (B, n, 3), generator=g, dtype=torch.int32)
    idx[:, ::4, 1] = idx[:, ::4, 0]                                   # one point twice among the three
    w = torch.rand(B, n, 3, generator=g)
    go = torch.randn(B, c, n, generator=g)
    f, i, wd, gd = feat.cuda(), idx.cuda(), w.cuda(), go.cuda()
    out, gf = _profiled(lambda: (ops.three_interpolate(f, i, wd), ops.three_interpolate_grad(gd, i, wd, m)))
    rows = _gather_rows(feat.transpose(1, 2).double(), idx.view(B, -1)).view(B, n, 3, c)
    _check_sum(f"{case.name} out", out, (rows * w.double()[..., None]).sum(2).transpose(1, 2), INTERP_BAR)
    src = (go.transpose(1, 2).double()[:, :, None, :] * w.double()[..., None]).reshape(B, n * 3, c)
    _check_sum(f"{case.name} dfeat", gf, _scatter_rows(src, idx.view(B, -1), m).transpose(1, 2), SUM_BAR)
    _assert_kernels(case)


def _weights_f32(d2):
    """the fused kernel's inverse-distance weights, step by step in float32 (every step IEEE-rounded on both sides)"""
    d2 = d2.numpy().astype(np.float32)
    r = np.float32(1.0) / (np.sqrt(d2) + np.float32(1e-8))
    norm = (r[..., 0] + r[..., 1]) + r[..., 2]
    return torch.from_numpy(r / norm[..., None])


@pytest.mark.gpu
@pytest.mark.parametrize("case", FNN_CASES, ids=[c.name for c in FNN_CASES])
def test_three_nn_interpolate_path(case):
    g = _gen(case)
    B, n, m, c = case.B, case.n, case.m, case.c
    unknown, known = _nn_clouds(case, g)
    kf = torch.randn(B, m, c, generator=g)
    go = torch.randn(B, n, c, generator=g)
    u, k, f, gd = unknown.cuda(), known.cuda(), kf.cuda(), go.cuda()

    def step():
        out, idx, w = ops.three_nn_interpolate(u, k, f)
        return out, idx, w, ops.three_nn_interpolate_grad(gd, idx, w, m)

    out, idx, w, gk = _profiled(step)
    wd2, widx = oops.three_nn(unknown, known)
    assert torch.equal(idx.cpu(), widx)
    ww = _weights_f32(wd2)
    assert torch.equal(w.cpu(), ww)
    assert ((ww * (wd2 == 0)).sum(-1)[:, ::5] > 0.99).all()           # coincident known points take (almost) all the weight
    rows = _gather_rows(kf.double(), widx.view(B, -1)).view(B, n, 3, c)
    _check_sum(f"{case.name} out", out, (rows * ww.double()[..., None]).sum(2), INTERP_BAR)
    src = (go.double()[:, :, None, :] * ww.double()[..., None]).reshape(B, n * 3, c)
    _check_sum(f"{case.name} dfeat", gk, _scatter_rows(src, widx.view(B, -1), m), SUM_BAR)
    _assert_kernels(case)


# ---------------------------------------------------------------------------------------------- BoxAware top-k
@pytest.mark.gpu
@pytest.mark.parametrize("case", TOPK_CASES, ids=[c.name for c in TOPK_CASES])
def test_boxaware_topk_path(case):
    g = _gen(case)
    B, M, N, D, k = case.B, case.M, case.N, case.D, case.k
    t = torch.randint(0, 48, (B, M, D), generator=g).float() / 64
    s = torch.randint(0, 48, (B, N, D), generator=g).float() / 64
    if M >= 6:
        t[:, M // 2:M // 2 + 3] = t[:, 0:3]                           # duplicated template points: exact ties
    tc, sc = t.cuda(), s.cuda()
    got = _profiled(lambda: ops.boxaware_topk(tc, sc, k)).cpu()
    d2 = ((t[:, :, None, :].double() - s[:, None, :, :].double()) ** 2).sum(-1)        # (B, M, N), exact
    want = torch.argsort(d2, dim=1, stable=True)[:, :k, :].transpose(1, 2).int()     # ties: ascending template index
    assert torch.equal(got, want)
    _assert_kernels(case)


# ---------------------------------------------------------------------------------------------- P2B cosine map
def _cosine_map(t, s, eps=1e-8):
    """(B, n2, n1) cosine map with the norms clamped to eps by a differentiable clamp: below eps a row's term is x / eps, linear,
    whose derivative is the kernel's.  F.cosine_similarity computes the same values, but it clamps its norms in place without
    recording the clamp, so its gradient for a row with 0 < |x| <= eps is not the derivative of what it computes; everywhere
    else the two gradients agree (asserted below)."""
    tn = t / t.norm(dim=-1, keepdim=True).clamp_min(eps)
    sn = s / s.norm(dim=-1, keepdim=True).clamp_min(eps)
    return sn @ tn.transpose(1, 2)


@pytest.mark.gpu
@pytest.mark.parametrize("case", P2B_CASES, ids=[c.name for c in P2B_CASES])
def test_p2b_cosine_path(case):
    g = _gen(case)
    B, n1, n2, C = case.B, case.n1, case.n2, case.C
    t = torch.randn(B, n1, C, generator=g)
    s = torch.randn(B, n2, C, generator=g)
    t[0, 0] = 0.0                                                     # zero-norm rows
    s[0, n2 - 1] = 0.0
    t[B - 1, n1 - 1] *= 1e-9                                          # tiny rows: 1e-9 * sqrt(C), clamped up to C = 100
    s[B - 1, 0] *= 1e-9
    w = torch.randn(B, n2, n1, generator=g)
    tc, sc, wc = t.cuda().requires_grad_("t" in case.need), s.cuda().requires_grad_("s" in case.need), w.cuda()

    def step():
        sim, tn, sn = ops.p2b_cosine(tc.detach(), sc.detach())
        if not case.need:
            return sim, tn, sn, ()
        out = fused._P2BCosine.apply(tc, sc)
        return sim, tn, sn, torch.autograd.grad((out * wc).sum(), [x for x in (tc, sc) if x.requires_grad])

    sim, tn, sn, grads = _profiled(step)
    td, sd = t.double().requires_grad_(True), s.double().requires_grad_(True)
    ref = _cosine_map(td, sd)
    torch_ref = F.cosine_similarity(td.transpose(1, 2).unsqueeze(-1), sd.transpose(1, 2).unsqueeze(2), dim=1).transpose(1, 2)
    assert float((ref - torch_ref).detach().abs().max()) < 1e-12
    e = float((sim.cpu().double() - ref.detach()).abs().max())
    print(f"[{case.name}] sim max abs {e:.1e} (bar {SIM_BAR:.0e})")
    assert e < SIM_BAR
    for tag, got, x in (("tnorm", tn, t), ("snorm", sn, s)):
        want = x.double().norm(dim=-1)
        e = float(((got.cpu().double() - want).abs() / want.clamp_min(1e-30)).max())
        print(f"[{case.name}] {tag} max rel {e:.1e} (bar {NORM_BAR:.0e})")
        assert e < NORM_BAR, (tag, e)
    if case.need:
        want = torch.autograd.grad((ref * w.double()).sum(), [td, sd])
        want_torch = torch.autograd.grad((torch_ref * w.double()).sum(), [td, sd])
        taken = [(tag, x, wt, wtt) for tag, x, wt, wtt in zip("ts", (t, s), want, want_torch) if tag in case.need]
        for (tag, x, wt, wtt), got in zip(taken, grads):
            got, nrm = got.cpu().double(), x.double().norm(dim=-1)
            # each kind of row on its own: the clamped ones are scaled by 1 / eps = 1e8 and would swamp the others
            for kind, rows in (("zero", nrm == 0), ("clamped", (nrm > 0) & (nrm <= 1e-8)), ("tiny", (nrm > 1e-8) & (nrm < 1e-6)),
                               ("unit", nrm >= 1e-6)):
                if rows.any():
                    _check_sum(f"{case.name} d{tag} {kind} rows", got[rows], wt[rows], P2B_GRAD_BAR)
                    if kind != "clamped":
                        assert float((wt[rows] - wtt[rows]).norm() / wt[rows].norm().clamp_min(1e-30)) < 1e-12
    _assert_kernels(case)
