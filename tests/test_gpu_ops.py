"""GPU parity of the sm_90a kernels (through the C ABI) against the oracle: bit-exact indices, 1e-4-relative
floats (north_star).  Edge cases per SURVEY.md §8c: duplicates, near-origin points, all-zero clouds, N not a
multiple of the block, N < block, empty balls, on-radius points, > nsample hits, m < 3, repeated indices."""
import numpy as np
import pytest
import torch

from open3dsot_b200 import ops
from open3dsot_b200.datasets.synthetic import synthetic_siamese_batch
from oracle import ops as oops

pytestmark = pytest.mark.gpu
RTOL = 1e-4


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def dup_cloud(B, N, seed, frac_unique=0.2, near_origin=True):
    g = torch.Generator().manual_seed(seed)
    U = max(4, int(N * frac_unique))
    base = (torch.rand(B, U, 3, generator=g) - 0.5) * 4
    if near_origin:
        base[:, 0] = 0.01
        base[:, 1] = torch.tensor([0.0316, 0.0, 0.0])  # |p|^2 = 0.00099856 <= 1e-3 -> skipped
    sel = torch.randint(0, U, (B, N), generator=g)
    return torch.gather(base, 1, sel.unsqueeze(-1).expand(-1, -1, 3)).contiguous()


@pytest.mark.parametrize("N,npoint", [(37, 20), (100, 50), (128, 128), (256, 128), (512, 256), (700, 300),
                                      (1024, 512), (2048, 256), (3000, 64), (5000, 32)])
def test_fps_bit_exact_duplicates(N, npoint):
    xyz = dup_cloud(3, N, seed=N)
    got = ops.furthest_point_sampling(xyz.cuda(), npoint).cpu()
    assert torch.equal(got, oops.furthest_point_sampling(xyz, npoint))


def test_fps_random_allzero_and_kitti_shaped():
    g = torch.Generator().manual_seed(0)
    xyz = torch.randn(4, 1024, 3, generator=g)
    assert torch.equal(ops.furthest_point_sampling(xyz.cuda(), 512).cpu(), oops.furthest_point_sampling(xyz, 512))
    z = torch.zeros(2, 512, 3)
    assert ops.furthest_point_sampling(z.cuda(), 64).eq(0).all()
    b = synthetic_siamese_batch(48, 512, 1024, seed=20260924)          # BASELINE configs[1] sizes
    for key, npnt in (("template_points", 256), ("search_points", 512)):
        got = ops.furthest_point_sampling(b[key].cuda(), npnt).cpu()
        assert torch.equal(got, oops.furthest_point_sampling(b[key], npnt)), key


def test_fps_properties_at_full_size():
    # size-independent properties: starts at 0, indices in range, no repeats while unique points remain
    g = torch.Generator().manual_seed(3)
    xyz = torch.rand(64, 1024, 3, generator=g) + 1.0
    idx = ops.furthest_point_sampling(xyz.cuda(), 512).cpu()
    assert idx[:, 0].eq(0).all() and idx.min() >= 0 and idx.max() < 1024
    assert all(len(set(r.tolist())) == 512 for r in idx)


@pytest.mark.parametrize("N,M,r,ns", [(512, 256, 0.3, 32), (1024, 512, 0.3, 32), (256, 128, 0.5, 32),
                                      (128, 64, 0.7, 32), (128, 64, 0.3, 16), (100, 37, 0.4, 5), (1023, 77, 0.25, 64)])
def test_ball_query_bit_exact(N, M, r, ns):
    xyz = dup_cloud(3, N, seed=N + M, frac_unique=0.5, near_origin=False)
    new_xyz = xyz[:, :M].contiguous()
    got = ops.ball_query(new_xyz.cuda(), xyz.cuda(), r, ns).cpu()
    assert torch.equal(got, oops.ball_query(new_xyz, xyz, r, ns))


def test_ball_query_edge_cases():
    xyz = torch.tensor([[[0., 0, 0], [0.5, 0, 0], [1.0, 0, 0], [0.2, 0, 0], [0.9, 0, 0], [100., 0, 0]]])
    new_xyz = torch.tensor([[[0., 0, 0], [50., 0, 0], [100., 0, 0]]])
    idx = ops.ball_query(new_xyz.cuda(), xyz.cuda(), 1.0, 4).cpu()
    assert idx[0].tolist() == [[0, 1, 3, 4], [0, 0, 0, 0], [5, 5, 5, 5]]
    assert ops.ball_query(new_xyz[:, :1].contiguous().cuda(), xyz.cuda(), 0.3, 4).cpu()[0, 0].tolist() == [0, 3, 0, 0]


def test_ball_query_kitti_shaped_full_batch():
    b = synthetic_siamese_batch(48, 512, 1024, seed=5)
    xyz = b["search_points"]
    new_xyz = xyz[:, :512].contiguous()
    got = ops.ball_query(new_xyz.cuda(), xyz.cuda(), 0.3, 32).cpu()
    assert torch.equal(got, oops.ball_query(new_xyz, xyz, 0.3, 32))
    u = synthetic_siamese_batch(8, 512, 1024, seed=6, uniform=True)["search_points"]   # sparse balls -> heavy padding
    got = ops.ball_query(u[:, :512].contiguous().cuda(), u.cuda(), 0.3, 32).cpu()
    assert torch.equal(got, oops.ball_query(u[:, :512].contiguous(), u, 0.3, 32))


def test_gather_group_forward_exact_and_grads():
    g = torch.Generator().manual_seed(1)
    feat = torch.randn(3, 19, 130, generator=g)
    idx = torch.randint(0, 130, (3, 40), generator=g, dtype=torch.int32)
    assert torch.equal(ops.gather_points(feat.cuda(), idx.cuda()).cpu(), oops.gather_points(feat, idx))
    go = torch.randn(3, 19, 40, generator=g)
    assert rel(ops.gather_points_grad(go.cuda(), idx.cuda(), 130), oops.gather_points_grad(go, idx, 130)) < 1e-6
    gidx = torch.randint(0, 130, (3, 21, 7), generator=g, dtype=torch.int32)
    gidx[:, :, 1] = gidx[:, :, 0]                                              # repeated indices
    assert torch.equal(ops.group_points(feat.cuda(), gidx.cuda()).cpu(), oops.group_points(feat, gidx))
    gidx4 = torch.randint(0, 130, (3, 16, 32), generator=g, dtype=torch.int32)  # vectorised path (L % 4 == 0)
    assert torch.equal(ops.group_points(feat.cuda(), gidx4.cuda()).cpu(), oops.group_points(feat, gidx4))
    gg = torch.randn(3, 19, 21, 7, generator=g)
    assert rel(ops.group_points_grad(gg.cuda(), gidx.cuda(), 130), oops.group_points_grad(gg, gidx, 130)) < 1e-6


@pytest.mark.parametrize("n,m", [(64, 2), (100, 3), (512, 128), (1000, 257)])
def test_three_nn_bit_exact(n, m):
    unknown = dup_cloud(2, n, seed=n, frac_unique=0.5, near_origin=False)
    known = dup_cloud(2, m, seed=m, frac_unique=0.5, near_origin=False)
    d2, idx = ops.three_nn(unknown.cuda(), known.cuda())
    wd2, widx = oops.three_nn(unknown, known)
    assert torch.equal(idx.cpu(), widx)
    assert torch.equal(d2.cpu(), wd2)            # same fp32 op order -> identical bits (inf for m < 3)


def test_three_interpolate_and_grad():
    g = torch.Generator().manual_seed(2)
    feat = torch.randn(2, 24, 50, generator=g)
    idx = torch.randint(0, 50, (2, 70, 3), generator=g, dtype=torch.int32)
    w = torch.rand(2, 70, 3, generator=g)
    assert rel(ops.three_interpolate(feat.cuda(), idx.cuda(), w.cuda()), oops.three_interpolate(feat, idx, w)) < 1e-7
    go = torch.randn(2, 24, 70, generator=g)
    assert rel(ops.three_interpolate_grad(go.cuda(), idx.cuda(), w.cuda(), 50),
               oops.three_interpolate_grad(go, idx, w, 50)) < 1e-6


@pytest.mark.parametrize("C,norm", [(0, False), (8, False), (128, False), (256, True)])
def test_fused_ballquery_group_matches_composition(C, norm):
    N, M, S, r = 256, 128, 32, 0.5
    xyz = dup_cloud(2, N, seed=C + 1, frac_unique=0.6, near_origin=False)
    new_xyz = xyz[:, :M].contiguous()
    g = torch.Generator().manual_seed(C)
    feat_cl = torch.randn(2, N, C, generator=g) if C else None
    grouped, idx = ops.ballquery_group(xyz.cuda(), new_xyz.cuda(), feat_cl.cuda() if C else None, r, S, norm)
    widx = oops.ball_query(new_xyz, xyz, r, S)
    assert torch.equal(idx.cpu(), widx)
    gx = oops.group_points(xyz.transpose(1, 2).contiguous(), widx) - new_xyz.transpose(1, 2).unsqueeze(-1)
    if norm:
        gx = gx / r
    grouped = grouped.cpu()
    assert torch.equal(grouped[..., C:C + 3], gx.permute(0, 2, 3, 1))
    assert grouped[..., C + 3].eq(0).all()
    if C:
        gf = oops.group_points(feat_cl.transpose(1, 2).contiguous(), widx)
        assert torch.equal(grouped[..., :C], gf.permute(0, 2, 3, 1))
    # backward: scatter-add to features / xyz / centres
    gg = torch.randn(2, M, S, C + 4, generator=g)
    gf, gxyz, gnew = ops.ballquery_group_grad(gg.cuda(), idx, N, r, norm, need_feat=bool(C), need_xyz=True,
                                              need_new_xyz=True)
    scale = (1.0 / r) if norm else 1.0
    want_xyz = oops.group_points_grad(gg[..., C:C + 3].permute(0, 3, 1, 2).contiguous() * scale, widx, N)
    assert rel(gxyz.cpu().transpose(1, 2), want_xyz) < 1e-5
    assert rel(gnew.cpu(), -(gg[..., C:C + 3] * scale).sum(2)) < 1e-5
    if C:
        want_f = oops.group_points_grad(gg[..., :C].permute(0, 3, 1, 2).contiguous(), widx, N)
        assert rel(gf.cpu().transpose(1, 2), want_f) < 1e-5


def test_fused_three_nn_interpolate():
    unknown = dup_cloud(2, 300, seed=9, frac_unique=0.7, near_origin=False)
    known = dup_cloud(2, 64, seed=10, frac_unique=0.7, near_origin=False)
    g = torch.Generator().manual_seed(4)
    kf = torch.randn(2, 64, 32, generator=g)
    out, idx, w = ops.three_nn_interpolate(unknown.cuda(), known.cuda(), kf.cuda())
    d2, widx = oops.three_nn(unknown, known)
    assert torch.equal(idx.cpu(), widx)
    r = 1.0 / (torch.sqrt(d2) + 1e-8)
    ww = r / r.sum(2, keepdim=True)
    assert rel(w, ww) < 1e-6
    want = oops.three_interpolate(kf.transpose(1, 2).contiguous(), widx, ww)
    assert rel(out.cpu().transpose(1, 2), want) < 1e-6
    go = torch.randn(2, 300, 32, generator=g)
    gk = ops.three_nn_interpolate_grad(go.cuda(), idx, w, 64)
    want_g = oops.three_interpolate_grad(go.transpose(1, 2).contiguous(), widx, ww, 64)
    assert rel(gk.cpu().transpose(1, 2), want_g) < 1e-5


def test_wrong_dtype_or_layout_raises():
    x = torch.zeros(1, 8, 3, device="cuda")
    with pytest.raises(RuntimeError, match="contiguous"):
        ops.furthest_point_sampling(x.transpose(1, 2).transpose(1, 2)[:, ::2], 2)
    with pytest.raises(RuntimeError, match="float"):
        ops.furthest_point_sampling(x.double(), 2)
    with pytest.raises(RuntimeError, match="int"):
        ops.gather_points(torch.zeros(1, 2, 8, device="cuda"), torch.zeros(1, 3, device="cuda", dtype=torch.int64))


def test_kernels_are_cuda_graph_capturable():
    xyz = dup_cloud(2, 512, seed=1).cuda()
    want = ops.furthest_point_sampling(xyz, 64)
    out = torch.empty_like(want)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            tmp = ops.furthest_point_sampling(xyz, 64)
            bq = ops.ball_query(xyz[:, :64].contiguous(), xyz, 0.5, 16)
            out.copy_(tmp)
        g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, want) and bq.shape == (2, 64, 16)
