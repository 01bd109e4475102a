"""PointNet++ primitives with the reference's names, signatures and return conventions.

Mirror of pointnet2/utils/pointnet2_utils.py: FurthestPointSampling (:35-65), GatherOperation (:68-102),
ThreeNN (:105-134), ThreeInterpolate (:137-191), GroupingOperation (:194-242), BallQuery (:245-277),
QueryAndGroup (:280-339), GroupAll (:342-385), knn_point (:388-402).  Every op dispatches to the sm_90a
kernels behind the C ABI (open3dsot_b200._ext == the `pointnet2_ops._ext` call surface); there is no
PyTorch or CPU fallback — CPU tensors raise RuntimeError exactly like upstream ("CPU not supported").
"""
import torch
import torch.nn as nn
from torch.autograd import Function

from ... import _ext
from ... import ops as _ops


class FurthestPointSampling(Function):
    @staticmethod
    def forward(ctx, xyz, npoint):
        """xyz (B,N,3) f32, npoint -> (B,npoint) i32; non-differentiable."""
        inds = _ext.furthest_point_sampling(xyz, npoint)
        ctx.mark_non_differentiable(inds)
        return inds

    @staticmethod
    def backward(ctx, a=None):
        return None, None


furthest_point_sample = FurthestPointSampling.apply


class GatherOperation(Function):
    @staticmethod
    def forward(ctx, features, idx):
        """features (B,C,N), idx (B,npoint) i32 -> (B,C,npoint)."""
        ctx.for_backwards = (idx, features.size(1), features.size(2))
        return _ext.gather_points(features, idx)

    @staticmethod
    def backward(ctx, grad_out):
        idx, C, N = ctx.for_backwards
        return _ext.gather_points_grad(grad_out.contiguous(), idx, N), None


gather_operation = GatherOperation.apply


class ThreeNN(Function):
    @staticmethod
    def forward(ctx, unknown, known):
        """unknown (B,n,3), known (B,m,3) -> dist (B,n,3) (square-rooted), idx (B,n,3) i32."""
        dist2, idx = _ext.three_nn(unknown, known)
        ctx.mark_non_differentiable(idx)
        return torch.sqrt(dist2), idx

    @staticmethod
    def backward(ctx, a=None, b=None):
        return None, None


three_nn = ThreeNN.apply


class ThreeInterpolate(Function):
    @staticmethod
    def forward(ctx, features, idx, weight):
        """features (B,c,m), idx (B,n,3), weight (B,n,3) -> (B,c,n)."""
        ctx.three_interpolate_for_backward = (idx, weight, features.size(2))
        return _ext.three_interpolate(features, idx, weight)

    @staticmethod
    def backward(ctx, grad_out):
        idx, weight, m = ctx.three_interpolate_for_backward
        return _ext.three_interpolate_grad(grad_out.contiguous(), idx, weight, m), None, None


three_interpolate = ThreeInterpolate.apply


class GroupingOperation(Function):
    @staticmethod
    def forward(ctx, features, idx):
        """features (B,C,N), idx (B,npoint,nsample) i32 -> (B,C,npoint,nsample)."""
        ctx.for_backwards = (idx, features.size(2))
        return _ext.group_points(features, idx)

    @staticmethod
    def backward(ctx, grad_out):
        idx, N = ctx.for_backwards
        return _ext.group_points_grad(grad_out.contiguous(), idx, N), None


grouping_operation = GroupingOperation.apply


class BallQuery(Function):
    @staticmethod
    def forward(ctx, radius, nsample, xyz, new_xyz):
        """radius, nsample, xyz (B,N,3), new_xyz (B,npoint,3) -> (B,npoint,nsample) i32; non-differentiable."""
        inds = _ext.ball_query(new_xyz, xyz, radius, nsample)
        ctx.mark_non_differentiable(inds)
        return inds

    @staticmethod
    def backward(ctx, a=None):
        return None, None, None, None


ball_query = BallQuery.apply


class _QueryAndGroupCL(Function):
    """Fused QueryAndGroup on channels-last features: one kernel forward, one backward."""

    @staticmethod
    def forward(ctx, xyz, new_xyz, feat_cl, radius, nsample, normalize_xyz):
        grouped, idx = _ops.ballquery_group(xyz, new_xyz, feat_cl, radius, nsample, normalize_xyz)
        ctx.save_for_backward(idx)
        ctx.cfg = (xyz.shape[1], radius, normalize_xyz, feat_cl is not None)
        ctx.mark_non_differentiable(idx)
        return grouped, idx

    @staticmethod
    def backward(ctx, g_grouped, _g_idx):
        (idx,) = ctx.saved_tensors
        N, radius, normalize_xyz, has_feat = ctx.cfg
        need = ctx.needs_input_grad
        gf, gx, gn = _ops.ballquery_group_grad(g_grouped.contiguous(), idx, N, radius, normalize_xyz,
                                               need_feat=has_feat and need[2], need_xyz=need[0], need_new_xyz=need[1])
        return gx, gn, gf, None, None, None


def query_and_group_cl(xyz, new_xyz, feat_cl, radius, nsample, normalize_xyz=False):
    """(B,N,3),(B,M,3),(B,N,C)|None -> grouped (B,M,S,C+4) = [features | dx dy dz 0], idx (B,M,S)."""
    return _QueryAndGroupCL.apply(xyz, new_xyz, feat_cl, radius, nsample, normalize_xyz)


class QueryAndGroup(nn.Module):
    """Ball-query grouping; returns (B, 3+C, npoint, nsample) with channel order [xyz, features]."""

    def __init__(self, radius, nsample, use_xyz=True, return_idx=False, normalize_xyz=False):
        super().__init__()
        self.radius, self.nsample, self.use_xyz = radius, nsample, use_xyz
        self.return_idx = return_idx
        self.normalize_xyz = normalize_xyz

    def forward(self, xyz, new_xyz, features=None):
        idx = ball_query(self.radius, self.nsample, xyz, new_xyz)
        xyz_trans = xyz.transpose(1, 2).contiguous()
        grouped_xyz = grouping_operation(xyz_trans, idx) - new_xyz.transpose(1, 2).unsqueeze(-1)
        if self.normalize_xyz:
            grouped_xyz = grouped_xyz / self.radius
        if features is not None:
            new_features = grouping_operation(features.contiguous(), idx)
            if self.use_xyz:
                new_features = torch.cat([grouped_xyz, new_features], dim=1)
        else:
            assert self.use_xyz, "Cannot have not features and not use xyz as a feature!"
            new_features = grouped_xyz
        if self.return_idx:
            return new_features, idx
        return new_features


class GroupAll(nn.Module):
    """Groups every point into one set: (B, 3+C, 1, N)."""

    def __init__(self, use_xyz=True):
        super().__init__()
        self.use_xyz = use_xyz

    def forward(self, xyz, new_xyz, features=None):
        grouped_xyz = xyz.transpose(1, 2).unsqueeze(2)
        if features is None:
            return grouped_xyz
        grouped_features = features.unsqueeze(2)
        return torch.cat([grouped_xyz, grouped_features], dim=1) if self.use_xyz else grouped_features


def knn_point(k, points1, points2):
    """k nearest points of points2 (B,n2,d) for every point of points1 (B,n1,d) -> (B,n1,k) i32."""
    dist_matrix = torch.cdist(points1, points2)
    return torch.argsort(dist_matrix, dim=-1)[:, :, :k].int().contiguous()
