"""PointNet++ set-abstraction / feature-propagation modules with the reference's constructor and
forward signatures.

Mirror of pointnet2/utils/pointnet2_modules.py: _PointnetSAModuleBase.forward (:31-79),
PointnetSAModuleMSG (:82-117), PointnetSAModule (:120-149), PointnetFPModule (:152-212).
(FlowEmbedding / PointNetSetUpConv, :215-334, are unused by every model and broken upstream; they are kept
importable as thin compositions of the same primitives.)

Two execution modes, both on the sm_90a kernels (there is no CPU path):
  * fused   (default) — open3dsot_b200.fused: ball-query + gather feed the point-wise MLP kernels directly
              (channels-last activations, BN statistics and max-pool in the GEMM epilogues);
  * composed — the reference's op-by-op composition over the nine `_ext` kernels + torch conv/BN, kept as
              the on-device cross-check of the fused path (tests/test_gpu_modules.py).
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import pointnet2_utils
from . import pytorch_utils as pt_utils
from ... import runtime


class _PointnetSAModuleBase(nn.Module):
    def __init__(self, use_fps=False):
        super().__init__()
        self.groupers = None
        self.mlps = None
        self.use_fps = use_fps

    def forward(self, xyz, features, npoint, return_idx=False, sample_idxs=None):
        """xyz (B,N,3), features (B,C,N)|None -> new_xyz (B,npoint,3), new_features (B,sum C_out,npoint)
        [, sample_idxs (B,npoint) i32].  `sample_idxs` (extension): centre indices computed ahead of time (e.g. FPS
        overlapped with other work on a side stream); must equal what this layer would compute itself."""
        self.npoint = npoint
        if sample_idxs is not None:
            pass
        elif self.use_fps:
            sample_idxs = pointnet2_utils.furthest_point_sample(xyz, self.npoint)
        else:
            sample_idxs = torch.arange(self.npoint, dtype=torch.int32, device=xyz.device).repeat(xyz.size(0), 1)

        if runtime.fused_enabled():
            from ... import fused
            new_xyz, outs = fused.sa_forward(self, xyz, features, sample_idxs)
        else:
            xyz_flipped = xyz.transpose(1, 2).contiguous()
            new_xyz = pointnet2_utils.gather_operation(xyz_flipped, sample_idxs).transpose(1, 2).contiguous()
            outs = []
            for grouper, mlp in zip(self.groupers, self.mlps):
                new_features = mlp(grouper(xyz, new_xyz, features))           # (B, C_out, npoint, nsample)
                new_features = F.max_pool2d(new_features, kernel_size=[1, new_features.size(3)]).squeeze(-1)
                outs.append(new_features)
        new_features = outs[0] if len(outs) == 1 else torch.cat(outs, dim=1)
        if return_idx:
            return new_xyz, new_features, sample_idxs
        return new_xyz, new_features


class PointnetSAModuleMSG(_PointnetSAModuleBase):
    """Set abstraction with multi-scale grouping.  Like the reference, `mlps[i][0]` is incremented in place
    by 3 when `use_xyz` (callers' lists are mutated, pointnet2_modules.py:113-115)."""

    def __init__(self, radii, nsamples, mlps, bn=True, use_xyz=True, use_fps=False, normalize_xyz=False):
        super().__init__(use_fps=use_fps)
        assert len(radii) == len(nsamples) == len(mlps)
        self.groupers = nn.ModuleList()
        self.mlps = nn.ModuleList()
        for radius, nsample, mlp_spec in zip(radii, nsamples, mlps):
            self.groupers.append(
                pointnet2_utils.QueryAndGroup(radius, nsample, use_xyz=use_xyz, normalize_xyz=normalize_xyz))
            if use_xyz:
                mlp_spec[0] += 3
            self.mlps.append(pt_utils.SharedMLP(mlp_spec, bn=bn))


class PointnetSAModule(PointnetSAModuleMSG):
    """Single-scale set abstraction."""

    def __init__(self, mlp, radius=None, nsample=None, bn=True, use_xyz=True, use_fps=False, normalize_xyz=False):
        super().__init__(mlps=[mlp], radii=[radius], nsamples=[nsample], bn=bn, use_xyz=use_xyz, use_fps=use_fps,
                         normalize_xyz=normalize_xyz)


class PointnetFPModule(nn.Module):
    """Feature propagation: 3-NN inverse-distance interpolation (+ skip features) -> SharedMLP."""

    def __init__(self, mlp, bn=True):
        super().__init__()
        self.mlp = pt_utils.SharedMLP(mlp, bn=bn)

    def forward(self, unknown, known, unknow_feats, known_feats):
        """unknown (B,n,3), known (B,m,3), unknow_feats (B,C1,n)|None, known_feats (B,C2,m) -> (B,mlp[-1],n)."""
        if runtime.fused_enabled() and known is not None:
            from ... import fused
            return fused.fp_forward(self, unknown, known, unknow_feats, known_feats)
        if known is not None:
            dist, idx = pointnet2_utils.three_nn(unknown, known)
            dist_recip = 1.0 / (dist + 1e-8)
            weight = dist_recip / torch.sum(dist_recip, dim=2, keepdim=True)
            interpolated_feats = pointnet2_utils.three_interpolate(known_feats.contiguous(), idx, weight)
        else:
            interpolated_feats = known_feats.expand(*(list(known_feats.size()[0:2]) + [unknown.size(1)]))
        new_features = interpolated_feats if unknow_feats is None else torch.cat([interpolated_feats, unknow_feats], 1)
        return self.mlp(new_features.unsqueeze(-1)).squeeze(-1)


class FlowEmbedding(nn.Module):
    """Unused by BAT/P2B/M2-Track (pointnet2_modules.py:215-269); knn grouping + concat correlation + MLP + pool."""

    def __init__(self, radius, nsample, in_channel, mlp, pooling='max', corr_func='concat', knn=True):
        super().__init__()
        self.radius, self.nsample, self.knn, self.pooling, self.corr_func = radius, nsample, knn, pooling, corr_func
        self.mlp_convs, self.mlp_bns = nn.ModuleList(), nn.ModuleList()
        last_channel = in_channel * 2 + 3
        for out_channel in mlp:
            self.mlp_convs.append(nn.Conv2d(last_channel, out_channel, 1, bias=False))
            self.mlp_bns.append(nn.BatchNorm2d(out_channel))
            last_channel = out_channel

    def _group_idx(self, query, support):
        if self.knn:
            return pointnet2_utils.knn_point(self.nsample, query, support)
        return pointnet2_utils.ball_query(self.radius, self.nsample, support.contiguous(), query.contiguous())

    def forward(self, xyz1, xyz2, feature1, feature2):
        B, N, _ = xyz1.shape
        idx = self._group_idx(xyz1, xyz2)
        pos_diff = pointnet2_utils.grouping_operation(xyz2.transpose(1, 2).contiguous(), idx) \
            - xyz1.transpose(1, 2).unsqueeze(-1)
        feat2_grouped = pointnet2_utils.grouping_operation(feature2.contiguous(), idx)
        feat = torch.cat([pos_diff, feat2_grouped, feature1.unsqueeze(-1).expand(-1, -1, -1, self.nsample)], dim=1)
        for conv, bn in zip(self.mlp_convs, self.mlp_bns):
            feat = F.relu(bn(conv(feat)))
        return xyz1, feat.max(dim=-1)[0]


class PointNetSetUpConv(nn.Module):
    """Unused by BAT/P2B/M2-Track (pointnet2_modules.py:272-334)."""

    def __init__(self, nsample, radius, f1_channel, f2_channel, mlp, mlp2, knn=True):
        super().__init__()
        self.nsample, self.radius, self.knn = nsample, radius, knn
        self.mlp1_convs, self.mlp2_convs = nn.ModuleList(), nn.ModuleList()
        last_channel = f2_channel + 3
        for out_channel in mlp:
            self.mlp1_convs.append(nn.Sequential(nn.Conv2d(last_channel, out_channel, 1, bias=False),
                                                 nn.BatchNorm2d(out_channel), nn.ReLU(inplace=False)))
            last_channel = out_channel
        last_channel = (mlp[-1] if len(mlp) else last_channel) + f1_channel
        for out_channel in mlp2:
            self.mlp2_convs.append(nn.Sequential(nn.Conv1d(last_channel, out_channel, 1, bias=False),
                                                 nn.BatchNorm1d(out_channel), nn.ReLU(inplace=False)))
            last_channel = out_channel

    def forward(self, xyz1, xyz2, feature1, feature2):
        if self.knn:
            idx = pointnet2_utils.knn_point(self.nsample, xyz1, xyz2)
        else:
            idx = pointnet2_utils.ball_query(self.radius, self.nsample, xyz2.contiguous(), xyz1.contiguous())
        pos_diff = pointnet2_utils.grouping_operation(xyz2.transpose(1, 2).contiguous(), idx) \
            - xyz1.transpose(1, 2).unsqueeze(-1)
        feat = torch.cat([pointnet2_utils.grouping_operation(feature2.contiguous(), idx), pos_diff], dim=1)
        for conv in self.mlp1_convs:
            feat = conv(feat)
        feat = feat.max(dim=-1)[0]
        if feature1 is not None:
            feat = torch.cat([feat, feature1], dim=1)
        for conv in self.mlp2_convs:
            feat = conv(feat)
        return feat
