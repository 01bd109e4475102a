"""M2-Track (motion-centric tracker).  Mirror of models/m2track.py: __init__ (:17-71), forward (:73-151),
compute_loss (:153-231), training_step (:233-266).  No pointnet2 ops: a per-point segmentation net over the stacked
2 x point_sample_size cloud, a global-feature net, four small MLP heads and closed-form box transforms.  The dense
per-point stacks run on the same fused point-wise kernels as the SA layers (fused.seq_forward); metric objects
(torchmetrics Accuracy) of the reference are logging-only and omitted."""
import torch
import torch.nn.functional as F
from torch import nn

from . import base_model
from .backbone.pointnet import MiniPointNet, SegPointNet
from ..datasets import points_utils
from .. import runtime


def _head(out_dim):
    return nn.Sequential(nn.Linear(256, 128), nn.BatchNorm1d(128), nn.ReLU(), nn.Linear(128, 128), nn.BatchNorm1d(128),
                         nn.ReLU(), nn.Linear(128, out_dim))


class M2TRACK(base_model.MotionBaseModel):
    def __init__(self, config, **kwargs):
        super().__init__(config, **kwargs)
        self.box_aware = getattr(config, 'box_aware', False)
        self.use_motion_cls = getattr(config, 'use_motion_cls', True)
        self.use_second_stage = getattr(config, 'use_second_stage', True)
        self.use_prev_refinement = getattr(config, 'use_prev_refinement', True)
        bc = 9 if self.box_aware else 0
        self.seg_pointnet = SegPointNet(input_channel=3 + 1 + 1 + bc, per_point_mlp1=[64, 64, 64, 128, 1024],
                                        per_point_mlp2=[512, 256, 128, 128], output_size=2 + bc)
        self.mini_pointnet = MiniPointNet(input_channel=3 + 1 + bc, per_point_mlp=[64, 128, 256, 512],
                                          hidden_mlp=[512, 256], output_size=-1)
        if self.use_second_stage:
            self.mini_pointnet2 = MiniPointNet(input_channel=3 + bc, per_point_mlp=[64, 128, 256, 512],
                                               hidden_mlp=[512, 256], output_size=-1)
            self.box_mlp = _head(4)
        if self.use_prev_refinement:
            self.final_mlp = _head(4)
        if self.use_motion_cls:
            self.motion_state_mlp = _head(2)
        self.motion_mlp = _head(4)

    def _mlp(self, module, x):
        """(B,256) -> head output, on the fused kernels when enabled."""
        if runtime.fused_enabled() and x.is_cuda:
            from .. import fused
            return fused.rows_forward(module, x)
        return module(x)

    def forward(self, input_dict):
        """input_dict: points (B,N,3+1+1) = [xyz, timestamp, prior mask], candidate_bc (B,N,9) -> dict with boxes (B,4)."""
        output_dict = {}
        x = input_dict["points"].transpose(1, 2)
        if self.box_aware:
            x = torch.cat([x, input_dict["candidate_bc"].transpose(1, 2)], dim=1)
        B, _, N = x.shape

        seg_out = self.seg_pointnet(x)
        seg_logits = seg_out[:, :2, :]
        # the point mask and the motion state are arg-max decisions on computed logits: routed through runtime.choose so that a
        # parity test can hold them fixed (a no-op otherwise)
        pred_cls = runtime.choose("m2_segment", {"N": N}, lambda: torch.argmax(seg_logits, dim=1, keepdim=True))   # (B,1,N)
        mask_points = x[:, :4, :] * pred_cls
        mask_xyz_t0 = mask_points[:, :3, :N // 2]
        mask_xyz_t1 = mask_points[:, :3, N // 2:]
        if self.box_aware:
            pred_bc = seg_out[:, 2:, :]
            mask_pred_bc = pred_bc * pred_cls
            mask_points = torch.cat([mask_points, mask_pred_bc], dim=1)
            output_dict['pred_bc'] = pred_bc.transpose(1, 2)

        point_feature = self.mini_pointnet(mask_points)

        motion_pred = self._mlp(self.motion_mlp, point_feature)                       # (B,4)
        if self.use_motion_cls:
            motion_state_logits = self._mlp(self.motion_state_mlp, point_feature)     # (B,2)
            motion_mask = runtime.choose("m2_motion_state", {}, lambda: torch.argmax(motion_state_logits, dim=1, keepdim=True))
            motion_pred_masked = motion_pred * motion_mask
            output_dict['motion_cls'] = motion_state_logits
        else:
            motion_pred_masked = motion_pred
        if self.use_prev_refinement:
            prev_boxes = self._mlp(self.final_mlp, point_feature)
            output_dict["estimation_boxes_prev"] = prev_boxes[:, :4]
        else:
            prev_boxes = torch.zeros_like(motion_pred)

        aux_box = points_utils.get_offset_box_tensor(prev_boxes, motion_pred_masked)  # 1st-stage prediction

        if self.use_second_stage:
            moved = points_utils.get_offset_points_tensor(mask_xyz_t0.transpose(1, 2), prev_boxes[:, :4],
                                                          motion_pred_masked).transpose(1, 2)
            mask_xyz_t01 = torch.cat([moved, mask_xyz_t1], dim=-1)                   # (B,3,N)
            mask_xyz_t01 = points_utils.remove_transform_points_tensor(mask_xyz_t01.transpose(1, 2), aux_box).transpose(1, 2)
            if self.box_aware:
                mask_xyz_t01 = torch.cat([mask_xyz_t01, mask_pred_bc], dim=1)
            output_offset = self._mlp(self.box_mlp, self.mini_pointnet2(mask_xyz_t01))
            output_dict["estimation_boxes"] = points_utils.get_offset_box_tensor(aux_box, output_offset)
        else:
            output_dict["estimation_boxes"] = aux_box
        output_dict.update({"seg_logits": seg_logits, "motion_pred": motion_pred, 'aux_estimation_boxes': aux_box})
        return output_dict

    def compute_loss(self, data, output):
        c = self.config
        loss_total = 0.0
        loss_dict = {}
        aux_boxes, motion_pred, seg_logits = output['aux_estimation_boxes'], output['motion_pred'], output['seg_logits']
        with torch.no_grad():
            seg_label = data['seg_label']
            box_label, box_label_prev, motion_label = data['box_label'], data['box_label_prev'], data['motion_label']
            motion_state_label = data['motion_state_label']
            center_label, angle_label = box_label[:, :3], torch.sin(box_label[:, 3])
            center_label_prev, angle_label_prev = box_label_prev[:, :3], torch.sin(box_label_prev[:, 3])
            center_label_motion, angle_label_motion = motion_label[:, :3], torch.sin(motion_label[:, 3])
            seg_w = torch.stack([torch.full((), 0.5, device=seg_logits.device), torch.full((), 2.0, device=seg_logits.device)])

        loss_seg = F.cross_entropy(seg_logits, seg_label, weight=seg_w)
        if self.use_motion_cls:
            loss_motion_cls = F.cross_entropy(output['motion_cls'], motion_state_label)
            loss_total = loss_total + loss_motion_cls * c.motion_cls_seg_weight
            loss_dict['loss_motion_cls'] = loss_motion_cls
            lcm = F.smooth_l1_loss(motion_pred[:, :3], center_label_motion, reduction='none')
            loss_center_motion = (motion_state_label * lcm.mean(dim=1)).sum() / (motion_state_label.sum() + 1e-6)
            lam = F.smooth_l1_loss(torch.sin(motion_pred[:, 3]), angle_label_motion, reduction='none')
            loss_angle_motion = (motion_state_label * lam).sum() / (motion_state_label.sum() + 1e-6)
        else:
            loss_center_motion = F.smooth_l1_loss(motion_pred[:, :3], center_label_motion)
            loss_angle_motion = F.smooth_l1_loss(torch.sin(motion_pred[:, 3]), angle_label_motion)

        if self.use_second_stage:
            boxes = output['estimation_boxes']
            loss_center = F.smooth_l1_loss(boxes[:, :3], center_label)
            loss_angle = F.smooth_l1_loss(torch.sin(boxes[:, 3]), angle_label)
            loss_total = loss_total + loss_center * c.center_weight + loss_angle * c.angle_weight
            loss_dict["loss_center"], loss_dict["loss_angle"] = loss_center, loss_angle
        if self.use_prev_refinement:
            prev = output['estimation_boxes_prev']
            loss_center_prev = F.smooth_l1_loss(prev[:, :3], center_label_prev)
            loss_angle_prev = F.smooth_l1_loss(torch.sin(prev[:, 3]), angle_label_prev)
            loss_total = loss_total + loss_center_prev * c.center_weight + loss_angle_prev * c.angle_weight
            loss_dict["loss_center_prev"], loss_dict["loss_angle_prev"] = loss_center_prev, loss_angle_prev

        loss_center_aux = F.smooth_l1_loss(aux_boxes[:, :3], center_label)
        loss_angle_aux = F.smooth_l1_loss(torch.sin(aux_boxes[:, 3]), angle_label)
        loss_total = (loss_total + loss_seg * c.seg_weight
                      + loss_center_aux * c.center_weight + loss_angle_aux * c.angle_weight
                      + loss_center_motion * c.center_weight + loss_angle_motion * c.angle_weight)
        loss_dict.update({"loss_total": loss_total, "loss_seg": loss_seg, "loss_center_aux": loss_center_aux,
                          "loss_center_motion": loss_center_motion, "loss_angle_aux": loss_angle_aux,
                          "loss_angle_motion": loss_angle_motion})
        if self.box_aware:
            bc_label = torch.cat([data['prev_bc'], data['this_bc']], dim=1)
            loss_bc = F.smooth_l1_loss(output['pred_bc'], bc_label)
            loss_total = loss_total + loss_bc * c.bc_weight
            loss_dict.update({"loss_total": loss_total, "loss_bc": loss_bc})
        return loss_dict

    def training_step(self, batch, batch_idx):
        output = self(batch)
        loss_dict = self.compute_loss(batch, output)
        for k, v in loss_dict.items():
            self.log(f'{k}/train', v.detach(), on_step=True, on_epoch=True, prog_bar=False, logger=True)
        return loss_dict['loss_total']
