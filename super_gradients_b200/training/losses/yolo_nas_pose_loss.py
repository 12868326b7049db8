"""YoloNASPoseLoss (reference: training/losses/yolo_nas_pose_loss.py:280-682) on the sm_90a path.

forward(outputs, targets) -> (loss, log_items[6] = cls, iou, dfl, pose_cls, pose_reg, total) with the reference's
semantics: OKS-aware task-aligned assigner with crowd handling, focal / BCE person classification normalised by
max(sum(assigned_scores), 1), CIoU / GIoU + DFL on the positive anchors, OKS keypoint regression and joint-visibility
classification (optionally rescaled by the assigned score).  The flat targets are padded on the host to a FIXED n_max
(static shapes, CUDA-graph friendly); the assigner (4 small kernels) and the fused forward+backward (1 kernel) replace the
reference's eager graph.
"""
from typing import List, Tuple, Union

import numpy as np
import torch
from torch import Tensor, nn

from ... import kernels as K
from ...common.registry import register_loss
from .ppyolo_loss import host_out


def _same_instances(img, joints, crowd):
    # the reference selects boxes, joints and crowd flags per image by THEIR OWN image index column, in order
    j_img, c_img = joints[:, 0, 0].astype(np.int64), crowd[:, 0].astype(np.int64)
    if not (np.array_equal(j_img, img) and np.array_equal(c_img, img)):
        raise ValueError("boxes, joints and crowd rows must describe the same instances in the same order")


def max_pose_targets_host(targets: Tuple[Tensor, Tensor, Tensor]) -> int:
    """Largest number of instances one image of the batch holds: (boxes [N, 5], joints [N, J, 4], crowd [N, 2]) host targets, each
    with the image index first, numpy only.  Raises ValueError as pad_pose_targets_host does when the three disagree."""
    boxes, joints, crowd = (t.detach().float().numpy() for t in targets)
    if not boxes.shape[0]:
        return 0
    img = boxes[:, 0].astype(np.int64)
    _same_instances(img, joints, crowd)
    return int(np.bincount(img).max())


def pad_pose_targets_host(targets: Tuple[Tensor, Tensor, Tensor], batch_size: int, n_max: int, out=None) -> Tuple[Tensor, Tensor, Tensor, Tensor]:
    """(boxes [N, 5] = img, x1, y1, x2, y2; joints [N, J, 4] = img, x, y, visibility; crowd [N, 2] = img, is_crowd) ->
    gt_boxes [B, n_max, 4], gt_poses [B, n_max, J, 3], gt_crowd [B, n_max] uint8, gt_valid [B, n_max] uint8
    (YoloNASPoseLoss._unpack_flat_targets, yolo_nas_pose_loss.py:343-401).  Instances keep their order within an image.
    out: caller-owned host tensors of those shapes and dtypes, written (and returned) instead of new ones."""
    boxes, joints, crowd = (t.detach().float().cpu().numpy() for t in targets)
    J = joints.shape[1]
    gt_boxes, gt_poses, gt_crowd, gt_valid = host_out(out, (((batch_size, n_max, 4), np.float32), ((batch_size, n_max, J, 3), np.float32),
                                                            ((batch_size, n_max), np.uint8), ((batch_size, n_max), np.uint8)))  # fmt: skip
    if boxes.shape[0]:
        img = boxes[:, 0].astype(np.int64)
        order = np.argsort(img, kind="stable")
        first = np.searchsorted(img[order], np.arange(batch_size))
        slot = np.empty_like(img)
        slot[order] = np.arange(img.shape[0]) - first[img[order]]
        if slot.max() >= n_max:
            raise ValueError(f"an image has {slot.max() + 1} instances but n_max={n_max}")
        _same_instances(img, joints, crowd)
        gt_boxes[img, slot] = boxes[:, 1:5]
        gt_poses[img, slot] = joints[:, :, 1:4]
        gt_crowd[img, slot] = (crowd[:, 1] != 0).astype(np.uint8)
        gt_valid[img, slot] = (boxes[:, 1:5].sum(1) > 0).astype(np.uint8)
    return tuple(out) if out is not None else (torch.from_numpy(gt_boxes), torch.from_numpy(gt_poses), torch.from_numpy(gt_crowd), torch.from_numpy(gt_valid))


class _FusedPoseLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, cls_logits, reg_distri, pose_coords, pose_logits, anchor_points, stride_tensor, gt_boxes, gt_poses, gt_crowd, gt_valid, sigmas, desc, sync):
        cls_logits, reg_distri = cls_logits.contiguous().float(), reg_distri.contiguous().float()
        pose_coords, pose_logits = pose_coords.contiguous().float(), pose_logits.contiguous().float()
        sums = torch.zeros(8, dtype=torch.float64, device=cls_logits.device)
        agt, asc = K.pose_tal_assign(desc, cls_logits, reg_distri, pose_coords, anchor_points, stride_tensor, gt_boxes, gt_poses, gt_crowd, gt_valid, sigmas, sums)
        if sync:
            import torch.distributed as dist

            dist.all_reduce(sums[3:4])
            sums[3:4] /= dist.get_world_size()
        items, gc, gr, gp, gl = K.pose_loss(desc, cls_logits, reg_distri, pose_coords, pose_logits, anchor_points, stride_tensor, gt_boxes, gt_poses, sigmas, agt, asc, sums)
        ctx.save_for_backward(gc, gr, gp, gl)
        ctx.mark_non_differentiable(items)
        return items[5].clone(), items

    @staticmethod
    def backward(ctx, gloss, _gitems):
        gc, gr, gp, gl = ctx.saved_tensors
        return (gc * gloss, gr * gloss, gp * gloss, gl * gloss) + (None,) * 9


@register_loss(name="YoloNASPoseLoss")
class YoloNASPoseLoss(nn.Module):
    def __init__(
        self,
        oks_sigmas: Union[List[float], np.ndarray, Tensor],
        classification_loss_type: str = "focal",
        regression_iou_loss_type: str = "ciou",
        classification_loss_weight: float = 1.0,
        iou_loss_weight: float = 2.5,
        dfl_loss_weight: float = 0.5,
        pose_cls_loss_weight: float = 1.0,
        pose_reg_loss_weight: float = 1.0,
        pose_classification_loss_type: str = "bce",
        bbox_assigner_topk: int = 13,
        bbox_assigned_alpha: float = 1.0,
        bbox_assigned_beta: float = 6.0,
        assigner_multiply_by_pose_oks: bool = False,
        rescale_pose_loss_with_assigned_score: bool = False,
        average_losses_in_ddp: bool = False,
        max_targets_per_image: int = 0,
    ):
        super().__init__()
        self.cls_type = {"focal": 0, "bce": 1}[classification_loss_type]
        self.iou_type = {"giou": 0, "ciou": 1}[regression_iou_loss_type]
        self.pose_cls_type = {"bce": 0, "focal": 1}[pose_classification_loss_type]
        self.classification_loss_type = classification_loss_type
        self.pose_classification_loss_type = pose_classification_loss_type
        self.classification_loss_weight = classification_loss_weight
        self.iou_loss_weight = iou_loss_weight
        self.dfl_loss_weight = dfl_loss_weight
        self.pose_cls_loss_weight = pose_cls_loss_weight
        self.pose_reg_loss_weight = pose_reg_loss_weight
        self.num_keypoints = len(oks_sigmas)
        self.num_classes = 1  # one class (person) in the pose task
        self.register_buffer("oks_sigmas", torch.as_tensor(oks_sigmas, dtype=torch.float32).clone(), persistent=False)
        self.topk, self.alpha, self.beta = bbox_assigner_topk, bbox_assigned_alpha, bbox_assigned_beta
        self.assigner_multiply_by_pose_oks = assigner_multiply_by_pose_oks
        self.rescale_pose_loss_with_assigned_score = rescale_pose_loss_with_assigned_score
        self.average_losses_in_ddp = average_losses_in_ddp
        self.max_targets_per_image = max_targets_per_image
        self._n_max = max_targets_per_image

    @property
    def component_names(self):
        return ["loss_cls", "loss_iou", "loss_dfl", "loss_pose_cls", "loss_pose_reg", "loss"]

    # The padded-target interface of the captured train step (sg_trainer.TrainStep.run_padded)
    def max_targets(self, targets) -> int:
        return max_pose_targets_host(targets)

    def pad_targets(self, targets, batch_size: int, n_max: int, out=None) -> Tuple[Tensor, Tensor, Tensor, Tensor]:
        return pad_pose_targets_host(targets, batch_size, n_max, out)

    def forward(self, outputs, targets) -> Tuple[Tensor, Tensor]:
        _, predictions = outputs
        cls_logits, reg_distri, pose_coords, pose_logits, _anchors, anchor_points, _num_anchors_list, stride_tensor = predictions
        K.require_cuda(cls_logits, "predictions")
        B, L, _ = cls_logits.shape
        J = pose_logits.shape[-1]
        if J != self.num_keypoints:
            raise ValueError(f"the model predicts {J} joints but the loss was built with {self.num_keypoints} oks_sigmas")
        reg_max = reg_distri.shape[-1] // 4 - 1
        dev = cls_logits.device
        if len(targets) == 4:  # already padded on the device: (gt_boxes, gt_poses, gt_crowd, gt_valid)
            gt_boxes, gt_poses, gt_crowd, gt_valid = targets
            n_max = gt_boxes.shape[1]
        else:
            boxes = targets[0]
            counts = torch.bincount(boxes[:, 0].long().cpu(), minlength=B) if boxes.numel() else torch.zeros(B, dtype=torch.long)
            self._n_max = max(self._n_max, int(counts.max()) if boxes.numel() else 0)  # grow-only: static shapes across steps
            n_max = self._n_max
            padded = pad_pose_targets_host(targets, B, max(n_max, 1))
            gt_boxes, gt_poses, gt_crowd, gt_valid = (t.to(dev, non_blocking=True) for t in padded)
        desc = K.pose_loss_desc(B, L, J, reg_max, n_max, topk=self.topk, alpha=self.alpha, beta=self.beta, w_cls=self.classification_loss_weight, w_iou=self.iou_loss_weight,
                                w_dfl=self.dfl_loss_weight, w_pose_cls=self.pose_cls_loss_weight, w_pose_reg=self.pose_reg_loss_weight, iou_type=self.iou_type,
                                cls_type=self.cls_type, pose_cls_type=self.pose_cls_type, multiply_by_oks=self.assigner_multiply_by_pose_oks,
                                rescale_with_score=self.rescale_pose_loss_with_assigned_score)  # fmt: skip
        sync = self.average_losses_in_ddp and torch.distributed.is_available() and torch.distributed.is_initialized()
        sigmas = self.oks_sigmas.to(dev)
        loss, items = _FusedPoseLoss.apply(cls_logits, reg_distri, pose_coords, pose_logits, anchor_points, stride_tensor.reshape(-1).contiguous(), gt_boxes, gt_poses,
                                           gt_crowd, gt_valid, sigmas, desc, sync)  # fmt: skip
        return loss, items.detach()
