"""PPYoloELoss (reference: training/losses/ppyolo_loss.py:640-1084) on the sm_90a path.

forward(outputs, targets) -> (loss, log_items[4]) with the reference's semantics (task-aligned assigner, varifocal +
GIoU + DFL, normalisation by max(sum(assigned_scores), 1), weights 1.0 / 2.5 / 0.5).  Target padding is done on the
host with a FIXED n_max (static shapes, CUDA-graph friendly) instead of the reference's per-image Python loop; the
assigner (3 small kernels) and the fused loss forward+backward (1 kernel) replace ~60 eager kernels and 3 host syncs.

Both assigners of the reference are served: the task-aligned one (`use_static_assigner=False`, the YOLO-NAS recipes) by
`sgb_tal_assign`, the ATSS static one (`use_static_assigner=True`, the constructor default as in the reference) by `sgb_atss_assign`;
`use_varifocal_loss=False` swaps the classification term for the focal pass (`sgb_focal_cls_fwd_bwd`).  All of them are parity-tested on
the GPU against the reference's recorded values (tests/test_zz_pose_train_gpu.py).  Deviation (DESIGN.md section 4): under DDP the
normaliser is per rank unless `sync_normaliser=True` (SURVEY.md D4).
"""
from typing import Optional, Tuple, Union

import numpy as np
import torch
from torch import Tensor, nn

from ... import kernels as K
from ...common.registry import register_loss


def host_out(out, specs):
    """numpy arrays to pad into: fresh zeros (out None), or the caller-owned CPU tensors `out`, checked against `specs` ((shape,
    numpy dtype) per tensor) and zeroed, so the slots a batch does not fill hold no earlier batch's targets."""
    if out is None:
        return [np.zeros(shape, dtype) for shape, dtype in specs]
    if len(out) != len(specs):
        raise ValueError(f"out must hold {len(specs)} tensors, got {len(out)}")
    arrays = []
    for t, (shape, dtype) in zip(out, specs):
        if t.is_cuda or not t.is_contiguous() or tuple(t.shape) != tuple(shape) or t.numpy().dtype != np.dtype(dtype):
            raise ValueError(f"out tensors must be contiguous host tensors of the padded shapes: expected {shape} {np.dtype(dtype)}, got {tuple(t.shape)} {t.dtype}")
        a = t.numpy()
        a.fill(0)
        arrays.append(a)
    return arrays


def max_targets_host(targets: Tensor) -> int:
    """Largest number of targets one image of the batch holds: flat [N, 6] (img, cls, cx, cy, w, h) host targets, numpy only."""
    img = targets.detach().float().numpy().reshape(-1, 6)[:, 0].astype(np.int64)
    return int(np.bincount(img).max()) if img.size else 0


def pad_targets_host(targets: Tensor, batch_size: int, n_max: int, out=None) -> Tuple[Tensor, Tensor, Tensor]:
    """flat [N, 6] (img, cls, cx, cy, w, h) -> gt_boxes [B, n_max, 4] xyxy, gt_labels [B, n_max] int32,
    gt_valid [B, n_max] uint8  (ppyolo_loss.py:726-775).  Vectorised numpy on the host copy of the targets.
    out: caller-owned host tensors of those shapes and dtypes, written (and returned) instead of new ones."""
    t = targets.detach().float().cpu().numpy().reshape(-1, 6)
    boxes, labels, valid = host_out(out, (((batch_size, n_max, 4), np.float32), ((batch_size, n_max), np.int32), ((batch_size, n_max), np.uint8)))
    if t.shape[0]:
        img = t[:, 0].astype(np.int64)
        order = np.argsort(img, kind="stable")
        img, t = img[order], t[order]
        first = np.searchsorted(img, np.arange(batch_size))
        slot = np.arange(t.shape[0]) - first[img]
        if slot.max() >= n_max:
            raise ValueError(f"an image has {slot.max() + 1} boxes but n_max={n_max}")
        xyxy = np.stack([t[:, 2] - t[:, 4] * 0.5, t[:, 3] - t[:, 5] * 0.5, t[:, 2] + t[:, 4] * 0.5, t[:, 3] + t[:, 5] * 0.5], 1)
        boxes[img, slot] = xyxy
        labels[img, slot] = t[:, 1].astype(np.int32)
        valid[img, slot] = (xyxy.sum(1) > 0).astype(np.uint8)
    return tuple(out) if out is not None else (torch.from_numpy(boxes), torch.from_numpy(labels), torch.from_numpy(valid))


class _FusedDetectionLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, cls_logits, reg_distri, anchor_points, stride_tensor, gt_boxes, gt_labels, gt_valid, desc, sync, static=None, focal_alpha=None):
        """static: None (task-aligned assigner) or (anchor boxes [L, 4], num_anchors_list) for the ATSS assigner;
        focal_alpha: None (varifocal classification term) or the focal term's alpha."""
        cls_logits, reg_distri = cls_logits.contiguous().float(), reg_distri.contiguous().float()
        sums = torch.zeros(4, dtype=torch.float64, device=cls_logits.device)
        if static is None:
            al, ab, asc = K.tal_assign(desc, cls_logits, reg_distri, anchor_points, stride_tensor, gt_boxes, gt_labels, gt_valid, sums)
        else:
            al, ab, asc = K.atss_assign(desc, reg_distri, static[0], anchor_points, stride_tensor, static[1], gt_boxes, gt_labels, gt_valid, sums)
        if sync:
            import torch.distributed as dist

            dist.all_reduce(sums[3:4])
            sums[3:4] /= dist.get_world_size()
        items, gc, gr = K.dfl_iou_loss(desc, cls_logits, reg_distri, anchor_points, stride_tensor, al, ab, asc, sums, focal_alpha=focal_alpha)
        ctx.save_for_backward(gc, gr)
        ctx.mark_non_differentiable(items)
        return items[3].clone(), items

    @staticmethod
    def backward(ctx, gloss, _gitems):
        gc, gr = ctx.saved_tensors
        return gc * gloss, gr * gloss, None, None, None, None, None, None, None, None, None


@register_loss(name="PPYoloELoss", deprecated_name="ppyoloe_loss")
class PPYoloELoss(nn.Module):
    def __init__(
        self,
        num_classes: int,
        use_varifocal_loss: bool = True,
        use_static_assigner: bool = True,
        reg_max=None,
        classification_loss_weight: float = 1.0,
        iou_loss_weight: float = 2.5,
        dfl_loss_weight: float = 0.5,
        use_batched_assignment: bool = True,
        max_targets_per_image: int = 0,
        sync_normaliser: bool = False,
        iou_type: str = "giou",
    ):
        super().__init__()
        self.use_varifocal_loss = use_varifocal_loss  # False: focal term, alpha 0.25 behind ATSS / none behind TAL (:820, :832-838)
        self.use_static_assigner = use_static_assigner  # ATSS (topk 9 per level) instead of the task-aligned assigner (:681-683)
        self.num_classes = num_classes
        self.classification_loss_weight = classification_loss_weight
        self.iou_loss_weight = iou_loss_weight
        self.dfl_loss_weight = dfl_loss_weight
        self.max_targets_per_image = max_targets_per_image
        self.sync_normaliser = sync_normaliser
        self.iou_type = {"giou": 0, "ciou": 1}[iou_type]
        self._n_max = max_targets_per_image

    @property
    def component_names(self):
        return ["loss_cls", "loss_iou", "loss_dfl", "loss"]

    # The padded-target interface of the captured train step (sg_trainer.TrainStep.run_padded)
    def max_targets(self, targets: Tensor) -> int:
        return max_targets_host(targets)

    def pad_targets(self, targets: Tensor, batch_size: int, n_max: int, out=None) -> Tuple[Tensor, Tensor, Tensor]:
        return pad_targets_host(targets, batch_size, n_max, out)

    def forward(self, outputs: Union[Tuple, Tuple[Tuple[Tensor, Tensor], Tuple]], targets: Tensor) -> Tuple[Tensor, Tensor]:
        if isinstance(outputs, tuple) and len(outputs) == 2:
            _, predictions = outputs
        else:
            predictions = outputs
        cls_logits, reg_distri, anchors, anchor_points, num_anchors_list, stride_tensor = predictions
        K.require_cuda(cls_logits, "predictions")
        B, L, C = cls_logits.shape
        reg_max = reg_distri.shape[-1] // 4 - 1
        dev = cls_logits.device
        if isinstance(targets, (tuple, list)) and len(targets) == 3:
            gt_boxes, gt_labels, gt_valid = targets  # already padded on the device
            n_max = gt_boxes.shape[1]
        else:
            t = targets
            counts = torch.bincount(t[:, 0].long().cpu(), minlength=B) if t.numel() else torch.zeros(B, dtype=torch.long)
            need = int(counts.max()) if t.numel() else 0
            # grow-only padding keeps the shapes static across steps
            self._n_max = max(self._n_max, need)
            n_max = self._n_max
            gt_boxes, gt_labels, gt_valid = pad_targets_host(t, B, max(n_max, 1))
            gt_boxes, gt_labels, gt_valid = gt_boxes.to(dev, non_blocking=True), gt_labels.to(dev, non_blocking=True), gt_valid.to(dev, non_blocking=True)
        desc = K.loss_desc(B, L, C, reg_max, n_max, topk=9 if self.use_static_assigner else 13, w_cls=self.classification_loss_weight, w_iou=self.iou_loss_weight,
                           w_dfl=self.dfl_loss_weight, iou_type=self.iou_type)  # fmt: skip
        sync = self.sync_normaliser and torch.distributed.is_available() and torch.distributed.is_initialized()
        static = (anchors.detach().float().contiguous(), [int(v) for v in num_anchors_list]) if self.use_static_assigner else None
        loss, items = _FusedDetectionLoss.apply(cls_logits, reg_distri, anchor_points, stride_tensor.reshape(-1).contiguous(), gt_boxes, gt_labels, gt_valid, desc, sync, static,
                                                None if self.use_varifocal_loss else (0.25 if self.use_static_assigner else -1.0))  # fmt: skip
        return loss, items.detach()
