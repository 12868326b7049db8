"""Train-time loading for the GPU pose augmentation.

`PoseAugmentDataset` wraps any map-style dataset with `__len__` and `load_sample(index)` returning a PoseEstimationSample-like
object (image uint8 H x W x 3, joints [N, J, 3], areas, bboxes_xywh, is_crowd): the contract of the reference's
AbstractPoseEstimationDataset.  In DataLoader workers it runs the host half of the keypoint transforms the way the reference's
KeypointsCompose.apply_to_sample does: sanitize, then the transforms, loading a mosaic's three extra samples with
random.randrange and passing each through the transforms applied so far.  `PoseAugmentCollateFN` packs a batch into one uint8
buffer (table + images) plus YoloNASPoseCollateFN's targets, touching no CUDA state; `PackedPoseBatch.to_model_input(device)`
then makes the model input with one copy and one kernel call.  With `with_gt_samples` (the validation datasets) each item also
carries the transformed sample's ground truth, and `YoloNASPoseAugmentCollateFN` delivers it as YoloNASPoseCollateFN does, in the
batch's `extras` {"gt_samples": [...]}, which PoseEstimationMetrics reads."""
import random
from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

from ....common.registry import register_collate_function
from ...transforms.keypoints import KeypointsImageStandardize, PoseHostSample, check_pose_pipeline
from ...transforms.keypoints_augment import PosePlan, pack_into, packed_size, run_packed
from .yolo_nas_pose_collate_fn import flat_collate_tensors_with_batch_index


@dataclass
class PoseGroundTruth:
    """One transformed sample as YoloNASPoseCollateFN leaves it in gt_samples (set_image_to_none): joints [N, J, 3], areas [N] or
    None, bboxes_xywh [N, 4] or None, is_crowd [N] or None; no image or mask."""

    joints: np.ndarray
    areas: Optional[np.ndarray]
    bboxes_xywh: Optional[np.ndarray]
    is_crowd: Optional[np.ndarray]
    image: None = None
    mask: None = None
    additional_samples: None = None


class PoseAugmentDataset(torch.utils.data.Dataset):
    """with_gt_samples: items are (plan, targets, PoseGroundTruth), else (plan, targets)."""

    def __init__(self, dataset, transforms: Sequence, with_gt_samples: bool = False):
        self.output_size = check_pose_pipeline(transforms)
        self.dataset, self.transforms, self.with_gt_samples = dataset, list(transforms), bool(with_gt_samples)
        self.max_value = float([t for t in self.transforms if isinstance(t, KeypointsImageStandardize)][0].max_value)

    def __len__(self) -> int:
        return len(self.dataset)

    def _load(self, index: int) -> PoseHostSample:
        return PoseHostSample.from_sample(self.dataset.load_sample(index))

    def _apply(self, sample: PoseHostSample, transforms) -> PoseHostSample:
        applied = []
        for t in transforms:
            if not t.may_require_additional_samples:
                sample = t.apply_to_sample(sample)
                applied.append(t)
            else:
                extra = [self._load(random.randrange(0, len(self.dataset))) for _ in range(t.get_number_of_additional_samples())]
                sample.additional_samples = [self._apply(s, applied) for s in extra]
                sample = t.apply_to_sample(sample)
        return sample

    def __getitem__(self, index: int) -> Tuple[PosePlan, Tuple[np.ndarray, np.ndarray, np.ndarray]]:
        """(plan of the pixel work, (boxes [n, 4] xyxy, joints [n, J, 3], is_crowd [n, 1])) of sample `index` after the transforms:
        the targets YoloNASPoseCollateFN takes from the reference's sample."""
        s = self._apply(self._load(index).sanitize_sample(), self.transforms)
        xywh = np.asarray(s.bboxes_xywh)
        xyxy = np.concatenate([xywh[..., :2], xywh[..., :2] + xywh[..., 2:4]], axis=-1)
        is_crowd = np.zeros(len(xyxy)) if s.is_crowd is None else s.is_crowd
        targets = (xyxy, s.joints, is_crowd.astype(int).reshape((-1, 1)))
        if self.with_gt_samples:
            return s.plan, targets, PoseGroundTruth(s.joints, s.areas, s.bboxes_xywh, s.is_crowd)
        return s.plan, targets


class PackedPoseBatch:
    """A collated batch: `buffer` (uint8: the int64 per-sample table, then the images), YoloNASPoseCollateFN's targets
    (boxes [N, 5], joints [N, J, 4], is_crowd [N, 2], each with the sample index first) and `extras`, the additional batch items
    the metrics receive ({"gt_samples": [...]} from YoloNASPoseAugmentCollateFN)."""

    def __init__(self, buffer: torch.Tensor, batch: int, targets, output_size: int, max_value: float, extras=None):
        self.buffer, self.batch, self.targets, self.output_size, self.max_value = buffer, batch, targets, output_size, max_value
        self.extras = extras if extras is not None else {}

    def pin_memory(self) -> "PackedPoseBatch":
        """Called by DataLoader(pin_memory=True) in the main process, so the copy to the device is asynchronous."""
        return PackedPoseBatch(self.buffer.pin_memory(), self.batch, self.targets, self.output_size, self.max_value, self.extras)

    @property
    def input_shape(self) -> Tuple[int, int, int, int]:
        """Shape of the model input to_model_input makes."""
        return (self.batch, 16, self.output_size, self.output_size)

    def to_model_input(self, device, out=None):
        """(images bf16 NHWC [B, 16, S, S], (boxes, joints, is_crowd)): one copy and one augmentation call, no host synchronisation.
        out: a bf16 channels_last tensor of input_shape the images are written into instead of a new one."""
        return run_packed(self.buffer, self.batch, device, self.output_size, self.max_value, out=out), self.targets


@register_collate_function()
class PoseAugmentCollateFN:
    """Collates PoseAugmentDataset items into a PackedPoseBatch."""

    def __init__(self, output_size: int = 640, max_value: float = 255.0):
        self.output_size, self.max_value = int(output_size), float(max_value)

    @classmethod
    def for_dataset(cls, dataset: PoseAugmentDataset) -> "PoseAugmentCollateFN":
        return cls(dataset.output_size, dataset.max_value)

    def __call__(self, data: List[Tuple[PosePlan, tuple]]) -> PackedPoseBatch:
        plans = [d[0] for d in data]
        buf = torch.empty(packed_size(plans), dtype=torch.uint8)
        pack_into(plans, buf.numpy())
        targets = tuple(flat_collate_tensors_with_batch_index([torch.from_numpy(d[1][k]) for d in data]) for k in range(3))
        return PackedPoseBatch(buf, len(plans), targets, self.output_size, self.max_value)


@register_collate_function()
class YoloNASPoseAugmentCollateFN(PoseAugmentCollateFN):
    """Collates PoseAugmentDataset(with_gt_samples=True) items into a PackedPoseBatch whose extras are YoloNASPoseCollateFN's
    {"gt_samples": [...]} (reference datasets/pose_estimation_datasets/yolo_nas_pose_collate_fn.py:28-70)."""

    def __call__(self, data: List[Tuple[PosePlan, tuple, PoseGroundTruth]]) -> PackedPoseBatch:
        if any(len(d) != 3 for d in data):
            raise ValueError("YoloNASPoseAugmentCollateFN takes (plan, targets, ground truth) items: build the dataset with with_gt_samples=True")
        batch = super().__call__([d[:2] for d in data])
        batch.extras = {"gt_samples": [d[2] for d in data]}
        return batch
