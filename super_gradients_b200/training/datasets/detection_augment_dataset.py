"""Train-time loading for the GPU detection augmentation.

`DetectionAugmentDataset` wraps any map-style dataset with `__len__` and `get_sample(index)` returning the reference's raw sample
dict (`image` uint8 H x W x 3, `target` [n, 5] xyxy + label, optional `crowd_target`).  In DataLoader workers it runs the host half
of the transforms the way the reference's DetectionDataset.apply_transforms does (detection_dataset.py:394-450): the draws, the
mosaic's three and the mixup's one extra sample index, the box arithmetic.  `DetectionAugmentCollateFN` packs a batch into one uint8 buffer (table + images) plus
the targets, touching no CUDA state; `PackedDetectionBatch.to_model_input(device)` then makes the model input with one copy and
one kernel launch.  With `with_crowd` (the validation datasets) each item also carries its crowd targets, and
`CrowdDetectionAugmentCollateFN` delivers them as CrowdDetectionCollateFN does, in the batch's `extras`."""
import random
from typing import List, Sequence, Tuple

import numpy as np
import torch

from ...common.registry import register_collate_function
from ..transforms.detection_augment import AugmentPlan, pack_into, packed_size, run_packed
from ..transforms.transforms import DetectionPaddedRescale, DetectionPadToSize, DetectionStandardize, DetectionTargetsFormatTransform, HostSample, check_order


class DetectionAugmentDataset(torch.utils.data.Dataset):
    """with_crowd: items are (plan, target, crowd_target), the reference's output_fields of a with_crowd dataset (the raw samples
    then hold `crowd_target`); else (plan, target)."""

    def __init__(self, dataset, transforms: Sequence, with_crowd: bool = False):
        check_order(transforms)
        self.dataset, self.transforms, self.with_crowd = dataset, list(transforms), bool(with_crowd)
        size = [t for t in self.transforms if isinstance(t, (DetectionPaddedRescale, DetectionPadToSize))][0]
        std = [t for t in self.transforms if isinstance(t, DetectionStandardize)]
        self.input_dim = size.input_dim if isinstance(size, DetectionPaddedRescale) else size.output_size
        self.pad_value = int(size.pad_value)
        self.max_value = std[0].max_value if std else 0.0
        if not std:
            raise ValueError("DetectionStandardize must be in the pipeline: the model input is written standardized")

    def __len__(self) -> int:
        return len(self.dataset)

    def _random_sample(self) -> HostSample:
        return HostSample.from_dict(self.dataset.get_sample(random.randint(0, len(self.dataset) - 1)))

    def __getitem__(self, index: int) -> Tuple[AugmentPlan, np.ndarray]:
        """(plan of the pixel work, targets [n, 5] label + cxcywh[, crowd targets [m, 5]]) of sample `index` after the transforms."""
        sample = HostSample.from_dict(self.dataset.get_sample(index))
        fmt = None
        for t in self.transforms:
            n = t.get_number_of_additional_samples() if t.may_require_additional_samples else 0
            sample.additional_samples = [self._random_sample() for _ in range(n)]
            sample = t.apply_to_sample(sample)
            sample.additional_samples = None
            if isinstance(t, DetectionTargetsFormatTransform):
                fmt = t
        out = sample.to_dict(include_crowd_target=self.with_crowd)
        if fmt is not None:
            out = {k: fmt.apply_on_targets(v) for k, v in out.items()}
        if self.with_crowd:
            return sample.plan, out["target"], out["crowd_target"]
        return sample.plan, out["target"]


class PackedDetectionBatch:
    """A collated batch: `buffer` (uint8: the int64 per-image table, then the images), `targets` [N, 6] (sample index first) and
    `extras`, the additional batch items the metrics receive ({"crowd_targets": [M, 6]} from CrowdDetectionAugmentCollateFN)."""

    def __init__(self, buffer: torch.Tensor, batch: int, targets: torch.Tensor, input_dim, pad_value: int, max_value: float, extras=None):
        self.buffer, self.batch, self.targets = buffer, batch, targets
        self.input_dim, self.pad_value, self.max_value = tuple(input_dim), pad_value, max_value
        self.extras = extras if extras is not None else {}

    def pin_memory(self) -> "PackedDetectionBatch":
        """Called by DataLoader(pin_memory=True) in the main process, so the copy to the device is asynchronous."""
        return PackedDetectionBatch(self.buffer.pin_memory(), self.batch, self.targets, self.input_dim, self.pad_value, self.max_value, self.extras)

    @property
    def input_shape(self) -> Tuple[int, int, int, int]:
        """Shape of the model input to_model_input makes."""
        return (self.batch, 16, *self.input_dim)

    def to_model_input(self, device, out=None) -> Tuple[torch.Tensor, torch.Tensor]:
        """(images bf16 NHWC [B, 16, H, W], targets [N, 6]): one copy and one augmentation launch, no host synchronisation.  out: a
        bf16 channels_last tensor of input_shape the images are written into instead of a new one."""
        return run_packed(self.buffer, self.batch, device, self.input_dim, self.pad_value, self.max_value, out=out), self.targets


@register_collate_function()
class DetectionAugmentCollateFN:
    """Collates DetectionAugmentDataset items into a PackedDetectionBatch; its targets are DetectionCollateFN's."""

    def __init__(self, input_dim=(640, 640), pad_value: int = 114, max_value: float = 255.0):
        self.input_dim, self.pad_value, self.max_value = (int(input_dim[0]), int(input_dim[1])), int(pad_value), float(max_value)

    @classmethod
    def for_dataset(cls, dataset: DetectionAugmentDataset) -> "DetectionAugmentCollateFN":
        return cls(dataset.input_dim, dataset.pad_value, dataset.max_value)

    def __call__(self, data: List[Tuple[AugmentPlan, np.ndarray]]) -> PackedDetectionBatch:
        plans = [d[0] for d in data]
        buf = torch.empty(packed_size(plans), dtype=torch.uint8)
        pack_into(plans, buf.numpy())
        return PackedDetectionBatch(buf, len(plans), _format_targets([d[1] for d in data]), self.input_dim, self.pad_value, self.max_value)


def _format_targets(targets: Sequence[np.ndarray]) -> torch.Tensor:
    """DetectionCollateFN._format_targets: [n_i, 5] per sample -> [sum n_i, 6] with the sample index first."""
    rows = []
    for i, t in enumerate(targets):
        t = torch.as_tensor(t)
        rows.append(torch.cat((t.new_full((t.shape[0], 1), i), t), dim=-1))
    return torch.cat(rows, 0)


@register_collate_function()
class CrowdDetectionAugmentCollateFN(DetectionAugmentCollateFN):
    """Collates DetectionAugmentDataset(with_crowd=True) items into a PackedDetectionBatch whose extras are CrowdDetectionCollateFN's
    {"crowd_targets": [M, 6]} (reference utils/collate_fn/crowd_detection_collate_fn.py:11)."""

    def __call__(self, data: List[Tuple[AugmentPlan, np.ndarray, np.ndarray]]) -> PackedDetectionBatch:
        if any(len(d) != 3 for d in data):
            raise ValueError("CrowdDetectionAugmentCollateFN takes (plan, target, crowd_target) items: build the dataset with with_crowd=True")
        batch = super().__call__([d[:2] for d in data])
        batch.extras = {"crowd_targets": _format_targets([d[2] for d in data])}
        return batch
