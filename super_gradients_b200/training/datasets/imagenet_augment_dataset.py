"""Train-time loading for the GPU ImageNet augmentation.

`ImageNetAugmentDataset` wraps any dataset returning (PIL RGB image or uint8 H x W x 3 RGB array, label).  In DataLoader workers it
makes the draws of the ResNet-50 recipe's train chain (RandomResizedCropAndInterpolation -> RandomHorizontalFlip -> RandAugment, see
transforms/imagenet_augment.py) and returns the plan with only the crop window's bytes.  `ImageNetAugmentCollateFN` packs a batch into
one uint8 buffer and draws the batch's mixup / cutmix parameters as the reference's CollateMixup does in batch mode
(datasets/mixup.py:179-206, 89-100), touching no CUDA state; `PackedImageNetBatch.to_model_input(device)` then makes the bf16 NHWC
model input with one copy and one kernel launch, and the [B, num_classes] soft targets with a few small torch ops on the device.

`ImageNetValidationDataset` / `ImageNetValidationCollateFN` do the same for the recipe's validation chain Resize(236) ->
CenterCrop(224) -> ToTensor -> Normalize: the workers only pack the decoded images, and `PackedImageNetValidationBatch` makes the
model input with one copy and one launch of the predict() resize-and-crop kernel (kernels.resample_crop_u8)."""
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

from ... import kernels as K
from ...common.registry import register_collate_function
from ..transforms.imagenet_augment import ImageNetPlan, RandAugmentConfig, draw_plan, pack_into, packed_size, run_packed, workspace_size

IMAGENET_MEAN = (0.485, 0.456, 0.406)
IMAGENET_STD = (0.229, 0.224, 0.225)


def _as_rgb_array(image) -> np.ndarray:
    if isinstance(image, np.ndarray):
        if image.dtype != np.uint8 or image.ndim != 3 or image.shape[2] != 3:
            raise ValueError(f"images must be uint8 H x W x 3 RGB arrays, got {image.dtype} {image.shape}")
        return image
    if getattr(image, "mode", None) != "RGB":
        raise ValueError(f"images must be PIL RGB images or uint8 H x W x 3 arrays, got {type(image).__name__} {getattr(image, 'mode', '')}")
    return np.asarray(image)


class ImageNetAugmentDataset(torch.utils.data.Dataset):
    """The recipe's RandomResizedCropAndInterpolation(size, interpolation), RandomHorizontalFlip and
    RandAugmentTransform(config_str, crop_size=size, img_mean), drawn on the host; the pixels are the kernel's.  interpolation:
    'random' (bilinear or bicubic per sample) or 'default' (bilinear); config_str None: no RandAugment."""

    def __init__(self, dataset, size: int = 224, interpolation: str = "random", config_str: Optional[str] = "rand-m7-mstd0.5", img_mean=IMAGENET_MEAN,
                 img_std=IMAGENET_STD):  # fmt: skip
        if interpolation not in ("random", "default"):
            raise ValueError(f"interpolation must be 'random' or 'default', got {interpolation!r}")
        self.dataset, self.size = dataset, int(size)
        self.random_interpolation = interpolation == "random"
        self.rand_augment = RandAugmentConfig.parse(config_str) if config_str is not None else None
        self.img_mean, self.img_std = tuple(float(m) for m in img_mean), tuple(float(s) for s in img_std)
        self.fill = tuple(min(255, round(255 * m)) for m in self.img_mean)  # rand_augment_transform's img_mean hparam

    def __len__(self) -> int:
        return len(self.dataset)

    def __getitem__(self, index: int) -> ImageNetPlan:
        image, label = self.dataset[index]
        return draw_plan(_as_rgb_array(image), int(label), self.size, self.random_interpolation, self.rand_augment)


class PackedImageNetBatch:
    """A collated batch: `buffer` (uint8: the int64 per-image table, then the crop windows), the labels and the batch's mix draws."""

    def __init__(self, buffer, batch, labels, workspace_bytes, size, fill, mean, std, lam, use_cutmix, box, num_classes, label_smoothing):
        self.buffer, self.batch, self.labels, self.workspace_bytes = buffer, batch, labels, workspace_bytes
        self.size, self.fill, self.mean, self.std = size, fill, mean, std
        self.lam, self.use_cutmix, self.box = lam, use_cutmix, box
        self.num_classes, self.label_smoothing = num_classes, label_smoothing

    def _replace(self, buffer) -> "PackedImageNetBatch":
        return PackedImageNetBatch(buffer, self.batch, self.labels, self.workspace_bytes, self.size, self.fill, self.mean, self.std, self.lam, self.use_cutmix, self.box,
                                   self.num_classes, self.label_smoothing)  # fmt: skip

    def pin_memory(self) -> "PackedImageNetBatch":
        """Called by DataLoader(pin_memory=True) in the main process, so the copy to the device is asynchronous."""
        return self._replace(self.buffer.pin_memory())

    @property
    def mix_mode(self) -> int:
        return 0 if self.lam == 1.0 else (2 if self.use_cutmix else 1)

    def targets(self, device) -> torch.Tensor:
        """CollateMixup's mixup_target: [B, num_classes] float32 smoothed two-hot targets, partner B - 1 - i."""
        off = self.label_smoothing / self.num_classes
        on = 1.0 - self.label_smoothing + off
        x = self.labels.to(device, non_blocking=True).long().view(-1, 1)
        y1 = torch.full((x.size(0), self.num_classes), off, device=device).scatter_(1, x, on)
        y2 = torch.full((x.size(0), self.num_classes), off, device=device).scatter_(1, x.flip(0), on)
        return y1 * self.lam + y2 * (1.0 - self.lam)

    @property
    def input_shape(self) -> Tuple[int, int, int, int]:
        """Shape of the model input to_model_input makes."""
        return (self.batch, 16, self.size, self.size)

    def to_model_input(self, device, out=None) -> Tuple[torch.Tensor, torch.Tensor]:
        """(images bf16 NHWC [B, 16, S, S], targets [B, num_classes]): one copy and one augmentation launch, no host synchronisation.
        out: a bf16 channels_last tensor of input_shape the images are written into instead of a new one."""
        images = run_packed(self.buffer, self.batch, self.workspace_bytes, device, self.size, self.fill, self.mean, self.std, self.mix_mode, self.lam, self.box, out=out)
        return images, self.targets(device)


@register_collate_function()
class ImageNetAugmentCollateFN:
    """Collates ImageNetAugmentDataset plans into a PackedImageNetBatch; the mix draws and targets are CollateMixup's in batch mode.
    The per-element modes ('elem', 'pair', 'half') and cutmix_minmax are refused."""

    def __init__(self, mixup_alpha: float = 1.0, cutmix_alpha: float = 0.0, cutmix_minmax: Optional[List[float]] = None, prob: float = 1.0, switch_prob: float = 0.5,
                 mode: str = "batch", correct_lam: bool = True, label_smoothing: float = 0.1, num_classes: int = 1000, size: int = 224, img_mean=IMAGENET_MEAN,
                 img_std=IMAGENET_STD):  # fmt: skip
        if mode != "batch":
            raise ValueError(f"only CollateMixup's 'batch' mode runs on the GPU path, got {mode!r}")
        if cutmix_minmax is not None:
            raise ValueError("cutmix_minmax is not supported on the GPU path")
        if mixup_alpha <= 0.0 and cutmix_alpha <= 0.0:
            raise ValueError("one of mixup_alpha > 0, cutmix_alpha > 0 must hold")
        self.mixup_alpha, self.cutmix_alpha, self.mix_prob, self.switch_prob = mixup_alpha, cutmix_alpha, prob, switch_prob
        self.correct_lam, self.label_smoothing, self.num_classes = correct_lam, label_smoothing, num_classes
        self.mixup_enabled = True  # the train loop may switch mixing off, as on CollateMixup
        self.size, self.img_mean, self.img_std = int(size), tuple(img_mean), tuple(img_std)
        self.fill = tuple(min(255, round(255 * m)) for m in self.img_mean)

    @classmethod
    def for_dataset(cls, dataset: ImageNetAugmentDataset, **kwargs) -> "ImageNetAugmentCollateFN":
        return cls(size=dataset.size, img_mean=dataset.img_mean, img_std=dataset.img_std, **kwargs)

    def _params_per_batch(self) -> Tuple[float, bool]:
        lam, use_cutmix = 1.0, False
        if self.mixup_enabled and torch.rand(1) < self.mix_prob:
            if self.mixup_alpha > 0.0 and self.cutmix_alpha > 0.0:
                use_cutmix = bool(torch.rand(1) < self.switch_prob)
                alpha = self.cutmix_alpha if use_cutmix else self.mixup_alpha
            elif self.mixup_alpha > 0.0:
                alpha = self.mixup_alpha
            else:
                use_cutmix, alpha = True, self.cutmix_alpha
            lam = float(torch.distributions.beta.Beta(alpha, alpha).sample())
        return lam, use_cutmix

    def _cutmix_box(self, lam: float) -> Tuple[Tuple[int, int, int, int], float]:
        """cutmix_bbox_and_lam / rand_bbox on the S x S output: the box (yl, yh, xl, xh) and the corrected lam."""
        s = self.size
        ratio = np.sqrt(1 - lam)
        cut = int(s * ratio), int(s * ratio)
        cy, cx = np.random.randint(0, s), np.random.randint(0, s)
        yl, yh = np.clip(cy - cut[0] // 2, 0, s), np.clip(cy + cut[0] // 2, 0, s)
        xl, xh = np.clip(cx - cut[1] // 2, 0, s), np.clip(cx + cut[1] // 2, 0, s)
        if self.correct_lam:
            lam = 1.0 - (yh - yl) * (xh - xl) / float(s * s)
        return (int(yl), int(yh), int(xl), int(xh)), float(lam)

    def __call__(self, plans: Sequence[ImageNetPlan]) -> PackedImageNetBatch:
        if len(plans) % 2:
            raise ValueError("the batch size must be even: image i mixes with image B - 1 - i")
        buf = torch.empty(packed_size(plans), dtype=torch.uint8)
        pack_into(plans, buf.numpy(), self.size)
        lam, use_cutmix = self._params_per_batch()
        box = (0, 0, 0, 0)
        if use_cutmix:
            box, lam = self._cutmix_box(lam)
        labels = torch.tensor([p.label for p in plans], dtype=torch.int32)
        return PackedImageNetBatch(buf, len(plans), labels, workspace_size(plans, self.size), self.size, self.fill, self.img_mean, self.img_std, lam, use_cutmix, box,
                                   self.num_classes, self.label_smoothing)  # fmt: skip


class ImageNetValidationDataset(torch.utils.data.Dataset):
    """The recipe's validation chain torchvision Resize(resize) (Pillow bilinear, antialiased) -> CenterCrop(size) -> ToTensor ->
    Normalize(img_mean, img_std) over any dataset returning (PIL RGB image or uint8 H x W x 3 RGB array, label).  Items are the
    uint8 image and the label; every pixel is the kernel's."""

    def __init__(self, dataset, resize: int = 236, size: int = 224, img_mean=IMAGENET_MEAN, img_std=IMAGENET_STD):
        if int(resize) < int(size):
            raise ValueError(f"Resize({resize}) must not be smaller than CenterCrop({size}): the GPU path does not pad")
        self.dataset, self.resize, self.size = dataset, int(resize), int(size)
        self.img_mean, self.img_std = tuple(float(m) for m in img_mean), tuple(float(s) for s in img_std)

    def __len__(self) -> int:
        return len(self.dataset)

    def __getitem__(self, index: int) -> Tuple[np.ndarray, int]:
        image, label = self.dataset[index]
        return _as_rgb_array(image), int(label)


def validation_geometry(height: int, width: int, resize: int, size: int) -> Tuple[Tuple[int, int], Tuple[int, int]]:
    """torchvision's Resize(resize) output size (shorter side resize, longer side truncated) and CenterCrop(size)'s top-left
    corner (rounded half to even) -> ((resized h, w), (top, left))."""
    short, long = (width, height) if width <= height else (height, width)
    new_long = int(resize * long / short)
    rh, rw = (new_long, resize) if width <= height else (resize, new_long)
    return (rh, rw), (int(round((rh - size) / 2.0)), int(round((rw - size) / 2.0)))


class PackedImageNetValidationBatch:
    """A collated batch: `buffer` (uint8: the int64 [B, RS_FIELDS] table, then the images) and the int64 labels."""

    def __init__(self, buffer: torch.Tensor, batch: int, labels: torch.Tensor, size: int, mean, std):
        self.buffer, self.batch, self.labels, self.size, self.mean, self.std = buffer, batch, labels, size, mean, std

    def pin_memory(self) -> "PackedImageNetValidationBatch":
        """Called by DataLoader(pin_memory=True) in the main process, so the copy to the device is asynchronous."""
        return PackedImageNetValidationBatch(self.buffer.pin_memory(), self.batch, self.labels, self.size, self.mean, self.std)

    @property
    def input_shape(self) -> Tuple[int, int, int, int]:
        """Shape of the model input to_model_input makes."""
        return (self.batch, 16, self.size, self.size)

    def to_model_input(self, device, out=None) -> Tuple[torch.Tensor, torch.Tensor]:
        """(images bf16 NHWC [B, 16, S, S], labels [B]): one copy and one resize-and-crop launch, no host synchronisation.  out: a
        bf16 channels_last tensor of input_shape the images are written into instead of a new one."""
        head = self.batch * K.RS_FIELDS * 8
        dev = self.buffer.to(device, non_blocking=True)
        out = K.empty_nhwc(*self.input_shape, device) if out is None else K.require_nhwc_out(out, self.input_shape)
        table_host = self.buffer[:head].view(torch.int64).view(self.batch, K.RS_FIELDS)
        K.resample_crop_u8(table_host, dev[:head].view(torch.int64).view(self.batch, K.RS_FIELDS), dev[head:], out, max_value=255.0, mean=self.mean, std=self.std)
        return out, self.labels


@register_collate_function()
class ImageNetValidationCollateFN:
    """Collates ImageNetValidationDataset items into a PackedImageNetValidationBatch; the labels are default_collate's."""

    def __init__(self, resize: int = 236, size: int = 224, img_mean=IMAGENET_MEAN, img_std=IMAGENET_STD):
        self.resize, self.size, self.img_mean, self.img_std = int(resize), int(size), tuple(img_mean), tuple(img_std)

    @classmethod
    def for_dataset(cls, dataset: ImageNetValidationDataset) -> "ImageNetValidationCollateFN":
        return cls(dataset.resize, dataset.size, dataset.img_mean, dataset.img_std)

    def __call__(self, data: Sequence[Tuple[np.ndarray, int]]) -> PackedImageNetValidationBatch:
        images = [_as_rgb_array(d[0]) for d in data]
        B = len(images)
        head = B * K.RS_FIELDS * 8
        offsets = np.cumsum([0] + [im.nbytes for im in images])
        buf = torch.empty(head + int(offsets[-1]), dtype=torch.uint8)
        raw = buf.numpy()
        table = raw[:head].view(np.int64).reshape(B, K.RS_FIELDS)
        for b, im in enumerate(images):
            h, w = im.shape[:2]
            (rh, rw), (top, left) = validation_geometry(h, w, self.resize, self.size)
            table[b] = (offsets[b], h, w, w * 3, rh, rw, top, left)
            raw[head + offsets[b] : head + offsets[b + 1]] = np.ascontiguousarray(im).reshape(-1)
        labels = torch.tensor([int(d[1]) for d in data], dtype=torch.int64)
        return PackedImageNetValidationBatch(buf, B, labels, self.size, self.img_mean, self.img_std)
