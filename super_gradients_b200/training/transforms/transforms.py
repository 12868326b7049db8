"""The YOLO-NAS COCO and Roboflow fine-tuning train transforms (reference: training/transforms/transforms.py:490-1330, 1345-1554,
1579-1590, 1623-1634, transforms/utils.py:45-57, 183-226, utils/detection_utils.py:174-185, 738-785), split in two halves.

On the host, in DataLoader workers, each transform draws its random numbers from the global `random` / `np.random` in the
reference's order and transforms the boxes with the reference's numpy arithmetic.  The pixels are not touched: every transform
records its draws in the sample's `AugmentPlan`, and `BatchAugmenter` later turns a batch of plans into the model input with one
kernel launch (csrc/augment.cu).  The kernel applies the steps in the recipe's order, so a pipeline must list these transforms in
that order (`check_order`); DetectionMosaic, when present, comes first and the kernel reads its canvas as the chain's source."""
import math
import random
from numbers import Number
from typing import List, Optional, Tuple, Union

import cv2
import numpy as np

from ...common.registry import register_transform
from .detection_augment import AugmentPlan, MixupPlan, MosaicPlan, MosaicTile

RECIPE_ORDER = ("DetectionMosaic", "DetectionRandomAffine", "DetectionRGB2BGR", "DetectionHSV", "DetectionHorizontalFlip", "DetectionMixup",
                "DetectionPaddedRescale", "DetectionPadToSize", "DetectionStandardize", "DetectionImagePermute", "DetectionTargetsFormatTransform")  # fmt: skip
# DetectionPadToSize runs on the affine step of the kernel, so it only combines with the steps that commute with a pad of one grey
PAD_TO_SIZE_EXCLUDES = ("DetectionMosaic", "DetectionRandomAffine", "DetectionHSV", "DetectionHorizontalFlip", "DetectionMixup", "DetectionPaddedRescale")


def _tuple_of_two(v):
    if v is None:
        return None
    if isinstance(v, Number):
        return (int(v), int(v))
    return (int(v[0]), int(v[1]))


def clip_boxes_inplace(boxes: np.ndarray, shape: Tuple[int, int]) -> np.ndarray:
    """change_bbox_bounds_for_image_size_inplace: clip xyxy boxes to an image of shape (h, w)."""
    boxes[..., [0, 2]] = boxes[..., [0, 2]].clip(min=0, max=shape[1])
    boxes[..., [1, 3]] = boxes[..., [1, 3]].clip(min=0, max=shape[0])
    return boxes


class HostSample:
    """The reference's DetectionSample without pixels: the current image shape, the boxes (xyxy), labels and crowd flags, and the
    plan of the pixel work.  Construction sanitizes like DetectionSample: clip to the image and drop boxes of zero area."""

    def __init__(self, plan: AugmentPlan, shape: Tuple[int, int], bboxes_xyxy: np.ndarray, labels: np.ndarray, is_crowd: np.ndarray):
        self.plan, self.shape = plan, (int(shape[0]), int(shape[1]))
        self.bboxes_xyxy, self.labels, self.is_crowd = bboxes_xyxy, labels, is_crowd
        self.additional_samples: Optional[List["HostSample"]] = None
        self.sanitize()

    def sanitize(self) -> "HostSample":
        self.bboxes_xyxy = clip_boxes_inplace(self.bboxes_xyxy, self.shape)
        w = self.bboxes_xyxy[..., 2] - self.bboxes_xyxy[..., 0]
        h = self.bboxes_xyxy[..., 3] - self.bboxes_xyxy[..., 1]
        keep = np.stack([w, h], -1).prod(axis=-1) > 0
        self.bboxes_xyxy, self.labels, self.is_crowd = self.bboxes_xyxy[keep], self.labels[keep], self.is_crowd[keep]
        return self

    def replaced(self, **kw) -> "HostSample":
        a = dict(plan=self.plan, shape=self.shape, bboxes_xyxy=self.bboxes_xyxy, labels=self.labels, is_crowd=self.is_crowd)
        a.update(kw)
        return HostSample(**a)

    @classmethod
    def from_dict(cls, sample: dict) -> "HostSample":
        """LegacyDetectionTransformMixin.convert_input_dict_to_detection_sample of a raw sample (image, target, [crowd_target])."""
        image = sample["image"]
        if not isinstance(image, np.ndarray) or image.dtype != np.uint8 or image.ndim != 3 or image.shape[2] != 3:
            raise ValueError(f"raw samples must hold a uint8 H x W x 3 image, got {getattr(image, 'dtype', type(image))} {getattr(image, 'shape', '')}")
        target = sample["target"]
        if len(target) == 0:
            target = np.zeros((0, 5), dtype=np.float32)
        boxes, labels = target[:, 0:4].reshape(-1, 4), target[:, 4]
        is_crowd = np.zeros_like(labels, dtype=bool)
        if "crowd_target" in sample:
            crowd = sample["crowd_target"]
            if len(crowd) == 0:
                crowd = np.zeros((0, 5), dtype=np.float32)
            boxes = np.concatenate([boxes, crowd[:, 0:4].reshape(-1, 4)], axis=0)
            labels = np.concatenate([labels, crowd[:, 4]], axis=0)
            is_crowd = np.concatenate([is_crowd, np.ones_like(crowd[:, 4], dtype=bool)], axis=0)
        return cls(AugmentPlan(image, image.shape[:2]), image.shape[:2], boxes, labels, is_crowd)

    def to_dict(self, include_crowd_target: bool = False) -> dict:
        """convert_detection_sample_to_dict: what a dataset returns, `crowd_target` too when it was built with_crowd."""
        crowd = self.is_crowd > 0
        out = {"target": np.concatenate([self.bboxes_xyxy[~crowd], self.labels[~crowd][..., None]], axis=-1)}
        if include_crowd_target:
            out["crowd_target"] = np.concatenate([self.bboxes_xyxy[crowd], self.labels[crowd][..., None]], axis=-1)
        return out


class _Transform:
    def get_number_of_additional_samples(self) -> int:
        return 0

    @property
    def may_require_additional_samples(self) -> bool:
        return False

    def close(self):
        pass


def get_mosaic_coordinate(mosaic_index, xc, yc, w, h, input_h, input_w):
    """Where tile `mosaic_index` (0 top-left, 1 top-right, 2 bottom-left, 3 bottom-right) of a resized w x h image lands on the
    2 * input_h x 2 * input_w canvas: (x1, y1, x2, y2) on the canvas and (x1s, y1s, x2s, y2s) in the tile."""
    if mosaic_index == 0:
        x1, y1, x2, y2 = max(xc - w, 0), max(yc - h, 0), xc, yc
        small_coord = w - (x2 - x1), h - (y2 - y1), w, h
    elif mosaic_index == 1:
        x1, y1, x2, y2 = xc, max(yc - h, 0), min(xc + w, input_w * 2), yc
        small_coord = 0, h - (y2 - y1), min(w, x2 - x1), h
    elif mosaic_index == 2:
        x1, y1, x2, y2 = max(xc - w, 0), yc, xc, min(input_h * 2, yc + h)
        small_coord = w - (x2 - x1), 0, w, min(y2 - y1, h)
    else:
        x1, y1, x2, y2 = xc, yc, min(xc + w, input_w * 2), min(input_h * 2, yc + h)
        small_coord = 0, 0, min(w, x2 - x1), min(y2 - y1, h)
    return (x1, y1, x2, y2), small_coord


@register_transform()
class DetectionMosaic(_Transform):
    """Four samples (this one and three random others), each resized to fit input_dim, placed around a random centre of a
    2 * input_dim canvas of border_value.  The coin flip happens in get_number_of_additional_samples, so a failed flip (or a closed
    mosaic) leaves the sample as it is."""

    def __init__(self, input_dim, prob: float = 1.0, enable_mosaic: bool = True, border_value=114):
        self.prob, self.input_dim, self.enable_mosaic, self.border_value = prob, _tuple_of_two(input_dim), enable_mosaic, border_value

    def close(self):
        self.enable_mosaic = False

    def get_number_of_additional_samples(self) -> int:
        return 3 if self.enable_mosaic and random.random() < self.prob else 0

    @property
    def may_require_additional_samples(self) -> bool:
        return self.enable_mosaic

    def apply_to_sample(self, sample: HostSample) -> HostSample:
        if not sample.additional_samples or not self.enable_mosaic:
            return sample
        input_h, input_w = self.input_dim
        yc = int(random.uniform(0.5 * input_h, 1.5 * input_h))
        xc = int(random.uniform(0.5 * input_w, 1.5 * input_w))
        tiles, boxes, labels, is_crowd = [], [], [], []
        for i, s in enumerate([sample] + sample.additional_samples):
            h0, w0 = s.shape
            scale = min(1.0 * input_h / h0, 1.0 * input_w / w0)
            h, w = int(h0 * scale), int(w0 * scale)
            (l_x1, l_y1, l_x2, l_y2), (s_x1, s_y1, _, _) = get_mosaic_coordinate(i, xc, yc, w, h, input_h, input_w)
            tiles.append(MosaicTile(s.plan.image, (h, w), (l_x1, l_y1, l_x2, l_y2), (s_x1, s_y1)))
            padw, padh = l_x1 - s_x1, l_y1 - s_y1
            boxes.append(s.bboxes_xyxy * scale + np.array([[padw, padh, padw, padh]], dtype=np.float32))
            labels.append(s.labels)
            is_crowd.append(s.is_crowd)
        canvas = (input_h * 2, input_w * 2)
        sample.plan.mosaic = MosaicPlan(tiles, canvas, xc, yc, int(self.border_value))
        return HostSample(sample.plan, canvas, np.concatenate(boxes, 0), np.concatenate(labels, 0), np.concatenate(is_crowd, 0))


def get_aug_params(value: Union[tuple, float], center: float = 0) -> float:
    if isinstance(value, Number):
        return random.uniform(center - float(value), center + float(value))
    if len(value) == 2:
        return random.uniform(value[0], value[1])
    raise ValueError(f"Affine params should be either a sequence containing two values or single float values. Got {value}")


def get_affine_matrix(input_size, target_size, degrees, translate, scales, shear) -> np.ndarray:
    center_m = np.eye(3)
    center = (input_size[0] // 2, input_size[1] // 2)
    center_m[0, 2] = -center[1]
    center_m[1, 2] = -center[0]
    rotation_m = np.eye(3)
    rotation_m[:2] = cv2.getRotationMatrix2D(angle=get_aug_params(degrees), center=(0, 0), scale=get_aug_params(scales, center=1.0))
    shear_m = np.eye(3)
    shear_m[0, 1] = math.tan(get_aug_params(shear) * math.pi / 180)
    shear_m[1, 0] = math.tan(get_aug_params(shear) * math.pi / 180)
    translation_m = np.eye(3)
    translation_m[0, 2] = get_aug_params(translate, center=0.5) * target_size[1]
    translation_m[1, 2] = get_aug_params(translate, center=0.5) * target_size[0]
    return (translation_m @ shear_m @ rotation_m @ center_m)[:2]


def apply_affine_to_bboxes(targets: np.ndarray, target_size, M: np.ndarray) -> np.ndarray:
    """Corner warp of xyxy boxes (no segments), then the clip to target_size = (w, h) as the reference passes it."""
    n = len(targets)
    if n == 0:
        return targets
    twidth, theight = target_size
    corners = np.ones((n * 4, 3))
    corners[:, :2] = targets[:, [0, 1, 2, 3, 0, 3, 2, 1]].reshape(n * 4, 2)
    corners = (corners @ M.T).reshape(n, 8)
    xs, ys = corners[:, 0::2], corners[:, 1::2]
    targets[:, :4] = np.concatenate((np.min(xs, 1), np.min(ys, 1), np.max(xs, 1), np.max(ys, 1))).reshape(4, -1).T
    targets[:, [0, 2]] = targets[:, [0, 2]].clip(0, twidth)
    targets[:, [1, 3]] = targets[:, [1, 3]].clip(0, theight)
    return targets


def filter_box_candidates(original: np.ndarray, transformed: np.ndarray, wh_thr=2, ar_thr=20, area_thr=0.1) -> np.ndarray:
    original, transformed = original.T, transformed.T
    w1, h1 = original[2] - original[0], original[3] - original[1]
    w2, h2 = transformed[2] - transformed[0], transformed[3] - transformed[1]
    ar = np.maximum(w2 / (h2 + 1e-16), h2 / (w2 + 1e-16))
    return (w2 > wh_thr) & (h2 > wh_thr) & (w2 * h2 / (w1 * h1 + 1e-16) > area_thr) & (ar < ar_thr)


def _affine_targets(targets, target_size, M, filt, wh_thr, ar_thr, area_thr):
    if len(targets) == 0:
        return targets
    orig = targets.copy()
    targets = apply_affine_to_bboxes(targets, target_size, M)
    if filt:
        targets = targets[filter_box_candidates(orig[:, :4], targets[:, :4], wh_thr=wh_thr, ar_thr=ar_thr, area_thr=area_thr)]
    return targets


@register_transform()
class DetectionRandomAffine(_Transform):
    def __init__(self, degrees=10, translate=0.1, scales=0.1, shear=10, target_size=(640, 640), filter_box_candidates: bool = False, wh_thr: float = 2,
                 ar_thr: float = 20, area_thr: float = 0.1, border_value: int = 114):  # fmt: skip
        self.degrees, self.translate, self.scale, self.shear = degrees, translate, scales, shear
        self.target_size = _tuple_of_two(target_size)
        self.enable = True
        self.filter_box_candidates, self.wh_thr, self.ar_thr, self.area_thr = filter_box_candidates, wh_thr, ar_thr, area_thr
        self.border_value = border_value

    def close(self):
        self.enable = False

    def apply_to_sample(self, sample: HostSample) -> HostSample:
        if not self.enable:
            return sample
        crowd = sample.is_crowd > 0
        crowd_targets = np.concatenate([sample.bboxes_xyxy[crowd], sample.labels[crowd, None]], axis=1)
        targets = np.concatenate([sample.bboxes_xyxy[~crowd], sample.labels[~crowd, None]], axis=1)
        target_size = self.target_size or tuple(sample.shape)
        M = get_affine_matrix(sample.shape, target_size, self.degrees, self.translate, self.scale, self.shear)
        rows, cols = target_size[:2]
        args = (target_size, M, self.filter_box_candidates, self.wh_thr, self.ar_thr, self.area_thr)
        targets, crowd_targets = _affine_targets(targets, *args), _affine_targets(crowd_targets, *args)
        sample.plan.affine = (M, (rows, cols), int(self.border_value))
        is_crowd = np.array([0] * len(targets) + [1] * len(crowd_targets), dtype=bool)
        boxes = np.concatenate([targets[:, 0:4], crowd_targets[:, 0:4]], axis=0, dtype=sample.bboxes_xyxy.dtype)
        labels = np.concatenate([targets[:, 4], crowd_targets[:, 4]], axis=0, dtype=sample.labels.dtype)
        return sample.replaced(shape=(rows, cols), bboxes_xyxy=boxes, labels=labels, is_crowd=is_crowd)


@register_transform()
class DetectionRGB2BGR(_Transform):
    def __init__(self, prob: float = 0.5):
        self.prob = float(prob)

    def apply_to_sample(self, sample: HostSample) -> HostSample:
        if random.random() < self.prob:
            sample.plan.swap = not sample.plan.swap
            sample = sample.replaced()
        return sample


@register_transform()
class DetectionHSV(_Transform):
    def __init__(self, prob: float, hgain: float = 0.5, sgain: float = 0.5, vgain: float = 0.5, bgr_channels=(0, 1, 2)):
        self.prob, self.hgain, self.sgain, self.vgain = prob, hgain, sgain, vgain
        self.bgr_channels = tuple(int(c) for c in bgr_channels)
        if sorted(self.bgr_channels) != [0, 1, 2]:
            raise ValueError(f"bgr_channels must be a permutation of (0, 1, 2) for 3-channel images, got {bgr_channels}")

    def apply_to_sample(self, sample: HostSample) -> HostSample:
        if random.random() < self.prob:
            gains = np.random.uniform(-1, 1, 3) * [self.hgain, self.sgain, self.vgain]
            gains *= np.random.randint(0, 2, 3)
            g = gains.astype(np.int16)
            sample.plan.hsv = (int(g[0]), int(g[1]), int(g[2]), self.bgr_channels)
            sample = sample.replaced()
        return sample


@register_transform()
class DetectionHorizontalFlip(_Transform):
    def __init__(self, prob: float):
        self.prob = float(prob)

    def apply_to_sample(self, sample: HostSample) -> HostSample:
        if random.random() < self.prob:
            boxes = sample.bboxes_xyxy
            boxes[..., [0, 2]] = sample.shape[1] - boxes[..., [2, 0]]
            sample.plan.flip = True
            sample = sample.replaced(bboxes_xyxy=boxes)
        return sample


@register_transform()
class DetectionMixup(_Transform):
    def __init__(self, input_dim, mixup_scale: tuple, prob: float = 1.0, enable_mixup: bool = True, flip_prob: float = 0.5, border_value: int = 114):
        self.input_dim = _tuple_of_two(input_dim)
        self.mixup_scale, self.prob, self.enable_mixup, self.flip_prob, self.border_value = mixup_scale, prob, enable_mixup, flip_prob, border_value
        self.non_empty_targets = True

    def close(self):
        self.enable_mixup = False

    def get_number_of_additional_samples(self) -> int:
        return int(self.enable_mixup and random.random() < self.prob)

    @property
    def may_require_additional_samples(self) -> bool:
        return self.enable_mixup

    def apply_to_sample(self, sample: HostSample) -> HostSample:
        if not sample.additional_samples or not self.enable_mixup:
            return sample
        (cp,) = sample.additional_samples
        target_dim = self.input_dim if self.input_dim is not None else sample.shape
        flip = random.random() < self.flip_prob
        cp_boxes = cp.bboxes_xyxy
        if flip:
            cp_boxes[..., [0, 2]] = cp.shape[1] - cp_boxes[..., [2, 0]]
            cp = cp.replaced(bboxes_xyxy=cp_boxes)
        jit_factor = random.uniform(*self.mixup_scale)
        ratio = min(target_dim[0] / cp.shape[0], target_dim[1] / cp.shape[1])
        resized = (int(cp.shape[0] * ratio), int(cp.shape[1] * ratio))
        jittered = (int(target_dim[0] * jit_factor), int(target_dim[1] * jit_factor))
        ratio *= jit_factor
        origin_h, origin_w = jittered
        target_h, target_w = sample.shape
        ph, pw = max(origin_h, target_h), max(origin_w, target_w)
        x_offset, y_offset = 0, 0
        if ph > target_h:
            y_offset = random.randint(0, ph - target_h - 1)
        if pw > target_w:
            x_offset = random.randint(0, pw - target_w - 1)
        boxes = clip_boxes_inplace(cp.bboxes_xyxy[:, :4].copy() * ratio + np.array([[0, 0, 0, 0]]), (origin_h, origin_w))
        boxes = boxes.copy()
        boxes[:, [0, 2]] = boxes[:, [0, 2]] - x_offset
        boxes[:, [1, 3]] = boxes[:, [1, 3]] - y_offset
        boxes = clip_boxes_inplace(boxes, (target_h, target_w))
        sample.plan.mixup = MixupPlan(cp.plan.image, flip, resized, tuple(target_dim), jittered, x_offset, y_offset, int(self.border_value))
        return sample.replaced(bboxes_xyxy=np.concatenate([sample.bboxes_xyxy, boxes], axis=0), labels=np.concatenate([sample.labels, cp.labels], axis=0),
                               is_crowd=np.concatenate([sample.is_crowd, cp.is_crowd], axis=0))  # fmt: skip


@register_transform()
class DetectionPaddedRescale(_Transform):
    def __init__(self, input_dim, swap: Tuple[int, ...] = (2, 0, 1), max_targets: Optional[int] = None, pad_value: int = 114):
        self.swap, self.input_dim, self.pad_value = swap, _tuple_of_two(input_dim), pad_value
        if tuple(swap) != (2, 0, 1):
            raise ValueError("the model input is written channels-first (swap=(2, 0, 1)); other layouts are not supported")

    def apply_to_sample(self, sample: HostSample) -> HostSample:
        r = min(self.input_dim[0] / sample.shape[0], self.input_dim[1] / sample.shape[1])
        sample.plan.rescaled = (int(sample.shape[0] * r), int(sample.shape[1] * r))
        boxes = sample.bboxes_xyxy.astype(np.float32, copy=True)
        boxes[:, :4] *= np.array([[r, r, r, r]], dtype=boxes.dtype)
        sample.bboxes_xyxy = boxes
        sample.shape = self.input_dim
        return sample


@register_transform()
class DetectionPadToSize(_Transform):
    """Center padding to output_size (rows, cols) without a rescale (DetectionPadIfNeeded in "center" mode, detection_pad_if_needed.py);
    the boxes move by the pad's top-left offsets.  The pixels are the kernel's affine step with the integer translation
    (pad_left, pad_top), whose border is the pad value: cv2's fixed-point warp reads every output pixel from exactly one source pixel
    there.  An image larger than output_size would make the reference's output larger than output_size, so it raises ValueError."""

    def __init__(self, output_size, pad_value):
        self.output_size = _tuple_of_two(output_size)
        values = [pad_value] if isinstance(pad_value, Number) else list(pad_value)
        if len(set(values)) != 1 or not float(values[0]).is_integer() or not 0 <= values[0] <= 255:
            raise ValueError(f"pad_value must be one integer in [0, 255] (or the same one for every channel), got {pad_value}")
        self.pad_value = int(values[0])

    def apply_to_sample(self, sample: HostSample) -> HostSample:
        (h, w), (oh, ow) = sample.shape, self.output_size
        if h > oh or w > ow:
            raise ValueError(f"DetectionPadToSize({self.output_size}) received a {h}x{w} image: the GPU path writes a fixed {oh}x{ow} batch")
        top, left = (oh - h) // 2, (ow - w) // 2
        sample.plan.affine = (np.array([[1.0, 0.0, left], [0.0, 1.0, top]]), (oh, ow), self.pad_value)
        sample.plan.rescaled = (oh, ow)
        boxes = sample.bboxes_xyxy[:, :4].copy()  # _shift_bboxes_xyxy (transforms/utils.py)
        boxes[:, [0, 2]] += left
        boxes[:, [1, 3]] += top
        return sample.replaced(shape=(oh, ow), bboxes_xyxy=np.concatenate((boxes, sample.bboxes_xyxy[:, 4:]), 1))


@register_transform()
class DetectionImagePermute(_Transform):
    """HWC -> CHW of the reference's image; the kernel writes the NHWC model input, so only the default dims (2, 0, 1) are accepted."""

    def __init__(self, dims=(2, 0, 1)):
        if tuple(dims) != (2, 0, 1):
            raise ValueError(f"only dims (2, 0, 1) are supported on the GPU path, got {dims}")

    def apply_to_sample(self, sample: HostSample) -> HostSample:
        return sample


@register_transform()
class DetectionStandardize(_Transform):
    def __init__(self, max_value: float = 255.0):
        self.max_value = float(max_value)

    def apply_to_sample(self, sample: HostSample) -> HostSample:
        return sample


@register_transform()
class DetectionTargetsFormatTransform(_Transform):
    """The recipe's form only: XYXY_LABEL in, LABEL_CXCYWH out (pixels), boxes with an edge <= min_bbox_edge_size dropped."""

    def __init__(self, input_dim=None, input_format="XYXY_LABEL", output_format="LABEL_CXCYWH", min_bbox_edge_size: float = 1, max_targets: Optional[int] = None):
        if str(input_format) != "XYXY_LABEL" or str(output_format) != "LABEL_CXCYWH":
            raise ValueError("only input_format XYXY_LABEL and output_format LABEL_CXCYWH are supported")
        self.min_bbox_edge_size = min_bbox_edge_size

    def apply_to_sample(self, sample: HostSample) -> HostSample:
        return sample

    def apply_on_targets(self, targets: np.ndarray) -> np.ndarray:
        keep = np.minimum(targets[:, 2] - targets[:, 0], targets[:, 3] - targets[:, 1]) > self.min_bbox_edge_size
        t = targets[keep]
        x1, y1, x2, y2 = t[..., 0], t[..., 1], t[..., 2], t[..., 3]
        w, h = x2 - x1, y2 - y1
        out = np.concatenate([t[:, 4:5], np.stack([x1 + 0.5 * w, y1 + 0.5 * h, w, h], axis=-1)], axis=-1)
        return np.ascontiguousarray(out, dtype=np.float32)


def check_order(transforms) -> None:
    """The kernel applies the pixel steps in the recipe's order: each transform may appear once, in that order."""
    names = [type(t).__name__ for t in transforms]
    for n in names:
        if n not in RECIPE_ORDER:
            raise ValueError(f"{n} has no GPU pixel path; supported: {RECIPE_ORDER}")
    pos = [RECIPE_ORDER.index(n) for n in names]
    if pos != sorted(set(pos)):
        raise ValueError(f"the transforms must appear at most once each and in the order {RECIPE_ORDER}, got {names}")
    if "DetectionPaddedRescale" not in names and "DetectionPadToSize" not in names:
        raise ValueError("DetectionPaddedRescale or DetectionPadToSize must be in the pipeline: it fixes the model input size")
    if "DetectionPadToSize" in names and any(n in PAD_TO_SIZE_EXCLUDES for n in names):
        raise ValueError(f"DetectionPadToSize combines only with DetectionRGB2BGR, DetectionStandardize, DetectionImagePermute and "
                         f"DetectionTargetsFormatTransform, got {names}")  # fmt: skip
