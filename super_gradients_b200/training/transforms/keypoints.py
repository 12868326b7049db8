"""The YOLO-NAS-POSE train transforms (reference: training/transforms/keypoints/*.py, KeypointsCompose._apply_transforms,
samples/pose_estimation_sample.py), split in two halves.

On the host, in DataLoader workers, each transform draws its random numbers from the global `random` / `np.random` in the
reference's order and transforms the joints, boxes, areas and crowd flags with the reference's numpy arithmetic.  The pixels are
not touched: every transform records its draws in the sample's `PosePlan`, and the batch is later turned into the model input by
csrc/pose_augment.cu.  The kernels apply the steps in POSE_ORDER, so a pipeline must list these transforms in that order
(`check_pose_pipeline`).  The only pixel statistic the host computes is KeypointsBrightnessContrast's channel mean, with the reference's
own expression: numpy's float32 sum depends on the pixel order, which no other order reproduces."""
import random
from typing import Iterable, List, Optional

import cv2
import numpy as np

from ...common.registry import register_transform
from .keypoints_augment import PosePlan, colour

POSE_ORDER = ("KeypointsRandomHorizontalFlip", "KeypointsBrightnessContrast", "KeypointsReverseImageChannels", "KeypointsHSV", "KeypointsRandomRotate90",
              "KeypointsRandomAffineTransform", "KeypointsMosaic", "KeypointsLongestMaxSize", "KeypointsPadIfNeeded", "KeypointsImageStandardize",
              "KeypointsRemoveSmallObjects")  # fmt: skip


def xywh_to_xyxy(b: np.ndarray) -> np.ndarray:
    return np.stack([b[..., 0], b[..., 1], b[..., 0] + b[..., 2], b[..., 1] + b[..., 3]], axis=-1)


def xyxy_to_xywh(b: np.ndarray) -> np.ndarray:
    return np.stack([b[..., 0], b[..., 1], b[..., 2] - b[..., 0], b[..., 3] - b[..., 1]], axis=-1)


class PoseHostSample:
    """The reference's PoseEstimationSample without pixels or mask: the current image shape (h, w), joints [N, J, 3], areas [N]
    or None, boxes [N, 4] xywh or None, crowd flags [N], the plan of the pixel work and the additional samples of a mosaic."""

    def __init__(self, plan: PosePlan, shape, joints, areas, bboxes_xywh, is_crowd, additional_samples=None):
        self.plan, self.shape = plan, (int(shape[0]), int(shape[1]))
        self.joints, self.areas, self.bboxes_xywh, self.is_crowd = joints, areas, bboxes_xywh, is_crowd
        self.additional_samples: Optional[List["PoseHostSample"]] = additional_samples

    @classmethod
    def from_sample(cls, sample) -> "PoseHostSample":
        """From a PoseEstimationSample-like object (image uint8 H x W x 3, joints, areas, bboxes_xywh, is_crowd)."""
        image = sample.image
        if not isinstance(image, np.ndarray) or image.dtype != np.uint8 or image.ndim != 3 or image.shape[2] != 3:
            raise ValueError(f"samples must hold a uint8 H x W x 3 image, got {getattr(image, 'dtype', type(image))} {getattr(image, 'shape', '')}")
        return cls(PosePlan.single(image), image.shape[:2], sample.joints, sample.areas, sample.bboxes_xywh, sample.is_crowd)

    @property
    def tile(self):
        return self.plan.tiles[0]

    def sanitize_sample(self) -> "PoseHostSample":
        h, w = self.shape
        outside = (self.joints[:, :, 0] < 0) | (self.joints[:, :, 1] < 0) | (self.joints[:, :, 0] >= w) | (self.joints[:, :, 1] >= h)
        self.joints[outside, 2] = 0
        if self.bboxes_xywh is not None:
            boxes = xywh_to_xyxy(self.bboxes_xywh)
            boxes[..., [0, 2]] = boxes[..., [0, 2]].clip(min=0, max=w)
            boxes[..., [1, 3]] = boxes[..., [1, 3]].clip(min=0, max=h)
            boxes = xyxy_to_xywh(boxes)
            if self.areas is not None:
                self.areas = self.areas * (boxes[..., 2:4].prod(axis=-1) / (self.bboxes_xywh[..., 2:4].prod(axis=-1) + 1e-6))
            self.bboxes_xywh = boxes
        return self

    def filter_by_mask(self, keep) -> "PoseHostSample":
        self.joints, self.is_crowd = self.joints[keep], self.is_crowd[keep]
        if self.bboxes_xywh is not None:
            self.bboxes_xywh = self.bboxes_xywh[keep]
        if self.areas is not None:
            self.areas = self.areas[keep]
        return self

    @staticmethod
    def joints_box_area(joints) -> np.ndarray:
        vis = joints[:, :, 2] > 0
        xmax = np.max(joints[:, :, 0], axis=-1, where=vis, initial=joints[:, :, 0].min())
        xmin = np.min(joints[:, :, 0], axis=-1, where=vis, initial=joints[:, :, 0].max())
        ymax = np.max(joints[:, :, 1], axis=-1, where=vis, initial=joints[:, :, 1].min())
        ymin = np.min(joints[:, :, 1], axis=-1, where=vis, initial=joints[:, :, 1].max())
        return np.clip((xmax - xmin) * (ymax - ymin), a_min=0, a_max=None) * (vis.sum(axis=-1, keepdims=False) > 1)


class _Transform:
    def get_number_of_additional_samples(self) -> int:
        return 0

    @property
    def may_require_additional_samples(self) -> bool:
        return False


@register_transform()
class KeypointsRandomHorizontalFlip(_Transform):
    def __init__(self, flip_index: List[int], prob: float = 0.5):
        self.flip_index, self.prob = flip_index, prob

    def apply_to_sample(self, sample: PoseHostSample) -> PoseHostSample:
        if random.random() < self.prob:
            sample.tile.flip = True
            cols = sample.shape[1]
            joints = sample.joints.copy()[:, self.flip_index]
            joints[:, :, 0] = cols - joints[:, :, 0] - 1
            sample.joints = joints
            if sample.bboxes_xywh is not None:
                boxes = sample.bboxes_xywh.copy()
                boxes[:, 0] = cols - (boxes[:, 0] + boxes[:, 2])
                sample.bboxes_xywh = boxes
        return sample


@register_transform()
class KeypointsBrightnessContrast(_Transform):
    def __init__(self, prob: float, brightness_range, contrast_range):
        if len(brightness_range) != 2:
            raise ValueError("Brightness range must be a tuple of two elements, got: " + str(brightness_range))
        if len(contrast_range) != 2:
            raise ValueError("Contrast range must be a tuple of two elements, got: " + str(contrast_range))
        self.prob, self.brightness_range, self.contrast_range = prob, tuple(brightness_range), tuple(contrast_range)

    def apply_to_sample(self, sample: PoseHostSample) -> PoseHostSample:
        if random.random() < self.prob:
            contrast_gain = random.uniform(self.contrast_range[0], self.contrast_range[1])
            brightness_gain = random.uniform(self.brightness_range[0], self.brightness_range[1])
            t = sample.tile
            image = np.ascontiguousarray(np.fliplr(t.image)) if t.flip else t.image  # the image the reference averages
            t.bc = (np.mean(image.astype(np.float32), axis=(0, 1)), contrast_gain, brightness_gain)
        return sample


@register_transform()
class KeypointsReverseImageChannels(_Transform):
    def __init__(self, prob: float):
        self.prob = prob

    def apply_to_sample(self, sample: PoseHostSample) -> PoseHostSample:
        if random.random() < self.prob:
            sample.tile.reverse = True
        return sample


@register_transform()
class KeypointsHSV(_Transform):
    def __init__(self, prob: float, hgain: float, sgain: float, vgain: float):
        self.prob, self.hgain, self.sgain, self.vgain = prob, hgain, sgain, vgain

    def apply_to_sample(self, sample: PoseHostSample) -> PoseHostSample:
        if random.random() < self.prob:  # augment_hsv's draws
            gains = np.random.uniform(-1, 1, 3) * [self.hgain, self.sgain, self.vgain]
            gains *= np.random.randint(0, 2, 3)
            g = gains.astype(np.int16)
            sample.tile.hsv = (int(g[0]), int(g[1]), int(g[2]))
        return sample


@register_transform()
class KeypointsRandomRotate90(_Transform):
    def __init__(self, prob: float = 0.5):
        self.prob = prob

    def apply_to_sample(self, sample: PoseHostSample) -> PoseHostSample:
        if random.random() < self.prob:
            factor = random.randint(0, 3)
            rows, cols = sample.shape
            sample.tile.rot = factor
            x, y, v = sample.joints[:, :, 0], sample.joints[:, :, 1], sample.joints[:, :, 2]
            sample.joints = np.stack([(x, y, v), (y, cols - x - 1, v), (cols - x - 1, rows - y - 1, v), (rows - y - 1, x, v)][factor], axis=-1)
            if sample.bboxes_xywh is not None:
                b = xywh_to_xyxy(sample.bboxes_xywh)
                x0, y0, x1, y1 = b[:, 0], b[:, 1], b[:, 2], b[:, 3]
                b = [(x0, y0, x1, y1), (y0, cols - x1, y1, cols - x0), (cols - x1, rows - y1, cols - x0, rows - y0), (rows - y1, x0, rows - y0, x1)][factor]
                sample.bboxes_xywh = xyxy_to_xywh(np.stack(b, axis=1))
            sample.shape = (cols, rows) if factor % 2 else (rows, cols)
            sample.plan.canvas = sample.shape
        return sample


@register_transform()
class KeypointsRandomAffineTransform(_Transform):
    def __init__(self, max_rotation: float, min_scale: float, max_scale: float, max_translate: float, image_pad_value, mask_pad_value: float,
                 interpolation_mode=cv2.INTER_LINEAR, prob: float = 0.5):  # fmt: skip
        self.max_rotation, self.min_scale, self.max_scale, self.max_translate = max_rotation, min_scale, max_scale, max_translate
        self.image_pad_value, self.mask_pad_value, self.prob = image_pad_value, mask_pad_value, prob
        self.interpolation_mode = tuple(interpolation_mode) if isinstance(interpolation_mode, Iterable) else (interpolation_mode,)
        if any(int(m) not in (0, 1, 2, 3, 4) for m in self.interpolation_mode):
            raise ValueError(f"interpolation_mode must be among cv2's INTER_NEAREST .. INTER_LANCZOS4 (0 .. 4), got {interpolation_mode}")
        self.border = colour(image_pad_value)

    def apply_to_sample(self, sample: PoseHostSample) -> PoseHostSample:
        if random.random() < self.prob:
            angle = random.uniform(-self.max_rotation, self.max_rotation)
            scale = random.uniform(self.min_scale, self.max_scale)
            dx = random.uniform(-self.max_translate, self.max_translate)
            dy = random.uniform(-self.max_translate, self.max_translate)
            interpolation = random.choice(self.interpolation_mode)
            height, width = sample.shape
            mat = cv2.getRotationMatrix2D((width / 2 + dx * width, height / 2 + dy * height), angle, scale)[:2]
            sample.tile.affine = (mat, int(interpolation), self.border)
            kp = sample.joints.copy()
            xy = kp[:, :, 0:2]
            shape, dtype = xy.shape, xy.dtype
            xy = xy.reshape(-1, 2)
            xy = np.dot(np.concatenate((xy, xy[:, 0:1] * 0 + 1), axis=1), mat.T).reshape(shape)
            outside = (xy[:, :, 0] < 0) | (xy[:, :, 1] < 0) | (xy[:, :, 0] >= width) | (xy[:, :, 1] >= height)
            kp[:, :, 0:2] = xy
            kp[outside, 2] = 0
            sample.joints = kp.astype(dtype, copy=False)
            if sample.bboxes_xywh is not None and len(sample.bboxes_xywh):
                out = []
                for box in xywh_to_xyxy(sample.bboxes_xywh):
                    x_min, y_min, x_max, y_max = box[:4]
                    pts = np.vstack([np.array([x_min, x_max, x_max, x_min]), np.array([y_min, y_min, y_max, y_max]), np.ones(4)]).transpose()
                    tr = mat.dot(pts.T).T
                    out.append(np.array([min(tr[:, 0]), min(tr[:, 1]), max(tr[:, 0]), max(tr[:, 1])]))
                sample.bboxes_xywh = xyxy_to_xywh(np.array(out)).astype(sample.bboxes_xywh.dtype)
            if sample.areas is not None:
                sample.areas = (sample.areas * abs(np.linalg.det(mat[:2, :2]))).astype(sample.areas.dtype)
            sample = sample.sanitize_sample()
        return sample


def _concat(a, b, shape_if_empty):
    if a is None and b is None:
        return None
    a = np.zeros(shape_if_empty, dtype=np.float32) if a is None else a
    b = np.zeros(shape_if_empty, dtype=np.float32) if b is None else b
    return np.concatenate([a, b], axis=0)


@register_transform()
class KeypointsMosaic(_Transform):
    def __init__(self, prob: float, pad_value=(127, 127, 127)):
        self.prob, self.pad_value = prob, tuple(pad_value)
        self.colour = colour(self.pad_value)

    def get_number_of_additional_samples(self) -> int:
        return 3 if random.random() < self.prob else 0

    @property
    def may_require_additional_samples(self) -> bool:
        return True

    def apply_to_sample(self, sample: PoseHostSample) -> PoseHostSample:
        if sample.additional_samples is None or len(sample.additional_samples) == 0:
            return sample
        for s in [sample] + sample.additional_samples:
            if len(s.plan.tiles) != 1:
                raise ValueError("a mosaic tile cannot itself be a mosaic")
        tl, tr, bl, br = [sample] + sample.additional_samples
        out = self._stack_v(self._stack_h(tl, tr, True), self._stack_h(bl, br, False))
        out.plan = PosePlan([s.tile for s in (tl, tr, bl, br)], [tuple(p) for p in out.positions], out.shape, self.colour)
        del out.positions
        return out

    @staticmethod
    def _pad(s, top=0, left=0, bottom=0, right=0):
        s.joints[:, :, 0] += left
        s.joints[:, :, 1] += top
        s.bboxes_xywh[:, 0] += left
        s.bboxes_xywh[:, 1] += top
        s.shape = (s.shape[0] + top + bottom, s.shape[1] + left + right)
        s.positions = [[y + top, x + left] for y, x in s.positions]
        return s

    def _stack_h(self, left, right, pad_from_top):
        for s in (left, right):
            if not hasattr(s, "positions"):
                s.positions = [[0, 0]]
        hmax = max(left.shape[0], right.shape[0])
        if pad_from_top:
            left, right = self._pad(left, top=hmax - left.shape[0]), self._pad(right, top=hmax - right.shape[0])
        else:
            left, right = self._pad(left, bottom=hmax - left.shape[0]), self._pad(right, bottom=hmax - right.shape[0])
        lw = left.shape[1]
        rb = right.bboxes_xywh if right.bboxes_xywh is not None else np.zeros((0, 4), dtype=np.float32)
        joints = np.concatenate([left.joints, right.joints + np.array([lw, 0, 0], dtype=right.joints.dtype).reshape((1, 1, 3))], axis=0)
        boxes = _concat(left.bboxes_xywh, rb + np.array([lw, 0, 0, 0], dtype=rb.dtype).reshape((1, 4)), (0, 4))
        s = PoseHostSample(None, (hmax, lw + right.shape[1]), joints, _concat(left.areas, right.areas, (0,)), boxes,
                           np.concatenate([left.is_crowd, right.is_crowd], axis=0))  # fmt: skip
        s.positions = left.positions + [[y, x + lw] for y, x in right.positions]
        return s

    def _stack_v(self, top, bottom):
        wmax = max(top.shape[1], bottom.shape[1])
        pl = (wmax - top.shape[1]) // 2
        top = self._pad(top, left=pl, right=wmax - top.shape[1] - pl)
        pl = (wmax - bottom.shape[1]) // 2
        bottom = self._pad(bottom, left=pl, right=wmax - bottom.shape[1] - pl)
        th = top.shape[0]
        bb = bottom.bboxes_xywh if bottom.bboxes_xywh is not None else np.zeros((0, 4), dtype=np.float32)
        joints = np.concatenate([top.joints, bottom.joints + np.array([0, th, 0], dtype=bottom.joints.dtype).reshape((1, 1, 3))], axis=0)
        boxes = _concat(top.bboxes_xywh, bb + np.array([0, th, 0, 0], dtype=bb.dtype).reshape((1, 4)), (0, 4))
        s = PoseHostSample(None, (th + bottom.shape[0], wmax), joints, _concat(top.areas, bottom.areas, (0,)), boxes,
                           np.concatenate([top.is_crowd, bottom.is_crowd], axis=0))  # fmt: skip
        s.positions = top.positions + [[y + th, x] for y, x in bottom.positions]
        return s


@register_transform()
class KeypointsLongestMaxSize(_Transform):
    def __init__(self, max_height: int, max_width: int, interpolation: int = cv2.INTER_LINEAR, prob: float = 1.0):
        self.max_height, self.max_width, self.interpolation, self.prob = max_height, max_width, interpolation, prob

    def apply_to_sample(self, sample: PoseHostSample) -> PoseHostSample:
        if random.random() < self.prob:
            height, width = sample.shape
            scale = min(self.max_height / height, self.max_width / width)
            if scale != 1.0:
                sample.shape = (int(height * scale + 0.5), int(width * scale + 0.5))
            sample.plan.resized = sample.shape
            if sample.shape[0] != self.max_height and sample.shape[1] != self.max_width:
                raise RuntimeError(f"Image shape is not as expected (scale={scale}, input_shape={height, width}, resized_shape={sample.shape})")
            if sample.shape[0] > self.max_height or sample.shape[1] > self.max_width:
                raise RuntimeError(f"Image shape is not as expected (scale={scale}, input_shape={height, width}, resized_shape={sample.shape}")
            joints = sample.joints.astype(np.float32, copy=True)
            joints[:, :, 0:2] *= scale
            sample.joints = joints
            if sample.bboxes_xywh is not None:
                sample.bboxes_xywh = np.multiply(sample.bboxes_xywh, scale, dtype=np.float32)
            if sample.areas is not None:
                sample.areas = np.multiply(sample.areas, scale**2, dtype=np.float32)
        return sample


@register_transform()
class KeypointsPadIfNeeded(_Transform):
    def __init__(self, min_height: int, min_width: int, image_pad_value, mask_pad_value: float, padding_mode: str = "bottom_right"):
        if padding_mode not in ("bottom_right", "center"):
            raise ValueError(f"Unknown padding mode: {padding_mode}. Supported modes: 'bottom_right', 'center'")
        self.min_height, self.min_width, self.image_pad_value, self.mask_pad_value, self.padding_mode = min_height, min_width, image_pad_value, mask_pad_value, padding_mode
        self.colour = colour(image_pad_value)

    def apply_to_sample(self, sample: PoseHostSample) -> PoseHostSample:
        height, width = sample.shape
        if self.padding_mode == "bottom_right":
            pad_left = pad_top = 0
        else:
            pad_left, pad_top = max(0, (self.min_width - width) // 2), max(0, (self.min_height - height) // 2)
        pad_bottom, pad_right = max(0, self.min_height - height - pad_top), max(0, self.min_width - width - pad_left)
        sample.plan.pad, sample.plan.pad_value = (pad_top, pad_left), self.colour
        sample.shape = (height + pad_top + pad_bottom, width + pad_left + pad_right)
        joints = sample.joints.copy()
        joints[:, :, 0] += pad_left
        joints[:, :, 1] += pad_top
        sample.joints = joints
        if sample.bboxes_xywh is not None:
            boxes = sample.bboxes_xywh.copy()
            boxes[:, 0] += pad_left
            boxes[:, 1] += pad_top
            sample.bboxes_xywh = boxes
        return sample


@register_transform()
class KeypointsImageStandardize(_Transform):
    def __init__(self, max_value: float = 255.0):
        self.max_value = max_value

    def apply_to_sample(self, sample: PoseHostSample) -> PoseHostSample:
        return sample


@register_transform()
class KeypointsRemoveSmallObjects(_Transform):
    def __init__(self, min_visible_keypoints: int = 0, min_instance_area: int = 0, min_bbox_area: int = 0):
        self.min_visible_keypoints, self.min_instance_area, self.min_bbox_area = min_visible_keypoints, min_instance_area, min_bbox_area

    def apply_to_sample(self, sample: PoseHostSample) -> PoseHostSample:
        if self.min_visible_keypoints:
            sample = sample.filter_by_mask(np.sum(sample.joints[:, :, 2] > 0, axis=-1) >= self.min_visible_keypoints)
        if self.min_instance_area:
            if sample.areas is not None:
                areas = sample.areas
            elif sample.bboxes_xywh is not None:
                areas = sample.bboxes_xywh[..., 2:4].prod(axis=-1, keepdims=False) * 0.53
            else:
                areas = PoseHostSample.joints_box_area(sample.joints)
            sample = sample.filter_by_mask(areas >= self.min_instance_area)
        if self.min_bbox_area:
            area = PoseHostSample.joints_box_area(sample.joints) if sample.bboxes_xywh is None else sample.bboxes_xywh[..., 2:4].prod(axis=-1)
            sample = sample.filter_by_mask(area >= self.min_bbox_area)
        return sample


def check_pose_pipeline(transforms) -> int:
    """The kernels apply the pixel steps in POSE_ORDER: each transform at most once, in that order, ending in a fixed S x S output
    (KeypointsLongestMaxSize with prob >= 1 into KeypointsPadIfNeeded's min_height == min_width == S).  Returns S."""
    names = [type(t).__name__ for t in transforms]
    for n in names:
        if n not in POSE_ORDER:
            raise ValueError(f"{n} has no GPU pixel path; supported: {POSE_ORDER}")
    pos = [POSE_ORDER.index(n) for n in names]
    if pos != sorted(set(pos)):
        raise ValueError(f"the transforms must appear at most once each and in the order {POSE_ORDER}, got {names}")
    by = {type(t).__name__: t for t in transforms}
    lms, pad = by.get("KeypointsLongestMaxSize"), by.get("KeypointsPadIfNeeded")
    if lms is None or pad is None or lms.prob < 1 or pad.min_height != pad.min_width or lms.max_height > pad.min_height or lms.max_width > pad.min_width:
        raise ValueError("KeypointsLongestMaxSize (prob 1) and KeypointsPadIfNeeded (min_height == min_width, at least the max size) must fix an S x S output")
    if "KeypointsImageStandardize" not in by:
        raise ValueError("KeypointsImageStandardize must be in the pipeline: the model input is written standardized")
    return int(pad.min_height)
