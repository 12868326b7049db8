"""predict() pre/post-processing on the GPU (SURVEY.md section 8(f) N3).  Same class names, constructor arguments and order of
operations as the reference's training/processing/processing.py, but a ComposeProcessing does not run five numpy / cv2 passes per
image on the host: it folds its chain into ONE kernel launch per image (csrc/preprocess.cu: OpenCV's fixed-point INTER_LINEAR
resize, constant padding, channel reversal, standardisation, mean / std, bf16 NHWC store straight into the batch tensor) and undoes
padding and rescaling on the prediction tensors with the reference's float32 arithmetic.

Supported chains, each step optional, in this order:
  detection (the YOLO-NAS / YOLO-NAS-POSE defaults, processing.py:960-980, 1060-1075): ReverseImageChannels, one *Rescale, one
  *Padding, StandardizeImage, NormalizeImage, ImagePermute((2, 0, 1)) -- one launch per image (csrc/preprocess.cu); for
  predict(skip_image_resizing=True) a DetectionAutoPadding first instead of the rescale and padding steps;
  classification (the ImageNet default, processing.py:1142-1151): ReverseImageChannels, Resize, CenterCrop, StandardizeImage,
  NormalizeImage, ImagePermute((2, 0, 1)) -- Pillow's antialiased bilinear resize evaluated inside the crop window, ONE launch per
  batch (csrc/resample.cu).
Anything else raises NotImplementedError."""
from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

from ... import kernels as K


@dataclass
class ImageGeometry:
    """Per-image record of what the chain did (the reference's RescaleMetadata + DetectionPadToSizeMetadata)."""

    original_shape: Tuple[int, int]
    scale_factor_h: float
    scale_factor_w: float
    resized_shape: Tuple[int, int]
    pad_top: int
    pad_left: int


class Processing:
    resizes_image = False


class ReverseImageChannels(Processing):
    pass


class StandardizeImage(Processing):
    def __init__(self, max_value: float = 255.0):
        self.max_value = float(max_value)


class NormalizeImage(Processing):
    def __init__(self, mean: List[float], std: List[float]):
        self.mean = np.array(mean, dtype=np.float32).reshape(-1)
        self.std = np.array(std, dtype=np.float32).reshape(-1)


class ImagePermute(Processing):
    def __init__(self, permutation: Tuple[int, int, int] = (2, 0, 1)):
        self.permutation = tuple(permutation)
        if self.permutation != (2, 0, 1):
            raise NotImplementedError("only the HWC -> CHW permutation (2, 0, 1) is supported")


class _Rescale(Processing):
    resizes_image = True
    keep_aspect = False

    def __init__(self, output_shape: Tuple[int, int]):
        self.output_shape = tuple(output_shape)

    def target(self, height: int, width: int):
        """-> (new_h, new_w, scale_h, scale_w) exactly as the reference computes them (processing.py:516-550)."""
        if self.keep_aspect:
            scale = min(self.output_shape[0] / height, self.output_shape[1] / width)
            if scale != 1.0:
                return round(height * scale), round(width * scale), scale, scale
            return height, width, scale, scale
        return self.output_shape[0], self.output_shape[1], self.output_shape[0] / height, self.output_shape[1] / width


class DetectionRescale(_Rescale):
    pass


class DetectionLongestMaxSizeRescale(_Rescale):
    keep_aspect = True


class KeypointsLongestMaxSizeRescale(DetectionLongestMaxSizeRescale):
    pass


class _Padding(Processing):
    resizes_image = True
    center = False

    def __init__(self, output_shape: Tuple[int, int], pad_value: int):
        self.output_shape = tuple(output_shape)
        self.pad_value = pad_value

    def top_left(self, height: int, width: int) -> Tuple[int, int]:
        pad_h, pad_w = self.output_shape[0] - height, self.output_shape[1] - width
        if pad_h < 0 or pad_w < 0:
            raise ValueError(f"image {height}x{width} is larger than the padded shape {self.output_shape}")
        return (pad_h // 2, pad_w // 2) if self.center else (0, 0)


class DetectionCenterPadding(_Padding):
    center = True


class DetectionBottomRightPadding(_Padding):
    pass


class KeypointsBottomRightPadding(DetectionBottomRightPadding):
    pass


class DetectionAutoPadding(Processing):
    """processing.py:443-470: pads bottom / right with `pad_value` up to the next multiple of `shape_multiple` (H, W); the image
    stays at the top-left corner.  In a chain it comes first (get_equivalent_compose_without_resizing).  Like the reference's
    AutoPadding (processing.py:128-130) it does not count as resizing."""

    resizes_image = False

    def __init__(self, shape_multiple: Tuple[int, int], pad_value: int):
        self.shape_multiple = tuple(shape_multiple)
        self.pad_value = pad_value

    def padded_shape(self, height: int, width: int) -> Tuple[int, int]:
        mh, mw = self.shape_multiple
        return ((height + mh - 1) // mh) * mh, ((width + mw - 1) // mw) * mw


class Resize(Processing):
    """processing.py:614-644: scales the shorter side to `size` with PIL's bilinear filter (no-op when the scale is exactly 1)."""

    resizes_image = True

    def __init__(self, size: int = 224):
        self.size = int(size)

    def target(self, height: int, width: int) -> Tuple[int, int, float]:
        """-> (new_h, new_w, scale) in Python float, as the reference computes them."""
        scale = max(self.size / height, self.size / width)
        if scale != 1.0:
            return int(height * scale), int(width * scale), scale
        return height, width, scale


class CenterCrop(Processing):
    """processing.py:647-680: the size x size window starting at ((H - size) // 2, (W - size) // 2).  A window larger than the image
    raises ValueError (the reference's numpy slicing returns a malformed image there)."""

    resizes_image = True

    def __init__(self, size: int = 224):
        self.size = int(size)

    def top_left(self, height: int, width: int) -> Tuple[int, int]:
        if height < self.size or width < self.size:
            raise ValueError(f"CenterCrop({self.size}) does not fit an image of {height}x{width}")
        return (height - self.size) // 2, (width - self.size) // 2


class ComposeProcessing(Processing):
    def __init__(self, processings: Sequence[Processing]):
        self.processings = list(processings)
        order = [DetectionAutoPadding, ReverseImageChannels, _Rescale, _Padding, Resize, CenterCrop, StandardizeImage, NormalizeImage, ImagePermute]
        pos = -1
        self.auto_padding = self.reverse = self.rescale = self.padding = self.resize = self.crop = self.standardize = self.normalize = None
        for p in self.processings:
            idx = next((i for i, t in enumerate(order) if isinstance(p, t)), None)
            if idx is None or idx <= pos:
                raise NotImplementedError(f"unsupported processing chain at {type(p).__name__}: supported order is [DetectionAutoPadding] [ReverseImageChannels] "
                                          "([Rescale] [Padding] | [Resize] [CenterCrop]) [StandardizeImage] [NormalizeImage] [ImagePermute]")  # fmt: skip
            pos = idx
            name = ("auto_padding", "reverse", "rescale", "padding", "resize", "crop", "standardize", "normalize", "permute")[idx]
            setattr(self, name, p)
        if self.auto_padding is not None and any(p is not None for p in (self.rescale, self.padding, self.resize, self.crop)):
            raise NotImplementedError("DetectionAutoPadding cannot be combined with a resizing or padding step")
        if (self.resize is not None or self.crop is not None) and (self.rescale is not None or self.padding is not None):
            raise NotImplementedError("Resize / CenterCrop (classification) cannot be combined with a detection Rescale / Padding step")
        if self.padding is None and self.rescale is not None and self.rescale.keep_aspect:
            raise NotImplementedError("an aspect-preserving rescale needs a padding step to give the batch one shape")
        self._staging = None  # pinned host buffer of the classification chain, reused while it is large enough
        self._staging_free = None  # event: the last copy out of the staging buffer has executed

    @property
    def resizes_image(self) -> bool:
        return any(p is not None for p in (self.rescale, self.padding, self.resize, self.crop))

    def get_equivalent_compose_without_resizing(self, auto_padding: DetectionAutoPadding) -> "ComposeProcessing":
        """processing.py:185-201: `auto_padding` first, then every step of this chain that does not resize the image."""
        return ComposeProcessing([auto_padding] + [p for p in self.processings if not p.resizes_image])

    def for_predict(self, skip_image_resizing: bool) -> "ComposeProcessing":
        """The chain a detector's predict() runs: this one, or with skip_image_resizing its equivalent without resizing behind
        DetectionAutoPadding((32, 32), 0) (the reference's _get_pipeline)."""
        if not skip_image_resizing:
            return self
        return self.get_equivalent_compose_without_resizing(auto_padding=DetectionAutoPadding(shape_multiple=(32, 32), pad_value=0))

    @property
    def classification(self) -> bool:
        return self.resize is not None or self.crop is not None

    def without_resizing(self) -> "ComposeProcessing":
        """The same chain without its Resize / CenterCrop steps (predict(skip_image_resizing=True))."""
        return ComposeProcessing([p for p in self.processings if not isinstance(p, (Resize, CenterCrop))])

    def crop_geometry(self, height: int, width: int) -> Tuple[Tuple[int, int], Tuple[int, int], Tuple[int, int]]:
        """Classification chain: -> (resized (h, w), crop (top, left), output (h, w))."""
        rh, rw, _ = self.resize.target(height, width) if self.resize is not None else (height, width, 1.0)
        if self.crop is None:
            return (rh, rw), (0, 0), (rh, rw)
        return (rh, rw), self.crop.top_left(rh, rw), (self.crop.size, self.crop.size)

    def preprocess_crop_batch(self, images: Sequence[np.ndarray], device) -> torch.Tensor:
        """Classification chain over uint8 H x W x 3 arrays of any sizes -> bf16 NHWC [B, 16, H, W] (channels >= 3 zero), in ONE kernel
        launch: the images and the per-image table are packed into one pinned staging buffer and sent with one copy."""
        for im in images:
            if not isinstance(im, np.ndarray) or im.dtype != np.uint8 or im.ndim != 3:
                raise ValueError("predict() images must be uint8 H x W x 3 arrays")
            if im.shape[2] != 3:  # PIL premultiplies the alpha of RGBA images; grayscale has another resize mode
                raise NotImplementedError(f"only 3-channel images are supported by the classification chain, got {im.shape[2]} channels")
        geos = [self.crop_geometry(im.shape[0], im.shape[1]) for im in images]
        shapes = sorted(set(g[2] for g in geos))
        if len(shapes) != 1:
            raise ValueError(f"the images of a batch must map to one input shape, got {shapes}")
        (oh, ow), B = shapes[0], len(images)
        head = B * K.RS_FIELDS * 8
        offsets = np.cumsum([0] + [im.nbytes for im in images])
        total = head + int(offsets[-1])
        on_gpu = torch.device(device).type == "cuda"
        if self._staging is None or self._staging.numel() < total:
            self._staging = torch.empty(total + total // 4, dtype=torch.uint8, pin_memory=on_gpu)
            self._staging_free = None
        elif self._staging_free is not None:
            self._staging_free.synchronize()  # the previous batch's copy has read the buffer
        raw = self._staging.numpy()
        table = raw[:head].view(np.int64).reshape(B, K.RS_FIELDS)
        for b, (im, ((rh, rw), (top, left), _)) in enumerate(zip(images, geos)):
            h, w = im.shape[:2]
            table[b] = (offsets[b], h, w, w * 3, rh, rw, top, left)
            raw[head + offsets[b] : head + offsets[b + 1]] = np.ascontiguousarray(im).reshape(-1)
        dev = self._staging[:total].to(device, non_blocking=True)
        if on_gpu:
            self._staging_free = torch.cuda.Event()
            self._staging_free.record()
        batch = K.empty_nhwc(B, 16, oh, ow, device)
        K.resample_crop_u8(self._staging[:head].view(torch.int64).view(B, K.RS_FIELDS), dev[:head].view(torch.int64).view(B, K.RS_FIELDS), dev[head:], batch,
                           max_value=self.standardize.max_value if self.standardize is not None else 0.0, reverse_channels=self.reverse is not None,
                           mean=self.normalize.mean if self.normalize is not None else None, std=self.normalize.std if self.normalize is not None else None)  # fmt: skip
        return batch

    def geometry(self, height: int, width: int) -> Tuple[ImageGeometry, Tuple[int, int]]:
        nh, nw, sh, sw = self.rescale.target(height, width) if self.rescale is not None else (height, width, 1.0, 1.0)
        if self.padding is not None:
            top, left = self.padding.top_left(nh, nw)
            canvas = self.padding.output_shape
        elif self.auto_padding is not None:
            top, left, canvas = 0, 0, self.auto_padding.padded_shape(nh, nw)
        else:
            top, left, canvas = 0, 0, (nh, nw)
        return ImageGeometry((height, width), sh, sw, (nh, nw), top, left), canvas

    def preprocess_batch(self, images: Sequence[np.ndarray], device) -> Tuple[torch.Tensor, List[ImageGeometry]]:
        """images: uint8 H x W x C arrays (any sizes).  Returns the model input -- bf16 NHWC [B, 16, H, W] with channels >= C
        zero, which the model mirrors consume as is -- and the per-image geometry for postprocess_*()."""
        geos, canvases = zip(*(self.geometry(im.shape[0], im.shape[1]) for im in images))
        if len(set(canvases)) != 1:
            raise ValueError(f"the images of a batch must map to one input shape, got {sorted(set(canvases))}")
        oh, ow = canvases[0]
        batch = K.empty_nhwc(len(images), 16, oh, ow, device)
        pad = self.padding or self.auto_padding
        for b, (im, g) in enumerate(zip(images, geos)):
            if im.dtype != np.uint8 or im.ndim != 3:
                raise ValueError("predict() images must be uint8 H x W x C arrays")
            src = torch.from_numpy(np.ascontiguousarray(im)).to(device, non_blocking=True)
            K.preprocess_u8(src, batch[b : b + 1], g.resized_shape, (g.pad_top, g.pad_left), pad_value=pad.pad_value if pad is not None else 0.0,
                            max_value=self.standardize.max_value if self.standardize is not None else 0.0, reverse_channels=self.reverse is not None,
                            mean=self.normalize.mean if self.normalize is not None else None, std=self.normalize.std if self.normalize is not None else None)  # fmt: skip
        return batch, list(geos)

    @staticmethod
    def batch_shift_scale(geos: Sequence[ImageGeometry], device) -> Tuple[torch.Tensor, torch.Tensor]:
        """Per-image (shift [B, 2] = (-pad_left, -pad_top), scale [B, 2] = float32(1 / scale_w), float32(1 / scale_h)): the operands
        of postprocess_boxes / postprocess_keypoints for a whole batch, so that undoing the padding / rescaling of every image is
        a handful of batched launches ((v + shift) * scale in float32: the same two roundings per coordinate as the per-image form)."""
        shift = torch.tensor([[-g.pad_left, -g.pad_top] for g in geos], dtype=torch.float32)
        scale = torch.tensor([[float(np.float32(1 / g.scale_factor_w)), float(np.float32(1 / g.scale_factor_h))] for g in geos], dtype=torch.float32)
        return shift.to(device, non_blocking=True), scale.to(device, non_blocking=True)

    @staticmethod
    def postprocess_boxes(boxes_xyxy: torch.Tensor, g: ImageGeometry) -> torch.Tensor:
        """[n, >= 4] rows whose first four columns are xyxy in model-input pixels -> original-image pixels: shift by the padding,
        then multiply by float32(1 / scale) (_shift_bboxes_xyxy, _rescale_bboxes: transforms/utils.py:47-62, 155-166)."""
        out = boxes_xyxy.float().clone()
        out[:, [0, 2]] += -g.pad_left
        out[:, [1, 3]] += -g.pad_top
        sx, sy = np.float32(1 / g.scale_factor_w), np.float32(1 / g.scale_factor_h)
        out[:, :4] *= torch.tensor([sx, sy, sx, sy], dtype=torch.float32, device=out.device)
        return out

    @staticmethod
    def postprocess_keypoints(poses: torch.Tensor, g: ImageGeometry) -> torch.Tensor:
        """[n, J, >= 2] keypoints (x, y, ...) -> original-image pixels (_shift_keypoints, _rescale_keypoints)."""
        out = poses.float().clone()
        out[..., 0] += -g.pad_left
        out[..., 1] += -g.pad_top
        out[..., 0] *= float(np.float32(1 / g.scale_factor_w))
        out[..., 1] *= float(np.float32(1 / g.scale_factor_h))
        return out


def default_yolo_nas_coco_processing_params() -> dict:
    """processing.py:960-980 (class names are dataset metadata and not part of this mirror)."""
    return dict(image_processor=ComposeProcessing([DetectionLongestMaxSizeRescale(output_shape=(636, 636)), DetectionCenterPadding(output_shape=(640, 640), pad_value=114),
                                                   StandardizeImage(max_value=255.0), ImagePermute(permutation=(2, 0, 1))]), iou=0.7, conf=0.25)  # fmt: skip


def default_imagenet_processing_params() -> dict:
    """processing.py:1142-1151 (the ImageNet class names are dataset metadata and not part of this mirror)."""
    return dict(image_processor=ComposeProcessing([Resize(size=256), CenterCrop(size=224), StandardizeImage(), NormalizeImage(mean=[0.485, 0.456, 0.406], std=[0.229, 0.224, 0.225]),
                                                   ImagePermute()]))  # fmt: skip


def default_yolo_nas_pose_coco_processing_params() -> dict:
    """processing.py:1060-1085."""
    return dict(image_processor=ComposeProcessing([ReverseImageChannels(), KeypointsLongestMaxSizeRescale(output_shape=(640, 640)),
                                                   KeypointsBottomRightPadding(output_shape=(640, 640), pad_value=127), StandardizeImage(max_value=255.0),
                                                   ImagePermute(permutation=(2, 0, 1))]), conf=0.5)  # fmt: skip
