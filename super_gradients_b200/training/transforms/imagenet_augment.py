"""Host half of the ImageNet train augmentation on the GPU: the draws of the ResNet-50 recipe's chain and the packed form the kernel
reads.

The chain (recipes/dataset_params/imagenet_resnet50_dataset_params.yaml) is RandomResizedCropAndInterpolation -> RandomHorizontalFlip
-> RandAugment -> ToTensor -> Normalize, then CollateMixup in batch mode.  `draw_plan` makes the reference's draws for one sample from
the same RNG streams in the same order (torch for the crop window and the flip, python `random` for the interpolation and the
RandAugment op draws, numpy for the op choice) and returns an `ImageNetPlan`: only the crop window's bytes and what the pixel work
needs.  `pack_into` writes a batch's int64 table (include/sgb200.h SGB_IN_*) and windows into one buffer; `run_packed` sends it with
one copy and runs one launch of csrc/imagenet_augment.cu."""
import math
import random
import re
from dataclasses import dataclass, field
from typing import List, Sequence, Tuple

import numpy as np
import torch

from super_gradients_b200 import kernels as K

# columns of the per-image table (include/sgb200.h SGB_IN_*)
OFFSET, H, W, FILTER, FLIP, WS_OFFSET, OP, OP_FIELDS, OPS = 0, 1, 2, 3, 4, 5, 6, 7, 2
OP_NONE, OP_AFFINE, OP_INVERT, OP_POSTERIZE, OP_SOLARIZE, OP_SOLARIZE_ADD, OP_BRIGHTNESS, OP_CONTRAST = 0, 1, 2, 3, 4, 5, 6, 7
OP_AUTOCONTRAST, OP_EQUALIZE, OP_COLOR, OP_SHARPNESS = 8, 9, 10, 11
BILINEAR, BICUBIC = 0, 1

MAX_MAGNITUDE = 10.0
# RandAugment's op list, in the order np.random.choice indexes it (auto_augment.py _RAND_TRANSFORMS)
RAND_TRANSFORMS = ("AutoContrast", "Equalize", "Invert", "Rotate", "Posterize", "Solarize", "SolarizeAdd", "Color", "Contrast", "Brightness", "Sharpness",
                   "ShearX", "ShearY", "TranslateXRel", "TranslateYRel")  # fmt: skip
_ENHANCE = {"Color": OP_COLOR, "Contrast": OP_CONTRAST, "Brightness": OP_BRIGHTNESS, "Sharpness": OP_SHARPNESS}
_PLAIN = {"AutoContrast": OP_AUTOCONTRAST, "Equalize": OP_EQUALIZE, "Invert": OP_INVERT}


@dataclass
class RandAugmentConfig:
    """rand_augment_transform's parsed config string: magnitude `m`, ops per image `n`, magnitude std `mstd`."""

    magnitude: float = MAX_MAGNITUDE
    num_layers: int = 2
    magnitude_std: float = 0.0

    @classmethod
    def parse(cls, config_str: str) -> "RandAugmentConfig":
        """Sections after the leading 'rand', as rand_augment_transform reads them.  'inc' and 'w' select op lists and weights that
        no shipped ResNet recipe uses; they are refused."""
        cfg = cls()
        sections = config_str.split("-")
        if sections[0] != "rand":
            raise ValueError(f"RandAugment config must start with 'rand', got {config_str!r}")
        for c in sections[1:]:
            cs = re.split(r"(\d.*)", c)
            if len(cs) < 2:
                continue
            key, val = cs[:2]
            if key == "mstd":
                cfg.magnitude_std = float(val)
            elif key == "m":
                cfg.magnitude = int(val)
            elif key == "n":
                cfg.num_layers = int(val)
            elif key in ("inc", "w"):
                raise ValueError(f"RandAugment section {key!r} ({config_str!r}) is not supported on the GPU path")
            else:
                raise ValueError(f"unknown RandAugment config section {c!r}")
        if cfg.num_layers != OPS:
            raise ValueError(f"the GPU path applies {OPS} RandAugment ops per image, got n{cfg.num_layers}")
        return cfg


@dataclass
class ImageNetPlan:
    """One sample's draws: the crop window (uint8 h x w x 3, RandomResizedCrop's), the resize filter (BILINEAR / BICUBIC), the flip,
    the RandAugment ops as (code, six int64 arguments) and the label."""

    window: np.ndarray
    filter: int
    flip: bool
    ops: List[Tuple[int, List[int]]] = field(default_factory=list)
    label: int = 0


def _f64_bits(*v) -> List[int]:
    return [int(x) for x in np.asarray(v, dtype=np.float64).view(np.int64)]


def _affine(*m) -> Tuple[int, List[int]]:
    return OP_AFFINE, _f64_bits(*m)


def rotate_matrix(degrees: float, w: int, h: int) -> Tuple[float, ...]:
    """The inverse matrix Image.rotate(degrees) passes to Image.transform (rotation about the centre, no expand)."""
    angle = -math.radians(degrees % 360.0)
    m = [round(math.cos(angle), 15), round(math.sin(angle), 15), 0.0, round(-math.sin(angle), 15), round(math.cos(angle), 15), 0.0]
    cx, cy = w / 2, h / 2
    m[2], m[5] = m[0] * -cx + m[1] * -cy + m[2], m[3] * -cx + m[4] * -cy + m[5]
    m[2] += cx
    m[5] += cy
    return tuple(m)


def _negate(v: float) -> float:
    return -v if random.random() > 0.5 else v


def op_plan(name: str, magnitude: float, size: int) -> Tuple[int, List[int]]:
    """(code, arguments) of RandAugment op `name` at `magnitude` on a size x size image, with its level-to-argument draws."""
    level = magnitude / MAX_MAGNITUDE
    if name in _PLAIN:
        return _PLAIN[name], [0] * 6
    if name == "Rotate":
        degrees = _negate(level * 30.0)
        if degrees % 360.0 == 0:  # Image.rotate's copy
            return OP_NONE, [0] * 6
        return _affine(*rotate_matrix(degrees, size, size))
    if name in ("ShearX", "ShearY"):
        f = _negate(level * 0.3)
        return _affine(1, f, 0, 0, 1, 0) if name == "ShearX" else _affine(1, 0, 0, f, 1, 0)
    if name in ("TranslateXRel", "TranslateYRel"):
        pixels = _negate(level * 0.45) * size
        return _affine(1, 0, pixels, 0, 1, 0) if name == "TranslateXRel" else _affine(1, 0, 0, 0, 1, pixels)
    if name == "Posterize":
        bits = int(level * 4)
        return (OP_NONE, [0] * 6) if bits >= 8 else (OP_POSTERIZE, [bits] + [0] * 5)
    if name == "Solarize":
        return OP_SOLARIZE, [int(level * 256)] + [0] * 5
    if name == "SolarizeAdd":
        return OP_SOLARIZE_ADD, [int(level * 110)] + [0] * 5
    if name in _ENHANCE:
        return _ENHANCE[name], _f64_bits(level * 1.8 + 0.1) + [0] * 5
    raise ValueError(f"unknown RandAugment op {name!r}")


def random_resized_crop_params(height: int, width: int, scale=(0.08, 1.0), ratio=(3.0 / 4.0, 4.0 / 3.0)) -> Tuple[int, int, int, int]:
    """torchvision RandomResizedCrop.get_params: (top, left, h, w) from the torch RNG, up to 10 tries, then the centre crop."""
    area = height * width
    log_ratio = torch.log(torch.tensor(ratio))
    for _ in range(10):
        target_area = area * torch.empty(1).uniform_(scale[0], scale[1]).item()
        aspect_ratio = torch.exp(torch.empty(1).uniform_(log_ratio[0], log_ratio[1])).item()
        w = int(round(math.sqrt(target_area * aspect_ratio)))
        h = int(round(math.sqrt(target_area / aspect_ratio)))
        if 0 < w <= width and 0 < h <= height:
            i = torch.randint(0, height - h + 1, size=(1,)).item()
            j = torch.randint(0, width - w + 1, size=(1,)).item()
            return i, j, h, w
    in_ratio = float(width) / float(height)
    if in_ratio < min(ratio):
        w = width
        h = int(round(w / min(ratio)))
    elif in_ratio > max(ratio):
        h = height
        w = int(round(h * max(ratio)))
    else:
        w, h = width, height
    return (height - h) // 2, (width - w) // 2, h, w


def draw_plan(image: np.ndarray, label: int, size: int, random_interpolation: bool, rand_augment: RandAugmentConfig) -> ImageNetPlan:
    """The reference chain's draws for one uint8 H x W x 3 RGB image, in its order; returns the plan with a copy of the window."""
    top, left, h, w = random_resized_crop_params(image.shape[0], image.shape[1])
    filt = random.choice((BILINEAR, BICUBIC)) if random_interpolation else BILINEAR
    flip = bool(torch.rand(1) < 0.5)
    ops = []
    if rand_augment is not None:
        for k in np.random.choice(len(RAND_TRANSFORMS), rand_augment.num_layers):
            if random.random() > 0.5:
                ops.append((OP_NONE, [0] * 6))
                continue
            m = rand_augment.magnitude
            if rand_augment.magnitude_std > 0:
                m = random.gauss(m, rand_augment.magnitude_std)
            ops.append(op_plan(RAND_TRANSFORMS[k], min(MAX_MAGNITUDE, max(0, m)), size))
    while len(ops) < OPS:
        ops.append((OP_NONE, [0] * 6))
    return ImageNetPlan(np.ascontiguousarray(image[top : top + h, left : left + w]), filt, flip, ops, int(label))


def _check_window(im):
    if not isinstance(im, np.ndarray) or im.dtype != np.uint8 or im.ndim != 3 or im.shape[2] != 3 or im.shape[0] < 1 or im.shape[1] < 1:
        raise ValueError(f"a crop window must be a non-empty uint8 H x W x 3 array, got {getattr(im, 'dtype', type(im))} {getattr(im, 'shape', '')}")


def packed_size(plans: Sequence[ImageNetPlan]) -> int:
    """Bytes of the packed form of `plans`: the int64 table, then every crop window."""
    return len(plans) * K.IN_FIELDS * 8 + sum(p.window.nbytes for p in plans)


def workspace_size(plans: Sequence[ImageNetPlan], size: int) -> int:
    """Device workspace bytes of the horizontal resize pass: every window's rows at the output width."""
    return sum(p.window.shape[0] * size * 3 for p in plans)


def pack_into(plans: Sequence[ImageNetPlan], raw: np.ndarray, size: int) -> None:
    """Writes the packed form of `plans` into the uint8 array `raw` (at least packed_size(plans) bytes)."""
    for p in plans:
        _check_window(p.window)
        if len(p.ops) != OPS:
            raise ValueError(f"a plan has {OPS} RandAugment ops, got {len(p.ops)}")
    head = len(plans) * K.IN_FIELDS * 8
    table = raw[:head].view(np.int64).reshape(len(plans), K.IN_FIELDS)
    table[:] = 0
    pos = ws = 0
    for b, p in enumerate(plans):
        h, w = p.window.shape[:2]
        raw[head + pos : head + pos + p.window.nbytes] = p.window.reshape(-1)
        t = table[b]
        t[OFFSET], t[H], t[W], t[FILTER], t[FLIP], t[WS_OFFSET] = pos, h, w, p.filter, int(p.flip), ws
        for k, (code, args) in enumerate(p.ops):
            t[OP + k * OP_FIELDS] = code
            t[OP + k * OP_FIELDS + 1 : OP + (k + 1) * OP_FIELDS] = args
        pos += p.window.nbytes
        ws += h * size * 3


def run_packed(host: torch.Tensor, batch: int, workspace_bytes: int, device, size: int, fill, mean, std, mix_mode=0, lam=1.0, box=(0, 0, 0, 0), out=None) -> torch.Tensor:
    """One copy of the packed uint8 buffer `host` to `device` and one augmentation launch -> bf16 NHWC [B, 16, size, size], written
    into `out` (e.g. a captured train step's static input) when given."""
    head = batch * K.IN_FIELDS * 8
    dev = host.to(device, non_blocking=True)
    ws = torch.empty(max(workspace_bytes, 1), dtype=torch.uint8, device=device)
    out = K.empty_nhwc(batch, 16, size, size, device) if out is None else K.require_nhwc_out(out, (batch, 16, size, size))
    K.imagenet_augment(host[:head].view(torch.int64).view(batch, K.IN_FIELDS), dev[:head].view(torch.int64).view(batch, K.IN_FIELDS), dev[head:], ws, out, fill, mean, std,
                       mix_mode=mix_mode, lam=lam, box=box)  # fmt: skip
    return out
