"""Pixels of the YOLO-NAS COCO train augmentation on the GPU.

An `AugmentPlan` holds the draws of one sample of the recipe chain DetectionMosaic -> DetectionRandomAffine -> DetectionRGB2BGR ->
DetectionHSV -> DetectionHorizontalFlip -> DetectionMixup -> DetectionPaddedRescale -> DetectionStandardize (the reference's
training/transforms/transforms.py); a mosaic sample carries its four source images.  `BatchAugmenter` (and `PackedDetectionBatch`, built by `DetectionAugmentCollateFN` in DataLoader
workers) packs the images and the per-image table of a batch into one buffer, sends it with one copy and runs one kernel launch (csrc/augment.cu) that writes the bf16 NHWC [B, 16, H, W] model input,
bit-exact with the reference's cv2 / numpy chain followed by DetectionCollateFN and functional.to_nhwc."""
from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

from super_gradients_b200 import kernels as K

# column of each field in the per-image table (include/sgb200.h SGB_AUG_*)
OFFSET, H, W, AFFINE, AFF_H, AFF_W, M, AFF_BORDER = 0, 1, 2, 3, 4, 5, 6, 12
SWAP, HSV, DH, DS, DV, BGR, FLIP = 13, 14, 15, 16, 17, 18, 19
MIX, MIX_OFFSET, MIX_H, MIX_W, MIX_FLIP, MIX_R1_H, MIX_R1_W, MIX_CANVAS_H, MIX_CANVAS_W, MIX_BORDER = 20, 21, 22, 23, 24, 25, 26, 27, 28, 29
MIX_R2_H, MIX_R2_W, MIX_X, MIX_Y, RS_H, RS_W = 30, 31, 32, 33, 34, 35
MOS, MOS_CANVAS_H, MOS_CANVAS_W, MOS_XC, MOS_YC, MOS_BORDER, MOS_TILE, MOS_TILE_FIELDS = 36, 37, 38, 39, 40, 41, 42, 11
# columns of a mosaic tile relative to MOS_TILE + i * MOS_TILE_FIELDS
T_OFFSET, T_H, T_W, T_RH, T_RW, T_X1, T_Y1, T_X2, T_Y2, T_SX, T_SY = range(11)


@dataclass
class MixupPlan:
    """DetectionMixup's draws: the partner image (uint8 H x W x 3, before its flip), its flip, the first resize size (fit into
    `canvas`), the canvas size (target_dim), the second resize size (jit_factor) and the crop offsets."""

    image: np.ndarray
    flip: bool
    resized: Tuple[int, int]
    canvas: Tuple[int, int]
    jittered: Tuple[int, int]
    x_offset: int
    y_offset: int
    border_value: int = 114


@dataclass
class MosaicTile:
    """One of DetectionMosaic's four images: the source (uint8 H x W x 3), its resized size (int(h0 * scale), int(w0 * scale)),
    its rectangle (x1, y1, x2, y2) on the canvas and the resized tile's pixel (sx, sy) placed at (x1, y1)
    (get_mosaic_coordinate's large and small coordinates)."""

    image: np.ndarray
    resized: Tuple[int, int]
    rect: Tuple[int, int, int, int]
    origin: Tuple[int, int]


@dataclass
class MosaicPlan:
    """DetectionMosaic's draws: the four tiles (top-left, top-right, bottom-left, bottom-right; tile 0 holds the sample's own
    image), the canvas size (2 * input_dim), the centre (xc, yc) and the border value."""

    tiles: List[MosaicTile]
    canvas: Tuple[int, int]
    xc: int
    yc: int
    border_value: int = 114


@dataclass
class AugmentPlan:
    """One sample's draws.  `mosaic`: DetectionMosaic's canvas (None: no mosaic; its tile 0 holds `image`); `affine`: the forward
    2 x 3 matrix of random_affine (None: DetectionRandomAffine closed) with its output size (rows, cols) and border value; `hsv`:
    the int16 gains (dh, ds, dv) with bgr_channels (None: not applied); `rescaled`: (int(h * r), int(w * r)) of
    DetectionPaddedRescale."""

    image: np.ndarray
    rescaled: Tuple[int, int]
    affine: Optional[Tuple[np.ndarray, Tuple[int, int], int]] = None
    swap: bool = False
    hsv: Optional[Tuple[int, int, int, Tuple[int, int, int]]] = None
    flip: bool = False
    mixup: Optional[MixupPlan] = None
    mosaic: Optional[MosaicPlan] = None

    def size_before_affine(self) -> Tuple[int, int]:
        return tuple(self.mosaic.canvas) if self.mosaic is not None else tuple(self.image.shape[:2])

    def size_after_affine(self) -> Tuple[int, int]:
        return tuple(self.affine[1]) if self.affine is not None else self.size_before_affine()

    def images(self) -> List[np.ndarray]:
        """The images the kernel reads, in packing order: the sample's, the mosaic's three others, the mixup partner."""
        out = [self.image]
        if self.mosaic is not None:
            out += [t.image for t in self.mosaic.tiles[1:]]
        if self.mixup is not None:
            out.append(self.mixup.image)
        return out


def _check_image(im, what):
    if not isinstance(im, np.ndarray) or im.dtype != np.uint8 or im.ndim != 3 or im.shape[2] != 3:
        raise ValueError(f"{what} must be a uint8 H x W x 3 array, got {getattr(im, 'dtype', type(im))} {getattr(im, 'shape', '')}")


def fill_table(plans: Sequence[AugmentPlan], offsets: Sequence[Sequence[int]], table: np.ndarray) -> None:
    """Writes the int64 [B, AUG_FIELDS] table of `plans`; offsets[b]: the byte offset of each of plans[b].images()."""
    table[:] = 0
    for b, (p, offs) in enumerate(zip(plans, offsets)):
        t = table[b]
        t[OFFSET], t[H], t[W] = offs[0], p.image.shape[0], p.image.shape[1]
        t[AFF_H], t[AFF_W] = p.size_after_affine()
        if p.affine is not None:
            m, _, border = p.affine
            t[AFFINE], t[AFF_BORDER] = 1, border
            t[M : M + 6] = np.ascontiguousarray(np.asarray(m, dtype=np.float64).reshape(6)).view(np.int64)
        t[SWAP], t[FLIP] = int(p.swap), int(p.flip)
        if p.hsv is not None:
            dh, ds, dv, bgr = p.hsv
            if sorted(bgr) != [0, 1, 2]:
                raise ValueError(f"bgr_channels must be a permutation of (0, 1, 2) for 3-channel images, got {bgr}")
            t[HSV], t[DH], t[DS], t[DV], t[BGR] = 1, dh, ds, dv, bgr[0] | bgr[1] << 2 | bgr[2] << 4
        if p.mixup is not None:
            x = p.mixup
            t[MIX], t[MIX_OFFSET], t[MIX_H], t[MIX_W], t[MIX_FLIP] = 1, offs[-1], x.image.shape[0], x.image.shape[1], int(x.flip)
            t[MIX_R1_H], t[MIX_R1_W] = x.resized
            t[MIX_CANVAS_H], t[MIX_CANVAS_W] = x.canvas
            t[MIX_BORDER] = x.border_value
            t[MIX_R2_H], t[MIX_R2_W] = x.jittered
            t[MIX_X], t[MIX_Y] = x.x_offset, x.y_offset
        t[RS_H], t[RS_W] = p.rescaled
        if p.mosaic is not None:
            mo = p.mosaic
            t[MOS], (t[MOS_CANVAS_H], t[MOS_CANVAS_W]), t[MOS_XC], t[MOS_YC], t[MOS_BORDER] = 1, mo.canvas, mo.xc, mo.yc, mo.border_value
            for i, (tile, off) in enumerate(zip(mo.tiles, offs)):
                k = t[MOS_TILE + i * MOS_TILE_FIELDS : MOS_TILE + (i + 1) * MOS_TILE_FIELDS]
                k[T_OFFSET], k[T_H], k[T_W] = off, tile.image.shape[0], tile.image.shape[1]
                k[T_RH], k[T_RW] = tile.resized
                k[T_X1], k[T_Y1], k[T_X2], k[T_Y2] = tile.rect
                k[T_SX], k[T_SY] = tile.origin


def packed_size(plans: Sequence[AugmentPlan]) -> int:
    """Bytes of the packed form of `plans`: the int64 table, then every image, mosaic tile and mixup partner."""
    return len(plans) * K.AUG_FIELDS * 8 + sum(im.nbytes for p in plans for im in p.images())


def pack_into(plans: Sequence[AugmentPlan], raw: np.ndarray) -> None:
    """Writes the packed form of `plans` into the uint8 array `raw` (at least packed_size(plans) bytes)."""
    for p in plans:
        _check_image(p.image, "the image")
        if p.mosaic is not None:
            if len(p.mosaic.tiles) != 4 or p.mosaic.tiles[0].image is not p.image:
                raise ValueError("a mosaic has four tiles, the first holding the sample's own image")
            for tile in p.mosaic.tiles[1:]:
                _check_image(tile.image, "a mosaic tile")
        if p.mixup is not None:
            _check_image(p.mixup.image, "the mixup image")
    head = len(plans) * K.AUG_FIELDS * 8
    offsets, pos = [], 0
    for p in plans:
        offs = []
        for im in p.images():
            offs.append(pos)
            raw[head + pos : head + pos + im.nbytes] = np.ascontiguousarray(im).reshape(-1)
            pos += im.nbytes
        offsets.append(offs)
    fill_table(plans, offsets, raw[:head].view(np.int64).reshape(len(plans), K.AUG_FIELDS))


def run_packed(host: torch.Tensor, batch: int, device, input_dim: Tuple[int, int], pad_value: int = 114, max_value: float = 255.0, out=None) -> torch.Tensor:
    """One copy of the packed uint8 buffer `host` to `device` and one augmentation launch -> bf16 NHWC [B, 16, H, W], written into
    `out` (e.g. a captured train step's static input) when given."""
    head = batch * K.AUG_FIELDS * 8
    dev = host.to(device, non_blocking=True)
    shape = (batch, 16, input_dim[0], input_dim[1])
    out = K.empty_nhwc(*shape, device) if out is None else K.require_nhwc_out(out, shape)
    K.detection_augment(host[:head].view(torch.int64).view(batch, K.AUG_FIELDS), dev[:head].view(torch.int64).view(batch, K.AUG_FIELDS), dev[head:], out,
                        pad_value=pad_value, max_value=max_value)  # fmt: skip
    return out


class BatchAugmenter:
    """Packs a batch of plans into one reusable pinned staging buffer (table first, then the images), sends it with one copy and
    runs the augmentation kernel: no host synchronisation except waiting, before the buffer is overwritten, for the previous
    batch's copy to have read it."""

    def __init__(self, input_dim: Tuple[int, int] = (640, 640), pad_value: int = 114, max_value: float = 255.0):
        self.input_dim = (int(input_dim[0]), int(input_dim[1]))
        self.pad_value = int(pad_value)
        self.max_value = float(max_value)
        self._staging = None
        self._staging_free = None

    def pack(self, plans: Sequence[AugmentPlan], pin: bool) -> Tuple[torch.Tensor, int]:
        """Returns (staging uint8 buffer, bytes used): the int64 table followed by every image."""
        used = packed_size(plans)
        if self._staging is None or self._staging.numel() < used:
            self._staging = torch.empty(used + used // 4, dtype=torch.uint8, pin_memory=pin)
            self._staging_free = None
        elif self._staging_free is not None:
            self._staging_free.synchronize()  # the previous batch's copy has read the buffer
        pack_into(plans, self._staging.numpy())
        return self._staging, used

    def __call__(self, plans: Sequence[AugmentPlan], device) -> torch.Tensor:
        """bf16 NHWC [B, 16, H, W] model input of the batch (channels >= 3 zero)."""
        staging, used = self.pack(plans, pin=torch.device(device).type == "cuda")
        out = run_packed(staging[:used], len(plans), device, self.input_dim, self.pad_value, self.max_value)
        if torch.device(device).type == "cuda":
            self._staging_free = torch.cuda.Event()
            self._staging_free.record()
        return out
