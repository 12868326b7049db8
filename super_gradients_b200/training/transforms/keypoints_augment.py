"""Pixels of the YOLO-NAS-POSE train augmentation on the GPU.

A `PosePlan` holds the draws of one sample of the keypoint chain KeypointsRandomHorizontalFlip -> KeypointsBrightnessContrast ->
KeypointsReverseImageChannels -> KeypointsHSV -> KeypointsRandomRotate90 -> KeypointsRandomAffineTransform -> KeypointsMosaic ->
KeypointsLongestMaxSize -> KeypointsPadIfNeeded -> KeypointsImageStandardize (the reference's training/transforms/keypoints/):
one `TilePlan` per source image (four after a mosaic) and the canvas geometry.  `pack_into` writes a batch of plans into one
uint8 buffer (the int64 table, then the images) and `run_packed` makes the bf16 NHWC [B, 16, S, S] model input with one copy and
one call of two kernel launches (csrc/pose_augment.cu), bit-exact with the reference's cv2 / numpy chain followed by
YoloNASPoseCollateFN and functional.to_nhwc."""
from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

from super_gradients_b200 import kernels as K

# columns of the per-sample table and of its tile records (include/sgb200.h SGB_POSE_*)
NSUB, CANVAS_H, CANVAS_W, MOSAIC_PAD, RS_H, RS_W, PAD_TOP, PAD_LEFT, PAD_VALUE, SUB, SUB_FIELDS = 0, 1, 2, 3, 4, 5, 6, 7, 8, 16, 32
S_OFFSET, S_H, S_W, S_FLIP, S_BC, S_MEAN, S_CONTRAST, S_BRIGHTNESS, S_REVERSE = 0, 1, 2, 3, 4, 5, 8, 9, 10
S_HSV, S_DH, S_DS, S_DV, S_ROT, S_AFFINE, S_M, S_MODE, S_BORDER, S_WS_OFFSET, S_Y, S_X, S_RH, S_RW = 11, 12, 13, 14, 15, 16, 17, 23, 24, 25, 26, 27, 28, 29


@dataclass
class TilePlan:
    """One source image's draws.  `bc`: (float32 channel means of the flipped image, contrast gain, brightness gain);
    `hsv`: int16 gains (dh, ds, dv); `rot`: np.rot90 count; `affine`: (forward 2 x 3 matrix, cv2 interpolation flag, border colour)."""

    image: np.ndarray
    flip: bool = False
    bc: Optional[Tuple[np.ndarray, float, float]] = None
    reverse: bool = False
    hsv: Optional[Tuple[int, int, int]] = None
    rot: int = 0
    affine: Optional[Tuple[np.ndarray, int, Tuple[int, int, int]]] = None

    def shape(self) -> Tuple[int, int]:
        h, w = self.image.shape[:2]
        return (w, h) if self.rot % 2 else (h, w)


@dataclass
class PosePlan:
    """The tiles with their positions in the canvas (one tile at (0, 0), or a mosaic's four), the canvas size and the mosaic pad
    colour, then LongestMaxSize's size and KeypointsPadIfNeeded's offsets and colour."""

    tiles: List[TilePlan]
    positions: List[Tuple[int, int]]
    canvas: Tuple[int, int]
    mosaic_pad: Tuple[int, int, int] = (127, 127, 127)
    resized: Optional[Tuple[int, int]] = None
    pad: Tuple[int, int] = (0, 0)
    pad_value: Tuple[int, int, int] = (127, 127, 127)

    @classmethod
    def single(cls, image: np.ndarray) -> "PosePlan":
        return cls([TilePlan(image)], [(0, 0)], tuple(image.shape[:2]))


def colour(v) -> Tuple[int, int, int]:
    """A scalar or a 3-sequence pad value as three uint8 channel values."""
    vals = [v] * 3 if np.isscalar(v) else list(v)
    if len(vals) != 3 or any(not float(x).is_integer() or not 0 <= float(x) <= 255 for x in vals):
        raise ValueError(f"pad colours must be one or three integers in [0, 255], got {v}")
    return tuple(int(x) for x in vals)


def _packed(c) -> int:
    return c[0] | c[1] << 8 | c[2] << 16


def _f32_bits(v) -> int:
    return int(np.float32(v).view(np.uint32))


def _check_image(im):
    if not isinstance(im, np.ndarray) or im.dtype != np.uint8 or im.ndim != 3 or im.shape[2] != 3:
        raise ValueError(f"images must be uint8 H x W x 3 arrays, got {getattr(im, 'dtype', type(im))} {getattr(im, 'shape', '')}")


def fill_table(plans: Sequence[PosePlan], offsets: Sequence[Sequence[int]], table: np.ndarray) -> None:
    """Writes the int64 [B, POSE_FIELDS] table; offsets[b][i]: byte offset of tile i's image in the source buffer, and of its rotated
    image in the workspace (the same size)."""
    table[:] = 0
    for b, p in enumerate(plans):
        t = table[b]
        t[NSUB], (t[CANVAS_H], t[CANVAS_W]), t[MOSAIC_PAD] = len(p.tiles), p.canvas, _packed(p.mosaic_pad)
        t[RS_H], t[RS_W] = p.resized if p.resized is not None else p.canvas
        t[PAD_TOP], t[PAD_LEFT], t[PAD_VALUE] = p.pad[0], p.pad[1], _packed(p.pad_value)
        for i, (tile, (y, x)) in enumerate(zip(p.tiles, p.positions)):
            s = t[SUB + i * SUB_FIELDS : SUB + (i + 1) * SUB_FIELDS]
            s[S_OFFSET], (s[S_H], s[S_W]) = offsets[b][i], tile.image.shape[:2]
            s[S_FLIP], s[S_REVERSE], s[S_ROT] = int(tile.flip), int(tile.reverse), tile.rot
            if tile.bc is not None:
                mean, cg, bg = tile.bc
                s[S_BC] = 1
                s[S_MEAN : S_MEAN + 3] = np.asarray(mean, dtype=np.float32).view(np.uint32)
                s[S_CONTRAST], s[S_BRIGHTNESS] = _f32_bits(cg), _f32_bits(bg)
            if tile.hsv is not None:
                s[S_HSV], s[S_DH], s[S_DS], s[S_DV] = 1, *tile.hsv
            if tile.affine is not None:
                m, mode, border = tile.affine
                s[S_AFFINE], s[S_MODE], s[S_BORDER] = 1, mode, _packed(border)
                s[S_M : S_M + 6] = np.ascontiguousarray(np.asarray(m, dtype=np.float64).reshape(6)).view(np.int64)
            s[S_WS_OFFSET], s[S_Y], s[S_X] = offsets[b][i], y, x
            s[S_RH], s[S_RW] = tile.shape()


def packed_size(plans: Sequence[PosePlan]) -> int:
    """Bytes of the packed form of `plans`: the int64 table, then every tile's image."""
    return len(plans) * K.POSE_FIELDS * 8 + sum(t.image.nbytes for p in plans for t in p.tiles)


def pack_into(plans: Sequence[PosePlan], raw: np.ndarray) -> None:
    """Writes the packed form of `plans` into the uint8 array `raw` (at least packed_size(plans) bytes).  Each tile's rotated image
    takes the same bytes in the workspace as its source image in the buffer."""
    for p in plans:
        for t in p.tiles:
            _check_image(t.image)
    head = len(plans) * K.POSE_FIELDS * 8
    offsets, pos = [], 0
    for p in plans:
        offs = []
        for t in p.tiles:
            offs.append(pos)
            raw[head + pos : head + pos + t.image.nbytes] = np.ascontiguousarray(t.image).reshape(-1)
            pos += t.image.nbytes
        offsets.append(offs)
    fill_table(plans, offsets, raw[:head].view(np.int64).reshape(len(plans), K.POSE_FIELDS))


def run_packed(host: torch.Tensor, batch: int, device, size: int, max_value: float = 255.0, out=None) -> torch.Tensor:
    """One copy of the packed uint8 buffer `host` to `device` and one pose augmentation call -> bf16 NHWC [B, 16, size, size], written
    into `out` (e.g. a captured train step's static input) when given."""
    head = batch * K.POSE_FIELDS * 8
    dev = host.to(device, non_blocking=True)
    ws = torch.empty(max(host.numel() - head, 1), dtype=torch.uint8, device=device)
    out = K.empty_nhwc(batch, 16, size, size, device) if out is None else K.require_nhwc_out(out, (batch, 16, size, size))
    K.pose_augment(host[:head].view(torch.int64).view(batch, K.POSE_FIELDS), dev[:head].view(torch.int64).view(batch, K.POSE_FIELDS), dev[head:], ws, out, max_value)
    return out
