"""Test infrastructure for DetectionMosaic in the detection train augmentation: a seeded stub dataset whose image sizes hit every
resize branch of a mosaic tile, the transform lists of the fixture tests/golden/detection_mosaic.pt, `oracle_canvas` (the
reference's mosaic canvas built with cv2 / numpy from a plan) and the g++ build of tests/host_kernels/detection_mosaic_host.cpp."""
import ctypes
import dataclasses
import os
import subprocess
import tempfile

import cv2
import numpy as np

from augment_cases import RECIPE, _image, oracle_u8
from super_gradients_b200.training.transforms.detection_augment import AugmentPlan

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_LIB = {}


def mosaic_lib():
    """g++ build of tests/host_kernels/detection_mosaic_host.cpp around the product header augment_math.cuh."""
    if "h" not in _LIB:
        d = tempfile.mkdtemp(prefix="sgb_mosaic_host_")
        so = os.path.join(d, "detection_mosaic_host.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", os.path.join(ROOT, "tests", "host_kernels", "detection_mosaic_host.cpp"), "-I",
                        os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "super_gradients_b200", "csrc"), "-o", so], check=True)  # fmt: skip
        h = ctypes.CDLL(so)
        P = ctypes.c_void_p
        h.mosaic_canvas_host.argtypes = [P, P, P]
        _LIB["h"] = h
    return _LIB["h"]


class StubMosaicDataset:
    """Seeded raw samples in the reference's get_sample() form.  Against a 640 mosaic input the sizes give every tile resize: the
    exact 2x downscale (1280 x 1280, 960 x 1280), a non-integer downscale (1000 x 750), scale 1 (640 x 640), upscales (333 x 500,
    250 x 600) and a x10 upscale (64 x 48).  Sample 3 has no targets; every third sample has a crowd box; boxes may cross the
    image border."""

    SIZES = [(1280, 1280), (960, 1280), (1000, 750), (640, 640), (333, 500), (250, 600), (64, 48), (480, 640)]

    def __init__(self, seed=0):
        rng = np.random.default_rng(seed)
        self.samples = []
        for i, (h, w) in enumerate(self.SIZES):
            n = 0 if i == 3 else int(rng.integers(2, 7))
            x1, y1 = rng.uniform(-0.1 * w, w * 0.8, n), rng.uniform(-0.1 * h, h * 0.8, n)
            bw, bh = rng.uniform(2, w * 0.5, n), rng.uniform(2, h * 0.5, n)
            boxes = np.stack([x1, y1, x1 + bw, y1 + bh, rng.integers(0, 4, n)], -1).astype(np.float32)
            crowd = boxes[:1].copy() if i % 3 == 1 else np.zeros((0, 5), np.float32)
            self.samples.append({"image": _image(rng, h, w), "target": boxes, "crowd_target": crowd})

    def __len__(self):
        return len(self.samples)

    def get_sample(self, index, ignore_empty_annotations=False):
        s = self.samples[index]
        return {k: v.copy() for k, v in s.items()}


# recipes/dataset_params/roboflow_detection_dataset_params.yaml's train transforms (the YOLO-NAS fine-tuning recipes)
ROBOFLOW = [
    ("DetectionMosaic", dict(input_dim=[640, 640], prob=1.0)),
    ("DetectionRandomAffine", dict(degrees=0.0, translate=0.1, scales=[0.5, 1.5], shear=0.0, target_size=[640, 640], filter_box_candidates=False, wh_thr=2, area_thr=0.1,
                                   ar_thr=20, border_value=128)),  # fmt: skip
    ("DetectionHSV", dict(prob=1.0, hgain=5, sgain=30, vgain=30)),
    ("DetectionHorizontalFlip", dict(prob=0.5)),
    ("DetectionPaddedRescale", dict(input_dim=[640, 640])),
    ("DetectionStandardize", dict(max_value=255.0)),
    ("DetectionTargetsFormatTransform", dict(input_dim=[640, 640], output_format="LABEL_CXCYWH")),
]
# mosaic with probability 0.5 before the COCO list: its target_size=None affine outputs the 1280 x 1280 canvas, then mixup,
# RGB2BGR and PaddedRescale's exact 2x downscale
MOSAIC_COCO = [("DetectionMosaic", dict(input_dim=[640, 640], prob=0.5))] + RECIPE
# the reference's own tests/unit_tests/detection_dataset_test.py mosaic size: a 768 x 768 canvas rescaled by 640 / 768
MOSAIC_384 = [("DetectionMosaic", dict(input_dim=384))] + RECIPE
# the Roboflow list with the mosaic closed (enable_mosaic=False, what close() sets)
ROBOFLOW_CLOSED = [(n, dict(kw, enable_mosaic=False) if n == "DetectionMosaic" else kw) for n, kw in ROBOFLOW]
GOLDEN_LISTS = {"roboflow": ROBOFLOW, "mosaic_coco": MOSAIC_COCO, "mosaic_384": MOSAIC_384, "roboflow_closed": ROBOFLOW_CLOSED}
GOLDEN_SEEDS = (0, 1, 2)

# canvases of the reference DetectionMosaic alone: (stub indices of the four tiles, input_dim, (yc, xc) the two random.uniform
# draws return).  Centres at both ends of the drawn range and on the canvas edges, where tiles are clipped or empty.
CANVAS_CASES = [
    ((0, 1, 2, 3), 640, (640.0, 640.0)),
    ((4, 5, 6, 7), 640, (320.0, 959.9)),
    ((6, 0, 5, 1), 640, (959.9, 320.0)),
    ((2, 6, 4, 0), 640, (0.0, 1280.0)),
    ((3, 2, 1, 6), 640, (1280.0, 0.0)),
    ((7, 4, 3, 5), 640, (1, 1279)),
    ((1, 3, 6, 2), 384, (200.5, 500.2)),
    ((5, 7, 0, 4), 384, (576.0, 192.0)),
]


def oracle_canvas(p: AugmentPlan) -> np.ndarray:
    """The uint8 canvas DetectionMosaic makes for plan p, with cv2.resize and numpy as the reference builds it."""
    mo = p.mosaic
    canvas = np.full((mo.canvas[0], mo.canvas[1], 3), mo.border_value, dtype=np.uint8)
    for tile in mo.tiles:
        img = cv2.resize(tile.image, (tile.resized[1], tile.resized[0]), interpolation=cv2.INTER_LINEAR)
        x1, y1, x2, y2 = tile.rect
        sx, sy = tile.origin
        canvas[y1:y2, x1:x2] = img[sy : sy + y2 - y1, sx : sx + x2 - x1]
    return canvas


def oracle_mosaic_u8(p: AugmentPlan) -> np.ndarray:
    """uint8 image DetectionStandardize receives for plan p (mosaic or not), computed with cv2 / numpy."""
    if p.mosaic is None:
        return oracle_u8(p)
    return oracle_u8(dataclasses.replace(p, image=oracle_canvas(p), mosaic=None))
