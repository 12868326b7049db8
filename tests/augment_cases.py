"""Test infrastructure for the detection train augmentation: seeded per-sample plans that cover the recipe chain's draws, and
`oracle_u8`, the reference's pixel operations (cv2.warpAffine, augment_hsv's cvtColor round trip, the flip, DetectionMixup's canvas
and blend, _rescale_and_pad_to_size) applied to a plan with cv2 and numpy, as transforms.py applies them."""
import ctypes
import math
import os
import subprocess
import tempfile

import cv2
import numpy as np

from super_gradients_b200.training.transforms.detection_augment import AugmentPlan, MixupPlan

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INPUT_DIM = (640, 640)
_LIB = {}


def host_lib():
    """g++ build of tests/host_kernels/augment_host.cpp around the product header augment_math.cuh."""
    if "h" not in _LIB:
        d = tempfile.mkdtemp(prefix="sgb_augment_host_")
        so = os.path.join(d, "augment_host.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", os.path.join(ROOT, "tests", "host_kernels", "augment_host.cpp"), "-I", os.path.join(ROOT, "include"),
                        "-I", os.path.join(ROOT, "super_gradients_b200", "csrc"), "-o", so], check=True)  # fmt: skip
        h = ctypes.CDLL(so)
        P, I, L = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64
        h.warp_affine_host.argtypes = [P, I, I, P, I, I, I, P]
        h.bgr2hsv_host.argtypes = [P, L, P]
        h.hsv2bgr_host.argtypes = [P, L, I, P]
        h.augment_host.argtypes = [P, P, I, I, I, I, I, P]
        _LIB["h"] = h
    return _LIB["h"]


def _p(a):
    return ctypes.c_void_p(a.ctypes.data)


def affine_matrix(rng, shape, target, degrees, translate, scales, shear):
    """The forward matrix of random_affine (transforms.py get_affine_matrix) from the given draws' ranges."""
    center = np.eye(3)
    center[0, 2], center[1, 2] = -(shape[1] // 2), -(shape[0] // 2)
    rot = np.eye(3)
    rot[:2] = cv2.getRotationMatrix2D(angle=rng.uniform(-degrees, degrees), center=(0, 0), scale=rng.uniform(*scales))
    sh = np.eye(3)
    sh[0, 1] = math.tan(rng.uniform(-shear, shear) * math.pi / 180)
    sh[1, 0] = math.tan(rng.uniform(-shear, shear) * math.pi / 180)
    tr = np.eye(3)
    tr[0, 2] = rng.uniform(0.5 - translate, 0.5 + translate) * target[1]
    tr[1, 2] = rng.uniform(0.5 - translate, 0.5 + translate) * target[0]
    return (tr @ sh @ rot @ center)[:2]


def _image(rng, h, w):
    """Smooth gradients plus noise: the resizes and the HSV round trip see every kind of neighbourhood."""
    yy, xx = np.mgrid[0:h, 0:w]
    base = np.stack([(xx * 255 // max(w - 1, 1)), (yy * 255 // max(h - 1, 1)), ((xx + yy) * 7) % 256], -1)
    noise = rng.integers(0, 256, (h, w, 3))
    return np.where(rng.random((h, w, 1)) < 0.3, noise, base).astype(np.uint8)


def make_plan(rng, h, w, degrees=0.0, shear=0.0, target_size=None, affine=True, swap=None, hsv=None, flip=None, mixup=None, mix_dim=None):
    img = _image(rng, h, w)
    tgt = target_size or (h, w)
    aff = (affine_matrix(rng, (h, w), tgt, degrees, 0.25, (0.5, 1.5), shear), tgt, 114) if affine else None
    th, tw = tgt if affine else (h, w)
    swap = bool(rng.random() < 0.5) if swap is None else swap
    if hsv is None:
        hsv = rng.random() < 0.5
    hsv_plan = None
    if hsv:
        g = (rng.uniform(-1, 1, 3) * [18, 30, 30] * rng.integers(0, 2, 3)).astype(np.int16)
        hsv_plan = (int(g[0]), int(g[1]), int(g[2]), (0, 1, 2) if hsv is True else hsv)
    flip = bool(rng.random() < 0.5) if flip is None else flip
    mix = None
    if mixup:
        mh, mw = mixup
        dim = mix_dim or (th, tw)
        ratio = min(dim[0] / mh, dim[1] / mw)
        r1 = (int(mh * ratio), int(mw * ratio))
        jit = rng.uniform(0.5, 1.5)
        r2 = (int(dim[0] * jit), int(dim[1] * jit))
        ph, pw = max(r2[0], th), max(r2[1], tw)
        y = int(rng.integers(0, ph - th)) if ph > th else 0  # random.randint(0, ph - th - 1)
        x = int(rng.integers(0, pw - tw)) if pw > tw else 0
        mix = MixupPlan(_image(rng, mh, mw), bool(rng.random() < 0.5), r1, tuple(dim), r2, x, y)
    r = min(INPUT_DIM[0] / th, INPUT_DIM[1] / tw)
    return AugmentPlan(img, (int(th * r), int(tw * r)), aff, swap, hsv_plan, flip, mix)


def cases(seed=0):
    """Sizes <= 640 in both orientations, one exactly 640 x 640, the recipe's draws (degrees 0, shear 0, target = image size)
    and the second list's (degrees 10, shear 5, target (640, 640)), mixups with and without a jittered crop, r != 1."""
    rng = np.random.default_rng(seed)
    return [
        make_plan(rng, 640, 640, hsv=True, flip=True, swap=True),
        make_plan(rng, 480, 640, mixup=(640, 427)),
        make_plan(rng, 640, 359, hsv=True, mixup=(333, 500)),
        make_plan(rng, 415, 333, hsv=(2, 1, 0), flip=False, mixup=(640, 640)),  # r != 1
        make_plan(rng, 233, 575, degrees=10, shear=5, target_size=(640, 640), hsv=True, mixup=(262, 638)),
        make_plan(rng, 638, 262, degrees=10, shear=5, target_size=(640, 640), hsv=True, flip=True, mixup=(480, 640), mix_dim=(640, 640)),
        make_plan(rng, 300, 500, affine=False, hsv=True, mixup=(500, 300)),
        make_plan(rng, 97, 61, degrees=10, shear=5, hsv=True, swap=True, flip=True),
    ]


def oracle_u8(p: AugmentPlan) -> np.ndarray:
    """uint8 image DetectionStandardize receives (the padded canvas, HWC) for plan p, computed with cv2 / numpy."""
    img = p.image.copy()
    if p.affine is not None:
        m, (rows, cols), border = p.affine
        img = cv2.warpAffine(img, m, dsize=(cols, rows), borderValue=(border, border, border))
    if p.swap:
        img = np.ascontiguousarray(img[..., ::-1])
    if p.hsv is not None:
        dh, ds, dv, bgr = p.hsv
        bgr = list(bgr)
        hsv = cv2.cvtColor(img[..., bgr], cv2.COLOR_BGR2HSV).astype(np.int16)
        hsv[..., 0] = (hsv[..., 0] + dh) % 180
        hsv[..., 1] = np.clip(hsv[..., 1] + ds, 0, 255)
        hsv[..., 2] = np.clip(hsv[..., 2] + dv, 0, 255)
        img[..., bgr] = cv2.cvtColor(hsv.astype(np.uint8), cv2.COLOR_HSV2BGR)
    if p.flip:
        img = img[:, ::-1]
    if p.mixup is not None:
        x = p.mixup
        cp = x.image[:, ::-1] if x.flip else x.image
        canvas = np.ones((x.canvas[0], x.canvas[1], 3), dtype=np.uint8) * x.border_value
        canvas[: x.resized[0], : x.resized[1]] = cv2.resize(np.ascontiguousarray(cp), (x.resized[1], x.resized[0]), interpolation=cv2.INTER_LINEAR)
        canvas = cv2.resize(canvas, (x.jittered[1], x.jittered[0]), interpolation=cv2.INTER_LINEAR)
        th, tw = img.shape[:2]
        padded = np.zeros((max(x.jittered[0], th), max(x.jittered[1], tw), 3), dtype=np.uint8)
        padded[: x.jittered[0], : x.jittered[1]] = canvas
        crop = padded[x.y_offset : x.y_offset + th, x.x_offset : x.x_offset + tw]
        img = (0.5 * img + 0.5 * crop).astype(np.uint8)
    out = np.full((INPUT_DIM[0], INPUT_DIM[1], 3), 114, dtype=np.uint8)
    rh, rw = p.rescaled
    out[:rh, :rw] = cv2.resize(np.ascontiguousarray(img), (rw, rh), interpolation=cv2.INTER_LINEAR)
    return out


class StubRawDataset:
    """Seeded raw samples in the reference's get_sample() form: sizes <= 640 in both orientations and one 640 x 640, crowd and
    non-crowd boxes, one image without targets, and thin / tiny boxes that the candidate and size filters drop."""

    SIZES = [(640, 640), (480, 640), (640, 427), (333, 500), (512, 384), (250, 600), (600, 250), (375, 375)]

    def __init__(self, seed=0):
        rng = np.random.default_rng(seed)
        self.samples = []
        for i, (h, w) in enumerate(self.SIZES):
            n = 0 if i == 3 else int(rng.integers(2, 9))
            x1, y1 = rng.uniform(0, w * 0.8, n), rng.uniform(0, h * 0.8, n)
            bw, bh = rng.uniform(2, w * 0.5, n), rng.uniform(2, h * 0.5, n)
            if n:
                bw[0], bh[-1] = 1.5, 0.8  # dropped by the box filters
            boxes = np.stack([x1, y1, np.minimum(x1 + bw, w), np.minimum(y1 + bh, h), rng.integers(0, 4, n)], -1).astype(np.float32)
            crowd = boxes[:1].copy() if i % 3 == 1 else np.zeros((0, 5), np.float32)
            self.samples.append({"image": _image(rng, h, w), "target": boxes, "crowd_target": crowd})

    def __len__(self):
        return len(self.samples)

    def get_sample(self, index, ignore_empty_annotations=False):
        s = self.samples[index]
        return {k: v.copy() for k, v in s.items()}


# the YOLO-NAS COCO recipe's train transforms (recipes/dataset_params/coco_detection_yolo_nas_dataset_params.yaml), and a second
# list with rotation, shear and a fixed affine target size
RECIPE = [
    ("DetectionRandomAffine", dict(degrees=0, translate=0.25, scales=[0.5, 1.5], shear=0, target_size=None, filter_box_candidates=True, wh_thr=2, area_thr=0.1, ar_thr=20)),
    ("DetectionRGB2BGR", dict(prob=0.5)),
    ("DetectionHSV", dict(prob=0.5, hgain=18, sgain=30, vgain=30)),
    ("DetectionHorizontalFlip", dict(prob=0.5)),
    ("DetectionMixup", dict(input_dim=None, mixup_scale=[0.5, 1.5], prob=0.5, flip_prob=0.5)),
    ("DetectionPaddedRescale", dict(input_dim=[640, 640], pad_value=114)),
    ("DetectionStandardize", dict(max_value=255)),
    ("DetectionTargetsFormatTransform", dict(input_format="XYXY_LABEL", output_format="LABEL_CXCYWH")),
]
SECOND = [(n, dict(kw, degrees=10, shear=5, target_size=(640, 640)) if n == "DetectionRandomAffine" else kw) for n, kw in RECIPE]
GOLDEN_LISTS = {"recipe": RECIPE, "second": SECOND}
GOLDEN_SEEDS = (0, 1, 2)
