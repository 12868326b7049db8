"""Test infrastructure for the pose train augmentation: the g++ build of the kernels' arithmetic, a seeded stub pose dataset in the
reference's load_sample() form, the three YOLO-NAS-POSE recipe lists, `oracle_u8` (the reference's pixel operations applied to a
plan with cv2 / numpy, as the keypoint transforms apply them) and `replay` (the loader on the stub under a seed)."""
import ctypes
import os
import random
import subprocess
import tempfile
import types

import cv2
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN_PATH = os.path.join(ROOT, "tests", "golden", "pose_augment.pt")
_LIB = {}


def host_lib():
    """g++ build of tests/host_kernels/pose_augment_host.cpp around the product header pose_augment_math.cuh."""
    if "h" not in _LIB:
        d = tempfile.mkdtemp(prefix="sgb_pose_augment_host_")
        so = os.path.join(d, "pose_augment_host.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", os.path.join(ROOT, "tests", "host_kernels", "pose_augment_host.cpp"), "-I",
                        os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "super_gradients_b200", "csrc"), "-o", so], check=True)  # fmt: skip
        h = ctypes.CDLL(so)
        P, I = ctypes.c_void_p, ctypes.c_int
        h.warp_affine_mode_host.argtypes = [P, I, I, P, I, P, I, I, P]
        h.pose_augment_host.argtypes = [P, P, P, I, I, I, P]
        _LIB["h"] = h
    return _LIB["h"]


def _p(a):
    return ctypes.c_void_p(a.ctypes.data)


def image(rng, h, w):
    """Smooth gradients plus noise: the warps, resizes and the HSV round trip see every kind of neighbourhood."""
    yy, xx = np.mgrid[0:h, 0:w]
    base = np.stack([(xx * 255 // max(w - 1, 1)), (yy * 255 // max(h - 1, 1)), ((xx + yy) * 7) % 256], -1)
    noise = rng.integers(0, 256, (h, w, 3))
    return np.where(rng.random((h, w, 1)) < 0.3, noise, base).astype(np.uint8)


FLIP_INDEX = [0, 2, 1, 4, 3, 6, 5, 8, 7, 10, 9, 12, 11, 14, 13, 16, 15]


class StubPoseDataset:
    """Seeded samples in AbstractPoseEstimationDataset.load_sample() form: 480 x 640 (several, so mosaics of four of them hit an exact
    2x downscale), 640 x 480, 427 x 640, an odd size and one smaller than 640 (upscaled); crowd instances, joints outside the image
    and invisible ones, and one sample without instances.  `sample_cls` builds the returned object (the reference's
    PoseEstimationSample, or a namespace)."""

    SIZES = [(480, 640), (640, 480), (427, 640), (333, 517), (200, 300), (480, 640), (480, 640), (480, 640)]

    def __init__(self, sample_cls=None, seed=0, num_joints=17):
        self.sample_cls = sample_cls or (lambda **kw: types.SimpleNamespace(**kw))
        rng = np.random.default_rng(seed)
        self.samples = []
        for i, (h, w) in enumerate(self.SIZES):
            n = 0 if i == 4 else int(rng.integers(1, 6))
            x, y = rng.uniform(-0.05 * w, 0.9 * w, n), rng.uniform(-0.05 * h, 0.9 * h, n)
            bw, bh = rng.uniform(4, 0.4 * w, n), rng.uniform(4, 0.4 * h, n)
            boxes = np.stack([x, y, bw, bh], -1).astype(np.float32)
            joints = np.zeros((n, num_joints, 3), np.float32)
            joints[..., 0] = x[:, None] + rng.uniform(-0.1, 1.1, (n, num_joints)) * bw[:, None]
            joints[..., 1] = y[:, None] + rng.uniform(-0.1, 1.1, (n, num_joints)) * bh[:, None]
            joints[..., 2] = rng.choice([0.0, 1.0, 2.0], (n, num_joints), p=[0.3, 0.2, 0.5])
            areas = (bw * bh * rng.uniform(0.3, 0.7, n)).astype(np.float32)
            crowd = (rng.random(n) < 0.2).astype(np.int64)
            self.samples.append(dict(image=image(rng, h, w), joints=joints, areas=areas, bboxes_xywh=boxes, is_crowd=crowd))

    def __len__(self):
        return len(self.samples)

    def load_sample(self, index):
        s = {k: v.copy() for k, v in self.samples[index].items()}
        return self.sample_cls(image=s["image"], mask=np.ones(s["image"].shape[:2], np.float32), joints=s["joints"], areas=s["areas"],
                               bboxes_xywh=s["bboxes_xywh"], is_crowd=s["is_crowd"], additional_samples=None)  # fmt: skip


_COMMON_TAIL = [
    ("KeypointsLongestMaxSize", dict(max_height=640, max_width=640)),
    ("KeypointsPadIfNeeded", dict(min_height=640, min_width=640, image_pad_value=[127, 127, 127], mask_pad_value=1, padding_mode="center")),
    ("KeypointsImageStandardize", dict(max_value=255)),
    ("KeypointsRemoveSmallObjects", dict(min_instance_area=1, min_visible_keypoints=1)),
]
# recipes/dataset_params/coco_pose_estimation_yolo_nas{,_mosaic,_mosaic_heavy}_dataset_params.yaml, train transforms verbatim
BASE = [
    ("KeypointsRandomHorizontalFlip", dict(flip_index=FLIP_INDEX, prob=0.5)),
    ("KeypointsBrightnessContrast", dict(brightness_range=[0.8, 1.2], contrast_range=[0.8, 1.2], prob=0.5)),
    ("KeypointsHSV", dict(hgain=20, sgain=20, vgain=20, prob=0.5)),
    ("KeypointsRandomAffineTransform", dict(max_rotation=5, min_scale=0.5, max_scale=1.5, max_translate=0.1, image_pad_value=127, mask_pad_value=1, prob=0.75,
                                            interpolation_mode=[0, 1, 2, 3, 4])),  # fmt: skip
] + _COMMON_TAIL
MOSAIC = BASE[:3] + [
    ("KeypointsRandomAffineTransform", dict(max_rotation=5, min_scale=0.75, max_scale=1.5, max_translate=0.1, image_pad_value=127, mask_pad_value=1, prob=0.75,
                                            interpolation_mode=[0, 1, 2, 3, 4])),  # fmt: skip
    ("KeypointsMosaic", dict(prob=0.5)),
] + _COMMON_TAIL
HEAVY = [
    ("KeypointsRandomHorizontalFlip", dict(flip_index=FLIP_INDEX, prob=0.5)),
    ("KeypointsBrightnessContrast", dict(brightness_range=[0.7, 1.3], contrast_range=[0.7, 1.3], prob=0.75)),
    ("KeypointsReverseImageChannels", dict(prob=0.5)),
    ("KeypointsHSV", dict(hgain=25, sgain=25, vgain=25, prob=0.75)),
    ("KeypointsRandomRotate90", dict(prob=0.5)),
    ("KeypointsRandomAffineTransform", dict(max_rotation=7, min_scale=0.6, max_scale=1.75, max_translate=0.1, image_pad_value=127, mask_pad_value=1, prob=0.75,
                                            interpolation_mode=[0, 1, 2, 3, 4])),  # fmt: skip
    ("KeypointsMosaic", dict(prob=0.5)),
] + _COMMON_TAIL
GOLDEN_LISTS = {"base": BASE, "mosaic": MOSAIC, "heavy": HEAVY}
GOLDEN_SEEDS = (0, 1, 2)


def build(spec, module):
    return [getattr(module, n)(**kw) for n, kw in spec]


def replay(name, seed):
    """(dataset, items) of the loader over the stub for one golden list and seed, samples in index order."""
    from super_gradients_b200.training.datasets.pose_estimation_datasets.pose_augment_dataset import PoseAugmentDataset
    from super_gradients_b200.training.transforms import keypoints as KP

    ds = PoseAugmentDataset(StubPoseDataset(), build(GOLDEN_LISTS[name], KP))
    random.seed(seed)
    np.random.seed(seed)
    return ds, [ds[i] for i in range(len(ds))]


def golden():
    return torch.load(GOLDEN_PATH, weights_only=False)


def tile_u8(t) -> np.ndarray:
    """A tile's image after flip -> brightness-contrast -> reversal -> HSV -> rot90 -> affine, with the reference's cv2 / numpy calls."""
    img = np.ascontiguousarray(np.fliplr(t.image)) if t.flip else t.image.copy()
    if t.bc is not None:
        mean, cg, bg = t.bc
        f = (img.astype(np.float32) - np.asarray(mean, np.float32)) * cg + np.asarray(mean, np.float32) * bg
        img = np.clip(f, a_min=0, a_max=255).astype(np.uint8)
    if t.reverse:
        img = np.ascontiguousarray(img[:, :, ::-1])
    if t.hsv is not None:
        hsv = cv2.cvtColor(img, cv2.COLOR_BGR2HSV).astype(np.int16)
        hsv[..., 0] = (hsv[..., 0] + t.hsv[0]) % 180
        hsv[..., 1] = np.clip(hsv[..., 1] + t.hsv[1], 0, 255)
        hsv[..., 2] = np.clip(hsv[..., 2] + t.hsv[2], 0, 255)
        img = cv2.cvtColor(hsv.astype(np.uint8), cv2.COLOR_HSV2BGR)
    img = np.ascontiguousarray(np.rot90(img, t.rot))
    if t.affine is not None:
        m, mode, border = t.affine
        img = cv2.warpAffine(img, m, dsize=(img.shape[1], img.shape[0]), flags=mode, borderValue=border, borderMode=cv2.BORDER_CONSTANT)
    return img


def oracle_u8(p, size=640) -> np.ndarray:
    """uint8 image KeypointsImageStandardize receives (HWC) for plan p."""
    canvas = np.empty((p.canvas[0], p.canvas[1], 3), np.uint8)
    canvas[:] = np.array(p.mosaic_pad, np.uint8)
    for t, (y, x) in zip(p.tiles, p.positions):
        img = tile_u8(t)
        canvas[y : y + img.shape[0], x : x + img.shape[1]] = img
    if p.resized is not None and tuple(p.resized) != tuple(p.canvas):
        canvas = cv2.resize(canvas, (p.resized[1], p.resized[0]), interpolation=cv2.INTER_LINEAR)
    out = np.empty((size, size, 3), np.uint8)
    out[:] = np.array(p.pad_value, np.uint8)
    out[p.pad[0] : p.pad[0] + canvas.shape[0], p.pad[1] : p.pad[1] + canvas.shape[1]] = canvas
    return out
