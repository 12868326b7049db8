"""Test infrastructure for the ImageNet train augmentation: the g++ build of its host driver, seeded images, `pil_op` (one RandAugment
op through Pillow, as datasets/auto_augment.py calls it) and the seeded stub dataset the goldens and the replay run over."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
from PIL import Image, ImageEnhance, ImageOps

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZE = 224
IMG_MEAN = [0.485, 0.456, 0.406]
IMG_STD = [0.229, 0.224, 0.225]
FILL = tuple(min(255, round(255 * m)) for m in IMG_MEAN)  # rand_augment_transform's img_mean hparam
CONFIG = "rand-m7-mstd0.5"
_LIB = {}


def host_lib():
    """g++ build of tests/host_kernels/imagenet_augment_host.cpp around the product headers."""
    if "h" not in _LIB:
        d = tempfile.mkdtemp(prefix="sgb_imagenet_augment_host_")
        so = os.path.join(d, "imagenet_augment_host.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", os.path.join(ROOT, "tests", "host_kernels", "imagenet_augment_host.cpp"), "-I",
                        os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "super_gradients_b200", "csrc"), "-o", so], check=True)  # fmt: skip
        h = ctypes.CDLL(so)
        P, I = ctypes.c_void_p, ctypes.c_int
        h.resize_host.argtypes = [P, I, I, I, I, I, P]
        h.op_host.argtypes = [P, I, P, P]
        h.augment_host.argtypes = [P, P, I, I, P, P]
        _LIB["h"] = h
    return _LIB["h"]


def _p(a):
    return ctypes.c_void_p(a.ctypes.data)


def image(rng, h, w):
    """Smooth gradients plus noise: the resizes and the filters see every kind of neighbourhood."""
    yy, xx = np.mgrid[0:h, 0:w]
    base = np.stack([(xx * 255 // max(w - 1, 1)), (yy * 255 // max(h - 1, 1)), ((xx + yy) * 7) % 256], -1)
    noise = rng.integers(0, 256, (h, w, 3))
    return np.where(rng.random((h, w, 1)) < 0.3, noise, base).astype(np.uint8)


def pil_op(img: Image.Image, name: str, magnitude: float, negate: bool, fill=FILL) -> Image.Image:
    """RandAugment op `name` at `magnitude` through Pillow, with _randomly_negate's outcome `negate`."""
    level = magnitude / 10.0
    sign = -1.0 if negate else 1.0
    kw = dict(resample=Image.BILINEAR, fillcolor=fill)
    if name == "AutoContrast":
        return ImageOps.autocontrast(img)
    if name == "Equalize":
        return ImageOps.equalize(img)
    if name == "Invert":
        return ImageOps.invert(img)
    if name == "Rotate":
        return img.rotate(sign * level * 30.0, **kw)
    if name == "Posterize":
        bits = int(level * 4)
        return img if bits >= 8 else ImageOps.posterize(img, bits)
    if name == "Solarize":
        return ImageOps.solarize(img, int(level * 256))
    if name == "SolarizeAdd":
        add = int(level * 110)
        return img.point([min(255, i + add) if i < 128 else i for i in range(256)] * 3)
    if name in ("Color", "Contrast", "Brightness", "Sharpness"):
        return getattr(ImageEnhance, name)(img).enhance(level * 1.8 + 0.1)
    if name == "ShearX":
        return img.transform(img.size, Image.AFFINE, (1, sign * level * 0.3, 0, 0, 1, 0), **kw)
    if name == "ShearY":
        return img.transform(img.size, Image.AFFINE, (1, 0, 0, sign * level * 0.3, 1, 0), **kw)
    if name == "TranslateXRel":
        return img.transform(img.size, Image.AFFINE, (1, 0, sign * level * 0.45 * img.size[0], 0, 1, 0), **kw)
    if name == "TranslateYRel":
        return img.transform(img.size, Image.AFFINE, (1, 0, 0, 0, 1, sign * level * 0.45 * img.size[1]), **kw)
    raise ValueError(name)


class StubImageDataset:
    """Seeded (uint8 H x W x 3 RGB, label) samples of mixed sizes: square, portrait and landscape, smaller than the 224 crop, one
    larger than 1000 on a side, and one so narrow that RandomResizedCrop falls back to its centre crop."""

    SIZES = [(375, 500), (500, 333), (224, 224), (120, 90), (60, 200), (1203, 817), (640, 480), (333, 1100), (31, 400), (256, 256)]

    def __init__(self, seed=0, length=None):
        rng = np.random.default_rng(seed)
        self.samples = [(image(rng, h, w), int(rng.integers(0, 1000))) for h, w in self.SIZES]
        self.length = length or len(self.samples)

    def __len__(self):
        return self.length

    def __getitem__(self, index):
        im, label = self.samples[index % len(self.samples)]
        return im.copy(), label


GOLDEN_BATCH = 256
# golden cases (collate parameters, seed): the recipe's CollateMixup at two seeds, and parameters that force a no-mix, a mixup and a
# cutmix batch
GOLDEN_CASES = (("recipe", 0), ("recipe", 1), ("nomix", 0), ("mixup", 0), ("cutmix", 0))
GOLDEN_MIX = {
    "recipe": dict(mixup_alpha=0.2, cutmix_alpha=1.0, label_smoothing=0.1),
    "nomix": dict(mixup_alpha=0.2, cutmix_alpha=1.0, prob=0.0, label_smoothing=0.1),
    "mixup": dict(mixup_alpha=0.2, cutmix_alpha=0.0, label_smoothing=0.1),
    "cutmix": dict(mixup_alpha=0.0, cutmix_alpha=1.0, label_smoothing=0.1),
}
