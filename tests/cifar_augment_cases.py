"""Test infrastructure for the CIFAR-10 augmentation: the g++ build of its host driver, seeded 32 x 32 images, torchvision's chain
with given draws, and the golden file tests/golden/cifar_augment.pt."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MEAN = (0.4914, 0.4822, 0.4465)
STD = (0.2023, 0.1994, 0.2010)
GOLDEN_PATH = os.path.join(ROOT, "tests", "golden", "cifar_augment.pt")
_LIB = {}


def golden():
    if "g" not in _LIB:
        _LIB["g"] = torch.load(GOLDEN_PATH, weights_only=False)
    return _LIB["g"]


def host_lib():
    """g++ build of tests/host_kernels/cifar_augment_host.cpp around the product headers."""
    if "h" not in _LIB:
        d = tempfile.mkdtemp(prefix="sgb_cifar_augment_host_")
        so = os.path.join(d, "cifar_augment_host.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", os.path.join(ROOT, "tests", "host_kernels", "cifar_augment_host.cpp"), "-I",
                        os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "super_gradients_b200", "csrc"), "-o", so], check=True)  # fmt: skip
        h = ctypes.CDLL(so)
        P = ctypes.c_void_p
        h.augment_host.argtypes = [P, P, ctypes.c_int, P, P, P, P]
        h.bf16_host.argtypes = [P, ctypes.c_int, P]
        _LIB["h"] = h
    return _LIB["h"]


def _p(a):
    return ctypes.c_void_p(a.ctypes.data)


def host_augment(table, images, mean=MEAN, std=STD):
    """The host build of the kernel: (float32 [B, 3, 32, 32], bf16 bits int16 [B, 3, 32, 32]) for an int32 [B, 4] table over uint8
    [N, 32, 32, 3] images."""
    table = np.ascontiguousarray(table, np.int32)
    images = np.ascontiguousarray(images, np.uint8)
    B = len(table)
    f32, bf = np.empty((B, 3, 32, 32), np.float32), np.empty((B, 3, 32, 32), np.int16)
    m, s = np.array(mean, np.float32), np.array(std, np.float32)
    host_lib().augment_host(_p(table), _p(images), B, _p(m), _p(s), _p(f32), _p(bf))
    return f32, bf


def images(n, seed=0):
    """Seeded uint8 32 x 32 x 3 images: noise over gradients, with saturated 0 / 255 patches."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:32, 0:32]
    base = np.stack([xx * 8, yy * 8, (xx + yy) * 4], -1)
    out = np.where(rng.random((n, 32, 32, 1)) < 0.5, rng.integers(0, 256, (n, 32, 32, 3)), base[None]).astype(np.uint8)
    out[:, :4, :4] = 0
    out[:, -4:, -4:] = 255
    return out


def all_values_images():
    """Eight 32 x 32 x 3 images in which every channel takes every uint8 value (four times each, in a seeded order)."""
    rng = np.random.default_rng(1)
    return np.stack([np.stack([rng.permutation(np.repeat(np.arange(256), 4)) for _ in range(3)], -1).reshape(32, 32, 3) for _ in range(8)]).astype(np.uint8)


def torchvision_chain(image: np.ndarray, top: int, left: int, flip: bool, mean=MEAN, std=STD) -> torch.Tensor:
    """torchvision's RandomCrop(32, padding=4) -> RandomHorizontalFlip -> ToTensor -> Normalize on a PIL image with the given draws
    (the functional ops the transforms call after their draws)."""
    import torchvision.transforms.functional as TF
    from PIL import Image

    img = TF.crop(TF.pad(Image.fromarray(image), 4, 0, "constant"), top, left, 32, 32)
    if flip:
        img = TF.hflip(img)
    return TF.normalize(TF.to_tensor(img), list(mean), list(std))
