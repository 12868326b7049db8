"""CPU checks of the ImageNet train augmentation: the g++ build of csrc/imagenet_augment_math.cuh and the bicubic filter of
resample_math.cuh (the arithmetic of the CUDA kernel) is bit-exact with the installed Pillow for every RandAugment op and the
crop resize; CrossEntropyLoss takes the [B, C] probability targets CollateMixup makes."""
import random

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from PIL import Image

from imagenet_augment_cases import FILL, SIZE, _p, host_lib, image, pil_op
from super_gradients_b200.training.losses.cross_entropy import CrossEntropyLoss
from super_gradients_b200.training.transforms import imagenet_augment as IA


def _host_op(img, name, magnitude, negate, monkeypatch):
    monkeypatch.setattr(IA.random, "random", lambda: 0.9 if negate else 0.1)  # _randomly_negate's draw
    code, args = IA.op_plan(name, magnitude, img.shape[1])
    out = img.copy()
    host_lib().op_host(_p(out), img.shape[1], _p(np.array([code] + args, np.int64)), _p(np.array(FILL, np.int32)))
    return out


@pytest.mark.parametrize("name", IA.RAND_TRANSFORMS)
@pytest.mark.parametrize("magnitude", [0, 7, 10, 6.37])
@pytest.mark.parametrize("negate", [False, True])
def test_op_matches_pillow(name, magnitude, negate, monkeypatch):
    img = image(np.random.default_rng(IA.RAND_TRANSFORMS.index(name) * 10 + int(magnitude)), SIZE, SIZE)
    ref = np.asarray(pil_op(Image.fromarray(img), name, magnitude, negate))
    out = _host_op(img, name, magnitude, negate, monkeypatch)
    assert np.array_equal(out, ref), int((out != ref).any(-1).sum())


@pytest.mark.parametrize("name", ["Rotate", "ShearX", "ShearY"])
def test_fill_reaches_the_corners(name, monkeypatch):
    img = image(np.random.default_rng(5), SIZE, SIZE)
    out = _host_op(img, name, 10, True, monkeypatch)
    assert any(tuple(out[y, x]) == FILL for y in (0, SIZE - 1) for x in (0, SIZE - 1))
    assert np.array_equal(out, np.asarray(pil_op(Image.fromarray(img), name, 10, True)))


def test_autocontrast_flat_channel_and_equalize_one_value(monkeypatch):
    img = image(np.random.default_rng(7), SIZE, SIZE)
    img[..., 1] = 77  # flat channel: AutoContrast leaves it alone
    img[..., 2] = 200  # one-value histogram: Equalize leaves it alone
    for name in ("AutoContrast", "Equalize"):
        out = _host_op(img, name, 7, False, monkeypatch)
        assert np.array_equal(out, np.asarray(pil_op(Image.fromarray(img), name, 7, False))), name
        assert (out[..., 1] == 77).all() and (out[..., 2] == 200).all()


def test_equalize_two_values_and_contrast_of_a_flat_image(monkeypatch):
    img = np.zeros((SIZE, SIZE, 3), np.uint8)
    img[: SIZE // 3] = 240
    for name in ("Equalize", "Contrast", "Sharpness", "Color"):
        for m in (0, 10):
            assert np.array_equal(_host_op(img, name, m, False, monkeypatch), np.asarray(pil_op(Image.fromarray(img), name, m, False))), (name, m)


@pytest.mark.parametrize("filt", [IA.BILINEAR, IA.BICUBIC])
@pytest.mark.parametrize("hw", [(1, 1), (3, 5), (7, 2), (224, 224), (224, 97), (300, 224), (1000, 950), (1203, 817), (4000, 240), (150, 2900)])
def test_crop_resize_matches_pillow(filt, hw):
    """Upscales of a few-pixel crop, unchanged axes, and downscales by up to ~18x (more than 4x on some axis)."""
    h, w = hw
    img = image(np.random.default_rng(h * 7 + w), h, w)
    ref = np.asarray(Image.fromarray(img).resize((SIZE, SIZE), Image.BICUBIC if filt == IA.BICUBIC else Image.BILINEAR))
    out = np.empty((SIZE, SIZE, 3), np.uint8)
    host_lib().resize_host(_p(img), h, w, SIZE, SIZE, filt, _p(out))
    assert np.array_equal(out, ref), int((out != ref).any(-1).sum())


def test_plan_rotate_matrix_is_pillows():
    """Image.rotate's matrix, through Image.transform, gives Image.rotate's pixels (both signs, the fast path at 0 degrees)."""
    img = Image.fromarray(image(np.random.default_rng(3), SIZE, SIZE))
    for deg in (-30.0, -13.7, 0.0, 21.0):
        m = IA.rotate_matrix(deg, SIZE, SIZE)
        a = np.asarray(img.transform(img.size, Image.AFFINE, m, resample=Image.BILINEAR, fillcolor=FILL))
        assert np.array_equal(a, np.asarray(img.rotate(deg, resample=Image.BILINEAR, fillcolor=FILL))), deg


def test_cross_entropy_probability_targets_match_the_reference_formula():
    """The reference's cross_entropy with float targets is -(target * log_softmax(x)).sum(-1).mean(); the product's loss gives the
    same loss and gradient for CollateMixup's [B, C] two-hot smoothed targets."""
    g = torch.Generator().manual_seed(0)
    x = torch.randn(16, 1000, generator=g, dtype=torch.float64)
    labels = torch.randint(0, 1000, (16,), generator=g)
    off, lam = 0.1 / 1000, 0.73
    y1 = torch.full((16, 1000), off, dtype=torch.float64).scatter_(1, labels.view(-1, 1), 0.9 + off)
    target = y1 * lam + y1.flip(0) * (1 - lam)
    a, b = x.clone().requires_grad_(), x.clone().requires_grad_()
    loss, item = CrossEntropyLoss()(a, target)
    ref = -(target * F.log_softmax(b, dim=-1)).sum(-1).mean()
    loss.backward()
    ref.backward()
    assert torch.allclose(loss.double(), ref, rtol=1e-6, atol=0) and item.shape == (1,)
    assert torch.allclose(a.grad, b.grad, rtol=1e-5, atol=1e-9)
