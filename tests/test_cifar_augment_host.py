"""CPU checks of the CIFAR-10 augmentation's arithmetic: the g++ build of csrc/cifar_augment_math.cuh (what the CUDA kernel computes)
reproduces every float32 value of the reference chains' golden bit for bit, its bf16 rounding is torch's, and every crop corner
with and without the flip matches torchvision's functional chain."""
import numpy as np
import pytest
import torch

from cifar_augment_cases import _p, all_values_images, golden, host_augment, host_lib, images, torchvision_chain


def _bits(x: torch.Tensor) -> np.ndarray:
    return x.bfloat16().view(torch.int16).numpy()


def test_train_golden_bit_for_bit():
    g = golden()["train"]
    table = np.concatenate([np.arange(len(g["draws"]), dtype=np.int32)[:, None], g["draws"].numpy()], 1)
    f32, bf = host_augment(table, g["images"].numpy())
    assert np.array_equal(f32.view(np.int32), g["output"].numpy().view(np.int32))
    assert np.array_equal(bf, _bits(g["output"]))


def test_validation_golden_every_value_bit_for_bit():
    g = golden()["val"]
    assert np.array_equal(g["images"].numpy(), all_values_images())
    table = np.array([(b, 4, 4, 0) for b in range(len(g["images"]))], np.int32)
    f32, bf = host_augment(table, g["images"].numpy())
    assert np.array_equal(f32.view(np.int32), g["output"].numpy().view(np.int32))
    assert np.array_equal(bf, _bits(g["output"]))


@pytest.mark.parametrize("flip", [0, 1])
def test_every_crop_corner_matches_torchvision(flip):
    ims = images(81, seed=3)
    table = np.array([(k, k // 9, k % 9, flip) for k in range(81)], np.int32)
    f32, bf = host_augment(table, ims)
    ref = torch.stack([torchvision_chain(ims[k], k // 9, k % 9, bool(flip)) for k in range(81)])
    assert np.array_equal(f32.view(np.int32), ref.numpy().view(np.int32))
    assert np.array_equal(bf, _bits(ref))


def test_bf16_rounding_is_torchs():
    """Round-to-nearest-even at ties both ways, the carry into the exponent, the largest finite value, infinities, NaN, zeros,
    subnormals and a million random bit patterns, as tensor.to(torch.bfloat16) rounds them."""
    special = np.array([0x3F808000, 0x3F818000, 0x3F80FFFF, 0x3FFFFFFF, 0x7F7FFFFF, 0x7F800000, 0xFF800000, 0x7FC00001, 0x80000000, 0x00000001, 0xBF808001], np.uint32)
    bits = np.concatenate([special, np.random.default_rng(0).integers(0, 2**32, 1 << 20, dtype=np.uint32)])
    vals = bits.view(np.float32)
    got = np.empty(len(vals), np.int16)
    host_lib().bf16_host(_p(vals), len(vals), _p(got))
    want = torch.from_numpy(vals.copy()).bfloat16().view(torch.int16).numpy()
    nan = np.isnan(vals)
    assert np.array_equal(got[~nan], want[~nan])
    assert (got[nan] & 0x7FFF == 0x7FC0).all()
