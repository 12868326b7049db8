"""CPU checks of the detection train augmentation: the g++ build of csrc/augment_math.cuh (the arithmetic of the CUDA kernel) is
bit-exact with cv2 for warpAffine, every BGR -> HSV colour and every HSV -> BGR triple on both of cv2's code paths, and
for the whole per-sample chain; the batch packing writes the table the kernel reads."""
import cv2
import numpy as np
import pytest

from augment_cases import _image, _p, affine_matrix, cases, host_lib, oracle_u8
from super_gradients_b200 import kernels as K
from super_gradients_b200.training.transforms import detection_augment as DA


def _warp_matrices():
    rng = np.random.default_rng(1)
    ms = []
    for degrees, shear, scales in ((10, 0, (0.58, 0.6)), (0, 5, (1.1, 1.16)), (30, 8, (0.3, 0.4)), (0, 0, (1.5, 2.0)), (170, 3, (0.9, 1.1))):
        ms.append(affine_matrix(rng, (333, 517), (400, 600), degrees, 0.25, scales, shear))
    far = np.array([[1.0, 0.0, 5000.5], [0.0, 1.0, -3000.25]])  # the whole output is border
    edge = np.array([[0.75, 0.1, -200.0], [-0.05, 1.25, -120.0]])  # part of the output is border
    return ms + [far, edge]


@pytest.mark.parametrize("i", range(7))
def test_warp_affine_matches_cv2(i):
    m = np.ascontiguousarray(_warp_matrices()[i], dtype=np.float64)
    img = _image(np.random.default_rng(i), 333, 517)
    oh, ow = 400, 600
    ref = cv2.warpAffine(img, m, dsize=(ow, oh), borderValue=(114, 114, 114))
    out = np.empty((oh, ow, 3), np.uint8)
    host_lib().warp_affine_host(_p(img), 333, 517, _p(m), 114, oh, ow, _p(out))
    assert np.array_equal(out, ref), int((out != ref).sum())


def test_bgr2hsv_every_colour():
    v = np.arange(1 << 24, dtype=np.uint32)
    bgr = np.stack([v & 255, (v >> 8) & 255, v >> 16], -1).astype(np.uint8)
    out = np.empty_like(bgr)
    host_lib().bgr2hsv_host(_p(bgr), bgr.shape[0], _p(out))
    for width in (4096, 1 << 24, 1):  # cv2's vector blocks, one long row, and its scalar path
        ref = cv2.cvtColor(bgr.reshape(-1, width, 3), cv2.COLOR_BGR2HSV).reshape(-1, 3)
        assert np.array_equal(out, ref), (width, int((out != ref).any(1).sum()))


@pytest.mark.parametrize("vec", [1, 0])
def test_hsv2bgr_every_triple(vec):
    h, s, v = np.meshgrid(np.arange(180), np.arange(256), np.arange(256), indexing="ij")
    hsv = np.ascontiguousarray(np.stack([h, s, v], -1).astype(np.uint8).reshape(-1, 3))
    out = np.empty_like(hsv)
    host_lib().hsv2bgr_host(_p(hsv), hsv.shape[0], vec, _p(out))
    width = 256 if vec else 1  # rows of whole vector blocks, or rows short enough that every pixel takes the scalar tail
    ref = cv2.cvtColor(hsv.reshape(-1, width, 3), cv2.COLOR_HSV2BGR).reshape(-1, 3)
    assert np.array_equal(out, ref), int((out != ref).any(1).sum())


def test_hsv2bgr_vector_block_is_32_pixels():
    """Columns below w - w % 32 take cv2's vector path; a row of 65 pixels has one scalar column."""
    rng = np.random.default_rng(3)
    hsv = np.stack([rng.integers(0, 180, (64, 65)), rng.integers(0, 256, (64, 65)), rng.integers(0, 256, (64, 65))], -1).astype(np.uint8)
    ref = cv2.cvtColor(hsv, cv2.COLOR_HSV2BGR)
    flat = np.ascontiguousarray(hsv.reshape(-1, 3))
    vec, sca = np.empty_like(flat), np.empty_like(flat)
    host_lib().hsv2bgr_host(_p(flat), flat.shape[0], 1, _p(vec))
    host_lib().hsv2bgr_host(_p(flat), flat.shape[0], 0, _p(sca))
    in_block = (np.arange(65) < 65 - 65 % K.HSV_SIMD_BLOCK)[None, :, None]
    want = np.where(in_block, vec.reshape(64, 65, 3), sca.reshape(64, 65, 3))
    assert np.array_equal(want, ref)


def _pack(plans):
    aug = DA.BatchAugmenter()
    staging, used = aug.pack(plans, pin=False)
    head = len(plans) * K.AUG_FIELDS * 8
    raw = staging.numpy()[:used]
    return raw[:head].view(np.int64).reshape(len(plans), K.AUG_FIELDS).copy(), np.ascontiguousarray(raw[head:])


def test_whole_chain_matches_cv2_numpy():
    plans = cases()
    table, src = _pack(plans)
    out = np.empty((len(plans), 640, 640, 3), np.uint8)
    host_lib().augment_host(_p(table), _p(src), len(plans), 640, 640, 114, K.HSV_SIMD_BLOCK, _p(out))
    for b, p in enumerate(plans):
        ref = oracle_u8(p)
        assert np.array_equal(out[b], ref), (b, int((out[b] != ref).any(-1).sum()))


def test_table_layout():
    plans = cases()[:3]
    table, src = _pack(plans)
    m = plans[1].affine[0]
    assert np.array_equal(table[1, DA.M : DA.M + 6].view(np.float64), m.reshape(6))
    off = int(table[2, DA.MIX_OFFSET])
    mh, mw = plans[2].mixup.image.shape[:2]
    assert np.array_equal(src[off : off + mh * mw * 3].reshape(mh, mw, 3), plans[2].mixup.image)
    assert tuple(table[0, [DA.RS_H, DA.RS_W]]) == (640, 640) and table[0, DA.MIX] == 0


def test_bad_input_raises():
    p = cases()[0]
    with pytest.raises(ValueError):
        DA.BatchAugmenter().pack([DA.AugmentPlan(p.image.astype(np.float32), p.rescaled)], pin=False)
    with pytest.raises(ValueError):
        DA.BatchAugmenter().pack([DA.AugmentPlan(p.image[..., :2].copy(), p.rescaled)], pin=False)
    with pytest.raises(ValueError):
        DA.BatchAugmenter().pack([DA.AugmentPlan(p.image, p.rescaled, hsv=(0, 0, 0, (0, 0, 1)))], pin=False)
