"""CPU checks of the pose train augmentation: the g++ build of csrc/pose_augment_math.cuh (the arithmetic of the two CUDA kernels)
is bit-exact with cv2.warpAffine in all five interpolation modes and with the reference's brightness-contrast, rot90, mosaic, pad and
resize; the host replay of the loader reproduces every reference target, and its plans every reference uint8 image, both through
a cv2 / numpy restatement and through the kernels' arithmetic."""
import hashlib

import cv2
import numpy as np
import pytest
import torch

from pose_augment_cases import GOLDEN_LISTS, _p, golden, host_lib, image, oracle_u8, replay
from super_gradients_b200 import kernels as K
from super_gradients_b200.training.transforms import keypoints as KP
from super_gradients_b200.training.transforms import keypoints_augment as PA


def _matrices():
    """The recipes' draws (rotation <= 7 degrees, scale 0.5 .. 1.75, translation <= 10 %), and maps that reach past the border."""
    rng = np.random.default_rng(7)
    h, w = 333, 517
    ms = [cv2.getRotationMatrix2D((w / 2 + rng.uniform(-0.1, 0.1) * w, h / 2 + rng.uniform(-0.1, 0.1) * h), rng.uniform(-7, 7), rng.uniform(0.5, 1.75))
          for _ in range(10)]  # fmt: skip
    ms.append(np.array([[1.0, 0.0, -400.3], [0.0, 1.0, 200.7]]))  # most of the output is border
    ms.append(np.array([[0.37, 0.91, -120.13], [-0.88, 0.41, 390.77]]))  # a large rotation: every tap crosses the border somewhere
    ms.append(np.array([[1.0, 0.0, 5000.5], [0.0, 1.0, -3000.25]]))  # the whole output is border
    return [np.ascontiguousarray(m, dtype=np.float64) for m in ms]


@pytest.mark.parametrize("mode", [0, 1, 2, 3, 4])
def test_warp_affine_every_mode_matches_cv2(mode):
    img = image(np.random.default_rng(mode), 333, 517)
    border = np.array([127, 30, 200], np.int32)
    phases = set()
    for m in _matrices():
        ref = cv2.warpAffine(img, m, dsize=(517, 333), flags=mode, borderMode=cv2.BORDER_CONSTANT, borderValue=tuple(int(b) for b in border))
        out = np.empty_like(ref)
        host_lib().warp_affine_mode_host(_p(img), 333, 517, _p(m), mode, _p(border), 333, 517, _p(out))
        assert np.array_equal(out, ref), int((out != ref).sum())
        inv = cv2.invertAffineTransform(m)
        yy, xx = np.mgrid[0:333, 0:517]
        phases |= set(np.unique((np.rint((inv[0, 0] * xx + inv[0, 1] * yy + inv[0, 2]) * 32).astype(np.int64) & 31) * 32
                                + (np.rint((inv[1, 0] * xx + inv[1, 1] * yy + inv[1, 2]) * 32).astype(np.int64) & 31)).tolist())  # fmt: skip
    assert len(phases) == 32 * 32  # every cv2 sub-pixel phase (every table row) was exercised


def _plan(rng, shapes, **tile):
    """A plan of len(shapes) tiles laid out as the mosaic does, each with the same draws."""
    tiles = [PA.TilePlan(image(rng, h, w), **tile) for h, w in shapes]
    if len(tiles) == 1:
        return PA.PosePlan(tiles, [(0, 0)], tiles[0].shape())
    (h0, w0), (h1, w1), (h2, w2), (h3, w3) = [t.shape() for t in tiles]
    ht, hb, W = max(h0, h1), max(h2, h3), max(w0 + w1, w2 + w3)
    lt, lb = (W - w0 - w1) // 2, (W - w2 - w3) // 2
    return PA.PosePlan(tiles, [(ht - h0, lt), (ht - h1, lt + w0), (ht, lb), (ht, lb + w2)], (ht + hb, W), (10, 20, 30))


def _host_chain(plans, size=640):
    raw = np.empty(PA.packed_size(plans), np.uint8)
    PA.pack_into(plans, raw)
    head = len(plans) * K.POSE_FIELDS * 8
    table, src = raw[:head].view(np.int64).reshape(len(plans), K.POSE_FIELDS).copy(), np.ascontiguousarray(raw[head:])
    ws = np.zeros(max(src.size, 1), np.uint8)
    out = np.empty((len(plans), size, size, 3), np.uint8)
    host_lib().pose_augment_host(_p(table), _p(src), _p(ws), len(plans), size, K.HSV_SIMD_BLOCK, _p(out))
    return out


def _check(plans):
    out = _host_chain(plans)
    for b, p in enumerate(plans):
        ref = oracle_u8(p)
        assert np.array_equal(out[b], ref), (b, int((out[b] != ref).any(-1).sum()))


def test_brightness_contrast_matches_numpy():
    rng = np.random.default_rng(1)
    plans = []
    for cg, bg in ((0.7, 1.3), (1.3, 0.7), (1.2, 1.2), (0.8134, 0.9261)):
        p = _plan(rng, [(97, 131)], flip=bool(rng.random() < 0.5))
        t = p.tiles[0]
        img = np.ascontiguousarray(np.fliplr(t.image)) if t.flip else t.image
        t.bc = (np.mean(img.astype(np.float32), axis=(0, 1)), cg, bg)
        p.resized, p.pad = (97, 131), (0, 0)
        plans.append(p)
    _check(plans)


@pytest.mark.parametrize("k", [0, 1, 2, 3])
def test_rot90_reverse_hsv_are_exact(k):
    rng = np.random.default_rng(k)
    p = _plan(rng, [(123, 211)], rot=k, reverse=True, hsv=(7, -11, 13), flip=k % 2 == 1)
    _check([p])


def test_mosaic_resize_and_center_pad_are_exact():
    """Four tiles of different sizes (rotated, warped with each mode), LongestMaxSize down to 640 and a center pad."""
    rng = np.random.default_rng(2)
    p = _plan(rng, [(300, 420), (250, 333), (411, 290), (199, 401)], rot=1)
    for i, t in enumerate(p.tiles):
        h, w = t.shape()
        t.affine = (cv2.getRotationMatrix2D((w / 2, h / 2), 5.0 * i - 7, 0.8 + 0.2 * i), i % 5, (127, 127, 127))
    s = min(640 / p.canvas[0], 640 / p.canvas[1])
    p.resized = (int(p.canvas[0] * s + 0.5), int(p.canvas[1] * s + 0.5))
    p.pad, p.pad_value = ((640 - p.resized[0]) // 2, (640 - p.resized[1]) // 2), (1, 2, 3)
    _check([p])


def test_exact_2x_mosaic_downscale():
    """Four 480 x 640 images make a 960 x 1280 mosaic that LongestMaxSize halves: cv2 runs that as INTER_AREA."""
    rng = np.random.default_rng(3)
    p = _plan(rng, [(480, 640)] * 4)
    assert p.canvas == (960, 1280)
    p.resized, p.pad = (480, 640), (80, 0)
    _check([p])
    canvas = np.concatenate([np.concatenate([t.image for t in p.tiles[:2]], 1), np.concatenate([t.image for t in p.tiles[2:]], 1)], 0)
    a = cv2.resize(canvas, (640, 480), interpolation=cv2.INTER_LINEAR)
    b = ((canvas[0::2, 0::2].astype(int) + canvas[0::2, 1::2] + canvas[1::2, 0::2] + canvas[1::2, 1::2] + 2) >> 2).astype(np.uint8)
    assert np.array_equal(a, b)


def test_upscale_and_bottom_right_pad_are_exact():
    rng = np.random.default_rng(4)
    p = _plan(rng, [(200, 301)], hsv=(-3, 20, -20))
    p.resized, p.pad = (425, 640), (0, 0)
    _check([p])


@pytest.mark.parametrize("case", sorted(golden()["cases"]))
def test_replay_matches_reference_goldens(case):
    """The loader's host half on the stub reproduces every reference target exactly, and its plans the reference's uint8 images,
    both through the cv2 / numpy restatement and through the kernels' arithmetic."""
    ref = golden()["cases"][case]
    _, items = replay(*case)
    out = _host_chain([plan for plan, _ in items])
    for i, ((plan, (boxes, joints, crowd)), r) in enumerate(zip(items, ref)):
        assert torch.equal(torch.from_numpy(boxes), r["boxes"]), (case, i)
        assert torch.equal(torch.from_numpy(joints), r["joints"]), (case, i)
        assert torch.equal(torch.from_numpy(crowd), r["is_crowd"]), (case, i)
        assert hashlib.sha256(oracle_u8(plan).tobytes()).hexdigest() == r["u8_sha256"], (case, i)
        assert hashlib.sha256(out[i].tobytes()).hexdigest() == r["u8_sha256"], (case, i)


def test_goldens_cover_mosaics_rotations_and_every_mode():
    seen = {"mosaic": 0, "rot": 0, "modes": set(), "bc": 0}
    for case in sorted(golden()["cases"]):
        for plan, _ in replay(*case)[1]:
            seen["mosaic"] += len(plan.tiles) == 4
            for t in plan.tiles:
                seen["rot"] += t.rot != 0
                seen["bc"] += t.bc is not None
                if t.affine is not None:
                    seen["modes"].add(t.affine[1])
    assert seen["mosaic"] >= 3 and seen["rot"] >= 3 and seen["bc"] >= 3 and seen["modes"] == {0, 1, 2, 3, 4}, seen


def test_bad_pipelines_raise():
    tail = [KP.KeypointsLongestMaxSize(640, 640), KP.KeypointsPadIfNeeded(640, 640, 127, 1), KP.KeypointsImageStandardize()]
    assert KP.check_pose_pipeline(tail) == 640
    with pytest.raises(ValueError):  # out of order
        KP.check_pose_pipeline([tail[1], tail[0], tail[2]])
    with pytest.raises(ValueError):  # no fixed square output
        KP.check_pose_pipeline([KP.KeypointsLongestMaxSize(640, 640), KP.KeypointsPadIfNeeded(640, 480, 127, 1), tail[2]])
    with pytest.raises(ValueError):
        KP.check_pose_pipeline([KP.KeypointsLongestMaxSize(640, 640, prob=0.5), tail[1], tail[2]])
    with pytest.raises(ValueError):
        KP.check_pose_pipeline(tail[1:])
    with pytest.raises(ValueError):  # a transform without a GPU pixel path
        KP.check_pose_pipeline([object()] + tail)
    with pytest.raises(ValueError):
        KP.KeypointsRandomAffineTransform(5, 0.5, 1.5, 0.1, 127, 1, interpolation_mode=[5])
    with pytest.raises(ValueError):
        PA.pack_into([PA.PosePlan.single(np.zeros((8, 8), np.uint8))], np.empty(10**4, np.uint8))


def test_registered_under_reference_names():
    from super_gradients_b200.common.registry import COLLATE_FUNCTIONS, TRANSFORMS

    for n, _ in GOLDEN_LISTS["heavy"]:
        assert n in TRANSFORMS, n
    assert "PoseAugmentCollateFN" in COLLATE_FUNCTIONS
