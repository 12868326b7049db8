"""CPU checks of DetectionMosaic in the detection train augmentation against tests/golden/detection_mosaic.pt (the unmodified
reference on the seeded StubMosaicDataset): the host build of augment_math.cuh's mosaic canvas equals the reference
DetectionMosaic image pixel for pixel; the product's transforms, DetectionAugmentDataset and DetectionAugmentCollateFN reproduce
every target of the four fixture lists and the host build of the kernel every uint8 image's sha256; the transform's
registration, constructor, close() and place in the list; DataLoader workers collate mosaic batches without CUDA."""
import hashlib
import os
import random
from unittest import mock

import numpy as np
import pytest
import torch

from augment_cases import _p, host_lib
from mosaic_cases import CANVAS_CASES, GOLDEN_LISTS, StubMosaicDataset, mosaic_lib, oracle_canvas
from super_gradients_b200 import kernels as K
from super_gradients_b200.common.registry import TRANSFORMS
from super_gradients_b200.training.datasets.detection_augment_dataset import DetectionAugmentCollateFN, DetectionAugmentDataset, PackedDetectionBatch
from super_gradients_b200.training.transforms import detection_augment as DA
from super_gradients_b200.training.transforms import transforms as T

GOLDEN = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "detection_mosaic.pt"), weights_only=False)


def make_dataset(name):
    return DetectionAugmentDataset(StubMosaicDataset(), [TRANSFORMS[n](**kw) for n, kw in GOLDEN_LISTS[name]])


def replay(name, seed):
    ds = make_dataset(name)
    random.seed(seed)
    np.random.seed(seed)
    return ds, [ds[i] for i in range(len(ds))]


def packed(plans):
    raw = np.empty(DA.packed_size(plans), np.uint8)
    DA.pack_into(plans, raw)
    head = len(plans) * K.AUG_FIELDS * 8
    return raw[:head].view(np.int64).reshape(len(plans), K.AUG_FIELDS).copy(), np.ascontiguousarray(raw[head:])


def host_canvas(plan) -> np.ndarray:
    table, src = packed([plan])
    out = np.empty((plan.mosaic.canvas[0], plan.mosaic.canvas[1], 3), np.uint8)
    mosaic_lib().mosaic_canvas_host(_p(table[0]), _p(src), _p(out))
    return out


def mosaic_sample(indices, input_dim, draws, stub=None):
    """The product's DetectionMosaic on the stub samples `indices` with random.uniform returning `draws` (yc, then xc)."""
    stub = stub or StubMosaicDataset()
    sample = T.HostSample.from_dict(stub.get_sample(indices[0]))
    sample.additional_samples = [T.HostSample.from_dict(stub.get_sample(j)) for j in indices[1:]]
    with mock.patch("random.uniform", side_effect=list(draws)):
        return T.DetectionMosaic(input_dim=input_dim).apply_to_sample(sample)


@pytest.mark.parametrize("k", range(len(CANVAS_CASES)))
def test_canvas_matches_reference_mosaic(k):
    ref = GOLDEN["canvases"][k]
    s = mosaic_sample(*CANVAS_CASES[k])
    canvas = host_canvas(s.plan)
    assert canvas.shape == ref["shape"] and s.shape == ref["shape"][:2]
    assert hashlib.sha256(canvas.tobytes()).hexdigest() == ref["canvas_sha256"]
    assert np.array_equal(canvas, oracle_canvas(s.plan))
    assert s.bboxes_xyxy.dtype == ref["bboxes"].numpy().dtype and torch.equal(torch.from_numpy(s.bboxes_xyxy), ref["bboxes"])
    assert torch.equal(torch.from_numpy(s.labels), ref["labels"]) and torch.equal(torch.from_numpy(s.is_crowd), ref["is_crowd"])


def test_canvas_at_random_centres():
    """Random tiles and centres anywhere on the canvas, edges included: the host kernel's canvas is cv2's, pixel for pixel."""
    rng = np.random.default_rng(7)
    stub = StubMosaicDataset()
    for it in range(12):
        input_dim = int(rng.choice([640, 384, 100]))
        yc, xc = (float(rng.integers(0, 2 * input_dim + 1)) for _ in range(2))
        if it < 4:
            yc, xc = [(0.0, 0.0), (2.0 * input_dim, 2.0 * input_dim), (0.0, 2.0 * input_dim), (2.0 * input_dim, 0.0)][it]
        s = mosaic_sample([int(i) for i in rng.integers(0, len(stub), 4)], input_dim, (yc, xc), stub)
        assert np.array_equal(host_canvas(s.plan), oracle_canvas(s.plan)), (it, input_dim, yc, xc)


def host_u8(batch: PackedDetectionBatch) -> np.ndarray:
    raw = batch.buffer.numpy()
    head = batch.batch * K.AUG_FIELDS * 8
    table, src = raw[:head].view(np.int64).copy(), np.ascontiguousarray(raw[head:])
    out = np.empty((batch.batch, 640, 640, 3), np.uint8)
    host_lib().augment_host(_p(table), _p(src), batch.batch, 640, 640, batch.pad_value, K.HSV_SIMD_BLOCK, _p(out))
    return out


@pytest.mark.parametrize("case", sorted(GOLDEN["cases"]), ids=lambda c: f"{c[0]}-{c[1]}")
def test_replay_matches_reference(case):
    ds, items = replay(*case)
    ref = GOLDEN["cases"][case]
    for i, ((_, target), r) in enumerate(zip(items, ref)):
        assert target.dtype == np.float32 and torch.equal(torch.from_numpy(target), r["target"]), (case, i)
    mosaics = sum(p.mosaic is not None for p, _ in items)
    if case[0] == "roboflow_closed":
        assert mosaics == 0
    elif case[0] != "mosaic_coco":
        assert mosaics == len(items)
    batch = DetectionAugmentCollateFN.for_dataset(ds)(items)
    u8 = host_u8(batch)
    for i, r in enumerate(ref):
        assert hashlib.sha256(u8[i].tobytes()).hexdigest() == r["u8_sha256"], (case, i)
    rows = torch.cat([torch.cat((torch.full((len(r["target"]), 1), float(i)), r["target"]), 1) for i, r in enumerate(ref)])
    assert torch.equal(batch.targets, rows)


def test_mosaic_coco_mixes_both_kinds_in_one_batch():
    _, items = replay("mosaic_coco", 0)
    kinds = {p.mosaic is not None for p, _ in items}
    assert kinds == {True, False}
    assert any(p.mosaic is not None and p.mixup is not None for p, _ in items)


def test_registered_constructor_and_close():
    assert TRANSFORMS["DetectionMosaic"] is T.DetectionMosaic
    m = T.DetectionMosaic(input_dim=384)
    assert m.input_dim == (384, 384) and m.prob == 1.0 and m.enable_mosaic and m.border_value == 114 and m.may_require_additional_samples
    m = T.DetectionMosaic([640, 512], prob=0.25, enable_mosaic=True, border_value=0)
    assert m.input_dim == (640, 512) and m.prob == 0.25 and m.border_value == 0
    random.seed(3)
    draws = [m.get_number_of_additional_samples() for _ in range(200)]
    random.seed(3)
    assert draws == [3 if random.random() < 0.25 else 0 for _ in range(200)]
    m.close()
    assert not m.enable_mosaic and not m.may_require_additional_samples
    state = random.getstate()
    assert m.get_number_of_additional_samples() == 0 and random.getstate() == state  # a closed mosaic draws nothing
    ds = make_dataset("roboflow")
    for t in ds.transforms:
        t.close()
    random.seed(0)
    np.random.seed(0)
    assert all(ds[i][0].mosaic is None and ds[i][0].affine is None for i in range(len(ds)))


def test_order_checked():
    rest = [T.DetectionPaddedRescale(640), T.DetectionStandardize()]
    DetectionAugmentDataset(StubMosaicDataset(), [T.DetectionMosaic(640), T.DetectionHSV(0.5)] + rest)
    with pytest.raises(ValueError):  # not first
        DetectionAugmentDataset(StubMosaicDataset(), [T.DetectionHSV(0.5), T.DetectionMosaic(640)] + rest)
    with pytest.raises(ValueError):
        DetectionAugmentDataset(StubMosaicDataset(), [T.DetectionRandomAffine(), T.DetectionMosaic(640)] + rest)
    with pytest.raises(ValueError):  # twice
        DetectionAugmentDataset(StubMosaicDataset(), [T.DetectionMosaic(640), T.DetectionMosaic(640)] + rest)


def test_pack_refuses_a_mosaic_without_the_samples_image():
    s = mosaic_sample((0, 1, 2, 3), 640, (640.0, 640.0))
    s.plan.mosaic.tiles[0].image = s.plan.mosaic.tiles[0].image.copy()
    with pytest.raises(ValueError):
        DA.pack_into([s.plan], np.empty(DA.packed_size([s.plan]), np.uint8))


def test_dataloader_workers_collate_without_cuda():
    ds = make_dataset("roboflow")
    loader = torch.utils.data.DataLoader(ds, batch_size=4, num_workers=2, collate_fn=DetectionAugmentCollateFN.for_dataset(ds))
    batches = list(loader)
    assert len(batches) == 2 and all(isinstance(b, PackedDetectionBatch) and b.batch == 4 for b in batches)
    for b in batches:
        table = b.buffer[: b.batch * K.AUG_FIELDS * 8].view(torch.int64).view(b.batch, K.AUG_FIELDS)
        assert bool((table[:, DA.MOS] == 1).all())
