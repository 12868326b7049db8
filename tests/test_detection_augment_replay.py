"""CPU replay of tests/golden/detection_augment.pt (the unmodified reference transforms on the seeded stub dataset): the product's
transforms, DetectionAugmentDataset and DetectionAugmentCollateFN reproduce every target exactly, and the host build of the
augmentation kernel reproduces every uint8 image's sha256."""
import hashlib
import os
import random

import numpy as np
import pytest
import torch

from augment_cases import GOLDEN_LISTS, StubRawDataset, _p, host_lib
from super_gradients_b200 import kernels as K
from super_gradients_b200.common.registry import COLLATE_FUNCTIONS, TRANSFORMS
from super_gradients_b200.training.datasets.detection_augment_dataset import DetectionAugmentCollateFN, DetectionAugmentDataset, PackedDetectionBatch
from super_gradients_b200.training.transforms import transforms as T

GOLDEN = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "detection_augment.pt"), weights_only=False)


def make_dataset(name):
    return DetectionAugmentDataset(StubRawDataset(), [TRANSFORMS[n](**kw) for n, kw in GOLDEN_LISTS[name]])


def replay(name, seed):
    ds = make_dataset(name)
    random.seed(seed)
    np.random.seed(seed)
    return ds, [ds[i] for i in range(len(ds))]


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
    batch = DetectionAugmentCollateFN.for_dataset(ds)(items)
    u8 = host_u8(batch)
    for i, r in enumerate(ref):
        assert hashlib.sha256(u8[i].tobytes()).hexdigest() == r["u8_sha256"], (case, i)
    rows = torch.cat([torch.cat((torch.full((len(r["target"]), 1), float(i)), r["target"]), 1) for i, r in enumerate(ref)])
    assert torch.equal(batch.targets, rows)  # DetectionCollateFN's [N, 6]
    if case == ("recipe", 0):
        assert torch.equal(torch.from_numpy(u8[-1][::8, ::8].copy()), GOLDEN["full_u8"])


def test_registered_and_order_checked():
    assert "DetectionAugmentCollateFN" in COLLATE_FUNCTIONS
    assert all(n in TRANSFORMS for n, _ in GOLDEN_LISTS["recipe"])
    with pytest.raises(ValueError):
        DetectionAugmentDataset(StubRawDataset(), [T.DetectionHorizontalFlip(0.5), T.DetectionHSV(0.5), T.DetectionPaddedRescale(640), T.DetectionStandardize()])
    with pytest.raises(ValueError):
        DetectionAugmentDataset(StubRawDataset(), [T.DetectionHSV(0.5), T.DetectionStandardize()])


def test_close_switches_affine_and_mixup_off():
    ds = make_dataset("recipe")
    for t in ds.transforms:
        t.close()
    random.seed(0)
    np.random.seed(0)
    plans = [ds[i][0] for i in range(len(ds))]
    assert all(p.affine is None and p.mixup is None for p in plans)


def test_dataloader_workers_collate_without_cuda():
    ds = make_dataset("recipe")
    loader = torch.utils.data.DataLoader(ds, batch_size=4, num_workers=2, collate_fn=DetectionAugmentCollateFN.for_dataset(ds))
    batches = list(loader)
    assert len(batches) == 2 and all(isinstance(b, PackedDetectionBatch) and b.batch == 4 for b in batches)
