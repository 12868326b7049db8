"""CPU checks of the GPU validation chains against tests/golden/validation_chains.pt (the unmodified reference's YOLO-NAS COCO,
YOLO-NAS-POSE and ResNet-50 validation transforms and collates): the targets, crowd targets, gt_samples and labels of the packed
collates; the model input of the kernels' arithmetic (the g++ builds of augment_math.cuh, pose_augment_math.cuh and
resample_math.cuh over the packed buffers), bf16 for bf16; the refusals; and Trainer._evaluate handing the metrics the same fields
for a packed batch as for the reference's tuple batch."""
import hashlib

import numpy as np
import pytest
import torch

import host_classification
import validation_cases as VC
from augment_cases import host_lib as detection_host_lib
from pose_augment_cases import host_lib as pose_host_lib
from super_gradients_b200 import kernels as K


def _p(a):
    import ctypes

    return ctypes.c_void_p(a.ctypes.data)


def _sha_u8(u8_nhwc: np.ndarray):
    """sha256 per image of StandardizeImage(255) of a uint8 NHWC canvas, float32 CHW rounded to bf16 (the kernels' standardize:
    the uint8 value over the float64 255, cast to float32)."""
    f = (u8_nhwc / 255.0).astype(np.float32).transpose(0, 3, 1, 2)
    return [hashlib.sha256(torch.from_numpy(np.ascontiguousarray(x)).bfloat16().view(torch.int16).numpy().tobytes()).hexdigest() for x in f]


def _split(buffer: torch.Tensor, batch: int, fields: int):
    raw = buffer.numpy()
    head = batch * fields * 8
    return raw[:head].view(np.int64).reshape(batch, fields).copy(), np.ascontiguousarray(raw[head:])


@pytest.fixture(scope="module")
def golden():
    return VC.golden()


def test_detection_targets_and_crowd_targets(golden):
    ds = VC.detection_dataset()
    batch = VC.collates()[0]([ds[i] for i in range(len(ds))])
    g = golden["detection"]
    assert torch.equal(batch.targets, g["targets"]) and batch.targets.dtype == g["targets"].dtype
    assert torch.equal(batch.extras["crowd_targets"], g["crowd_targets"])
    for i, row in enumerate(g["rows"]):
        _, t, c = ds[i]
        assert np.array_equal(t, row["target"].numpy()) and np.array_equal(c, row["crowd_target"].numpy())


def test_detection_host_pixels(golden):
    ds = VC.detection_dataset()
    batch = VC.collates()[0]([ds[i] for i in range(len(ds))])
    table, src = _split(batch.buffer, batch.batch, K.AUG_FIELDS)
    out = np.empty((batch.batch, 640, 640, 3), np.uint8)
    detection_host_lib().augment_host(_p(table), _p(src), batch.batch, 640, 640, 114, K.HSV_SIMD_BLOCK, _p(out))
    assert _sha_u8(out) == [r["input_sha256"] for r in golden["detection"]["rows"]]


def test_pose_targets_and_gt_samples(golden):
    ds = VC.pose_dataset()
    batch = VC.collates()[1]([ds[i] for i in range(len(ds))])
    g = golden["pose"]
    for got, want in zip(batch.targets, g["targets"]):
        assert torch.equal(got, want) and got.dtype == want.dtype
    assert len(batch.extras["gt_samples"]) == len(g["gt_samples"])
    for s, want in zip(batch.extras["gt_samples"], g["gt_samples"]):
        for k, v in want.items():
            got = getattr(s, k)
            assert (got is None) == (v is None) and (v is None or (np.array_equal(got, v) and got.dtype == v.dtype)), k
        assert s.image is None and s.mask is None


def test_pose_host_pixels(golden):
    ds = VC.pose_dataset()
    batch = VC.collates()[1]([ds[i] for i in range(len(ds))])
    table, src = _split(batch.buffer, batch.batch, K.POSE_FIELDS)
    ws = np.zeros(max(src.size, 1), np.uint8)
    out = np.empty((batch.batch, 640, 640, 3), np.uint8)
    pose_host_lib().pose_augment_host(_p(table), _p(src), _p(ws), batch.batch, 640, K.HSV_SIMD_BLOCK, _p(out))
    assert _sha_u8(out) == [r["input_sha256"] for r in golden["pose"]["rows"]]


@pytest.mark.parametrize("pil", [True, False])
def test_imagenet_labels_and_host_pixels(golden, pil):
    ds = VC.imagenet_dataset(pil=pil)
    batch = VC.collates()[2]([ds[i] for i in range(len(ds))])
    assert torch.equal(batch.labels, golden["imagenet"]["labels"]) and batch.labels.dtype == golden["imagenet"]["labels"].dtype
    table, src = _split(batch.buffer, batch.batch, K.RS_FIELDS)
    out = torch.empty((batch.batch, 16, VC.CROP, VC.CROP), dtype=torch.bfloat16)
    host_classification.resample_crop_u8(torch.from_numpy(table), None, torch.from_numpy(src), out, max_value=255.0, mean=batch.mean, std=batch.std)
    got = [hashlib.sha256(x[:3].contiguous().view(torch.int16).numpy().tobytes()).hexdigest() for x in out]
    assert got == [r["input_sha256"] for r in golden["imagenet"]["rows"]]


def test_standardize_rounds_like_totensor():
    """The resize-and-crop kernel's (float)((double)u / 255.0) equals ToTensor's float32 u / 255 for every uint8 value, so Normalize
    after it sees the same operand in both chains."""
    u = np.arange(256)
    assert np.array_equal((u / 255.0).astype(np.float32), u.astype(np.float32) / np.float32(255.0))


def test_validation_geometry_is_torchvision():
    from torchvision.transforms import functional as F

    from super_gradients_b200.training.datasets.imagenet_augment_dataset import validation_geometry

    for h, w in VC.StubImageNetDataset.SIZES + [(1, 1000), (1000, 3), (237, 236)]:
        rh, rw = F._compute_resized_output_size((h, w), [VC.RESIZE])
        assert validation_geometry(h, w, VC.RESIZE, VC.CROP) == ((rh, rw), (int(round((rh - VC.CROP) / 2.0)), int(round((rw - VC.CROP) / 2.0))))


def test_refusals():
    from super_gradients_b200.training.datasets.imagenet_augment_dataset import ImageNetValidationDataset
    from super_gradients_b200.training.transforms import transforms as T

    ds = VC.detection_dataset(VC.StubDetectionDataset(sizes=[(400, 641)]))
    with pytest.raises(ValueError, match="fixed 640x640"):
        ds[0]
    with pytest.raises(ValueError, match="combines only"):
        T.check_order([T.DetectionRandomAffine(), T.DetectionPadToSize(640, 114), T.DetectionStandardize()])
    with pytest.raises(ValueError, match="combines only"):
        T.check_order([T.DetectionPaddedRescale(640), T.DetectionPadToSize(640, 114), T.DetectionStandardize()])
    with pytest.raises(ValueError):
        T.DetectionPadToSize(640, (114, 0, 114))
    with pytest.raises(ValueError):
        T.DetectionImagePermute((1, 2, 0))
    with pytest.raises(ValueError):
        ImageNetValidationDataset(VC.StubImageNetDataset(), resize=200, size=224)
    with pytest.raises(ValueError, match="with_crowd"):
        VC.collates()[0]([d[:2] for d in (VC.detection_dataset()[0],)])


def test_collates_are_registered():
    from super_gradients_b200.common.registry import COLLATE_FUNCTIONS

    VC.collates()
    for name in ("CrowdDetectionAugmentCollateFN", "YoloNASPoseAugmentCollateFN", "ImageNetValidationCollateFN"):
        assert COLLATE_FUNCTIONS[name].__name__ == name


class _Recorder:
    """A metric that records what update() receives."""

    def __init__(self):
        self.seen = []

    def reset(self):
        self.seen = []

    def update(self, preds, target, crowd_targets=None, gt_samples=None):
        self.seen.append({"target": target, "crowd_targets": crowd_targets, "gt_samples": gt_samples})

    def compute(self):
        return {"n": float(len(self.seen))}


class _Packed:
    """A packed batch as the collates make it, its input made on the host."""

    def __init__(self, images, targets, extras):
        self.images, self.targets, self.extras = images, targets, extras

    def to_model_input(self, device, out=None):
        return self.images, self.targets


def test_evaluate_passes_the_same_fields_for_packed_and_tuple_batches():
    from super_gradients_b200.training.sg_trainer import Trainer

    torch.manual_seed(0)
    images = torch.randn(2, 3, 4, 4)
    det_targets, crowd = torch.randn(3, 6), torch.randn(1, 6)
    gt = [object(), object()]
    trainer = Trainer.__new__(Trainer)
    trainer.net, trainer.criterion, trainer.device = torch.nn.Flatten(), None, torch.device("cpu")
    for targets, extras in ((det_targets, {"crowd_targets": crowd}), ((det_targets, det_targets), {"gt_samples": gt})):
        seen = []
        for loader in ([(images, targets, extras)], [_Packed(images, targets, extras)]):
            m = _Recorder()
            trainer._evaluate(loader, [m])
            seen.append(m.seen)
        (tup,), (packed,) = seen
        assert set(tup) == set(packed)
        for k in tup:
            a, b = tup[k], packed[k]
            if torch.is_tensor(a):
                assert torch.equal(a, b)
            elif isinstance(a, tuple):
                assert all(torch.equal(x, y) for x, y in zip(a, b))
            else:
                assert a is b
