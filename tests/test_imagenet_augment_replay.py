"""CPU replay of tests/golden/imagenet_augment.pt (the unmodified reference ImageNet train chain and CollateMixup on the seeded stub
dataset): with the same seeds, ImageNetAugmentDataset draws the crop window, interpolation, flip and RandAugment ops the reference
drew and leaves the python / numpy / torch RNG states where the reference left them; the host build of the kernel's arithmetic
reproduces every uint8 image, and its float32 ToTensor / Normalize / mix, rounded to bf16, every model input image and the targets."""
import hashlib
import os
import pickle
import random

import numpy as np
import pytest
import torch

from imagenet_augment_cases import CONFIG, GOLDEN_BATCH, GOLDEN_MIX, IMG_MEAN, IMG_STD, SIZE, FILL, StubImageDataset, _p, host_lib
from super_gradients_b200 import kernels as K
from super_gradients_b200.common.registry import COLLATE_FUNCTIONS
from super_gradients_b200.training.datasets.imagenet_augment_dataset import ImageNetAugmentCollateFN, ImageNetAugmentDataset, PackedImageNetBatch
from super_gradients_b200.training.transforms import imagenet_augment as IA

GOLDEN = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "imagenet_augment.pt"), weights_only=False)


def sha(b: bytes) -> str:
    return hashlib.sha256(b).hexdigest()


def replay(case, batch=GOLDEN_BATCH):
    name, seed = case
    random.seed(seed)
    np.random.seed(seed)
    torch.manual_seed(seed)
    stub = StubImageDataset(length=batch)
    ds = ImageNetAugmentDataset(stub, size=SIZE, interpolation="random", config_str=CONFIG, img_mean=IMG_MEAN, img_std=IMG_STD)
    plans = [ds[i] for i in range(len(ds))]
    return stub, plans, ImageNetAugmentCollateFN.for_dataset(ds, **GOLDEN_MIX[name])(plans)


def expected_op(name, args):
    """(code, arguments) the kernel needs for the op the reference applied with `args`."""
    if name == "Rotate":
        return (IA.OP_NONE, [0] * 6) if args[0] % 360.0 == 0 else IA._affine(*IA.rotate_matrix(args[0], SIZE, SIZE))
    if name in ("ShearX", "ShearY", "TranslateXRel", "TranslateYRel"):
        v = args[0] * SIZE if name.startswith("Translate") else args[0]
        m = {"ShearX": (1, v, 0, 0, 1, 0), "ShearY": (1, 0, 0, v, 1, 0), "TranslateXRel": (1, 0, v, 0, 1, 0), "TranslateYRel": (1, 0, 0, 0, 1, v)}[name]
        return IA._affine(*m)
    if name in IA._ENHANCE:
        return IA._ENHANCE[name], IA._f64_bits(args[0]) + [0] * 5
    if name in IA._PLAIN:
        return IA._PLAIN[name], [0] * 6
    code = {"Posterize": IA.OP_POSTERIZE, "Solarize": IA.OP_SOLARIZE, "SolarizeAdd": IA.OP_SOLARIZE_ADD}[name]
    return code, [int(args[0])] + [0] * 5


def host_u8(batch: PackedImageNetBatch) -> np.ndarray:
    raw = batch.buffer.numpy()
    head = batch.batch * K.IN_FIELDS * 8
    table, src = raw[:head].view(np.int64).copy(), np.ascontiguousarray(raw[head:])
    out = np.empty((batch.batch, SIZE, SIZE, 3), np.uint8)
    host_lib().augment_host(_p(table), _p(src), batch.batch, SIZE, _p(np.array(FILL, np.int32)), _p(out))
    return out


def host_model_input(batch: PackedImageNetBatch, u8: np.ndarray) -> torch.Tensor:
    """ToTensor, Normalize and the batch-mode mix in float32 numpy (NCHW), as the kernel computes them."""
    x = ((u8.transpose(0, 3, 1, 2).astype(np.float32) / np.float32(255) - np.array(IMG_MEAN, np.float32)[:, None, None]) / np.array(IMG_STD, np.float32)[:, None, None])
    xj = x[::-1]
    if batch.mix_mode == 1:
        x = x * np.float32(batch.lam) + xj * np.float32(1.0 - batch.lam)
    elif batch.mix_mode == 2:
        yl, yh, xl, xh = batch.box
        x = x.copy()
        x[:, :, yl:yh, xl:xh] = xj[:, :, yl:yh, xl:xh]
    return torch.from_numpy(np.float32(0) + x)


@pytest.mark.parametrize("case", sorted(GOLDEN["cases"]), ids=lambda c: f"{c[0]}-{c[1]}")
def test_replay_matches_reference(case):
    ref = GOLDEN["cases"][case]
    stub, plans, batch = replay(case)
    assert [p.label for p in plans] == ref["labels"]
    for i, (p, r) in enumerate(zip(plans, ref["samples"])):
        top, left, h, w = r["crop"]
        assert np.array_equal(p.window, stub[i][0][top : top + h, left : left + w]), (case, i)
        assert p.filter == {"bilinear": IA.BILINEAR, "bicubic": IA.BICUBIC}[r["interpolation"]] and p.flip == r["flip"], (case, i)
        want = [expected_op(n, a) for n, a in r["ops"]]
        assert [o for o in p.ops if o[0] != IA.OP_NONE] == [o for o in want if o[0] != IA.OP_NONE], (case, i)
    states = {"python": sha(pickle.dumps(random.getstate())), "numpy": sha(pickle.dumps(np.random.get_state())), "torch": sha(torch.get_rng_state().numpy().tobytes())}
    assert states == ref["rng"]
    u8 = host_u8(batch)
    for i, r in enumerate(ref["samples"]):
        assert sha(u8[i].tobytes()) == r["u8_sha256"], (case, i)
    x = host_model_input(batch, u8)
    bf = x.bfloat16().view(torch.int16).numpy()
    for i in range(len(bf)):
        assert sha(bf[i].tobytes()) == ref["input_sha256"][i], (case, i)
    assert torch.equal(x[0, :, ::16, ::16], ref["first_input"])
    assert sha(batch.targets("cpu").numpy().tobytes()) == ref["target_sha256"]


def test_every_mix_mode_is_covered():
    modes = {replay(c, batch=8)[2].mix_mode for c in (("nomix", 0), ("mixup", 0), ("cutmix", 0))}
    assert modes == {0, 1, 2}


def test_refusals():
    assert "ImageNetAugmentCollateFN" in COLLATE_FUNCTIONS
    for bad in ("rand-m9-inc1", "rand-m9-w0", "rand-m9-n3", "rand-m9-x1", "auto-m9"):
        with pytest.raises(ValueError):
            IA.RandAugmentConfig.parse(bad)
    assert IA.RandAugmentConfig.parse("rand-m9-n2-mstd1.5") == IA.RandAugmentConfig(9, 2, 1.5)
    with pytest.raises(ValueError):
        ImageNetAugmentCollateFN(mode="elem")
    with pytest.raises(ValueError):
        ImageNetAugmentCollateFN(cutmix_minmax=[0.2, 0.8])
    with pytest.raises(ValueError):
        ImageNetAugmentDataset(StubImageDataset(), interpolation="bicubic")
    ds = ImageNetAugmentDataset(StubImageDataset())
    with pytest.raises(ValueError):
        ImageNetAugmentCollateFN.for_dataset(ds)([ds[0]] * 3)  # odd batch
    with pytest.raises(ValueError):
        ImageNetAugmentDataset([(np.zeros((8, 8), np.uint8), 0)])[0]


def test_dataloader_workers_collate_without_cuda():
    ds = ImageNetAugmentDataset(StubImageDataset(length=16))
    loader = torch.utils.data.DataLoader(ds, batch_size=8, num_workers=2, collate_fn=ImageNetAugmentCollateFN.for_dataset(ds, mixup_alpha=0.2, cutmix_alpha=1.0))
    batches = list(loader)
    assert len(batches) == 2 and all(isinstance(b, PackedImageNetBatch) and b.batch == 8 for b in batches)
