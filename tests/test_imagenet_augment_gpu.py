"""GPU checks of the ImageNet train augmentation kernel (csrc/imagenet_augment.cu): at B = 256 the bf16 NHWC batch is, image by
image and bit for bit, the reference chain's float32 CollateMixup output rounded to bf16, and the soft targets are the reference's,
for mixup, cutmix and unmixed batches; bad tables are refused; a Trainer.train() of resnet50 fed by the packed loader runs."""
import hashlib

import numpy as np
import pytest
import torch

from imagenet_augment_cases import FILL, IMG_MEAN, IMG_STD, StubImageDataset
from super_gradients_b200 import kernels as K
from super_gradients_b200 import lib as L
from super_gradients_b200.training.datasets.imagenet_augment_dataset import ImageNetAugmentCollateFN, ImageNetAugmentDataset
from super_gradients_b200.training.transforms import imagenet_augment as IA
from test_imagenet_augment_replay import GOLDEN, replay

pytestmark = pytest.mark.gpu


def sha(b: bytes) -> str:
    return hashlib.sha256(b).hexdigest()


@pytest.mark.parametrize("case", sorted(GOLDEN["cases"]), ids=lambda c: f"{c[0]}-{c[1]}")
def test_batch_matches_reference_goldens(case):
    ref = GOLDEN["cases"][case]
    _, _, batch = replay(case)
    images, targets = batch.pin_memory().to_model_input("cuda")
    torch.cuda.synchronize()
    assert images.shape == (256, 16, 224, 224) and images.dtype == torch.bfloat16
    assert bool((images[:, 3:] == 0).all())
    x = images[:, :3].contiguous().view(torch.int16).cpu().numpy()
    bad = [i for i in range(len(x)) if sha(x[i].tobytes()) != ref["input_sha256"][i]]
    assert not bad, (case, batch.mix_mode, bad[:8])
    assert targets.shape == (256, 1000) and sha(targets.cpu().numpy().tobytes()) == ref["target_sha256"]


def _run(table_host, src_bytes=64 * 64 * 3, ws_bytes=64 * 224 * 3, batch_box=(0, 0, 0, 0), mix=0):
    src = torch.zeros(src_bytes, dtype=torch.uint8, device="cuda")
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
    out = K.empty_nhwc(table_host.shape[0], 16, 224, 224, "cuda")
    K.imagenet_augment(table_host, table_host.cuda(), src, ws, out, FILL, IMG_MEAN, IMG_STD, mix_mode=mix, lam=0.5, box=batch_box)


def _table(n=2):
    t = torch.zeros(n, K.IN_FIELDS, dtype=torch.int64)
    t[:, IA.H] = t[:, IA.W] = 32
    t[1, IA.OFFSET] = 32 * 32 * 3
    t[1, IA.WS_OFFSET] = 32 * 224 * 3
    return t


def test_refusals():
    _run(_table())
    torch.cuda.synchronize()
    cases = []
    t = _table(); t[1, IA.OFFSET] = 64 * 64 * 3 - 8; cases.append(t)  # noqa: E702  the window would end past the buffer
    t = _table(); t[1, IA.WS_OFFSET] = 64 * 224 * 3 - 8; cases.append(t)  # noqa: E702  its resize rows would end past the workspace
    t = _table(); t[0, IA.OP] = 12; cases.append(t)  # noqa: E702  unknown op
    t = _table(); t[0, IA.OP], t[0, IA.OP + 1] = IA.OP_POSTERIZE, 8; cases.append(t)  # noqa: E702
    t = _table(); t[0, IA.OP + IA.OP_FIELDS] = IA.OP_AFFINE; t[0, IA.OP + IA.OP_FIELDS + 1] = torch.tensor([float("nan")], dtype=torch.float64).view(torch.int64)[0]; cases.append(t)  # noqa: E702,E501
    t = _table(); t[0, IA.FILTER] = 2; cases.append(t)  # noqa: E702
    t = _table(); t[0, IA.H] = 0; cases.append(t)  # noqa: E702
    for t in cases:
        with pytest.raises(L.SgbError):
            _run(t)
    with pytest.raises(L.SgbError):
        _run(_table(3)[:3].contiguous())  # odd batch
    with pytest.raises(L.SgbError):
        _run(_table(), batch_box=(0, 225, 0, 10), mix=2)
    with pytest.raises(L.SgbError):
        _run(_table(), mix=3)


def test_trainer_trains_resnet50_from_the_packed_loader(tmp_path):
    from super_gradients_b200.training import models
    from super_gradients_b200.training.losses import CrossEntropyLoss
    from super_gradients_b200.training.sg_trainer import Trainer

    ds = ImageNetAugmentDataset(StubImageDataset(length=16))
    collate = ImageNetAugmentCollateFN.for_dataset(ds, mixup_alpha=0.2, cutmix_alpha=1.0, label_smoothing=0.1)
    torch.manual_seed(0)
    loader = torch.utils.data.DataLoader(ds, batch_size=8, num_workers=0, collate_fn=collate, pin_memory=True)
    tp = dict(max_epochs=2, initial_lr=1e-3, lr_mode="constant", optimizer="SGD", loss=CrossEntropyLoss(), save_model=False, run_validation_freq=100)
    tr = Trainer("imagenet_aug", ckpt_root_dir=str(tmp_path))
    tr.train(models.get("resnet50", num_classes=1000).cuda().train(), tp, loader)
    assert len(tr.history["train_loss"]) == 2 and all(np.isfinite(v) for v in tr.history["train_loss"])
