"""GPU checks of the detection train augmentation kernel (csrc/augment.cu): the bf16 NHWC batch equals, bit for bit, what
DetectionStandardize + DetectionCollateFN + functional.to_nhwc make from the cv2 / numpy chain; bad tables are refused."""
import numpy as np
import pytest
import torch

from augment_cases import cases, oracle_u8
from super_gradients_b200 import kernels as K
from super_gradients_b200 import lib as L
from super_gradients_b200.training.transforms import detection_augment as DA

pytestmark = pytest.mark.gpu


def _expected(plans):
    x = torch.stack([torch.from_numpy((oracle_u8(p) / 255.0).astype(np.float32)).permute(2, 0, 1) for p in plans])  # reference float32 CHW
    return x.bfloat16()


def test_batch_matches_reference_chain():
    plans = cases()
    out = DA.BatchAugmenter()(plans, "cuda")
    torch.cuda.synchronize()
    assert out.shape == (len(plans), 16, 640, 640) and out.dtype == torch.bfloat16
    got = out.float().cpu()
    assert bool((got[:, 3:] == 0).all())
    exp = _expected(plans).float()
    for b in range(len(plans)):
        assert torch.equal(got[b, :3], exp[b]), (b, int((got[b, :3] != exp[b]).sum()))


def test_staging_buffer_is_reused_across_batches():
    aug = DA.BatchAugmenter()
    plans = cases(seed=5)
    first = aug(plans[:4], "cuda").float().cpu()
    second = aug(plans[4:], "cuda").float().cpu()
    exp = _expected(plans).float()
    assert torch.equal(first[:, :3], exp[:4]) and torch.equal(second[:, :3], exp[4:])


def _run(table_host, src_bytes=None):
    src = torch.zeros(src_bytes if src_bytes is not None else 64 * 64 * 3, dtype=torch.uint8, device="cuda")
    out = K.empty_nhwc(table_host.shape[0], 16, 64, 64, "cuda")
    K.detection_augment(table_host, table_host.cuda(), src, out)


def _table():
    t = torch.zeros(1, K.AUG_FIELDS, dtype=torch.int64)
    t[0, DA.H] = t[0, DA.W] = t[0, DA.AFF_H] = t[0, DA.AFF_W] = t[0, DA.RS_H] = t[0, DA.RS_W] = 64
    return t


def test_refusals():
    _run(_table())
    torch.cuda.synchronize()
    t = _table()
    t[0, DA.OFFSET] = 8  # the image would end past the buffer
    with pytest.raises(L.SgbError):
        _run(t)
    t = _table()
    t[0, DA.AFFINE] = 1
    t[0, DA.M : DA.M + 6] = torch.tensor([1.0, 2.0, 0.0, 2.0, 4.0, 0.0], dtype=torch.float64).view(torch.int64)  # determinant 0
    with pytest.raises(L.SgbError):
        _run(t)
    t = _table()
    t[0, DA.MIX], t[0, DA.MIX_H], t[0, DA.MIX_W] = 1, 64, 64
    t[0, DA.MIX_OFFSET] = 64 * 64 * 3  # the partner lies outside the buffer
    with pytest.raises(L.SgbError):
        _run(t)
    with pytest.raises(L.SgbError):
        _run(_table(), src_bytes=100)
    with pytest.raises(ValueError):
        DA.BatchAugmenter()([DA.AugmentPlan(np.zeros((8, 8), np.uint8), (8, 8))], "cuda")


def test_reference_goldens_on_the_gpu():
    """The model input the loader makes on the GPU has the sha256 of the reference's standardized output rounded to bf16."""
    import hashlib

    from test_detection_augment_replay import GOLDEN, replay

    from super_gradients_b200.training.datasets.detection_augment_dataset import DetectionAugmentCollateFN

    for case, ref in sorted(GOLDEN["cases"].items()):
        ds, items = replay(*case)
        images, targets = DetectionAugmentCollateFN.for_dataset(ds)(items).pin_memory().to_model_input("cuda")
        x = images[:, :3].contiguous().view(torch.int16).cpu().numpy()
        for i, r in enumerate(ref):
            assert hashlib.sha256(x[i].tobytes()).hexdigest() == r["input_sha256"], (case, i)
        assert int(targets.shape[0]) == sum(len(r["target"]) for r in ref)


def _tiny_yolo_nas():
    import copy
    import os

    from super_gradients_b200.training.models.detection_models.yolo_nas import YoloNAS

    g = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tiny_yolo_nas.pt"), weights_only=False)
    ap = copy.deepcopy(g["arch"])
    m = YoloNAS(backbone=ap["backbone"], neck=ap["neck"], heads=ap["heads"], num_classes=4, bn_eps=1e-3, bn_momentum=0.03, inplace_act=True, in_channels=3)
    m.load_state_dict({k: v.clone() for k, v in g["sd0"].items()}, strict=False)
    return m.cuda().train()


@pytest.mark.parametrize("cuda_graph", [False, True])
def test_trainer_with_packed_loader_matches_reference_batches(tmp_path, cuda_graph):
    """Trainer.train() fed by DetectionAugmentCollateFN batches gives the loss of the same batches made on the CPU by the cv2 / numpy
    chain + DetectionCollateFN and converted by functional.to_nhwc: an fp32 NCHW input reaches the stem by another path than a bf16 NHWC one, with other
    rounding, so both runs get the bf16 tensor the reference batch becomes."""
    from test_detection_augment_replay import replay

    from super_gradients_b200.functional import to_nhwc
    from super_gradients_b200.training.datasets.detection_augment_dataset import DetectionAugmentCollateFN
    from super_gradients_b200.training.losses import PPYoloELoss
    from super_gradients_b200.training.sg_trainer import Trainer
    from super_gradients_b200.training.utils.collate_fn.detection_collate_fn import DetectionCollateFN

    ds, items = replay("recipe", 0)
    collate = DetectionAugmentCollateFN.for_dataset(ds)
    packed = [collate(items[:4]).pin_memory(), collate(items[4:])]
    ref = [DetectionCollateFN()([((oracle_u8(p) / 255.0).astype(np.float32), t) for p, t in items[s : s + 4]]) for s in (0, 4)]
    ref = [(to_nhwc(x.cuda()), t) for x, t in ref]  # the model input DetectionCollateFN's float batch becomes
    for b, (x, _) in zip(packed, ref):
        assert torch.equal(b.to_model_input("cuda")[0], x)
    losses = []
    for k, loader in enumerate((packed, ref)):
        torch.manual_seed(0)
        tp = dict(max_epochs=2, initial_lr=1e-3, lr_mode="constant", optimizer="SGD", loss=PPYoloELoss(num_classes=4, use_static_assigner=False), cuda_graph=cuda_graph,
                  save_model=False, run_validation_freq=100)  # fmt: skip
        tr = Trainer(f"aug{k}", ckpt_root_dir=str(tmp_path))
        tr.train(_tiny_yolo_nas(), tp, loader)
        losses.append(tr.history["train_loss"])
    assert all(np.isfinite(v) for v in losses[0])
    assert losses[0] == pytest.approx(losses[1], rel=1e-4, abs=1e-6)
