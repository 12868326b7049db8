"""GPU checks of the pose train augmentation kernels (csrc/pose_augment.cu): the packed loader's model input has the sha256 of the
reference's standardized image rounded to bf16 for every golden sample; bad tables are refused; Trainer.train() fed by
PoseAugmentCollateFN gives the loss of the same batches made on the CPU by the cv2 chain + YoloNASPoseCollateFN + to_nhwc."""
import copy
import hashlib
import os
import random
import types

import numpy as np
import pytest
import torch

from pose_augment_cases import BASE, StubPoseDataset, build, golden, oracle_u8, replay
from super_gradients_b200 import kernels as K
from super_gradients_b200 import lib as L
from super_gradients_b200.training.datasets.pose_estimation_datasets.pose_augment_dataset import PoseAugmentCollateFN, PoseAugmentDataset
from super_gradients_b200.training.transforms import keypoints as KP
from super_gradients_b200.training.transforms import keypoints_augment as PA

pytestmark = pytest.mark.gpu


def test_reference_goldens_on_the_gpu():
    for case, ref in sorted(golden()["cases"].items()):
        ds, items = replay(*case)
        images, (boxes, joints, crowd) = PoseAugmentCollateFN.for_dataset(ds)(items).pin_memory().to_model_input("cuda")
        assert images.shape == (len(items), 16, 640, 640) and images.dtype == torch.bfloat16
        assert bool((images[:, 3:] == 0).all())
        x = images[:, :3].contiguous().view(torch.int16).cpu().numpy()
        for i, r in enumerate(ref):
            assert hashlib.sha256(x[i].tobytes()).hexdigest() == r["input_sha256"], (case, i)
        assert int(boxes.shape[0]) == int(joints.shape[0]) == int(crowd.shape[0]) == sum(len(r["boxes"]) for r in ref)


def _table(n=64):
    t = torch.zeros(1, K.POSE_FIELDS, dtype=torch.int64)
    t[0, PA.NSUB], t[0, PA.CANVAS_H], t[0, PA.CANVAS_W], t[0, PA.RS_H], t[0, PA.RS_W] = 1, n, n, n, n
    s = PA.SUB
    t[0, s + PA.S_H] = t[0, s + PA.S_W] = t[0, s + PA.S_RH] = t[0, s + PA.S_RW] = n
    return t


def _run(t, src_bytes=64 * 64 * 3, ws_bytes=64 * 64 * 3):
    src = torch.zeros(src_bytes, dtype=torch.uint8, device="cuda")
    ws = torch.zeros(ws_bytes, dtype=torch.uint8, device="cuda")
    out = K.empty_nhwc(t.shape[0], 16, 64, 64, "cuda")
    K.pose_augment(t, t.cuda(), src, ws, out)
    return out


def test_refusals():
    out = _run(_table())
    torch.cuda.synchronize()
    assert bool((out.float() == 0).all())
    bad = []
    t = _table()
    t[0, PA.SUB + PA.S_OFFSET] = 8  # the image would end past the buffer
    bad.append(t)
    t = _table()
    t[0, PA.SUB + PA.S_WS_OFFSET] = 3  # the rotated tile would end past the workspace
    bad.append(t)
    t = _table()
    t[0, PA.SUB + PA.S_AFFINE] = 1
    t[0, PA.SUB + PA.S_M : PA.SUB + PA.S_M + 6] = torch.tensor([1.0, 2.0, 0.0, 2.0, 4.0, 0.0], dtype=torch.float64).view(torch.int64)  # determinant 0
    bad.append(t)
    t = _table()
    t[0, PA.SUB + PA.S_AFFINE] = 1  # an identity matrix, but interpolation flag 5
    t[0, PA.SUB + PA.S_M : PA.SUB + PA.S_M + 6] = torch.tensor([1.0, 0.0, 0.0, 0.0, 1.0, 0.0], dtype=torch.float64).view(torch.int64)
    t[0, PA.SUB + PA.S_MODE] = 5
    bad.append(t)
    t = _table()
    t[0, PA.SUB + PA.S_ROT] = 4  # no rot90 count
    bad.append(t)
    t = _table()
    t[0, PA.NSUB] = 2
    bad.append(t)
    t = _table()
    t[0, PA.SUB + PA.S_BC], t[0, PA.SUB + PA.S_MEAN] = 1, 0x7FC00000  # NaN mean
    bad.append(t)
    t = _table()
    t[0, PA.PAD_TOP] = 1  # the canvas would leave the output
    bad.append(t)
    for t in bad:
        with pytest.raises(L.SgbError):
            _run(t)


def _tiny_pose(g0):
    from super_gradients_b200.training.models.pose_estimation_models import YoloNASPose

    ap = copy.deepcopy(g0["arch"])
    m = YoloNASPose(backbone=ap["backbone"], neck=ap["neck"], heads=ap["heads"], num_classes=5, bn_eps=1e-3, bn_momentum=0.03, inplace_act=True, in_channels=3)
    m.load_state_dict({k: v.clone() for k, v in g0["sd0"].items()}, strict=False)
    return m.cuda().train()


class _EpochLoader:
    def __init__(self, make):
        self.make, self.n = make, len(make())

    def __iter__(self):
        return iter(self.make())

    def __len__(self):
        return self.n


@pytest.mark.parametrize("cuda_graph", [False, True])
def test_trainer_with_packed_loader_matches_reference_batches(tmp_path, cuda_graph):
    from super_gradients_b200.functional import to_nhwc
    from super_gradients_b200.training.datasets.pose_estimation_datasets import YoloNASPoseCollateFN
    from super_gradients_b200.training.losses import YoloNASPoseLoss
    from super_gradients_b200.training.sg_trainer import Trainer

    here = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    g0 = torch.load(os.path.join(here, "tiny_yolo_nas_pose.pt"), weights_only=False)
    g = torch.load(os.path.join(here, "tiny_yolo_nas_pose_train.pt"), weights_only=False)
    spec = [(n, dict(kw, flip_index=[0, 2, 1, 4, 3]) if n == "KeypointsRandomHorizontalFlip" else kw) for n, kw in BASE]
    ds = PoseAugmentDataset(StubPoseDataset(num_joints=5), build(spec, KP))
    random.seed(0)
    np.random.seed(0)
    samples = [ds._apply(ds._load(i).sanitize_sample(), ds.transforms) for i in range(len(ds))]  # the host samples the items come from
    random.seed(0)
    np.random.seed(0)
    items = [ds[i] for i in range(len(ds))]
    collate = PoseAugmentCollateFN.for_dataset(ds)
    packed = [collate(items[:4]).pin_memory(), collate(items[4:])]
    ref = []
    for s0 in (0, 4):
        objs = [types.SimpleNamespace(image=(oracle_u8(s.plan) / 255.0).astype(np.float32), mask=np.ones((640, 640), np.float32), bboxes_xywh=s.bboxes_xywh,
                                      joints=s.joints, is_crowd=s.is_crowd, additional_samples=None) for s in samples[s0 : s0 + 4]]  # fmt: skip
        x, targets, _ = YoloNASPoseCollateFN()(objs)
        ref.append((to_nhwc(x.cuda()), targets))
    for b, (x, t) in zip(packed, ref):
        images, targets = b.to_model_input("cuda")
        assert torch.equal(images, x)
        assert all(torch.equal(a, c) for a, c in zip(targets, t))
    # each epoch gets freshly made batches on both sides, as a DataLoader gives them: a step may update its inputs in place
    fresh_packed = _EpochLoader(lambda: [collate(items[:4]).pin_memory(), collate(items[4:])])
    fresh_ref = _EpochLoader(lambda: [(x.clone(), tuple(t.clone() for t in tg)) for x, tg in ref])
    # one epoch (two steps, the second after an update): from the second epoch on, two runs of the tiny pose model on identical
    # batches can already differ by a discrete assignment flip
    losses = []
    for k, loader in enumerate((fresh_packed, fresh_ref)):
        torch.manual_seed(0)
        tp = dict(max_epochs=1, initial_lr=1e-3, lr_mode="constant", optimizer="SGD", loss=YoloNASPoseLoss(oks_sigmas=g["sigmas"], **g["kw"]), cuda_graph=cuda_graph,
                  save_model=False, run_validation_freq=100)  # fmt: skip
        tr = Trainer(f"pose_aug{k}", ckpt_root_dir=str(tmp_path))
        tr.train(_tiny_pose(g0), tp, loader)
        losses.append(tr.history["train_loss"])
    assert all(np.isfinite(v) for v in losses[0])
    assert losses[0] == pytest.approx(losses[1], rel=1e-4, abs=1e-6)
