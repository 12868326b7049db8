"""GPU checks of DetectionMosaic in the detection train augmentation kernel (csrc/augment.cu): the model input of every case of
tests/golden/detection_mosaic.pt has the reference's bf16 sha256; malformed mosaic tables are refused before any launch; a
Trainer fed by packed Roboflow-list batches gives the loss of the same batches made on the CPU by the cv2 chain."""
import hashlib

import numpy as np
import pytest
import torch

from mosaic_cases import oracle_mosaic_u8
from super_gradients_b200 import kernels as K
from super_gradients_b200 import lib as L
from super_gradients_b200.training.datasets.detection_augment_dataset import DetectionAugmentCollateFN
from super_gradients_b200.training.transforms import detection_augment as DA
from test_detection_mosaic_host import GOLDEN, replay

pytestmark = pytest.mark.gpu


def test_reference_goldens_on_the_gpu():
    for case, ref in sorted(GOLDEN["cases"].items()):
        ds, items = replay(*case)
        images, targets = DetectionAugmentCollateFN.for_dataset(ds)(items).pin_memory().to_model_input("cuda")
        x = images[:, :3].contiguous().view(torch.int16).cpu().numpy()
        for i, r in enumerate(ref):
            assert hashlib.sha256(x[i].tobytes()).hexdigest() == r["input_sha256"], (case, i)
        assert bool((images[:, 3:] == 0).all()) and int(targets.shape[0]) == sum(len(r["target"]) for r in ref)


def test_mosaic_and_affine_border_values_stay_apart():
    """The mosaic border fills the canvas outside the tiles, the affine border the output outside the canvas: a zoomed-out
    affine on a centre that leaves most of the canvas empty shows both, each with its own value."""
    from test_detection_mosaic_host import mosaic_sample

    from super_gradients_b200.training.transforms import transforms as T

    s = mosaic_sample((6, 6, 6, 6), 640, (1279.0, 1279.0))  # only tile 0 is visible; the rest of the canvas is border
    s.plan.mosaic.border_value = 7
    m = np.array([[0.4, 0.0, 64.0], [0.0, 0.4, 64.0]])  # the 1280 canvas shrinks to 512 at (64, 64) of the 640 output
    s.plan.affine = (m, (640, 640), 200)
    s.plan.rescaled = (640, 640)
    out = DA.BatchAugmenter()([s.plan], "cuda")
    exp = oracle_mosaic_u8(s.plan)
    assert torch.equal(out[0, :3].cpu(), torch.from_numpy((exp / 255.0).astype(np.float32)).permute(2, 0, 1).bfloat16())
    assert (exp[:60, :60] == 200).all() and (exp[80:240, 80:240] == 7).all()
    assert T.DetectionMosaic(640).border_value == 114


def _run(table_host, src_bytes=3 * 64 * 64 * 3):
    src = torch.zeros(src_bytes, dtype=torch.uint8, device="cuda")
    out = K.empty_nhwc(table_host.shape[0], 16, 64, 64, "cuda")
    K.detection_augment(table_host, table_host.cuda(), src, out)


def _table():
    """A valid 32 x 32 mosaic of four 16 x 16 images (the last shared) scaled x2 around the centre (16, 16), no affine."""
    t = torch.zeros(1, K.AUG_FIELDS, dtype=torch.int64)
    t[0, DA.H] = t[0, DA.W] = 16
    t[0, DA.AFF_H] = t[0, DA.AFF_W] = t[0, DA.RS_H] = t[0, DA.RS_W] = 32
    t[0, DA.MOS], t[0, DA.MOS_CANVAS_H], t[0, DA.MOS_CANVAS_W], t[0, DA.MOS_XC], t[0, DA.MOS_YC], t[0, DA.MOS_BORDER] = 1, 32, 32, 16, 16, 114
    for i in range(4):
        k = DA.MOS_TILE + i * DA.MOS_TILE_FIELDS
        x1, y1 = 16 * (i & 1), 16 * (i >> 1)
        t[0, k + DA.T_OFFSET] = min(i, 2) * 16 * 16 * 3
        t[0, k + DA.T_H] = t[0, k + DA.T_W] = 16
        t[0, k + DA.T_RH] = t[0, k + DA.T_RW] = 32
        t[0, k + DA.T_X1], t[0, k + DA.T_Y1], t[0, k + DA.T_X2], t[0, k + DA.T_Y2] = x1, y1, x1 + 16, y1 + 16
        t[0, k + DA.T_SX], t[0, k + DA.T_SY] = 16 - x1, 16 - y1
    return t


TILE1 = DA.MOS_TILE + DA.MOS_TILE_FIELDS


@pytest.mark.parametrize(
    "field, value",
    [
        (DA.MOS, 2),  # flag
        (TILE1 + DA.T_OFFSET, 3 * 64 * 64 * 3 - 100),  # tile outside src
        (TILE1 + DA.T_H, 0),
        (TILE1 + DA.T_RH, 0),  # resized size
        (TILE1 + DA.T_RW, 32768),
        (TILE1 + DA.T_SY, -1),  # a negative origin
        (DA.MOS_XC, 33),  # centre outside the canvas
        (DA.MOS_YC, -1),
        (DA.MOS_BORDER, 256),
        (DA.MOS_BORDER, -1),
        (DA.AFF_H, 16),  # without the affine the chain keeps the canvas size
    ],
)
def test_refusals(field, value):
    """Validation runs on the host table before the launch: a refused table launches nothing."""
    _run(_table())
    torch.cuda.synchronize()
    t = _table()
    t[0, field] = value
    with pytest.raises(L.SgbError):
        _run(t)


def _tile_cases():
    """Per tile of _table(), edits that break exactly one bound of its rectangle, each keeping the read inside the 32 x 32 resized
    tile (the origin moves with the edge), plus reads past the resized tile and an origin that overflows int64 arithmetic."""
    cases = []
    for i in range(4):
        right, bottom = i & 1, i >> 1
        if right:
            cases += [(i, "x1 left of the centre", {DA.T_X1: 15, DA.T_SX: 0}), (i, "x2 past the canvas", {DA.T_X2: 33})]
        else:
            cases += [(i, "x2 right of the centre", {DA.T_X2: 17, DA.T_SX: 15}), (i, "x1 before the canvas", {DA.T_X1: -1, DA.T_SX: 15})]
        if bottom:
            cases += [(i, "y1 above the centre", {DA.T_Y1: 15, DA.T_SY: 0}), (i, "y2 past the canvas", {DA.T_Y2: 33})]
        else:
            cases += [(i, "y2 below the centre", {DA.T_Y2: 17, DA.T_SY: 15}), (i, "y1 before the canvas", {DA.T_Y1: -1, DA.T_SY: 15})]
        cases += [(i, "x2 before x1", {DA.T_X1: 16 * right + 10, DA.T_X2: 16 * right + 9, DA.T_SX: 0}),
                  (i, "reads past the resized tile's right edge", {DA.T_SX: 17}), (i, "reads past its bottom edge", {DA.T_SY: 17}),
                  (i, "origin overflows", {DA.T_SX: 2**63 - 10}), (i, "origin overflows in y", {DA.T_SY: 2**63 - 10})]  # fmt: skip
    return cases


@pytest.mark.parametrize("tile, what, edits", _tile_cases(), ids=lambda v: str(v).replace(" ", "_") if isinstance(v, (int, str)) else "")
def test_tile_rectangle_refusals(tile, what, edits):
    t = _table()
    k = DA.MOS_TILE + tile * DA.MOS_TILE_FIELDS
    for f, v in edits.items():
        t[0, k + f] = v
    with pytest.raises(L.SgbError):
        _run(t)


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
def test_trainer_with_packed_roboflow_batches_matches_reference_batches(tmp_path, cuda_graph):
    """Trainer.train() fed by DetectionAugmentCollateFN batches of the Roboflow list gives the loss of the same batches made on the
    CPU by the cv2 / numpy chain + DetectionCollateFN, converted by functional.to_nhwc."""
    from super_gradients_b200.functional import to_nhwc
    from super_gradients_b200.training.losses import PPYoloELoss
    from super_gradients_b200.training.sg_trainer import Trainer
    from super_gradients_b200.training.utils.collate_fn.detection_collate_fn import DetectionCollateFN

    ds, items = replay("roboflow", 0)
    collate = DetectionAugmentCollateFN.for_dataset(ds)
    packed = [collate(items[:4]).pin_memory(), collate(items[4:])]
    ref = [DetectionCollateFN()([((oracle_mosaic_u8(p) / 255.0).astype(np.float32), t) for p, t in items[s : s + 4]]) for s in (0, 4)]
    ref = [(to_nhwc(x.cuda()), t) for x, t in ref]
    for b, (x, t) in zip(packed, ref):
        images, targets = b.to_model_input("cuda")
        assert torch.equal(images, x) and torch.equal(targets, t)
    losses = []
    for k, loader in enumerate((packed, ref)):
        torch.manual_seed(0)
        tp = dict(max_epochs=2, initial_lr=1e-3, lr_mode="constant", optimizer="SGD", loss=PPYoloELoss(num_classes=4, use_static_assigner=False), cuda_graph=cuda_graph,
                  save_model=False, run_validation_freq=100)  # fmt: skip
        tr = Trainer(f"mosaic{k}", ckpt_root_dir=str(tmp_path))
        tr.train(_tiny_yolo_nas(), tp, loader)
        losses.append(tr.history["train_loss"])
    assert all(np.isfinite(v) for v in losses[0])
    assert losses[0] == pytest.approx(losses[1], rel=1e-4, abs=1e-6)
