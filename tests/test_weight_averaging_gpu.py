"""Best-snapshot averaging on the GPU: sgb_average_snapshots is bit-exact with the reference's torch loop on the CPU for every slot
count up to 10, odd lengths, misaligned slots and float32 specials; bad arguments are refused; Trainer.train(average_best_models=True)
on the tiny YOLO-NAS writes the average of the EMA snapshots it validated into average_model.pth."""
import copy

import pytest
import torch

from weight_averaging_cases import assert_same_state, reference_average, same_bits

pytestmark = pytest.mark.gpu
DEV = "cuda"
SPECIAL = [float("nan"), float("inf"), -float("inf"), 1e-40, -3e-42, 1.4e-45, 1e38, -1e38, 3e38, 3.4e38]


def _slots(k, n, offset, seed):
    """k device slots of n values (`offset` floats into their allocation: offset 1 makes every slot 4-byte but not 16-byte aligned)."""
    g = torch.Generator().manual_seed(seed)
    host = []
    for j in range(k):
        v = torch.randn(n, generator=g) * 10.0 ** float(torch.randint(-30, 30, (1,), generator=g))
        idx = torch.randint(0, n, (min(n, 64),), generator=g)
        v[idx] = torch.tensor(SPECIAL)[torch.randint(0, len(SPECIAL), (len(idx),), generator=g)]
        host.append(v)
    dev = [torch.empty(n + offset, device=DEV)[offset:] for _ in range(k)]
    for d, h in zip(dev, host):
        d.copy_(h)
    return host, dev


@pytest.mark.parametrize("k", range(1, 11))
@pytest.mark.parametrize("n, offset", [(1, 0), (3, 0), (4097, 0), (1_000_003, 0), (4097, 1), (65_539, 3)])
def test_kernel_is_the_reference_loop(k, n, offset):
    from super_gradients_b200 import kernels as K

    host, dev = _slots(k, n, offset, seed=1000 * k + n + offset)
    table = torch.tensor([d.data_ptr() for d in dev], dtype=torch.int64, device=DEV)
    out = torch.empty(n + offset, device=DEV)[offset:]
    K.average_snapshots(table, k, out)
    want = reference_average([{"w": h} for h in host])["w"]
    assert same_bits(out.cpu(), want)


def test_kernel_refuses_bad_arguments():
    from super_gradients_b200 import kernels as K
    from super_gradients_b200 import lib as L

    _, dev = _slots(2, 16, 0, seed=0)
    table = torch.tensor([d.data_ptr() for d in dev] * 40, dtype=torch.int64, device=DEV)
    out = torch.empty(16, device=DEV)
    for k in (0, -1, 65):
        with pytest.raises(L.SgbError, match="k must be"):
            L.call("sgb_average_snapshots", K._ptr(table), k, 16, K._ptr(out), K._stream())
    with pytest.raises(L.SgbError, match="null"):
        L.call("sgb_average_snapshots", None, 2, 16, K._ptr(out), K._stream())
    with pytest.raises(L.SgbError):
        K.average_snapshots(table.int(), 2, out)
    L.call("sgb_average_snapshots", K._ptr(table), 2, 0, K._ptr(out), K._stream())  # n == 0: nothing to do


def test_trainer_average_model_is_the_average_of_its_snapshots(golden, tmp_path):
    from super_gradients_b200.training.losses import PPYoloELoss
    from super_gradients_b200.training.models.detection_models.yolo_nas import YoloNAS
    from super_gradients_b200.training.sg_trainer import Trainer

    g = golden("tiny_yolo_nas")
    ap = copy.deepcopy(g["arch"])
    m = YoloNAS(backbone=ap["backbone"], neck=ap["neck"], heads=ap["heads"], num_classes=4, bn_eps=1e-3, bn_momentum=0.03, inplace_act=True, in_channels=3)
    m.load_state_dict({k: v.clone() for k, v in g["sd0"].items()}, strict=False)
    loader = [(g["x"] * (1 + 0.1 * i), g["targets"]) for i in range(2)]
    tp = dict(max_epochs=4, initial_lr=2e-3, lr_mode="cosine", optimizer="AdamW", optimizer_params={"weight_decay": 1e-5}, zero_weight_decay_on_bias_and_bn=True, ema=True,
              ema_params={"decay": 0.9, "decay_type": "threshold"}, loss=PPYoloELoss(num_classes=4, use_static_assigner=False), average_best_models=True,
              save_ckpt_epoch_list=[0, 1, 2, 3])  # fmt: skip
    trainer = Trainer("avg_gpu", ckpt_root_dir=str(tmp_path))
    hist = trainer.train(m, tp, loader, valid_loader=loader[:1])
    d = tmp_path / "avg_gpu"
    assert not (d / "averaging_snapshots.pkl").exists() and torch.isfinite(torch.tensor(hist["average_model"]["valid_loss"]))
    losses = hist["valid_loss"]
    assert len(losses) == 4 and all(torch.isfinite(torch.tensor(losses)))  # four finite losses fill slots 0 .. 3 in epoch order
    snaps = [{k: v.cpu() for k, v in torch.load(d / f"ckpt_epoch_{e}.pth", weights_only=False)["ema_net"].items()} for e in range(4)]
    avg = torch.load(d / "average_model.pth", weights_only=False)
    assert "optimizer_state_dict" not in avg and "ema_net" not in avg and avg["epoch"] == 3
    assert_same_state(avg["net"], reference_average(snaps))
