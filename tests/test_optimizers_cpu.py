"""CPU checks of Adam, RMSprop, RMSpropTF, Lion and Lamb on the flat buffer: the g++ build of csrc/optim_math.cuh (the kernels'
arithmetic, tests/host_optim.py) stands in for the kernels and replays the unmodified reference's optimizers
(tests/golden/optimizers.pt); the constructor arguments resolve and refuse as the reference's build_optimizer and torch do."""
import pytest
import torch

import host_optim
from optimizer_cases import CASES, STEPS, ZERO_GRAD, ZERO_PARAM, assert_matches, is_live, replay, unpack

from super_gradients_b200.training import fused_optimizers as FO

@pytest.fixture
def host_kernels(monkeypatch):
    host_optim.install(monkeypatch)


@pytest.mark.parametrize("case", CASES)
def test_host_build_replays_the_reference(case, golden, host_kernels):
    want = golden("optimizers")["cases"][case]
    ref_no_decay = golden("optimizers")["no_decay"] if CASES[case][2] else []
    for step, got, ref, before, flat in replay(case, want):
        assert_matches(case, got, ref, before, step)
    no_decay = sorted(n for n, (off, k) in flat.offsets.items() if off >= flat.n_decay)
    assert no_decay == [n for n in ref_no_decay if is_live(n)]  # the flat buffer groups the live tensors as the reference does


def test_golden_covers_the_branches(golden):
    cases = golden("optimizers")["cases"]
    assert cases["lamb_default"]["group_weight_decay"] == [0.0]  # zero_wd grouping without weight_decay: no decay, no adaptation
    assert cases["lamb_default_no_zero_wd"]["group_weight_decay"] == [0.01]  # the class default
    last = unpack(cases["lion_default"], STEPS)
    assert all(torch.equal(last[n]["exp_avg"], torch.zeros_like(last[n]["exp_avg"])) for n in ZERO_GRAD)
    zp = unpack(cases["lamb_always_adapt"], STEPS)[ZERO_PARAM]["param"]
    assert torch.equal(zp, torch.zeros_like(zp))


@pytest.mark.parametrize("name", FO.NAMES)
def test_unknown_arguments_are_refused(name):
    with pytest.raises(TypeError, match="unexpected keyword argument 'nesterov_typo'"):
        FO.resolve(name, {"nesterov_typo": 1}, True)


@pytest.mark.parametrize("name, flag", [("Adam", "amsgrad"), ("Adam", "maximize"), ("RMSprop", "maximize"), ("Adam", "decoupled_weight_decay")])
def test_unsupported_flags_are_refused(name, flag):
    with pytest.raises(NotImplementedError, match=flag):
        FO.resolve(name, {flag: True}, False)
    FO.resolve(name, {flag: False, "foreach": True, **({"fused": False} if name == "Adam" else {})}, False)  # implementation selectors are accepted


def test_defaults_merge_like_build_optimizer():
    assert FO.resolve("Adam", {}, True)[1] == 1e-4 and FO.resolve("RMSprop", {}, False)[0]["momentum"] == 0.9
    assert FO.resolve("RMSpropTF", {"momentum": 0.0}, True)[0]["momentum"] == 0.0
    assert FO.resolve("Lamb", {}, True)[1] == 0.0 and FO.resolve("Lamb", {}, False)[1] == 0.01
    assert FO.resolve("Lion", {"weight_decay": 0.3}, True)[1] == 0.3


def test_lamb_chunk_table():
    t = FO.lamb_chunk_table([5, 0, 40000, 3], chunk=16384)
    assert t.tolist() == [[0, 5, 0, 1], [5, 16384, 1, 3], [16389, 16384, 1, 3], [32773, 7232, 1, 3], [40005, 3, 4, 1]]


def test_rmsprop_tf_square_avg_starts_at_one():
    flat = torch.zeros(7)
    op, _ = FO.resolve("RMSpropTF", {"centered": True}, True)
    st = FO.state_tensors("RMSpropTF", op, flat)
    assert len(st) == 3 and torch.equal(st[0], torch.ones(7)) and torch.equal(st[1], torch.zeros(7))
    assert len(FO.state_tensors("RMSprop", FO.resolve("RMSprop", {"momentum": 0.0}, True)[0], flat)) == 1


# ------------------------------------------------------------------------------------------------ Trainer.train()
TRAIN_CASES = {"Adam": {}, "RMSprop": {"centered": True}, "RMSpropTF": {"centered": True}, "Lion": {"weight_decay": 0.1}, "Lamb": {"weight_decay": 0.01}}


@pytest.fixture
def tiny_trainer(golden, monkeypatch):
    import copy

    import cpu_backend

    from super_gradients_b200.training import sg_trainer
    from super_gradients_b200.training.losses import PPYoloELoss
    from super_gradients_b200.training.models.detection_models.yolo_nas import YoloNAS

    cpu_backend.install_training(monkeypatch)
    host_optim.install(monkeypatch)
    monkeypatch.setattr(sg_trainer, "setup_device", lambda device=None: torch.device("cpu"))
    g = golden("tiny_yolo_nas")

    def build():
        torch.manual_seed(0)
        ap = copy.deepcopy(g["arch"])
        m = YoloNAS(backbone=ap["backbone"], neck=ap["neck"], heads=ap["heads"], num_classes=4, bn_eps=1e-3, bn_momentum=0.03, inplace_act=True, in_channels=3)
        m.load_state_dict({k: v.clone() for k, v in g["sd0"].items()}, strict=False)
        return m

    loader = [(g["x"] * (1 + 0.1 * i), g["targets"]) for i in range(2)]

    def tp(name, **kw):
        return {"max_epochs": 2, "initial_lr": 1e-3, "lr_mode": "constant", "optimizer": name, "optimizer_params": TRAIN_CASES[name], "zero_weight_decay_on_bias_and_bn": True,
                "batch_accumulate": 2 if name == "RMSpropTF" else 1, "loss": PPYoloELoss(num_classes=4, use_static_assigner=False), **kw}  # fmt: skip

    return build, loader, tp


@pytest.mark.parametrize("name", TRAIN_CASES)
def test_trainer_trains_and_resumes(name, tiny_trainer, tmp_path):
    """Trainer.train() with each optimizer on the CPU stand-in: the loss stays finite, the checkpoint holds the optimizer's state
    under its name, and a run resumed after epoch 0 ends bit-identical to the straight run (RMSpropTF keeps its saved square_avg)."""
    from super_gradients_b200.training.sg_trainer import Trainer

    build, loader, tp = tiny_trainer
    hist = Trainer("straight", ckpt_root_dir=str(tmp_path)).train(build(), tp(name, ema=True), loader)
    assert all(torch.isfinite(torch.tensor(hist["train_loss"])))
    Trainer("resumed", ckpt_root_dir=str(tmp_path)).train(build(), tp(name, ema=True, max_epochs=1), loader)
    first = torch.load(tmp_path / "resumed" / "ckpt_latest.pth", weights_only=False)["optimizer_state_dict"]
    assert first["name"] == name and len(first["state"]) == {"Adam": 2, "RMSprop": 3, "RMSpropTF": 3, "Lion": 1, "Lamb": 2}[name]
    if name == "RMSpropTF":
        assert not torch.equal(first["state"][0], torch.ones_like(first["state"][0]))
    Trainer("resumed", ckpt_root_dir=str(tmp_path)).train(build(), tp(name, ema=True, resume=True), loader)
    a = torch.load(tmp_path / "straight" / "ckpt_latest.pth", weights_only=False)
    b = torch.load(tmp_path / "resumed" / "ckpt_latest.pth", weights_only=False)
    assert all(torch.equal(a["net"][k], b["net"][k]) for k in a["net"]) and all(torch.equal(a["ema_net"][k], b["ema_net"][k]) for k in a["ema_net"])
    assert all(torch.equal(x, y) for x, y in zip(a["optimizer_state_dict"]["state"], b["optimizer_state_dict"]["state"]))


def test_trainer_refuses_a_checkpoint_of_another_state_layout(tiny_trainer, tmp_path):
    from super_gradients_b200.training.sg_trainer import Trainer

    build, loader, tp = tiny_trainer
    Trainer("r", ckpt_root_dir=str(tmp_path)).train(build(), tp("RMSprop", max_epochs=1), loader)
    with pytest.raises(ValueError, match="does not belong"):
        Trainer("r", ckpt_root_dir=str(tmp_path)).train(build(), tp("RMSprop", resume=True, optimizer_params={"centered": False}), loader)


def test_trainer_refuses_unknown_optimizer_arguments(tiny_trainer, tmp_path):
    from super_gradients_b200.training.sg_trainer import Trainer

    build, loader, tp = tiny_trainer
    with pytest.raises(TypeError, match="unexpected keyword argument"):
        Trainer("u", ckpt_root_dir=str(tmp_path)).train(build(), tp("Lion", optimizer_params={"eps": 1e-8}), loader)
    with pytest.raises(NotImplementedError, match="amsgrad"):
        Trainer("u", ckpt_root_dir=str(tmp_path)).train(build(), tp("Adam", optimizer_params={"amsgrad": True}), loader)


def test_trainer_world2_gloo(tmp_path):
    """Trainer.train() with every new optimizer on two gloo ranks (one NCCL-style flat all-reduce per step, 1/world folded into the
    kernels' grad_scale): the replicas stay identical."""
    import optimizer_trainer_cases

    codes, out = optimizer_trainer_cases.launch(str(tmp_path), 29571)
    assert codes == [0, 0], out[-4000:]
    assert out.count("optimizers ok") == 2, out[-4000:]
