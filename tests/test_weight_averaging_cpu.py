"""CPU checks of best-snapshot averaging and EarlyStop: the g++ build of csrc/weight_average_math.cuh (the CUDA kernel's arithmetic)
stands in for kernels.average_snapshots and is bit-exact with the unmodified reference's averages (tests/golden/weight_averaging.pt);
ModelWeightAveraging and EarlyStop replay the reference's sequences; Trainer.train(average_best_models=True) runs on the tiny YOLO-NAS
fixture with the CPU stand-in of tests/cpu_backend.py."""
import copy
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest
import torch

import cpu_backend
from weight_averaging_cases import AVERAGING_CASES, EARLY_STOP_CASES, assert_same_state, bn_model, reference_average, same_bits, snapshot_states

from super_gradients_b200 import kernels as K

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_LIB = {}


def host_lib():
    """g++ build of tests/host_kernels/weight_average_host.cpp; -ffp-contract=off keeps a * n + s two roundings, as on the device."""
    if "h" not in _LIB:
        d = tempfile.mkdtemp(prefix="sgb_weight_average_host_")
        so = os.path.join(d, "weight_average_host.so")
        subprocess.run(["g++", "-O3", "-ffp-contract=off", "-std=c++17", "-shared", "-fPIC", "-x", "c++", os.path.join(ROOT, "tests", "host_kernels", "weight_average_host.cpp"),
                        "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "super_gradients_b200", "csrc"), "-o", so], check=True)  # fmt: skip
        h = ctypes.CDLL(so)
        h.average_snapshots_host.argtypes = [ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_void_p]
        _LIB["h"] = h
    return _LIB["h"]


def average_snapshots(slot_ptr_table, k, out):
    """CPU stand-in of kernels.average_snapshots: the same table of slot addresses (host memory here) through the host build."""
    table = slot_ptr_table[:k].contiguous()
    host_lib().average_snapshots_host(ctypes.c_void_p(table.data_ptr()), int(k), out.numel(), ctypes.c_void_p(out.data_ptr()))


@pytest.mark.parametrize("k", range(1, 11))
@pytest.mark.parametrize("n", [1, 7, 1001])
def test_host_average_is_the_torch_loop(k, n):
    g = torch.Generator().manual_seed(k * 100 + n)
    slots = [torch.randn(n, generator=g) * 10.0 ** float(torch.randint(-40, 39, (1,), generator=g)) for _ in range(k)]
    special = torch.tensor([float("nan"), float("inf"), -float("inf"), 1e-40, -1.4e-45, 1e38, 3.4e38, -2e38])
    for j, s in enumerate(slots):
        s[: min(n, 3)] = special[(j + torch.arange(min(n, 3))) % len(special)]
    out = torch.empty(n)
    average_snapshots(torch.tensor([s.data_ptr() for s in slots]), k, out)
    assert same_bits(out, reference_average([{"w": s} for s in slots])["w"])


@pytest.mark.parametrize("case", AVERAGING_CASES)
def test_averaging_replays_the_reference(case, golden, tmp_path, monkeypatch):
    from super_gradients_b200.training.utils.weight_averaging_utils import ModelWeightAveraging

    monkeypatch.setattr(K, "average_snapshots", average_snapshots)
    ref = golden("weight_averaging")["averaging"][case]
    greater, metrics = AVERAGING_CASES[case]
    states, model = snapshot_states(), bn_model()
    mwa = ModelWeightAveraging(str(tmp_path), greater_is_better=greater, metric_to_watch="m")
    fresh = torch.load(mwa.averaging_snapshots_file, weights_only=False)
    assert all(fresh[f"snapshot{i}"] is None for i in range(10)) and fresh["snapshots_metric"].dtype == np.float64
    for epoch, (value, want) in enumerate(zip(metrics, ref["steps"])):
        model.load_state_dict(states[epoch])
        assert_same_state(mwa.get_average_model(model, validation_results_dict={"m": value}), want["average"])
        np.testing.assert_array_equal(mwa.snapshots_metric, want["snapshots_metric"])
    pkl = torch.load(mwa.averaging_snapshots_file, weights_only=False)
    assert list(pkl) == list(ref["pkl"])
    np.testing.assert_array_equal(pkl["snapshots_metric"], ref["pkl"]["snapshots_metric"])
    for i in range(10):
        assert_same_state(pkl[f"snapshot{i}"], ref["pkl"][f"snapshot{i}"])
    # a resumed run reads the same slots back from the file
    again = ModelWeightAveraging(str(tmp_path), greater_is_better=greater, metric_to_watch="m", load_checkpoint=True)
    assert_same_state(again.get_average_model(model), ref["steps"][-1]["average"])
    again.cleanup()
    assert not os.path.exists(mwa.averaging_snapshots_file)


def test_num_batches_tracked_turns_float32_after_two_snapshots(golden):
    steps = golden("weight_averaging")["averaging"]["loss"]["steps"]
    assert steps[0]["average"]["1.num_batches_tracked"].dtype == torch.int64
    nbt = steps[-1]["average"]["1.num_batches_tracked"]
    assert nbt.dtype == torch.float32 and float(nbt) != int(nbt)


@pytest.mark.parametrize("case", EARLY_STOP_CASES)
def test_early_stop_replays_the_reference(case, golden):
    from super_gradients_b200.training.utils.callbacks import PhaseContext
    from super_gradients_b200.training.utils.early_stopping import EarlyStop

    kwargs, values = EARLY_STOP_CASES[case]
    cb = EarlyStop(**kwargs)
    rows = []
    for v in values:
        ctx = PhaseContext(metrics_dict={} if v is None else {kwargs["monitor"]: v})
        cb(ctx)
        rows.append({"stop": bool(ctx.stop_training), "wait_count": cb.wait_count, "best_score": float(cb.best_score)})
    want = golden("weight_averaging")["early_stop"][case]
    assert [r["stop"] for r in rows] == [r["stop"] for r in want] and [r["wait_count"] for r in rows] == [r["wait_count"] for r in want]
    np.testing.assert_array_equal([r["best_score"] for r in rows], [r["best_score"] for r in want])
    if case == "pose_patience":
        assert [r["stop"] for r in rows].index(True) == 104  # the 100th check without a gain of min_delta


def test_early_stop_phase_forms_and_refusals():
    from super_gradients_b200.common.registry import CALLBACKS
    from super_gradients_b200.training.utils.callbacks import Phase
    from super_gradients_b200.training.utils.early_stopping import EarlyStop

    target = {"_target_": "super_gradients.training.utils.callbacks.base_callbacks.Phase", "value": "VALIDATION_EPOCH_END"}
    for phase in (Phase.VALIDATION_EPOCH_END, "VALIDATION_EPOCH_END", target):
        assert EarlyStop(phase, monitor="AP").phase is Phase.VALIDATION_EPOCH_END
    assert CALLBACKS["EarlyStop"] is EarlyStop
    with pytest.raises(ValueError):
        EarlyStop(Phase.TEST_END, monitor="AP")
    with pytest.raises(ValueError):
        EarlyStop("VALIDATION_EPOCH_END", monitor="AP", mode="median")
    with pytest.raises(RuntimeError, match="monitor"):
        from super_gradients_b200.training.utils.callbacks import PhaseContext

        EarlyStop("VALIDATION_EPOCH_END", monitor="AP")(PhaseContext(metrics_dict={"valid_loss": 1.0}))


# ------------------------------------------------------------------------------------------------ Trainer.train()
@pytest.fixture
def tiny(golden, monkeypatch):
    from super_gradients_b200.training import sg_trainer
    from super_gradients_b200.training.losses import PPYoloELoss
    from super_gradients_b200.training.models.detection_models.yolo_nas import YoloNAS

    cpu_backend.install_training(monkeypatch)
    monkeypatch.setattr(K, "average_snapshots", average_snapshots)
    monkeypatch.setattr(sg_trainer, "setup_device", lambda device=None: torch.device("cpu"))
    g = golden("tiny_yolo_nas")

    def build():
        torch.manual_seed(0)  # the unused rbr_reparam placeholders are not in the fixture: same random values in every build
        ap = copy.deepcopy(g["arch"])
        m = YoloNAS(backbone=ap["backbone"], neck=ap["neck"], heads=ap["heads"], num_classes=4, bn_eps=1e-3, bn_momentum=0.03, inplace_act=True, in_channels=3)
        m.load_state_dict({k: v.clone() for k, v in g["sd0"].items()}, strict=False)
        return m

    loader = [(g["x"] * (1 + 0.1 * i), g["targets"]) for i in range(2)]
    base = dict(max_epochs=3, initial_lr=2e-3, lr_mode="cosine", cosine_final_lr_ratio=0.1, optimizer="AdamW", optimizer_params={"weight_decay": 1e-5}, zero_weight_decay_on_bias_and_bn=True,
                ema=True, ema_params={"decay": 0.9, "decay_type": "threshold"})  # fmt: skip
    tp = lambda **kw: {**base, "loss": PPYoloELoss(num_classes=4, use_static_assigner=False), **kw}  # noqa: E731
    return build, loader, tp


def test_trainer_writes_and_validates_the_average(tiny, tmp_path):
    from super_gradients_b200.training.sg_trainer import Trainer
    from super_gradients_b200.training.utils.callbacks import Callback

    build, loader, tp = tiny
    events, live = [], {}
    trainer = Trainer("avg", ckpt_root_dir=str(tmp_path))

    class Rec(Callback):
        def on_average_best_models_validation_start(self, ctx):
            events.append("start")
            st = trainer.step
            live.update(params=st.flat.params.clone(), buffers=st.flat.buffers.clone(), nbt=[t.clone() for t in st._nbt])

        def on_average_best_models_validation_end(self, ctx):
            events.append(("end", dict(ctx.metrics_dict)))

        def on_training_end(self, ctx):
            events.append("training_end")

    model = build()
    hist = trainer.train(model, tp(average_best_models=True, save_ckpt_epoch_list=[0, 1, 2], phase_callbacks=[Rec()]), loader, valid_loader=loader[:1])
    d = tmp_path / "avg"
    assert not (d / "averaging_snapshots.pkl").exists()
    ck = torch.load(d / "average_model.pth", weights_only=False)
    assert set(ck) == {"net", "acc", "epoch", "metrics", "packages", "processing_params"} and ck["epoch"] == 2
    # every epoch's loss is finite, so the three EMA snapshots fill slots 0, 1, 2 in epoch order
    snaps = [torch.load(d / f"ckpt_epoch_{e}.pth", weights_only=False)["ema_net"] for e in range(3)]
    assert all(np.isfinite(hist["valid_loss"]))
    assert_same_state(ck["net"], reference_average(snaps))
    nbt = [k for k in ck["net"] if k.endswith("num_batches_tracked")]
    assert nbt and all(ck["net"][k].dtype == torch.float32 for k in nbt)  # torch.true_divide of the int64 counters, as the reference writes them
    # the final validation ran on the average, then the live weights came back bit for bit
    assert events[0] == "start" and events[1][0] == "end" and events[2] == "training_end"
    assert events[1][1] == hist["average_model"] and np.isfinite(hist["average_model"]["valid_loss"])
    st = trainer.step
    assert torch.equal(st.flat.params, live["params"]) and torch.equal(st.flat.buffers, live["buffers"]) and all(torch.equal(a, b) for a, b in zip(st._nbt, live["nbt"]))
    fresh = build()
    fresh.load_state_dict(ck["net"])
    res = Trainer("check", ckpt_root_dir=str(tmp_path)).test(model=fresh, test_loader=loader[:1], loss=tp()["loss"], silent_mode=True)
    assert res["loss"] == pytest.approx(hist["average_model"]["valid_loss"], rel=1e-6)


def test_trainer_average_survives_a_resume(tiny, tmp_path):
    from super_gradients_b200.training.sg_trainer import Trainer

    build, loader, tp = tiny

    class Interrupt(Exception):
        pass

    class TwoEpochLoader(list):
        passes = 0

        def __iter__(self):
            TwoEpochLoader.passes += 1
            if TwoEpochLoader.passes > 2:
                raise Interrupt()
            return super().__iter__()

    Trainer("straight", ckpt_root_dir=str(tmp_path)).train(build(), tp(average_best_models=True), loader, valid_loader=loader[:1])
    with pytest.raises(Interrupt):
        Trainer("resumed", ckpt_root_dir=str(tmp_path)).train(build(), tp(average_best_models=True), TwoEpochLoader(loader), valid_loader=loader[:1])
    pkl = torch.load(tmp_path / "resumed" / "averaging_snapshots.pkl", weights_only=False)
    assert [pkl[f"snapshot{i}"] is not None for i in range(3)] == [True, True, False]
    Trainer("resumed", ckpt_root_dir=str(tmp_path)).train(build(), tp(average_best_models=True, resume=True), loader, valid_loader=loader[:1])
    a = torch.load(tmp_path / "straight" / "average_model.pth", weights_only=False)["net"]
    b = torch.load(tmp_path / "resumed" / "average_model.pth", weights_only=False)["net"]
    assert_same_state(a, b)


def test_trainer_average_needs_save_model(tiny, tmp_path):
    from super_gradients_b200.training.sg_trainer import Trainer

    build, loader, tp = tiny
    with pytest.warns(UserWarning, match="average_best_models"):
        hist = Trainer("nosave", ckpt_root_dir=str(tmp_path)).train(build(), tp(max_epochs=1, average_best_models=True, save_model=False), loader, valid_loader=loader[:1])
    assert "average_model" not in hist and not (tmp_path / "nosave").exists()


def test_trainer_stops_on_the_pose_recipe_early_stop_entry(tiny, tmp_path):
    """The pose recipe's phase_callbacks entry (hydra's Phase target form) resolved through the CALLBACKS registry, watching the
    validation loss with mode max and patience 1: the run stops after the epoch a fresh EarlyStop fed the same losses stops at."""
    from super_gradients_b200.training.sg_trainer import Trainer
    from super_gradients_b200.training.utils.callbacks import PhaseContext
    from super_gradients_b200.training.utils.early_stopping import EarlyStop

    build, loader, tp = tiny
    entry = {"phase": {"_target_": "super_gradients.training.utils.callbacks.base_callbacks.Phase", "value": "VALIDATION_EPOCH_END"}, "monitor": "valid_loss", "mode": "max",
             "min_delta": 0.0001, "patience": 1, "verbose": True}  # fmt: skip
    hist = Trainer("es", ckpt_root_dir=str(tmp_path)).train(build(), tp(max_epochs=4, ema=False, phase_callbacks=[{"EarlyStop": entry}]), loader, valid_loader=loader[:1])
    replay, stop_at = EarlyStop(**entry), None
    for e, v in enumerate(hist["valid_loss"]):
        ctx = PhaseContext(metrics_dict={"valid_loss": v})
        replay(ctx)
        if ctx.stop_training:
            stop_at = e
            break
    assert stop_at is not None and len(hist["train_loss"]) == stop_at + 1 < 4
    with pytest.raises(ValueError, match="registered"):
        Trainer("es2", ckpt_root_dir=str(tmp_path)).train(build(), tp(max_epochs=1, phase_callbacks=[{"NoSuchCallback": {}}]), loader)


def test_trainer_without_the_new_keys_writes_the_same_files(tiny, tmp_path):
    from super_gradients_b200.training.sg_trainer import Trainer

    build, loader, tp = tiny
    hist = Trainer("plain", ckpt_root_dir=str(tmp_path)).train(build(), tp(max_epochs=2, save_ckpt_epoch_list=[1]), loader, valid_loader=loader[:1])
    assert sorted(os.listdir(tmp_path / "plain")) == ["ckpt_best.pth", "ckpt_epoch_1.pth", "ckpt_latest.pth"] and "average_model" not in hist
