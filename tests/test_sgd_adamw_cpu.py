"""SGD and AdamW on FlatOptimizer, checked on the CPU against the way TrainStep built them before they joined it: the merged
arguments and the decay group's weight decay, the state list checkpoints store, the hyper-parameter rows bit for bit as float32
(restated here from TrainStep.set_hyper_params as it was), and the per-step launch sequence on the CPU stand-in backend."""
import copy
import itertools

import pytest
import torch

from super_gradients_b200.training import fused_optimizers as FO

# TrainStep's OPTIMIZER_DEFAULTS for SGD and AdamW before they moved into fused_optimizers
OLD_DEFAULTS = {"SGD": {"weight_decay": 1e-4, "momentum": 0.9}, "AdamW": {"weight_decay": 1e-2}}


def old_op(name, params):
    return {**OLD_DEFAULTS[name], **dict(params)}


def old_rows(name, op, lr, t, gs):
    """The rows TrainStep.set_hyper_params wrote for SGD and AdamW, restated: one torch.tensor per row."""
    wd = float(op.get("weight_decay", 0.0))
    if name == "SGD":
        mu, nes = float(op.get("momentum", 0.0)), float(bool(op.get("nesterov", False)))
        return torch.stack([torch.tensor([lr, mu, wd, gs, nes]), torch.tensor([lr, mu, 0.0, gs, nes])])
    b1, b2 = op.get("betas", (0.9, 0.999))
    eps = float(op.get("eps", 1e-8))
    row = [lr, b1, b2, eps, wd, 1 - b1**t, 1 - b2**t, gs]
    r0 = torch.tensor(row)
    row[4] = 0.0
    return torch.stack([r0, torch.tensor(row)])


class FlatStub:
    """The one FlatState field FlatOptimizer reads for SGD and AdamW."""

    def __init__(self, n):
        self.params = torch.zeros(n)


SGD_PARAMS = [{"momentum": mu, "nesterov": nes, "weight_decay": wd} for mu, nes, wd in itertools.product((0.0, 0.9), (False, True), (0.0, 1e-4))]
ADAMW_PARAMS = [{}, {"weight_decay": 0.05}, {"betas": (0.8, 0.95), "eps": 1e-6}, {"betas": [0.5, 0.9], "eps": 1e-10, "weight_decay": 0.0}]
ROW_CASES = [("SGD", p) for p in SGD_PARAMS] + [("AdamW", p) for p in ADAMW_PARAMS]


@pytest.mark.parametrize("zero_wd", [True, False])
@pytest.mark.parametrize("name, params", ROW_CASES)
def test_rows_equal_the_old_formulas_bit_for_bit(name, params, zero_wd):
    op, wd = FO.resolve(name, params, zero_wd)
    opt = FO.FlatOptimizer(name, op, wd, FlatStub(7))
    assert opt.hp_len == FO.HP_LEN[name] == {"SGD": 5, "AdamW": 8}[name]
    for t, gs, lr in itertools.product(range(1, 6), (1.0, 0.5), (0.1, 3.7e-4, 0.01 * 0.5 * (1 + 0.3))):
        got = torch.tensor(opt.rows(lr, t, gs), dtype=torch.float32)
        want = old_rows(name, old_op(name, params), lr, t, gs)
        assert got.shape == (2, opt.hp_len)
        assert torch.equal(got.view(torch.int32), want.view(torch.int32)), (name, params, zero_wd, t, gs, lr, got, want)
        assert got[1, FO.GRAD_SCALE_COLUMN[name]] == gs and got[1, 2 if name == "SGD" else 4] == 0.0  # the zero-decay row


@pytest.mark.parametrize("zero_wd", [True, False])
@pytest.mark.parametrize("name, params", [("SGD", {}), ("AdamW", {}), ("SGD", {"weight_decay": 0.0, "momentum": 0.5, "nesterov": True}),
                                          ("AdamW", {"weight_decay": 3e-2, "betas": (0.8, 0.9)}), ("SGD", {"dampening": 0.1, "lr": 5.0, "foreach": True}),
                                          ("AdamW", {"amsgrad": True, "maximize": True, "no_such_key": 1})])  # fmt: skip
def test_resolution_is_unchanged(name, params, zero_wd):
    """The defaults merge under the user's arguments; the decay group takes the merged weight_decay whatever zero_wd says; unknown
    keys pass through, not refused."""
    op, wd = FO.resolve(name, params, zero_wd)
    assert op == old_op(name, params)
    assert wd == float(old_op(name, params).get("weight_decay", 0.0))
    assert name not in FO.NAMES and name in FO.ALL_NAMES


def test_unknown_optimizer_is_refused():
    with pytest.raises(NotImplementedError, match="optimizer SGDW has no fused kernel"):
        FO.resolve("SGDW", {}, True)


@pytest.mark.parametrize("name, params, n", [("SGD", {}, 1), ("SGD", {"momentum": 0.0}, 1), ("AdamW", {}, 2)])
def test_state(name, params, n):
    """Checkpoints store len(state): SGD keeps its momentum buffer even with momentum 0."""
    op, wd = FO.resolve(name, params, True)
    st = FO.FlatOptimizer(name, op, wd, FlatStub(11)).state
    assert len(st) == n and all(s.shape == (11,) and not s.any() for s in st)


# ------------------------------------------------------------------------------------------------ launches (CPU stand-in)
@pytest.fixture
def stand_in(golden, monkeypatch):
    import cpu_backend
    import host_clip

    from super_gradients_b200.training import sg_trainer

    cpu_backend.install_training(monkeypatch)
    host_clip.install(monkeypatch)
    monkeypatch.setattr(sg_trainer, "setup_device", lambda device=None: torch.device("cpu"))
    return golden("tiny_yolo_nas")


def _tiny_model(g):
    from super_gradients_b200.training.models.detection_models.yolo_nas import YoloNAS

    torch.manual_seed(0)
    ap = copy.deepcopy(g["arch"])
    m = YoloNAS(backbone=ap["backbone"], neck=ap["neck"], heads=ap["heads"], num_classes=4, bn_eps=1e-3, bn_momentum=0.03, inplace_act=True, in_channels=3)
    m.load_state_dict({k: v.clone() for k, v in g["sd0"].items()}, strict=False)
    return m


@pytest.mark.parametrize("clip", [None, 0.5])
@pytest.mark.parametrize("name, params", [("SGD", {"momentum": 0.9}), ("SGD", {"momentum": 0.0, "nesterov": True}), ("AdamW", {"betas": (0.8, 0.95)})])
def test_launch_sequence_is_unchanged(name, params, clip, stand_in, monkeypatch):
    """One TrainStep update on the stand-in: (clip,) the decay range, the zero-decay range, then EMA of the parameters and of the
    buffers -- every launch on the same slice as before, with the device rows of set_hyper_params."""
    from super_gradients_b200 import kernels as K
    from super_gradients_b200.training.losses import PPYoloELoss
    from super_gradients_b200.training.sg_trainer import TrainStep

    st = TrainStep(_tiny_model(stand_in), PPYoloELoss(num_classes=4, use_static_assigner=False), name, params, True, ema=True, clip_grad_norm=clip)
    f = st.flat
    assert 0 < f.n_decay < f.n_live and f.n_buf > 0
    calls = []

    def span(t, base):
        return (t.data_ptr() - base.data_ptr()) // t.element_size(), t.numel()

    def record(kernel):
        real = getattr(K, kernel)

        def fn(*args):
            if kernel == "ema_update":
                ema, p, _ = args
                base = f.params if p.data_ptr() == f.params.data_ptr() else f.buffers
                calls.append((kernel, "params" if base is f.params else "buffers", span(p, base), ema.numel()))
            elif kernel == "clip_grad_norm":
                calls.append((kernel, args[3]))
            else:
                p, hp = args[0], args[-1]
                row = 0 if hp.data_ptr() == st.hp[0].data_ptr() else 1
                calls.append((kernel, span(p, f.params), row))
            return real(*args)

        monkeypatch.setattr(K, kernel, fn)

    for kernel in ("sgd_step", "adamw_step", "ema_update", "clip_grad_norm"):
        record(kernel)
    for t in (1, 2):
        f.grads.copy_(torch.linspace(-1e-2, 1e-2, f.grads.numel()))
        st.set_hyper_params(1e-3 * t, 0.99)
        assert torch.equal(st.hp.view(torch.int32), old_rows(name, old_op(name, params), 1e-3 * t, t, 1.0).view(torch.int32))
        calls.clear()
        st._apply_update()
        st.opt_steps += 1
        kernel = "sgd_step" if name == "SGD" else "adamw_step"
        want = ([("clip_grad_norm", FO.GRAD_SCALE_COLUMN[name])] if clip else []) + [
            (kernel, (0, f.n_decay), 0),
            (kernel, (f.n_decay, f.n_live - f.n_decay), 1),
            ("ema_update", "params", (0, f.params.numel()), f.params.numel()),
            ("ema_update", "buffers", (0, f.buffers.numel()), f.buffers.numel()),
        ]
        assert calls == want, (t, calls)
