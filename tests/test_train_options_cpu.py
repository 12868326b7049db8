"""CPU checks of clip_grad_norm, precise_bn and batch_accumulate in Trainer.train(): the g++ build of the clip arithmetic in
csrc/optim_math.cuh (tests/host_clip.py) against torch.nn.utils.clip_grad_norm_, the grad_scale column it scales for every fused
optimizer, and the trainer glue on the CPU stand-in backend -- precise_bn against the reference's own compute_precise_bn_stats."""
import copy
import itertools
import math

import pytest
import torch

import host_clip
from oracle import ref_shim

from super_gradients_b200.training import fused_optimizers as FO

OPTIMIZERS = {"SGD": {}, "AdamW": {}, "Adam": {}, "RMSprop": {}, "RMSpropTF": {}, "Lion": {}, "Lamb": {}}


def _grads(kind):
    gen = torch.Generator().manual_seed(3)
    shapes = [(16, 3, 3, 3), (16,), (40000,), (7,), (0,), (5, 5)]
    gs = [torch.randn(s, generator=gen) for s in shapes]
    if kind == "clip":
        return gs, 0.5
    if kind == "no_clip":
        return gs, 1e4
    if kind == "zeros":
        return [torch.zeros_like(g) for g in gs], 1.0
    if kind == "tiny":
        return [g * 1e-30 for g in gs], 1.0
    if kind == "small":
        return [g * 1e-8 for g in gs], 1e-9
    if kind == "huge":
        return [g * 1e15 for g in gs], 1.0
    if kind == "overflow":
        return [g * 1e20 for g in gs], 1.0
    if kind in ("inf", "nan"):
        gs[2][123] = float(kind)
        return gs, 1.0
    raise AssertionError(kind)


def _host_clip(grads, max_norm, hp_len=8, gs_col=7, gs=1.0):
    g = torch.cat([x.reshape(-1) for x in grads]).contiguous()
    chunks = FO.lamb_chunk_table([x.numel() for x in grads])
    hp = torch.full((2, hp_len), 0.25)
    hp[:, gs_col] = gs
    partials = torch.zeros(chunks.shape[0], dtype=torch.float64)
    out = torch.zeros(2)
    host_clip.clip_grad_norm(g, chunks, hp, gs_col, max_norm, partials, out)
    return g, hp, out


def _torch_clip(grads, max_norm):
    ps = [torch.nn.Parameter(torch.zeros_like(x)) for x in grads]
    for p, x in zip(ps, grads):
        p.grad = x.clone()
    total = torch.nn.utils.clip_grad_norm_(ps, max_norm)
    return float(total), torch.cat([p.grad.reshape(-1) for p in ps])


@pytest.mark.parametrize("kind", ["clip", "no_clip", "zeros", "tiny", "small", "huge", "overflow", "inf", "nan"])
def test_clip_matches_torch(kind):
    """Total norm within 1e-6 (float64 sums here, float32 in torch; torch's float32 squares underflow for `tiny`), the coefficient
    bit-exact given torch's total, within 1e-6 given ours, and the scaled gradients g * grad_scale equal torch's clipped ones."""
    grads, max_norm = _grads(kind)
    g, hp, (total, coef) = _host_clip(grads, max_norm)
    t_total, t_clipped = _torch_clip(grads, max_norm)
    t_coef = float(torch.clamp(max_norm / (torch.tensor(t_total) + 1e-6), max=1.0))
    if kind == "nan":
        assert math.isnan(total) and math.isnan(t_total) and math.isnan(coef)
        assert torch.isnan(g * hp[0, 7]).all() and torch.isnan(t_clipped).all()
        return
    if kind in ("inf", "overflow"):
        assert math.isinf(total) and math.isinf(t_total) and coef == 0.0 == t_coef
    elif kind != "tiny":
        assert total == pytest.approx(t_total, rel=1e-6, abs=0.0)
    assert host_clip.coef(t_total, max_norm) == t_coef  # same float32 op order as torch
    assert coef == pytest.approx(t_coef, rel=1e-6, abs=0.0)
    assert hp[0, 7] == hp[1, 7] == coef and (hp[:, :7] == 0.25).all()  # only the grad_scale column of both rows moves
    clipped = g * hp[0, 7]
    tol = 0.0 if coef == t_coef else 1e-6
    torch.testing.assert_close(clipped, t_clipped, rtol=tol, atol=0.0, equal_nan=True)  # inf * 0 is NaN in both
    if kind in ("no_clip", "zeros", "tiny"):
        assert coef == 1.0


def test_clip_scales_the_existing_grad_scale():
    """Under data parallelism grad_scale is 1/world: the coefficient multiplies it, and the norm is that of g * grad_scale."""
    grads, _ = _grads("clip")
    g = torch.cat([x.reshape(-1) for x in grads])
    _, hp, (total, coef) = _host_clip(grads, 0.5, gs=0.25)
    assert total == pytest.approx(float((g.double() * 0.25).norm()), rel=1e-6)
    assert hp[0, 7] == torch.tensor(0.25) * coef


def _hp_rows(name, world, tiny_step):
    st = tiny_step(name)
    st.world = world
    st.set_hyper_params(1e-3, None)
    return st.hp.clone()


@pytest.mark.parametrize("name", OPTIMIZERS)
def test_grad_scale_column(name, tiny_step):
    """GRAD_SCALE_COLUMN names the one column of both hyper-parameter rows that carries grad_scale = 1/world, for every optimizer,
    and the clip multiplies exactly that column of both rows."""
    a, b = _hp_rows(name, 1, tiny_step), _hp_rows(name, 4, tiny_step)
    col = FO.GRAD_SCALE_COLUMN[name]
    assert a.shape[0] == 2 and (a != b).nonzero()[:, 1].unique().tolist() == [col]
    assert (a[:, col] == 1.0).all() and (b[:, col] == 0.25).all()
    grads, _ = _grads("clip")
    g = torch.cat([x.reshape(-1) for x in grads])
    chunks = FO.lamb_chunk_table([x.numel() for x in grads])
    hp, out = b.clone(), torch.zeros(2)
    host_clip.clip_grad_norm(g, chunks, hp, col, 0.5, torch.zeros(chunks.shape[0], dtype=torch.float64), out)
    keep = torch.ones_like(hp, dtype=torch.bool)
    keep[:, col] = False
    assert torch.equal(hp[keep], b[keep]) and (hp[:, col] == torch.tensor(0.25) * out[1]).all() and 0 < out[1] < 1


# ------------------------------------------------------------------------------------------------ Trainer glue (CPU stand-in)
@pytest.fixture
def stand_in(golden, monkeypatch):
    import cpu_backend
    import host_optim

    from super_gradients_b200.training import sg_trainer

    cpu_backend.install_training(monkeypatch)
    host_optim.install(monkeypatch)
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


@pytest.fixture
def tiny_step(stand_in):
    from super_gradients_b200.training.losses import PPYoloELoss
    from super_gradients_b200.training.sg_trainer import TrainStep

    def make(name, **kw):
        return TrainStep(_tiny_model(stand_in), PPYoloELoss(num_classes=4, use_static_assigner=False), name, OPTIMIZERS[name], True, **kw)

    return make


class Loader:
    """A train loader that records how many batches every fresh iteration drew."""

    def __init__(self, batches, batch_size):
        self.batches, self.batch_size, self.drawn = batches, batch_size, []

    def __len__(self):
        return len(self.batches)

    def __iter__(self):
        self.drawn.append(0)
        for b in self.batches:
            self.drawn[-1] += 1
            yield b


def _batches(g, n):
    return [(g["x"] * (1 + 0.1 * i), g["targets"]) for i in range(n)]


def _trainer(g, tmp_path, **kw):
    from super_gradients_b200.training.losses import PPYoloELoss
    from super_gradients_b200.training.sg_trainer import Trainer, TrainStep

    t = Trainer("pbn", ckpt_root_dir=str(tmp_path))
    t.net = _tiny_model(g).train()
    t.criterion = PPYoloELoss(num_classes=4, use_static_assigner=False)
    t.step = TrainStep(t.net, t.criterion, "SGD", {}, True, **kw)
    return t


@pytest.mark.parametrize("size, batch_size, n_batches, world, want", [(None, 4, 5, 1, 1), (None, 4, 5, 2, 2), (12, 4, 5, 1, 3), (30, 4, 5, 1, 5), (13, 2, 9, 2, 3), (3, 4, 5, 1, 0)])
def test_precise_bn_batch_count(size, batch_size, n_batches, world, want, stand_in, tmp_path, monkeypatch):
    """num_iter = int(precise_bn_batch_size / (batch_size * world)) with a size, else world; at most len(loader); one fresh
    iteration of the train loader.  The ranks' sums are averaged by one all-reduce of the flat buffer."""
    from super_gradients_b200.training import sg_trainer

    reduced = []
    if world > 1:
        monkeypatch.setattr(sg_trainer, "is_distributed", lambda: True)
        monkeypatch.setattr(torch.distributed, "get_world_size", lambda group=None: world)
        monkeypatch.setattr(torch.distributed, "all_reduce", lambda t, *a, **k: (reduced.append(t.numel()), t.mul_(world)))
    t = _trainer(stand_in, tmp_path)
    loader = Loader(_batches(stand_in, n_batches), batch_size)
    t._precise_bn(loader, {"precise_bn_batch_size": size})
    assert loader.drawn == ([want] if want else [])
    assert reduced == ([t.step.flat.n_buf] if world > 1 else [])


def test_precise_bn_matches_the_reference(stand_in, tmp_path, monkeypatch):
    """The same model and batches through the reference's compute_precise_bn_stats and through Trainer._precise_bn: identical
    statistics and num_batches_tracked, momenta restored, and the flat buffer's storage kept (the reference replaces the buffers)."""
    if not ref_shim.available():
        pytest.skip("reference tree not present")
    ref_shim.install()
    from super_gradients.training.utils.distributed_training_utils import compute_precise_bn_stats

    batches = _batches(stand_in, 4)
    t = _trainer(stand_in, tmp_path)
    bns = [m for m in t.net.modules() if isinstance(m, torch.nn.BatchNorm2d)]
    bns[0].momentum = 0.5  # restored per module
    ptrs = [(bn.running_mean.data_ptr(), bn.running_var.data_ptr()) for bn in bns]
    flat_ptr = t.step.flat.buffers.data_ptr()
    t._precise_bn(Loader(batches, 2), {"precise_bn_batch_size": 6})

    ref = _tiny_model(stand_in).train()
    ref_bns = [m for m in ref.modules() if isinstance(m, torch.nn.BatchNorm2d)]
    ref_bns[0].momentum = 0.5
    monkeypatch.setattr(torch.Tensor, "cuda", lambda self, *a, **k: self)
    compute_precise_bn_stats(ref, Loader(batches, 2), precise_bn_batch_size=6, num_gpus=1)

    assert [bn.momentum for bn in bns] == [bn.momentum for bn in ref_bns] and bns[0].momentum == 0.5
    assert [(bn.running_mean.data_ptr(), bn.running_var.data_ptr()) for bn in bns] == ptrs and t.step.flat.buffers.data_ptr() == flat_ptr
    sd, rsd = t.net.state_dict(), ref.state_dict()
    for k in rsd:
        if "running_" in k or k.endswith("num_batches_tracked"):
            assert torch.equal(sd[k], rsd[k]), k
    assert any(int(v) == 3 for k, v in sd.items() if k.endswith("num_batches_tracked"))


def test_precise_bn_live_then_ema_before_validation(stand_in, tmp_path, monkeypatch):
    """Trainer.train(precise_bn, ema): after every train epoch the pass runs on the live weights in train mode, then on the EMA
    weights in eval mode (the reference's EMA model is in eval mode), then validation; the pass leaves the weights alone."""
    from super_gradients_b200.training.losses import PPYoloELoss
    from super_gradients_b200.training.sg_trainer import Trainer

    calls, orig_pbn, orig_val = [], Trainer._precise_bn, Trainer._validate

    def pbn(self, loader, tp):
        calls.append(("precise_bn", self.net.training, self.step.flat.params.clone()))
        return orig_pbn(self, loader, tp)

    def val(self, *a, **k):
        calls.append(("validate",))
        return orig_val(self, *a, **k)

    monkeypatch.setattr(Trainer, "_precise_bn", pbn)
    monkeypatch.setattr(Trainer, "_validate", val)
    loader = Loader(_batches(stand_in, 2), 4)
    tp = {"max_epochs": 1, "initial_lr": 1e-3, "lr_mode": "constant", "ema": True, "precise_bn": True, "loss": PPYoloELoss(num_classes=4, use_static_assigner=False),
          "save_model": False, "batch_accumulate": 2, "clip_grad_norm": 0.1}  # fmt: skip
    tr = Trainer("order", ckpt_root_dir=str(tmp_path))
    tr.train(_tiny_model(stand_in), tp, loader, valid_loader=_batches(stand_in, 1))
    assert [c[:2] for c in calls] == [("precise_bn", True), ("precise_bn", False), ("validate",)]
    assert torch.equal(calls[0][2], tr.step.flat.params) and torch.equal(calls[1][2], tr.step.ema_params)
    assert loader.drawn == [2, 1, 1]  # the epoch, then one fresh iteration per pass
    total, coef = tr.step.clip_norm_coef.tolist()
    assert total > 0.1 and coef == pytest.approx(0.1 / total, rel=1e-6)


@pytest.mark.parametrize("value", [0, 0.0, -1.0])
def test_clip_grad_norm_must_be_positive(value, stand_in, tmp_path):
    from super_gradients_b200.training.sg_trainer import Trainer

    with pytest.raises(TypeError, match="Invalid clip_grad_norm"):
        Trainer("c", ckpt_root_dir=str(tmp_path)).train(_tiny_model(stand_in), {"clip_grad_norm": value, "loss": "ppyoloeloss"}, _batches(stand_in, 1))


def test_options_off_launch_nothing_new(stand_in, tmp_path, monkeypatch):
    """Unset, the three options add no call: no clip, no precise_bn pass."""
    from super_gradients_b200 import kernels as K
    from super_gradients_b200.training.losses import PPYoloELoss
    from super_gradients_b200.training.sg_trainer import Trainer

    def refuse(*a, **k):
        raise AssertionError("called with the options unset")

    monkeypatch.setattr(K, "clip_grad_norm", refuse)
    monkeypatch.setattr(Trainer, "_precise_bn", refuse)
    tp = {"max_epochs": 1, "initial_lr": 1e-3, "lr_mode": "constant", "loss": PPYoloELoss(num_classes=4, use_static_assigner=False), "save_model": False}
    hist = Trainer("off", ckpt_root_dir=str(tmp_path)).train(_tiny_model(stand_in), tp, _batches(stand_in, 2))
    assert math.isfinite(hist["train_loss"][0])


def test_clip_reaches_the_update(stand_in, tmp_path):
    """With SGD, lr 1 and no momentum or decay, the update of a clipped step is the gradient times the coefficient."""
    from super_gradients_b200.training.losses import PPYoloELoss
    from super_gradients_b200.training.sg_trainer import TrainStep

    x, tg = _batches(stand_in, 1)[0]
    st = TrainStep(_tiny_model(stand_in), PPYoloELoss(num_classes=4, use_static_assigner=False), "SGD", {"momentum": 0.0, "weight_decay": 0.0}, True, clip_grad_norm=1e-3)
    st.set_hyper_params(1.0, None)
    st.forward_backward(x, tg)
    g, p0 = st.flat.grads.clone(), st.flat.params.clone()
    st.optimizer_step()
    total, coef = st.clip_norm_coef.tolist()
    assert total == pytest.approx(float(g.double().norm()), rel=1e-6) and coef < 1
    torch.testing.assert_close(p0 - st.flat.params, g * coef, rtol=1e-5, atol=float(p0.abs().max()) * 2**-22)  # p - lr * update rounds at p's ulp
    assert float(st.hp[0, 3]) == coef  # grad_scale 1 times the coefficient; set_hyper_params rewrites it before the next step


def test_lamb_and_clip_share_the_flat_chunk_table(tiny_step):
    st = tiny_step("Lamb", clip_grad_norm=1.0)
    assert st.fused.chunks is st.flat.chunks and st.clip_partials.numel() == st.flat.chunks.shape[0]
    assert list(itertools.accumulate(st.flat.chunks[:, 1].tolist()))[-1] == st.flat.n_live
