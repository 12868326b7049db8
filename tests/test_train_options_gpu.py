"""clip_grad_norm, precise_bn and batch_accumulate under cuda_graph on the sm_90a path: the clip kernels against
torch.nn.utils.clip_grad_norm_ and against the same fused step on pre-clipped gradients, resnet18_cifar trained by Trainer.train()
against the unmodified reference's run (tests/golden/train_options.pt), accumulation under a captured graph against eager steps,
tiny YOLO-NAS / YOLO-NAS-POSE runs with all three options, and the launch list with the options unset."""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"


def rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-20))


def _tiny_yolo_nas(g):
    from super_gradients_b200.training.models.detection_models.yolo_nas import YoloNAS

    ap = copy.deepcopy(g["arch"])
    m = YoloNAS(backbone=ap["backbone"], neck=ap["neck"], heads=ap["heads"], num_classes=4, bn_eps=1e-3, bn_momentum=0.03, inplace_act=True, in_channels=3)
    m.load_state_dict({k: v.clone() for k, v in g["sd0"].items()}, strict=False)
    return m.to(DEV).train()


def _step(g, name, params=None, **kw):
    from super_gradients_b200.training.losses import PPYoloELoss
    from super_gradients_b200.training.sg_trainer import TrainStep

    return TrainStep(_tiny_yolo_nas(g), PPYoloELoss(num_classes=4, use_static_assigner=False), name, params or {}, True, **kw)


def _targets(g):
    from super_gradients_b200.training.losses import pad_targets_host

    gb, gl, gv = pad_targets_host(g["targets"], g["x"].shape[0], 16)
    return gb.to(DEV), gl.to(DEV), gv.to(DEV)


@pytest.mark.parametrize("name, params", [("SGD", {"momentum": 0.9, "weight_decay": 1e-4}), ("AdamW", {}), ("Lamb", {"weight_decay": 0.01, "max_grad_norm": 0.05})])
def test_one_step_clip(name, params, golden):
    """The same fp32 gradients in the flat buffer: the coefficient within 1e-6 of torch's clip_grad_norm_ (float64 sums here,
    float32 in torch), and the parameters and optimizer state after the step bit-identical to the same fused step run on gradients
    pre-multiplied by that coefficient with grad_scale 1 (SGD: within one rounding of the gradient term).  For Lamb both clips act: its own max_grad_norm sees the clipped gradient."""
    g = golden("tiny_yolo_nas")
    a, b = _step(g, name, params, clip_grad_norm=0.3), _step(g, name, params)
    gen = torch.Generator().manual_seed(1)
    grads = (torch.randn(a.flat.n_live, generator=gen) * 0.05).to(DEV)
    a.flat.grads.copy_(grads)
    p0 = a.flat.params.clone()
    a.set_hyper_params(1e-2)
    a.optimizer_step()
    total, coef = a.clip_norm_coef.tolist()
    ps = [torch.nn.Parameter(torch.zeros(k, device=DEV)) for _, k in a.flat.offsets.values()]
    for p, (o, k) in zip(ps, a.flat.offsets.values()):
        p.grad = grads[o : o + k].clone()
    t_total = torch.nn.utils.clip_grad_norm_(ps, 0.3)
    t_coef = float(torch.clamp(0.3 / (t_total + 1e-6), max=1.0))
    assert total == pytest.approx(float(t_total), rel=1e-6) and coef == pytest.approx(t_coef, rel=1e-6) and coef < 1
    b.flat.grads.copy_(grads * torch.tensor(coef, device=DEV))
    b.set_hyper_params(1e-2)
    b.optimizer_step()
    ulp = lambda t: torch.nextafter(t.abs(), torch.full_like(t, float("inf"))) - t.abs()  # noqa: E731
    gc = grads * coef  # the scaled gradient, rounded on its own in the pre-clipped run
    gr = gc + 1e-4 * p0  # SGD's decayed gradient
    for x, y in zip((a.flat.params, *a.state), (b.flat.params, *b.state)):
        if name == "SGD":
            # sgd_kernel contracts g * grad_scale + wd * p into one FMA, so the gradient term may differ by one rounding of
            # g * coef and one of the sum; the parameter and momentum carry that (lr < 1) plus their own rounding
            bound = ulp(x) + ulp(gc) + ulp(gr)
            assert bool(((x - y).abs() <= bound).all()), (name, float(((x - y).abs() / bound).max()))
        else:
            assert torch.equal(x, y), (name, int((x != y).sum()))


def test_resnet18_cifar_matches_reference_trajectory(golden, tmp_path):
    """Trainer.train() on resnet18_cifar with clip_grad_norm, batch_accumulate 2, precise_bn and EMA against the unmodified
    reference's run: per-micro-batch losses with the tolerances of test_resnet18_cifar_training_matches_reference_trajectory (2 % on
    the first, 10 % after), every step clipped with the reference's total norm to 10 %, and the live / EMA BatchNorm statistics."""
    import importlib.util
    import os

    spec = importlib.util.spec_from_file_location("make_train_options_goldens", os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "make_train_options_goldens.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    from super_gradients_b200.training import models
    from super_gradients_b200.training.losses import CrossEntropyLoss
    from super_gradients_b200.training.sg_trainer import Trainer

    gold = golden("train_options")
    cfg = gold["config"]
    torch.manual_seed(cfg["init_seed"])
    m = models.get("resnet18_cifar", num_classes=10)
    assert {k: float(v.double().sum()) for k, v in m.state_dict().items() if v.dtype.is_floating_point} == pytest.approx(gold["init_sums"], rel=1e-6, abs=1e-6)
    losses, norms = [], []

    class Record:
        def on_train_batch_loss_end(self, context):
            losses.append(float(context.loss_log_items.reshape(-1)[0]))

        def on_train_batch_gradient_step_end(self, context):
            norms.append(float(tr.step.clip_norm_coef[0]))

    tp = dict(max_epochs=1, initial_lr=cfg["lr"], lr_mode="constant", optimizer="SGD", optimizer_params={"momentum": cfg["momentum"], "weight_decay": cfg["weight_decay"]},
              batch_accumulate=cfg["batch_accumulate"], clip_grad_norm=cfg["clip_grad_norm"], precise_bn=True, precise_bn_batch_size=cfg["precise_bn_batch_size"], ema=True,
              ema_params={"decay": cfg["ema_decay"], "decay_type": "constant"}, loss=CrossEntropyLoss(), save_model=False, phase_callbacks=[Record()])  # fmt: skip
    tr = Trainer("options", ckpt_root_dir=str(tmp_path))
    tr.train(m, tp, gen.loader(cfg))
    want = gold["losses"]
    assert abs(losses[0] - want[0]) < 2e-2 * want[0], (losses, want)
    assert all(abs(a - b) < 0.1 * b for a, b in zip(losses[1:], want[1:])), (losses, want)
    assert len(norms) == len(gold["norms"]) and all(abs(a - b) < 0.1 * b for a, b in zip(norms, gold["norms"])), (norms, gold["norms"])
    sd = m.state_dict()
    for k in gold["bn"]:
        assert rel(sd[k].cpu(), gold["bn"][k]) < 0.1, (k, rel(sd[k].cpu(), gold["bn"][k]))
    tr.step.swap_ema()
    ema_sd = m.state_dict()
    for k in gold["ema_bn"]:
        assert rel(ema_sd[k].cpu(), gold["ema_bn"][k]) < 0.1, (k, rel(ema_sd[k].cpu(), gold["ema_bn"][k]))
    tr.step.swap_ema()
    nbt = {k: int(v) for k, v in sd.items() if k.endswith("num_batches_tracked")}
    assert nbt == gold["num_batches_tracked"]


def test_accumulation_under_cuda_graph_matches_eager(golden, tmp_path):
    """batch_accumulate 2 with clip_grad_norm: two micro-batches per step, captured (forward + backward graph replayed alone inside
    the window) against eager, with the tolerances of test_cuda_graph_replay_matches_eager; then precise_bn on both twins, and one
    more step: the in-place statistics reach the graph."""
    from super_gradients_b200.training.sg_trainer import Trainer

    g = golden("tiny_yolo_nas")
    x, t = g["x"].to(DEV), _targets(g)
    sa = _step(g, "SGD", {"weight_decay": 1e-5, "momentum": 0.9}, ema=True, batch_accumulate=2, clip_grad_norm=0.5)
    sb = _step(g, "SGD", {"weight_decay": 1e-5, "momentum": 0.9}, ema=True, batch_accumulate=2, clip_grad_norm=0.5)
    sb.set_hyper_params(1e-3, 0.99)
    sb.capture(x, t, warmup=2)
    assert sa.opt_steps == sb.opt_steps == 0 and torch.equal(sa.flat.params, sb.flat.params) and torch.equal(sa.flat.buffers, sb.flat.buffers)
    assert torch.equal(sb.flat.grads, torch.zeros_like(sb.flat.grads))

    def steps(n):
        for i in range(n):
            do_step = i % 2 == 1
            xi = x * (1 + 0.05 * i)
            sa.set_hyper_params(1e-3, 0.99)
            sb.set_hyper_params(1e-3, 0.99)
            la, _ = sa.run(xi, t, do_step)
            lb, _ = sb.run(xi, t, do_step)
            assert abs(float(la) - float(lb)) <= 2e-2 * abs(float(la)), (i, float(la), float(lb))
            if not do_step:
                assert rel(sb.flat.grads, sa.flat.grads) < 0.6  # accumulated, not applied
        assert rel(sb.flat.params, sa.flat.params) < 1e-3 and rel(sb.ema_params, sa.ema_params) < 1e-3
        assert float(sb.clip_norm_coef[1]) == pytest.approx(float(sa.clip_norm_coef[1]), rel=2e-2)

    steps(4)
    assert sa.opt_steps == sb.opt_steps == 2
    for st in (sa, sb):
        tr = Trainer("acc", ckpt_root_dir=str(tmp_path))
        tr.net, tr.step, tr.criterion = st.model, st, st.criterion
        before = st.flat.buffers.clone()
        tr._precise_bn([(x, t), (x * 0.5, t)], {"precise_bn_batch_size": None})
        assert not torch.equal(before, st.flat.buffers)
    assert rel(sb.flat.buffers, sa.flat.buffers) < 1e-2
    steps(2)


def _tiny_pose(g0):
    from super_gradients_b200.training.models.pose_estimation_models import YoloNASPose

    ap = copy.deepcopy(g0["arch"])
    m = YoloNASPose(backbone=ap["backbone"], neck=ap["neck"], heads=ap["heads"], num_classes=5, bn_eps=1e-3, bn_momentum=0.03, inplace_act=True, in_channels=3)
    m.load_state_dict({k: v.clone() for k, v in g0["sd0"].items()}, strict=False)
    return m


class _Loader(list):
    batch_size = 4


@pytest.mark.parametrize("task", ["detection", "pose"])
def test_tiny_models_train_with_all_options(task, golden, tmp_path):
    from super_gradients_b200.training.losses import PPYoloELoss, YoloNASPoseLoss
    from super_gradients_b200.training.sg_trainer import Trainer

    if task == "detection":
        g = golden("tiny_yolo_nas")
        model, crit = _tiny_yolo_nas(g), PPYoloELoss(num_classes=4, use_static_assigner=False)
    else:
        g0, g = golden("tiny_yolo_nas_pose"), golden("tiny_yolo_nas_pose_train")
        model, crit = _tiny_pose(g0), YoloNASPoseLoss(oks_sigmas=g["sigmas"], **g["kw"])
    loader = _Loader([(g["x"] * (1 + 0.1 * i), g["targets"]) for i in range(4)])
    tp = dict(max_epochs=2, initial_lr=1e-3, lr_mode="constant", optimizer="AdamW", loss=crit, ema=True, batch_accumulate=2, clip_grad_norm=1.0, precise_bn=True,
              precise_bn_batch_size=8, save_model=False)  # fmt: skip
    tr = Trainer(f"all_{task}", ckpt_root_dir=str(tmp_path))
    hist = tr.train(model, tp, loader)
    assert all(torch.isfinite(torch.tensor(hist["train_loss"]))), hist
    assert torch.isfinite(tr.step.flat.buffers).all() and torch.isfinite(tr.step.ema_buffers).all()
    assert 0 < float(tr.step.clip_norm_coef[1]) <= 1


def test_options_unset_launch_the_same_kernels(golden):
    """One eager step with the options unset issues exactly the launches of the same step with clip_grad_norm set, minus the clip."""
    from super_gradients_b200 import kernels as K

    g = golden("tiny_yolo_nas")
    x, t = g["x"].to(DEV), _targets(g)
    names = []
    for clip in (None, 0.5):
        st = _step(g, "SGD", {"momentum": 0.9}, clip_grad_norm=clip)
        st.set_hyper_params(1e-3)
        st.run(x, t)  # sizes the arena and builds the work tables
        st.set_hyper_params(1e-3)
        torch.cuda.synchronize()
        K.PROFILE.clear()
        K.PROFILE_ON[0] = True
        try:
            st.run(x, t)
            torch.cuda.synchronize()
        finally:
            K.PROFILE_ON[0] = False
        names.append([n for n, *_ in K.PROFILE])
        K.PROFILE.clear()
    off, on = names
    assert "sgb_clip_grad_norm" not in off and on.count("sgb_clip_grad_norm") == 1
    i = on.index("sgb_clip_grad_norm")
    assert on[:i] + on[i + 1 :] == off and on[i + 1] == "sgb_sgd_step"
