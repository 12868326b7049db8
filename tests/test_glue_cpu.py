"""The Python glue above kernels.py, run on the CPU through tests/cpu_backend.py (a stand-in for the kernel wrappers):
module wiring, head decoding, post-prediction callbacks and predict() of the detection and pose models against the
whole-graph oracle.  The CUDA kernels themselves are NOT exercised here (see the `-m gpu` tests)."""
import copy
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import sg_oracle as O
from oracle.yolo_nas_oracle import YoloNASOracle

import cpu_backend


def l2rel(a, b):
    a, b = a.detach().float(), b.detach().float()
    return float((a - b).norm() / b.norm().clamp_min(1e-12))


def _load(m, sd):
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not unexpected and all("rbr_reparam" in k for k in missing)
    return m.eval()


def test_yolo_nas_eval_glue_matches_oracle(golden, monkeypatch):
    from super_gradients_b200.training.models.detection_models.yolo_nas import YoloNAS

    cpu_backend.install(monkeypatch)
    g = golden("tiny_yolo_nas")
    ap = copy.deepcopy(g["arch"])
    m = YoloNAS(backbone=ap["backbone"], neck=ap["neck"], heads=ap["heads"], num_classes=4, bn_eps=1e-3, bn_momentum=0.03, inplace_act=True, in_channels=3)
    sd = {**g["sd0"], **g["running1"]}
    _load(m, sd)
    with torch.no_grad():
        (eb, es), raw = m(g["x"])
    with O.bf16_emulation():
        (ebe, ese), rawe = YoloNASOracle(g["arch"], {k: v.clone() for k, v in sd.items()}, training=False).forward(g["x"])
    assert l2rel(es, ese) < 2e-2 and l2rel(eb, ebe) < 2e-2 and l2rel(raw[1], rawe[1]) < 3e-2
    assert l2rel(es, g["eval_pred_scores"]) < 0.1 and l2rel(eb, g["eval_pred_bboxes"]) < 0.1  # the unmodified reference (fp32)
    torch.testing.assert_close(raw[3], rawe[3])  # anchor points


def test_yolo_nas_pose_eval_predict_glue_matches_oracle(golden, monkeypatch):
    from super_gradients_b200.training.models.pose_estimation_models import YoloNASPose, YoloNASPosePostPredictionCallback

    cpu_backend.install(monkeypatch)
    g = golden("tiny_yolo_nas_pose")
    ap = copy.deepcopy(g["arch"])
    m = YoloNASPose(backbone=ap["backbone"], neck=ap["neck"], heads=ap["heads"], num_classes=5, bn_eps=1e-3, bn_momentum=0.03, inplace_act=True, in_channels=3)
    _load(m, g["sd0"])
    with torch.no_grad():
        decoded, raw = m(g["x"])
    with O.bf16_emulation():
        dec_e, raw_e = YoloNASOracle(g["arch"], {k: v.clone() for k, v in g["sd0"].items()}, training=False).forward(g["x"])
    for name, a, b in zip(("boxes", "scores", "pose_coords", "pose_scores"), decoded, dec_e):
        assert tuple(a.shape) == tuple(b.shape), name
        assert l2rel(a, b) < 2e-2, (name, l2rel(a, b))
    for i in (0, 1, 3):
        assert l2rel(raw[i], raw_e[i]) < 3e-2, (i, l2rel(raw[i], raw_e[i]))
    for i in (4, 5, 7):
        torch.testing.assert_close(raw[i], raw_e[i])
    assert list(raw[6]) == list(raw_e[6])
    for name, a, b in zip(("boxes", "scores", "pose_coords", "pose_scores"), decoded, g["decoded"]):  # unmodified reference, fp32
        assert l2rel(a, b) < 0.1, (name, l2rel(a, b))
    # callback + predict() on the model's own outputs == the oracle post-processing of the same tensors
    cb = YoloNASPosePostPredictionCallback(**g["cb"])
    preds = cb((decoded, raw))
    ref, _ = O.yolo_nas_pose_postprocess(*decoded, **g["cb"])
    assert sum(r[0].shape[0] for r in ref) > 0
    for pr, (rposes, rscores, rboxes) in zip(preds, ref):
        np.testing.assert_array_equal(pr.scores.numpy(), rscores)
        np.testing.assert_array_equal(pr.bboxes_xyxy.numpy(), rboxes)
        np.testing.assert_array_equal(pr.poses.numpy(), rposes)
    out = m.predict(g["x"], conf=g["cb"]["pose_confidence_threshold"], iou=g["cb"]["nms_iou_threshold"], pre_nms_max_predictions=100, post_nms_max_predictions=20)
    assert [int(o.scores.shape[0]) for o in out] == [r[0].shape[0] for r in ref]


# ------------------------------------------------------------------------------------------------ TrainStep plumbing
def _train_step(g, monkeypatch, optimizer="SGD", **attrs):
    from super_gradients_b200.training.losses import PPYoloELoss
    from super_gradients_b200.training.models.detection_models.yolo_nas import YoloNAS
    from super_gradients_b200.training.sg_trainer import TrainStep

    ap = copy.deepcopy(g["arch"])
    m = YoloNAS(backbone=ap["backbone"], neck=ap["neck"], heads=ap["heads"], num_classes=4, bn_eps=1e-3, bn_momentum=0.03, inplace_act=True, in_channels=3)
    m.load_state_dict({k: v.clone() for k, v in g["sd0"].items()}, strict=False)
    m.train()
    params = {"weight_decay": 1e-5, "momentum": 0.9} if optimizer == "SGD" else {"weight_decay": 1e-5}
    st = TrainStep(m, PPYoloELoss(num_classes=4, use_static_assigner=False), optimizer, params, zero_wd_on_bias_and_bn=True, ema=True)
    for k, v in attrs.items():
        setattr(st, k, v)
    return m, st


def _padded_targets(g):
    from super_gradients_b200.training.losses import pad_targets_host

    return pad_targets_host(g["targets"], g["x"].shape[0], 16)


def _run(st, x, t, steps):
    out = []
    for _ in range(steps):
        st.set_hyper_params(1e-3, 0.99)
        loss, items = st.forward_backward(x, t)
        grads = st.flat.grads.clone()
        st.optimizer_step()
        st.opt_steps += 1
        out.append((float(loss), items.clone(), grads, st.flat.params.clone(), st.flat.buffers.clone(), st.ema_params.clone()))
    return out


def _same(a, b, what):
    for i, (ra, rb) in enumerate(zip(a, b)):
        assert ra[0] == rb[0], (what, i, ra[0], rb[0])
        for j in range(1, len(ra)):
            assert torch.equal(ra[j], rb[j]), (what, "step", i, "field", j, l2rel(ra[j], rb[j]))


@pytest.mark.parametrize("optimizer", ["SGD", "AdamW"])
def test_train_step_batched_plumbing_is_the_same_computation(golden, monkeypatch, optimizer):
    """With deterministic stand-in kernels the batched plumbing (step arena, batched filter refresh, deferred gradient
    layout change, foreach counters) must give BIT-IDENTICAL losses, gradients, parameters, running statistics and EMA to
    the per-layer launches: every difference here is a wiring bug (wrong work table, stale filter, lost gradient)."""
    cpu_backend.install_training(monkeypatch)
    g = golden("tiny_yolo_nas")
    x, t = g["x"], _padded_targets(g)
    ma, sa = _train_step(g, monkeypatch, optimizer, batched_plumbing=True)
    ra = _run(sa, x, t, 4)
    assert sa.arena.buf is not None and sa.arena.high > 0  # steps 2.. really ran from the arena
    table, n, _ = sa.ctx.weight_table
    assert n == sum(len(c.batch_entries()) for c in sa.ctx.caches.values()) and n > 50  # every filter of the model is in the batched refresh (a folded QARepVGG filter is two entries)
    assert all(c.key == c._key(*c.args) for c in sa.ctx.caches.values()) is False  # the optimizer step just invalidated them
    assert sa.ctx.wgrad_table is not None and sa.ctx.wgrad_table[1] > 50 and not sa.ctx.pending
    mb, sb = _train_step(g, monkeypatch, optimizer, batched_plumbing=False)
    rb = _run(sb, x, t, 4)
    _same(ra, rb, "batched vs per-layer")
    assert ra[0][0] != ra[3][0]  # the model really moved
    nbt = lambda m: {k: int(v) for k, v in m.state_dict().items() if k.endswith("num_batches_tracked")}  # noqa: E731
    assert nbt(ma) == nbt(mb) and set(nbt(ma).values()) == {4}
    # nothing is lost between the kernels' gradient slots and the flat buffer: the parameters with an all-zero gradient in
    # step 1 are exactly those of the unmodified reference (the regression branches of the two coarse levels, which have
    # no positive anchor in this fixture)
    dead = {n_ for n_, p in sa.flat.order if float(ra[0][2][slice(sa.flat.offsets[n_][0], sum(sa.flat.offsets[n_]))].abs().sum()) == 0.0}
    assert dead == {k for k, v in g["grad_sums"].items() if tuple(v) == (0.0, 0.0)} and len(dead) == 10


def test_two_interleaved_train_steps_do_not_share_state(golden, monkeypatch):
    """Two models stepped alternately in one process (each with its own TrainStep) reproduce, bit for bit, the same models
    stepped alone: no module-level cache, arena or work table leaks from one step object into another."""
    cpu_backend.install_training(monkeypatch)
    g = golden("tiny_yolo_nas")
    x, t = g["x"], _padded_targets(g)
    _, alone = _train_step(g, monkeypatch)
    ref = _run(alone, x, t, 3)
    (_, s1), (_, s2) = _train_step(g, monkeypatch), _train_step(g, monkeypatch)
    r1, r2 = [], []
    for _ in range(3):
        r1 += _run(s1, x, t, 1)
        r2 += _run(s2, x, t, 1)
    _same(r1, ref, "interleaved model 1 vs alone")
    _same(r2, ref, "interleaved model 2 vs alone")


def test_train_step_stand_in_tracks_the_whole_graph_oracle(golden, monkeypatch):
    """Sanity of the stand-in itself: its first-step loss and loss items agree with the bf16-emulating oracle's train step
    within the fixture's documented sensitivity, so the plumbing tests above run a meaningful computation."""
    from oracle.yolo_nas_oracle import train_step

    cpu_backend.install_training(monkeypatch)
    g = golden("tiny_yolo_nas")
    _, st = _train_step(g, monkeypatch, batched_plumbing=False)
    st.set_hyper_params(1e-3, 0.99)
    loss, items = st.forward_backward(g["x"], _padded_targets(g))
    live = [n for n, _ in st.flat.order]
    with O.bf16_emulation():
        loss_e, items_e, grads_e = train_step(g["arch"], {k: v.clone() for k, v in g["sd0"].items()}, g["x"], g["targets"], 4, live)
    assert abs(float(loss) - float(loss_e)) < 3e-2 * abs(float(loss_e)), (float(loss), float(loss_e))
    assert l2rel(items, items_e) < 5e-2
    # and against the unmodified reference (fp32): loss, and the gradients of the layers next to the loss (deeper layers are
    # dominated by the fixture's bf16 sensitivity, see test_bf16_emulation_sensitivity)
    assert abs(float(loss) - float(g["loss"])) < 5e-2 * abs(float(g["loss"]))
    for k in ("heads.head1.cls_pred.bias", "heads.head1.reg_pred.bias", "heads.head1.cls_pred.weight"):
        assert l2rel(st.flat.grad_of(k), g["grads"][k].reshape(-1)) < 0.15, (k, l2rel(st.flat.grad_of(k), g["grads"][k].reshape(-1)))


_DP_SCRIPT = r"""
import copy, os, sys, torch, torch.distributed as dist
root = sys.argv[1]
sys.path[:0] = [root, os.path.join(root, "tests")]
from _pytest.monkeypatch import MonkeyPatch
import cpu_backend
from super_gradients_b200.training.losses import PPYoloELoss, pad_targets_host
from super_gradients_b200.training.models.detection_models.yolo_nas import YoloNAS
from super_gradients_b200.training.sg_trainer import TrainStep

dist.init_process_group("gloo", init_method="env://")
rank, world = dist.get_rank(), dist.get_world_size()
mp = MonkeyPatch()
cpu_backend.install_training(mp)
g = torch.load(os.path.join(root, "tests", "golden", "tiny_yolo_nas.pt"), weights_only=False)
ap = copy.deepcopy(g["arch"])
m = YoloNAS(backbone=ap["backbone"], neck=ap["neck"], heads=ap["heads"], num_classes=4, bn_eps=1e-3, bn_momentum=0.03, inplace_act=True, in_channels=3)
m.load_state_dict({k: v.clone() for k, v in g["sd0"].items()}, strict=False)
m.train()
crit = PPYoloELoss(num_classes=4, use_static_assigner=False, sync_normaliser=(sys.argv[2] == "sync"))
st = TrainStep(m, crit, "SGD", {"weight_decay": 1e-5, "momentum": 0.9}, zero_wd_on_bias_and_bn=True, ema=True)
assert st.world == world == 2
x = g["x"] if rank == 0 else torch.flip(g["x"], dims=[0]) * 0.9      # each rank its own shard of the global batch
tg = g["targets"].clone()
if rank == 1:
    tg[:, 0] = (g["x"].shape[0] - 1) - tg[:, 0]
t = pad_targets_host(tg, x.shape[0], 16)
lr, wd = 1e-2, 1e-5
for step in range(3):
    p0, mom0 = st.flat.params.clone(), st.state[0].clone()
    st.set_hyper_params(lr, 0.99)
    loss, _ = st.forward_backward(x, t)
    local = st.flat.grads.clone()
    both = [torch.zeros_like(local) for _ in range(world)]
    dist.all_gather(both, local)
    assert not torch.equal(both[0], both[1]), "the two ranks must see different data"
    st.optimizer_step()            # ONE flat all-reduce (SUM), the 1/world average rides in the optimizer's grad_scale
    st.opt_steps += 1
    mean = (both[0] + both[1]) / world
    nd = st.flat.n_decay
    gg = mean.clone()
    gg[:nd] += wd * p0[:nd]
    mom = 0.9 * mom0 + gg
    torch.testing.assert_close(st.flat.params, p0 - lr * mom, rtol=1e-6, atol=1e-8)
    mine = [torch.zeros_like(st.flat.params) for _ in range(world)]
    dist.all_gather(mine, st.flat.params)
    assert torch.equal(mine[0], mine[1]), "replicas diverged"
    ema = [torch.zeros_like(st.ema_params) for _ in range(world)]
    dist.all_gather(ema, st.ema_params)
    assert torch.equal(ema[0], ema[1])
print("rank", rank, "ok", float(loss), flush=True)
dist.barrier()
dist.destroy_process_group()  # an orderly shutdown: a rank that exits while gloo's threads are alive can abort at interpreter exit
"""


@pytest.mark.parametrize("normaliser", ["local", "sync"])
def test_data_parallel_train_step_world2_gloo(tmp_path, normaliser):
    """The N>1 path of the training step on two CPU ranks (gloo): per-rank shards, one flat SUM all-reduce of the live
    gradients, the average applied through the optimizer's grad_scale, replicas (and their EMA) bit-identical afterwards;
    `sync` also exercises the loss normaliser's all-reduce."""
    script = tmp_path / "dp.py"
    script.write_text(_DP_SCRIPT)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    port = "29533" if normaliser == "local" else "29534"
    out = subprocess.run(
        [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1", "--master-port", port, str(script), root, normaliser],
        capture_output=True, text=True, timeout=600, env=dict(os.environ, OMP_NUM_THREADS="2"),
    )  # fmt: skip
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    assert out.stdout.count("ok") == 2


def test_tiny_yolo_nas_pose_train_step_glue(golden, monkeypatch):
    """Row L7 wiring without a GPU: the product's YoloNASPose in train mode (stand-in conv / BN kernels), its differentiable
    head decode, YoloNASPoseLoss on the host-compiled kernel arithmetic, backward into every parameter -- against the
    bf16-emulating whole-graph oracle (tight) and the unmodified reference's fp32 fixture (loose)."""
    from test_oracle_golden import pose_oracle_train_step

    from super_gradients_b200.training.losses import YoloNASPoseLoss
    from super_gradients_b200.training.models.pose_estimation_models import YoloNASPose

    cpu_backend.install_training(monkeypatch)
    g0, g = golden("tiny_yolo_nas_pose"), golden("tiny_yolo_nas_pose_train")
    ap = copy.deepcopy(g0["arch"])
    m = YoloNASPose(backbone=ap["backbone"], neck=ap["neck"], heads=ap["heads"], num_classes=5, bn_eps=1e-3, bn_momentum=0.03, inplace_act=True, in_channels=3)
    missing, unexpected = m.load_state_dict({k: v.clone() for k, v in g0["sd0"].items()}, strict=False)
    assert not unexpected and all("rbr_reparam" in k for k in missing)
    m.train()
    outs = m(g["x"])
    crit = YoloNASPoseLoss(oks_sigmas=g["sigmas"], **g["kw"])
    loss, items = crit(outs, g["targets"])
    loss.backward()
    with O.bf16_emulation():
        loss_e, items_e, raw_e, pe = pose_oracle_train_step(g0["arch"], g0["sd0"], g["x"], g["targets"], g["sigmas"], g["kw"])
    raw = outs[1]
    for i, tol in ((0, 2e-2), (1, 0.13), (2, 2e-2), (3, 5e-2)):  # reg_distri: same bound as the detection fixture (bf16 sensitivity)
        assert l2rel(raw[i], raw_e[i]) < tol, (i, l2rel(raw[i], raw_e[i]))
    # the assigned scores are iou^6 * oks of a randomly initialised model: bf16 rounding of the head outputs moves them by
    # tens of percent (the bf16-emulating oracle itself is 30 % away from the fp32 reference on this fixture), so only the
    # bf16-vs-bf16 comparison is meaningful for the loss values
    assert l2rel(items, items_e) < 0.1, (items, items_e)
    assert l2rel(items, g["items"]) < 0.4, (items, g["items"])
    # every parameter the reference trains receives a gradient here, and nothing else does
    params = dict(m.named_parameters())
    zero_ref = {k for k, v in g["grad_sums"].items() if tuple(v) == (0.0, 0.0)}
    for k in g["grad_sums"]:
        assert params[k].grad is not None, k
        assert (float(params[k].grad.abs().sum()) == 0.0) == (k in zero_ref), k
    assert all(p.grad is None for k, p in params.items() if "rbr_reparam" in k)
    # the layers next to the loss against the bf16-emulating oracle's gradients
    for k in ("heads.head1.cls_pred.bias", "heads.head1.pose_pred.bias", "heads.head1.reg_pred.bias", "heads.head1.pose_pred.weight"):
        assert l2rel(params[k].grad, pe[k].grad) < 0.25, (k, l2rel(params[k].grad, pe[k].grad))
    norms = sorted(abs(float(torch.log(params[k].grad.norm() / pe[k].grad.norm()))) for k in g["grad_sums"] if k not in zero_ref and g["grad_sums"][k][1] > 1e-4)
    assert norms[len(norms) // 2] < 0.1, norms[len(norms) // 2]


def test_trainer_train_end_to_end(golden, monkeypatch, tmp_path):
    """The reference-facing entry point itself, Trainer(...).train(model, training_params, train_loader, valid_loader), on the CPU
    stand-in: LR warm-up + cosine schedule reaches the optimizer, EMA decay schedule, validation on the EMA weights with the
    raw weights restored afterwards, rank-0 checkpoints with the reference's keys that load back into a fresh model."""
    from super_gradients_b200.training import sg_trainer
    from super_gradients_b200.training.losses import PPYoloELoss
    from super_gradients_b200.training.models.detection_models.yolo_nas import YoloNAS
    from super_gradients_b200.training.sg_trainer import Trainer, cosine_lr

    cpu_backend.install_training(monkeypatch)
    monkeypatch.setattr(sg_trainer, "setup_device", lambda device=None: torch.device("cpu"))
    g = golden("tiny_yolo_nas")

    def build():
        ap = copy.deepcopy(g["arch"])
        m = YoloNAS(backbone=ap["backbone"], neck=ap["neck"], heads=ap["heads"], num_classes=4, bn_eps=1e-3, bn_momentum=0.03, inplace_act=True, in_channels=3)
        m.load_state_dict({k: v.clone() for k, v in g["sd0"].items()}, strict=False)
        return m

    gen = torch.Generator().manual_seed(0)
    loader = [(g["x"] + 0.05 * i * torch.randn(g["x"].shape, generator=gen), g["targets"]) for i in range(3)]
    seen_lr = []
    orig = sg_trainer.TrainStep.set_hyper_params
    monkeypatch.setattr(sg_trainer.TrainStep, "set_hyper_params", lambda self, lr, d=None: (seen_lr.append((lr, d)), orig(self, lr, d))[1])
    tp = dict(max_epochs=2, initial_lr=2e-3, lr_mode="cosine", cosine_final_lr_ratio=0.1, lr_warmup_steps=2, optimizer="SGD", optimizer_params={"momentum": 0.9, "weight_decay": 1e-5},
              zero_weight_decay_on_bias_and_bn=True, ema=True, ema_params={"decay": 0.99, "decay_type": "threshold"}, loss=PPYoloELoss(num_classes=4, use_static_assigner=False),
              save_model=True, save_ckpt_epoch_list=[1])  # fmt: skip
    model = build()
    trainer = Trainer("glue", ckpt_root_dir=str(tmp_path))
    hist = trainer.train(model, tp, loader, valid_loader=loader[:1])
    assert len(hist["train_loss"]) == 2 and len(hist["valid_loss"]) == 2 and len(hist["lr"]) == 6
    assert all(np.isfinite(v) for v in hist["train_loss"] + hist["valid_loss"])
    # the schedule the reference's callbacks would leave in the optimizer (tests/test_host_logic.py pins lr_schedule against
    # traces of those callbacks): batch warm-up linspace(lr0 / 3, lr0, 2), then the cosine value computed after each step
    want = sg_trainer.lr_schedule({**sg_trainer.DEFAULT_TRAINING_PARAMS, **tp}, 3)
    np.testing.assert_allclose([lr for lr, _ in seen_lr], want, rtol=1e-12)
    np.testing.assert_allclose(want[:3], [2e-3 / 3, 2e-3, cosine_lr(0, 4, 2e-3, 0.1)], rtol=1e-12)
    assert want[-1] < 0.75 * 2e-3 and want[1:] == sorted(want[1:], reverse=True)  # decreasing after the warm-up
    np.testing.assert_allclose([d for _, d in seen_lr], [min(0.99, (1 + t) / (10 + t)) for t in range(1, 7)], rtol=1e-12)
    assert trainer.step.opt_steps == 6 and not np.allclose(hist["train_loss"][0], hist["train_loss"][1])
    ck = torch.load(tmp_path / "glue" / "ckpt_latest.pth", weights_only=False)
    assert {"net", "acc", "epoch", "metrics", "optimizer_state_dict", "scaler_state_dict", "processing_params", "ema_net"} <= set(ck) and ck["epoch"] == 1
    assert (tmp_path / "glue" / "ckpt_best.pth").exists() and (tmp_path / "glue" / "ckpt_epoch_1.pth").exists()
    assert list(ck["net"].keys()) == g["state_keys"] == list(ck["ema_net"].keys())
    # the live model holds the RAW weights again after validation; the checkpoint's ema_net differs from them
    torch.testing.assert_close(ck["net"]["heads.head1.cls_pred.weight"], model.state_dict()["heads.head1.cls_pred.weight"])
    assert not torch.equal(ck["net"]["heads.head1.cls_pred.weight"], ck["ema_net"]["heads.head1.cls_pred.weight"])
    fresh = build()
    fresh.load_state_dict(ck["ema_net"])  # strict
    fresh.eval()
    model.eval()
    trainer.step.swap_ema()
    with torch.no_grad():
        (b1, s1), _ = fresh(g["x"])
        (b2, s2), _ = model(g["x"])
    assert torch.equal(s1, s2) and torch.equal(b1, b2)  # checkpoint -> fresh model reproduces the EMA model bit for bit


def test_trainer_train_pose_model(golden, monkeypatch, tmp_path):
    """Trainer.train() with YoloNASPose + YoloNASPoseLoss built through the losses registry (flat (boxes, joints, crowd)
    targets stay on the host and are padded per step): two optimisation steps change the weights, losses stay finite."""
    from super_gradients_b200.training import sg_trainer
    from super_gradients_b200.training.models.pose_estimation_models import YoloNASPose
    from super_gradients_b200.training.sg_trainer import Trainer

    cpu_backend.install_training(monkeypatch)
    monkeypatch.setattr(sg_trainer, "setup_device", lambda device=None: torch.device("cpu"))
    g0, g = golden("tiny_yolo_nas_pose"), golden("tiny_yolo_nas_pose_train")
    ap = copy.deepcopy(g0["arch"])
    m = YoloNASPose(backbone=ap["backbone"], neck=ap["neck"], heads=ap["heads"], num_classes=5, bn_eps=1e-3, bn_momentum=0.03, inplace_act=True, in_channels=3)
    m.load_state_dict({k: v.clone() for k, v in g0["sd0"].items()}, strict=False)
    before = m.heads.head1.pose_pred.weight.detach().clone()
    # `yolo_nas_pose_loss` is how the shipped coco2017_yolo_nas_pose_train_params.yaml names the loss (fuzzy registry match)
    tp = dict(max_epochs=1, initial_lr=1e-3, lr_mode="constant", optimizer="AdamW", optimizer_params={"weight_decay": 1e-5}, zero_weight_decay_on_bias_and_bn=True, ema=False,
              loss="yolo_nas_pose_loss", criterion_params=dict(oks_sigmas=g["sigmas"], **g["kw"]), save_model=False)  # fmt: skip
    hist = Trainer("pose", ckpt_root_dir=str(tmp_path)).train(m, tp, [(g["x"], g["targets"]), (g["x"] * 0.9, g["targets"])])
    assert len(hist["train_loss"]) == 1 and np.isfinite(hist["train_loss"][0]) and hist["train_loss"][0] > 0
    assert not torch.equal(before, m.heads.head1.pose_pred.weight.detach())


def test_yolo_nas_predict_glue(golden, monkeypatch):
    """model.predict() of the detection mirror (eval switch, batching, PPYoloEPostPredictionCallback defaults and overrides) ==
    the oracle post-processing of the model's own decoded outputs."""
    from super_gradients_b200.training.models.detection_models.yolo_nas import YoloNAS

    cpu_backend.install(monkeypatch)
    g = golden("tiny_yolo_nas")
    ap = copy.deepcopy(g["arch"])
    m = YoloNAS(backbone=ap["backbone"], neck=ap["neck"], heads=ap["heads"], num_classes=4, bn_eps=1e-3, bn_momentum=0.03, inplace_act=True, in_channels=3)
    _load(m, {**g["sd0"], **g["running1"]})
    m.train()
    with torch.no_grad():
        m.eval()
        (boxes, scores), _ = m(g["x"])
        m.train()
    for kw in (dict(conf=0.008, iou=0.6), dict(conf=0.008, iou=0.5, multi_label_per_box=False, class_agnostic_nms=True, max_predictions=7)):
        out = m.predict(g["x"], batch_size=3, **kw)  # 4 images in batches of 3 + 1
        assert m.training  # predict() restores the mode
        ref, _ = O.ppyoloe_postprocess(boxes, scores, kw["conf"], kw["iou"], 1024, kw.get("max_predictions", 300), multi_label_per_box=kw.get("multi_label_per_box", True),
                                       class_agnostic_nms=kw.get("class_agnostic_nms", False))  # fmt: skip
        assert len(out) == 4 and sum(r.shape[0] for r in ref) > 0
        for mine, r in zip(out, ref):
            np.testing.assert_array_equal(mine.numpy(), r)


def test_trainer_train_resnet18_cifar_follows_the_reference_trajectory(golden, monkeypatch, tmp_path):
    """config[0] (the reference's own CPU-runnable case) through Trainer.train(): seeded resnet18_cifar from models.get, the
    fixture's four batches of 64, SGD(0.1, momentum 0.9, wd 1e-4 off for bias / BN) + CrossEntropyLoss from the registry.
    The per-step losses follow the unmodified reference's (bf16 activations here, fp32 there)."""
    from super_gradients_b200.training import models, sg_trainer
    from super_gradients_b200.training.losses import CrossEntropyLoss
    from super_gradients_b200.training.sg_trainer import Trainer

    cpu_backend.install_training(monkeypatch)
    monkeypatch.setattr(sg_trainer, "setup_device", lambda device=None: torch.device("cpu"))
    g = golden("resnet18_cifar_train")
    torch.manual_seed(0)
    m = models.get("resnet18_cifar", num_classes=10)
    gen = torch.Generator().manual_seed(6)
    X = torch.randn(256, 3, 32, 32, generator=gen)
    Y = torch.randint(0, 10, (256,), generator=gen)
    losses = []

    class Recording(CrossEntropyLoss):
        def forward(self, input, target):
            loss, item = super().forward(input, target)
            losses.append(float(loss.detach()))
            return loss, item

    tp = dict(max_epochs=1, initial_lr=0.1, lr_mode="constant", optimizer="SGD", optimizer_params={"momentum": 0.9, "weight_decay": 1e-4}, zero_weight_decay_on_bias_and_bn=True,
              loss=Recording(), save_model=False)  # fmt: skip
    Trainer("cifar", ckpt_root_dir=str(tmp_path)).train(m, tp, [(X[i * 64 : (i + 1) * 64], Y[i * 64 : (i + 1) * 64]) for i in range(4)])
    ref = [float(v) for v in g["losses"][:4]]
    assert len(losses) == 4
    assert abs(losses[0] - ref[0]) < 2e-2 * ref[0], (losses, ref)
    for mine, r in zip(losses[1:], ref[1:]):
        assert abs(mine - r) < 0.12 * r, (losses, ref)


@pytest.mark.parametrize("case", ["multi_conf", "multi_raw", "single", "agnostic", "one_empty_image", "nothing_passes"])
def test_yolox_non_max_suppression_glue(golden, monkeypatch, case):
    """Row N3 wiring (objectness filter folded into the scores, cxcywh -> xyxy, thresholds, None for empty images, the
    callback's truncation) on the stand-in NMS == the unmodified reference's rows."""
    from super_gradients_b200.lib import SgbError
    from super_gradients_b200.training.models.detection_models.yolo_base import YoloXPostPredictionCallback
    from super_gradients_b200.training.utils.detection_utils import non_max_suppression

    cpu_backend.install(monkeypatch)
    g = golden("yolox_nms")[case]
    res = non_max_suppression(g["pred"].clone(), **g["kw"])
    kw = g["kw"]
    cb = YoloXPostPredictionCallback(conf=kw["conf_thres"], iou=kw["iou_thres"], max_predictions=15, with_confidence=kw["with_confidence"], class_agnostic_nms=kw["class_agnostic_nms"],
                                     multi_label_per_box=kw["multi_label_per_box"])  # fmt: skip
    res_cb = cb((g["pred"].clone(), None))
    for mine, ref in list(zip(res, g["result"])) + list(zip(res_cb, g["callback"])):
        assert (mine is None) == (ref is None)
        if ref is not None:
            np.testing.assert_array_equal(mine.numpy(), ref.numpy())
    if case == "multi_raw":  # more candidates than the kernel's shared-memory IoU matrix holds: a loud error, not a truncation
        big = torch.cat([g["pred"]] * 8, 1)
        with pytest.raises(SgbError, match="candidates"):
            non_max_suppression(big, **{**kw, "conf_thres": 0.2})


def test_ppyoloe_loss_is_agnostic_to_the_head_output_form(golden, monkeypatch):
    """Row L0b: PPYOLOEHead's train mode returns the raw 6-tuple alone, NDFLHeads / eval mode return (decoded, raw); the loss
    accepts both (ppyolo_loss.py:959-964) and gives the same value and gradients."""
    from super_gradients_b200.training.losses import PPYoloELoss

    cpu_backend.install_training(monkeypatch)
    g = golden("tiny_yolo_nas")
    anchors, anchor_points, nums, strides = O.anchors_for_levels([(16, 16), (8, 8), (4, 4)], (8, 16, 32))
    res = []
    for wrap in (False, True):
        cl, rd = g["train_cls_logits"].clone().requires_grad_(True), g["train_reg_distri"].clone().requires_grad_(True)
        raw = (cl, rd, anchors, anchor_points, nums, strides)
        loss, items = PPYoloELoss(num_classes=4, use_static_assigner=False)(((g["train_pred_bboxes"], g["train_pred_scores"]), raw) if wrap else raw, g["targets"])
        loss.backward()
        res.append((loss.detach(), items, cl.grad, rd.grad))
    for a, b in zip(*res):
        assert torch.equal(a, b)
    torch.testing.assert_close(res[0][1], g["items"], rtol=1e-4, atol=1e-6)  # and it is the reference's value on the reference's own logits


def test_predict_on_raw_images_matches_the_reference_pipeline_steps(golden, monkeypatch):
    """predict() on raw uint8 images of different sizes: fused pre-processing (host build of the kernel arithmetic) -> model ->
    NMS -> boxes in original-image pixels == the oracle's chain (the reference's Pipeline steps) around the same model."""
    from super_gradients_b200.training import processing as P
    from super_gradients_b200.training.models.detection_models.yolo_nas import YoloNAS

    cpu_backend.install(monkeypatch)
    g = golden("tiny_yolo_nas")
    ap = copy.deepcopy(g["arch"])
    m = YoloNAS(backbone=ap["backbone"], neck=ap["neck"], heads=ap["heads"], num_classes=4, bn_eps=1e-3, bn_momentum=0.03, inplace_act=True, in_channels=3)
    _load(m, {**g["sd0"], **g["running1"]})
    m.set_dataset_processing_params(image_processor=P.ComposeProcessing([P.DetectionLongestMaxSizeRescale((120, 120)), P.DetectionCenterPadding((128, 128), pad_value=114),
                                                                         P.StandardizeImage(255.0), P.ImagePermute((2, 0, 1))]), conf=0.008, iou=0.6)  # fmt: skip
    rng = np.random.RandomState(4)
    images = [rng.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in ((90, 150), (200, 160), (128, 128))]
    out = m.predict(images, batch_size=2)
    assert len(out) == 3
    kw = dict(rescale=(120, 120), keep_aspect=True, pad_shape=(128, 128), pad_value=114, center=True)
    pres, metas = zip(*(O.preprocess_image(im, **kw) for im in images))
    x = torch.from_numpy(np.stack(pres))
    with torch.no_grad():
        (boxes, scores), _ = m(x)
    ref, _ = O.ppyoloe_postprocess(boxes, scores, 0.008, 0.6, 1024, 300)
    assert sum(r.shape[0] for r in ref) > 0
    for mine, r, meta in zip(out, ref, metas):
        np.testing.assert_array_equal(mine.numpy(), O.postprocess_boxes(r, meta))


def test_pose_predict_on_raw_images(golden, monkeypatch):
    """YoloNASPose.predict() on raw images: BGR->RGB + aspect-preserving rescale + bottom-right padding fused on the way in, poses
    and boxes mapped back to original pixels on the way out == the oracle chain around the same model."""
    from super_gradients_b200.training import processing as P
    from super_gradients_b200.training.models.pose_estimation_models import YoloNASPose

    cpu_backend.install(monkeypatch)
    g = golden("tiny_yolo_nas_pose")
    ap = copy.deepcopy(g["arch"])
    m = YoloNASPose(backbone=ap["backbone"], neck=ap["neck"], heads=ap["heads"], num_classes=5, bn_eps=1e-3, bn_momentum=0.03, inplace_act=True, in_channels=3)
    _load(m, g["sd0"])
    m.set_dataset_processing_params(image_processor=P.ComposeProcessing([P.ReverseImageChannels(), P.KeypointsLongestMaxSizeRescale((96, 96)), P.KeypointsBottomRightPadding((96, 96), pad_value=127),
                                                                         P.StandardizeImage(255.0), P.ImagePermute((2, 0, 1))]))  # fmt: skip
    rng = np.random.RandomState(8)
    images = [rng.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in ((60, 120), (150, 100))]
    cbkw = g["cb"]
    out = m.predict(images, conf=cbkw["pose_confidence_threshold"], iou=cbkw["nms_iou_threshold"], pre_nms_max_predictions=100, post_nms_max_predictions=20)
    kw = dict(rescale=(96, 96), keep_aspect=True, pad_shape=(96, 96), pad_value=127, center=False, reverse=True)
    pres, metas = zip(*(O.preprocess_image(im, **kw) for im in images))
    with torch.no_grad():
        decoded, _ = m(torch.from_numpy(np.stack(pres)))
    ref, _ = O.yolo_nas_pose_postprocess(*decoded, **cbkw)
    assert sum(r[0].shape[0] for r in ref) > 0
    for pr, (rposes, rscores, rboxes), meta in zip(out, ref, metas):
        np.testing.assert_array_equal(pr.scores.numpy(), rscores)
        np.testing.assert_array_equal(pr.bboxes_xyxy.numpy(), O.postprocess_boxes(rboxes, meta))
        exp = rposes.copy()
        exp[..., 0] = (exp[..., 0] - meta["pad_left"]) * np.float32(1 / meta["scale_w"])
        exp[..., 1] = (exp[..., 1] - meta["pad_top"]) * np.float32(1 / meta["scale_h"])
        np.testing.assert_array_equal(pr.poses.numpy(), exp)


def test_trainer_resume_continues_bit_exactly(golden, monkeypatch, tmp_path):
    """training_params.resume: network weights, optimizer moments, step counter (LR / EMA schedules) and EMA weights come back from
    ckpt_latest.pth -- one epoch + a resumed second epoch ends exactly where two uninterrupted epochs end."""
    from super_gradients_b200.training import sg_trainer
    from super_gradients_b200.training.losses import PPYoloELoss
    from super_gradients_b200.training.models.detection_models.yolo_nas import YoloNAS
    from super_gradients_b200.training.sg_trainer import Trainer

    cpu_backend.install_training(monkeypatch)
    monkeypatch.setattr(sg_trainer, "setup_device", lambda device=None: torch.device("cpu"))
    g = golden("tiny_yolo_nas")

    def build():
        ap = copy.deepcopy(g["arch"])
        m = YoloNAS(backbone=ap["backbone"], neck=ap["neck"], heads=ap["heads"], num_classes=4, bn_eps=1e-3, bn_momentum=0.03, inplace_act=True, in_channels=3)
        m.load_state_dict({k: v.clone() for k, v in g["sd0"].items()}, strict=False)
        return m

    loader = [(g["x"] * (1 + 0.1 * i), g["targets"]) for i in range(2)]
    tp = lambda **kw: dict(max_epochs=2, initial_lr=2e-3, lr_mode="cosine", cosine_final_lr_ratio=0.1, lr_warmup_steps=1, optimizer="AdamW", optimizer_params={"weight_decay": 1e-5},  # noqa: E731
                           zero_weight_decay_on_bias_and_bn=True, ema=True, ema_params={"decay": 0.9, "decay_type": "threshold"}, loss=PPYoloELoss(num_classes=4, use_static_assigner=False), **kw)  # fmt: skip
    straight = Trainer("straight", ckpt_root_dir=str(tmp_path))
    m_ref = build()
    straight.train(m_ref, tp(), loader)
    ck_dir = tmp_path / "resumed"
    # epoch 0 of the 2-epoch recipe, interrupted by an exception raised from the loader at the start of epoch 1
    class Interrupt(Exception):
        pass

    class OneEpochLoader(list):
        passes = 0

        def __iter__(self):
            OneEpochLoader.passes += 1
            if OneEpochLoader.passes > 1:
                raise Interrupt()
            return super().__iter__()

    broken = Trainer("resumed", ckpt_root_dir=str(tmp_path))
    with pytest.raises(Interrupt):
        broken.train(build(), tp(), OneEpochLoader(loader))
    assert (ck_dir / "ckpt_latest.pth").exists()
    resumed = Trainer("resumed", ckpt_root_dir=str(tmp_path))
    m_res = build()
    hist = resumed.train(m_res, tp(resume=True), loader)
    assert len(hist["train_loss"]) == 1 and resumed.step.opt_steps == straight.step.opt_steps == 4
    assert torch.equal(resumed.step.flat.params, straight.step.flat.params)
    assert torch.equal(resumed.step.ema_params, straight.step.ema_params) and torch.equal(resumed.step.flat.buffers, straight.step.flat.buffers)
    for a, b in zip(resumed.step.state, straight.step.state):
        assert torch.equal(a, b)
    with pytest.raises(ValueError, match="optimizer"):
        Trainer("resumed", ckpt_root_dir=str(tmp_path)).train(build(), {**tp(resume=True), "optimizer": "SGD", "optimizer_params": {}}, loader)


def test_folded_qarepvgg_path_is_the_same_block(golden, monkeypatch):
    """SGB_QAREP_FOLD experiment (the 1x1 branch as the centre tap of one 2K-channel 3x3 convolution): forward output, input
    gradient and every parameter gradient of a QARepVGG block agree with the two-convolution path, for a block with and without
    the identity / alpha, and a whole TrainStep of the tiny model stays on the unfolded trajectory."""
    from super_gradients_b200 import functional as SF
    from super_gradients_b200.modules import QARepVGGBlock

    cpu_backend.install_training(monkeypatch)

    def run(fold, cin, cout, use_alpha, seed=0):
        monkeypatch.setattr(SF, "QAREP_FOLD", [fold])
        torch.manual_seed(seed)
        blk = QARepVGGBlock(cin, cout, stride=1, use_alpha=use_alpha, use_residual_connection=cin == cout).train()
        with torch.no_grad():
            for p in blk.parameters():
                p.add_(0.05 * torch.randn_like(p))
        x = torch.randn(2, cin, 12, 12).bfloat16().contiguous(memory_format=torch.channels_last).requires_grad_(True)
        y = blk(x)
        (y.float() * torch.linspace(-1, 1, y.numel()).reshape(y.shape)).sum().backward()
        return y.detach().float(), x.grad.float(), {k: p.grad.clone() for k, p in blk.named_parameters() if p.grad is not None}

    for cin, cout, use_alpha in ((32, 32, True), (48, 48, False), (64, 32, True)):
        y0, dx0, g0 = run(False, cin, cout, use_alpha)
        y1, dx1, g1 = run(True, cin, cout, use_alpha)
        assert l2rel(y1, y0) < 4e-3 and l2rel(dx1, dx0) < 8e-3, (cin, cout, l2rel(y1, y0), l2rel(dx1, dx0))  # bf16 rounding of two GEMM orders
        assert set(g0) == set(g1)
        for k in g0:
            assert l2rel(g1[k], g0[k]) < 2e-2, (cin, cout, k, l2rel(g1[k], g0[k]))
    # a channel count without halo-kernel variants keeps the two-convolution path even with the switch on
    monkeypatch.setattr(SF, "QAREP_FOLD", [True])
    assert not SF.qarep_fold_supported(40, 40, 40, 1) and not SF.qarep_fold_supported(32, 32, 32, 2) and SF.qarep_fold_supported(96, 96, 96, 1)
    g = golden("tiny_yolo_nas")
    x, t = g["x"], _padded_targets(g)
    res = {}
    for fold in (False, True):
        monkeypatch.setattr(SF, "QAREP_FOLD", [fold])
        _, st = _train_step(g, monkeypatch)
        res[fold] = _run(st, x, t, 2)
    assert abs(res[True][0][0] - res[False][0][0]) < 2e-2 * abs(res[False][0][0])
    assert l2rel(res[True][1][3], res[False][1][3]) < 1e-3  # parameters after two steps


def test_patch_stem_is_the_same_block(golden, monkeypatch):
    """functional._QARepVGGStem (the stem as one 1 x 1 GEMM over gathered patches, both branches in one launch) against the
    two-convolution path of the same block: output, every parameter gradient, running statistics; then a whole TrainStep of the tiny
    model with and without it.  (GPU twin: tests/test_modules_gpu.py::test_patch_stem_matches_the_two_convolution_path.)"""
    from super_gradients_b200 import functional as SF
    from super_gradients_b200.modules import QARepVGGBlock

    cpu_backend.install_training(monkeypatch)

    def run(patches, seed=0):
        monkeypatch.setattr(SF, "STEM_PATCHES", [patches])
        torch.manual_seed(seed)
        blk = QARepVGGBlock(3, 16, stride=2, use_residual_connection=False).train()
        with torch.no_grad():
            for p in blk.parameters():
                p.add_(0.05 * torch.randn_like(p))
        x = torch.randn(2, 3, 22, 26).bfloat16().float()
        assert SF.stem_patches_supported(blk, x) == patches
        y = blk(x)
        (y.float() * torch.linspace(-1, 1, y.numel()).reshape(y.shape)).sum().backward()
        return y.detach().float(), {k: p.grad.clone() for k, p in blk.named_parameters() if p.grad is not None}, {k: v.clone() for k, v in blk.state_dict().items() if "running" in k}

    y0, g0, r0 = run(False)
    y1, g1, r1 = run(True)
    assert y0.shape == y1.shape == (2, 16, 11, 13) and l2rel(y1, y0) < 4e-3, l2rel(y1, y0)
    assert set(g0) == set(g1)
    for k in g0:
        assert l2rel(g1[k], g0[k]) < 2e-2 or float(g0[k].abs().max()) < 1e-4, (k, l2rel(g1[k], g0[k]))
    for k in r0:
        assert l2rel(r1[k], r0[k]) < 1e-3, k
    g = golden("tiny_yolo_nas")
    x, t = g["x"], _padded_targets(g)
    res = {}
    for patches in (False, True):
        monkeypatch.setattr(SF, "STEM_PATCHES", [patches])
        _, st = _train_step(g, monkeypatch)
        res[patches] = _run(st, x, t, 2)
    assert abs(res[True][0][0] - res[False][0][0]) < 2e-2 * abs(res[False][0][0])
    assert l2rel(res[True][1][3], res[False][1][3]) < 1e-3  # parameters after two steps


def test_resnet_blocks_with_drop_path_glue(golden, monkeypatch):
    """Drop-path wiring above the C ABI (the GPU twin is tests/test_modules_gpu.py::test_resnet_blocks_with_drop_path): the blocks
    hand the per-image scale to the fused bn + add + relu call and its backward; against the unmodified reference's fixture."""
    from super_gradients_b200.training.models.classification_models.resnet import BasicResNetBlock, Bottleneck

    cpu_backend.install_training(monkeypatch)
    G = golden("droppath")
    for name, mod in (("bottleneck_s2", Bottleneck(16, 8, stride=2, expansion=4, droppath_prob=0.4)), ("bottleneck_id", Bottleneck(32, 8, stride=1, expansion=4, droppath_prob=0.4)),
                      ("basic_s2", BasicResNetBlock(16, 24, stride=2, droppath_prob=0.5))):  # fmt: skip
        g = G[name]
        mod.load_state_dict(g["sd0"])
        mod.train()
        mod.drop_path.sample_scale = lambda x, g=g, mod=mod: g["scale"] if mod.training else None
        x = g["x"].bfloat16().contiguous(memory_format=torch.channels_last).requires_grad_(True)
        y = mod(x)
        y.backward(g["gy"].bfloat16())
        # tight: the oracle with the same rounding points; loose: the reference's fp32 fixture (as tests/test_modules_gpu.py::_run_block)
        fn, args = {"bottleneck_s2": (O.resnet_bottleneck, (2, True)), "bottleneck_id": (O.resnet_bottleneck, (1, False)), "basic_s2": (O.resnet_basic_block, (2, True))}[name]
        with O.bf16_emulation():
            pe = {k: v.clone() for k, v in g["sd0"].items()}
            for k in g["grads"]:
                pe[k].requires_grad_(True)
            xe = g["x"].clone().requires_grad_(True)
            ye = fn(O.q(xe), pe, "", args[0], args[1], True, sample_scale=g["scale"])
            ye.backward(g["gy"].bfloat16().float())
        assert l2rel(y, ye) < 5e-3 and l2rel(x.grad, xe.grad) < 2e-2, (name, l2rel(y, ye), l2rel(x.grad, xe.grad))
        for k in g["grads"]:
            assert l2rel(dict(mod.named_parameters())[k].grad, pe[k].grad) < 3e-2, (name, k)
        assert l2rel(y, g["y"]) < 1.5e-2 and l2rel(x.grad, g["gx"]) < 0.2, (name, l2rel(y, g["y"]), l2rel(x.grad, g["gx"]))
        assert int((g["scale"] == 0).sum()) > 0
        mod.eval()
        with torch.no_grad():
            assert l2rel(mod(x.detach()), g["y_eval"]) < 2e-2  # eval: no drop-path
    # the default stays exactly the plain block
    assert Bottleneck(16, 8).drop_path.sample_scale(torch.zeros(2, 1)) is None


@pytest.mark.parametrize("name,shape", [("resnet50", (2, 3, 64, 64)), ("resnet18", (2, 3, 64, 64))])
def test_resnet_imagenet_variants_wire_up(monkeypatch, name, shape):
    """configs[3] family (Bottleneck / BasicBlock ImageNet ResNets) through models.get(): forward + backward run on the stand-in,
    logits have the right shape, every parameter receives a finite gradient, eval mode is deterministic."""
    from super_gradients_b200.training import models

    cpu_backend.install_training(monkeypatch)
    torch.manual_seed(0)
    m = models.get(name, num_classes=7).train()
    x = torch.randn(*shape)
    logits = m(x)
    assert tuple(logits.shape) == (shape[0], 7) and logits.dtype == torch.float32
    torch.nn.functional.cross_entropy(logits, torch.tensor([1, 4])).backward()
    missing = [k for k, p in m.named_parameters() if p.grad is None or not torch.isfinite(p.grad).all()]
    assert not missing, missing[:5]
    m.eval()
    with torch.no_grad():
        a, b = m(x), m(x)
    assert torch.equal(a, b)


def test_trainer_accepts_the_shipped_yolo_nas_recipe_dict(golden, monkeypatch, tmp_path):
    """The training hyper-parameters of the reference's coco2017_yolo_nas_train_params.yaml (recipes/training_hyperparams), as the
    dict hydra would hand to Trainer.train(): registry-built loss with criterion_params, LinearBatchLRWarmup + CosineLRScheduler, AdamW,
    threshold EMA, sync_bn: True (a no-op on one device), the DetectionMetrics_050_095 entry of valid_metrics_list with its
    PPYoloEPostPredictionCallback and metric_to_watch on its mAP key."""
    from super_gradients_b200.training import sg_trainer
    from super_gradients_b200.training.models.detection_models.pp_yolo_e import PPYoloEPostPredictionCallback
    from super_gradients_b200.training.models.detection_models.yolo_nas import YoloNAS
    from super_gradients_b200.training.sg_trainer import Trainer

    cpu_backend.install_training(monkeypatch)
    monkeypatch.setattr(sg_trainer, "setup_device", lambda device=None: torch.device("cpu"))
    g = golden("tiny_yolo_nas")
    ap = copy.deepcopy(g["arch"])
    m = YoloNAS(backbone=ap["backbone"], neck=ap["neck"], heads=ap["heads"], num_classes=4, bn_eps=1e-3, bn_momentum=0.03, inplace_act=True, in_channels=3)
    m.load_state_dict({k: v.clone() for k, v in g["sd0"].items()}, strict=False)
    recipe = dict(max_epochs=2, warmup_mode="LinearBatchLRWarmup", warmup_initial_lr=1e-6, lr_warmup_steps=3, lr_warmup_epochs=0, initial_lr=2e-4, lr_mode="CosineLRScheduler",
                  cosine_final_lr_ratio=0.1, zero_weight_decay_on_bias_and_bn=True, batch_accumulate=1, save_ckpt_epoch_list=[100, 200, 250], loss="PPYoloELoss",
                  criterion_params={"use_static_assigner": False, "num_classes": 4}, optimizer="AdamW", optimizer_params={"weight_decay": 0.00001}, ema=True,
                  ema_params={"decay": 0.9997, "decay_type": "threshold"}, mixed_precision=False, sync_bn=True, pre_prediction_callback=None,
                  valid_metrics_list=[{"DetectionMetrics_050_095": {"score_thres": 0.1, "top_k_predictions": 300, "num_cls": 4, "normalize_targets": True,
                                                                   "post_prediction_callback": PPYoloEPostPredictionCallback(score_threshold=0.01, nms_top_k=1000, max_predictions=300, nms_threshold=0.7)}}],
                  metric_to_watch="mAP@0.50:0.95", greater_metric_to_watch_is_better=True)  # fmt: skip
    tr = Trainer("recipe", ckpt_root_dir=str(tmp_path))
    hist = tr.train(m, recipe, [(g["x"], g["targets"])] * 2, valid_loader=[(g["x"], g["targets"])])
    assert len(hist["train_loss"]) == 2 and all(np.isfinite(hist["train_loss"])) and len(hist["valid_loss"]) == 2
    np.testing.assert_allclose(hist["lr"][:2], [1e-6, 2e-4], rtol=1e-12)  # LinearBatchLRWarmup capped at the loader length (2 steps here)
    assert max(hist["lr"]) <= 2e-4 and tr.step.opt_name == "AdamW" and tr.step.ema_on
    assert {"mAP@0.50:0.95", "Recall@0.50:0.95", "valid_loss"} <= set(tr.valid_metric_values) | {"valid_loss"}
    with pytest.raises(ValueError, match="metric_to_watch"):  # the reference raises too when the watched metric is not produced (sg_trainer.py:588-593)
        Trainer("recipe2", ckpt_root_dir=str(tmp_path)).train(m, {**recipe, "valid_metrics_list": []}, [(g["x"], g["targets"])], valid_loader=[(g["x"], g["targets"])])


def test_phase_callbacks_fire_in_the_reference_order(golden, monkeypatch, tmp_path):
    """training_params.phase_callbacks: Callback subclasses get every on_<event>, PhaseCallbacks are called at their phase; the
    order is the reference training loop's (per batch: start, [fused step], loss_end, backward_end, gradient_step_start / _end,
    batch_end), validation runs on the EMA weights between loader_start / loader_end, and a callback can stop the run."""
    from super_gradients_b200.training import sg_trainer
    from super_gradients_b200.training.losses import PPYoloELoss
    from super_gradients_b200.training.models.detection_models.yolo_nas import YoloNAS
    from super_gradients_b200.training.sg_trainer import Trainer
    from super_gradients_b200.training.utils.callbacks import Callback, Phase, PhaseCallback

    cpu_backend.install_training(monkeypatch)
    monkeypatch.setattr(sg_trainer, "setup_device", lambda device=None: torch.device("cpu"))
    g = golden("tiny_yolo_nas")
    ap = copy.deepcopy(g["arch"])
    m = YoloNAS(backbone=ap["backbone"], neck=ap["neck"], heads=ap["heads"], num_classes=4, bn_eps=1e-3, bn_momentum=0.03, inplace_act=True, in_channels=3)
    m.load_state_dict({k: v.clone() for k, v in g["sd0"].items()}, strict=False)
    events = []

    class Recorder(Callback):
        pass

    for name in [n for n in dir(Callback) if n.startswith("on_")]:
        setattr(Recorder, name, (lambda n: lambda self, ctx: events.append((n, ctx.epoch, ctx.batch_idx)))(name))

    class StopAfterFirstEpoch(PhaseCallback):
        def __init__(self):
            super().__init__(Phase.VALIDATION_EPOCH_END)

        def __call__(self, ctx):
            events.append(("PHASE_VALIDATION_EPOCH_END", ctx.epoch, float(ctx.metrics_dict["valid_loss"])))
            ctx.stop_training = True

    tp = dict(max_epochs=3, initial_lr=1e-3, lr_mode="constant", optimizer="SGD", optimizer_params={}, ema=True, ema_params={"decay": 0.9, "decay_type": "constant"},
              loss=PPYoloELoss(num_classes=4, use_static_assigner=False), save_model=False, phase_callbacks=[Recorder(), StopAfterFirstEpoch()])  # fmt: skip
    hist = Trainer("cb", ckpt_root_dir=str(tmp_path)).train(m, tp, [(g["x"], g["targets"])] * 2, valid_loader=[(g["x"], g["targets"])])
    assert len(hist["train_loss"]) == 1  # stopped after the first epoch
    names = [e[0] for e in events]
    per_batch = ["on_train_batch_start", "on_train_batch_loss_end", "on_train_batch_backward_end", "on_train_batch_gradient_step_start", "on_train_batch_gradient_step_end",
                 "on_train_batch_end"]  # fmt: skip
    assert names == (["on_training_start", "on_train_loader_start"] + per_batch * 2 + ["on_train_loader_end", "on_validation_loader_start", "on_validation_batch_start",
                     "on_validation_batch_end", "on_validation_loader_end", "PHASE_VALIDATION_EPOCH_END", "on_training_end"])  # fmt: skip
    assert [e[2] for e in events if e[0] == "on_train_batch_start"] == [0, 1] and np.isfinite(events[-2][2])


def test_trainer_validation_metrics_and_metric_to_watch(golden, monkeypatch, tmp_path):
    """valid_metrics_list / metric_to_watch / greater_metric_to_watch_is_better (row (f)-N4): the Trainer feeds each validation
    batch to DetectionMetrics (NMS callback's batched output -> matching kernel stand-in), reports compute()'s keys next to the
    loss, selects ckpt_best by the watched metric, and the numbers equal the oracle's matching + summary on the same predictions."""
    from oracle import sg_oracle as O
    from super_gradients_b200.training import sg_trainer
    from super_gradients_b200.training.losses import PPYoloELoss
    from super_gradients_b200.training.models.detection_models.pp_yolo_e.post_prediction_callback import PPYoloEPostPredictionCallback
    from super_gradients_b200.training.models.detection_models.yolo_nas import YoloNAS
    from super_gradients_b200.training.sg_trainer import Trainer

    cpu_backend.install_training(monkeypatch)
    monkeypatch.setattr(sg_trainer, "setup_device", lambda device=None: torch.device("cpu"))
    g = golden("tiny_yolo_nas")
    ap = copy.deepcopy(g["arch"])
    model = YoloNAS(backbone=ap["backbone"], neck=ap["neck"], heads=ap["heads"], num_classes=4, bn_eps=1e-3, bn_momentum=0.03, inplace_act=True, in_channels=3)
    model.load_state_dict({k: v.clone() for k, v in g["sd0"].items()}, strict=False)
    callback = PPYoloEPostPredictionCallback(score_threshold=0.01, nms_threshold=0.7, nms_top_k=200, max_predictions=50)
    loader = [(g["x"], g["targets"]), (g["x"].flip(0), g["targets"])]
    tp = dict(max_epochs=2, initial_lr=1e-3, lr_mode="constant", optimizer="SGD", loss=PPYoloELoss(num_classes=4, use_static_assigner=False), save_model=True,
              valid_metrics_list=[{"DetectionMetrics_050": {"num_cls": 4, "post_prediction_callback": callback, "normalize_targets": True, "score_thres": 0.01}}],
              metric_to_watch="map@0.50", greater_metric_to_watch_is_better=True)  # fmt: skip
    trainer = Trainer("metrics", ckpt_root_dir=str(tmp_path))
    trainer.train(model, tp, loader[:1], valid_loader=loader)
    ck = torch.load(tmp_path / "metrics" / "ckpt_latest.pth", weights_only=False)
    assert {"valid_loss", "mAP@0.50", "Precision@0.50", "Recall@0.50", "F1@0.50", "Best_score_threshold"} <= set(ck["metrics"])
    # the same predictions through the oracle
    model.eval()
    info = []
    with torch.no_grad():
        for x, t in loader:
            rows = callback(model(x))
            info += O.detection_matching([r.numpy() for r in rows], t.numpy(), x.shape[2], x.shape[3], np.array([0.5], np.float32), None, 100, False)
    assert sum(len(i[0]) for i in info) > 0
    cat = [np.concatenate(c, 0) for c in zip(*info)]
    ap_, prec, rec, f1, classes, best, _ = O.detection_metrics(*cat, score_threshold=0.01)
    m = ck["metrics"]
    assert m["mAP@0.50"] == pytest.approx(float(ap_.mean()), abs=1e-6) and m["Recall@0.50"] == pytest.approx(float(rec.mean()), abs=1e-6)
    assert m["Precision@0.50"] == pytest.approx(float(prec.mean()), abs=1e-6) and m["F1@0.50"] == pytest.approx(float(f1.mean()), abs=1e-6)
    with pytest.raises(ValueError, match="metric_to_watch"):
        sg_trainer._match_metric_name("accuracy", list(m))


def test_trainer_test_returns_loss_items_and_metrics(golden, monkeypatch, tmp_path):
    """Trainer.test(model, test_loader, loss, test_metrics_list, test_phase_callbacks) with the reference's signature: a standalone
    evaluation (no train() before it) returns the loss components under the criterion's component_names plus the metrics' keys,
    fires the test-phase events, and leaves the trainer's own state untouched; after train() it evaluates the EMA weights."""
    from super_gradients_b200.training import sg_trainer
    from super_gradients_b200.training.losses import PPYoloELoss
    from super_gradients_b200.training.metrics import DetectionMetrics_050
    from super_gradients_b200.training.models.detection_models.pp_yolo_e.post_prediction_callback import PPYoloEPostPredictionCallback
    from super_gradients_b200.training.models.detection_models.yolo_nas import YoloNAS
    from super_gradients_b200.training.sg_trainer import Trainer
    from super_gradients_b200.training.utils.callbacks import Callback

    cpu_backend.install_training(monkeypatch)
    monkeypatch.setattr(sg_trainer, "setup_device", lambda device=None: torch.device("cpu"))
    g = golden("tiny_yolo_nas")
    ap = copy.deepcopy(g["arch"])
    model = YoloNAS(backbone=ap["backbone"], neck=ap["neck"], heads=ap["heads"], num_classes=4, bn_eps=1e-3, bn_momentum=0.03, inplace_act=True, in_channels=3)
    model.load_state_dict({k: v.clone() for k, v in g["sd0"].items()}, strict=False)
    events = []

    class Rec(Callback):
        def on_test_loader_start(self, context):
            events.append("start")

        def on_test_batch_end(self, context):
            events.append(("batch", context.batch_idx, context.preds is not None))

        def on_test_loader_end(self, context):
            events.append(("end", sorted(context.metrics_dict)))

    metric = DetectionMetrics_050(num_cls=4, normalize_targets=True, score_thres=0.01, post_prediction_callback=PPYoloEPostPredictionCallback(score_threshold=0.01, nms_threshold=0.7, nms_top_k=200, max_predictions=50))
    trainer = Trainer("test_api", ckpt_root_dir=str(tmp_path))
    loader = [(g["x"], g["targets"]), (g["x"].flip(0), g["targets"])]
    res = trainer.test(model=model, test_loader=loader, loss=PPYoloELoss(num_classes=4, use_static_assigner=False), test_metrics_list=[metric], test_phase_callbacks=[Rec()], silent_mode=True)
    assert list(res)[:4] == ["loss_cls", "loss_iou", "loss_dfl", "loss"] and {"mAP@0.50", "Recall@0.50", "Best_score_threshold"} <= set(res)
    assert res["loss"] == pytest.approx(res["loss_cls"] + res["loss_iou"] + res["loss_dfl"], rel=1e-5) and np.isfinite(list(res.values())).all()
    assert events[0] == "start" and events[1:3] == [("batch", 0, True), ("batch", 1, True)] and events[3][0] == "end" and "mAP@0.50" in events[3][1]
    assert getattr(trainer, "net", None) is None and model.training  # nothing sticks to the trainer; the model is back in train mode
    with pytest.raises(ValueError):
        Trainer("no_model", ckpt_root_dir=str(tmp_path)).test(test_loader=loader)
    # after training: test() without a model evaluates the EMA weights (use_ema_net=True) or the raw ones
    tp = dict(max_epochs=1, initial_lr=5e-3, lr_mode="constant", optimizer="SGD", loss=PPYoloELoss(num_classes=4, use_static_assigner=False), ema=True,
              ema_params={"decay": 0.5, "decay_type": "constant"}, save_model=False)  # fmt: skip
    trainer.train(model, tp, loader)
    ema, raw = trainer.test(test_loader=loader[:1], silent_mode=True), trainer.test(test_loader=loader[:1], silent_mode=True, use_ema_net=False)
    assert ema["loss"] != raw["loss"] and trainer.net is model
    again = trainer.test(test_loader=loader[:1], silent_mode=True, use_ema_net=False)
    assert again["loss"] == raw["loss"]  # the EMA swap was undone


def test_k_padded_prediction_conv_is_the_same_conv(monkeypatch):
    """functional.KPAD: a 68-channel 1x1 prediction convolution run with K rounded up to 80 (zero filter rows / bias) returns the
    same output, input gradient, weight and bias gradients as the unpadded call -- both when the incoming gradient's producer
    marked its padding as zero (the head-decode backward, no copy) and when it did not (copy into a zeroed buffer)."""
    from super_gradients_b200 import functional as SF

    cpu_backend.install_training(monkeypatch)

    def run(kpad, through_decode):
        monkeypatch.setattr(SF, "KPAD", [kpad])
        torch.manual_seed(5)
        w = (0.1 * torch.randn(68, 64, 1, 1)).requires_grad_(True)
        b = (0.1 * torch.randn(68)).requires_grad_(True)
        wc = (0.1 * torch.randn(80, 64, 1, 1)).requires_grad_(True)
        bc = torch.zeros(80, requires_grad=True)
        x = torch.randn(2, 64, 8, 8).bfloat16().contiguous(memory_format=torch.channels_last).requires_grad_(True)
        cache, cache_c = SF.WeightCache(), SF.WeightCache()
        reg = SF.conv_bias(x, w, b, stride=1, pad=0, cache=cache)
        assert tuple(reg.shape) == (2, 68, 8, 8)
        if through_decode:
            cls = SF.conv_bias(x, wc, bc, stride=1, pad=0, cache=cache_c)
            _pb, _ps, cl, rd = SF.dfl_decode([reg], [cls], [8], 80, 16, 0.5)
            loss = (rd * torch.linspace(-1, 1, rd.numel()).reshape(rd.shape)).sum() + cl.sum() * 0.01
        else:
            loss = (reg.float() * torch.linspace(-1, 1, reg.numel()).reshape(reg.shape)).sum()
        loss.backward()
        return reg.detach().float().clone(), x.grad.float().clone(), w.grad.clone(), b.grad.clone()

    for through_decode in (False, True):
        y0, dx0, dw0, db0 = run(False, through_decode)
        y1, dx1, dw1, db1 = run(True, through_decode)
        assert torch.equal(y0, y1)
        assert l2rel(dx1, dx0) < 1e-6 and l2rel(dw1, dw0) < 1e-6 and l2rel(db1, db0) < 1e-6, (through_decode, l2rel(dx1, dx0), l2rel(dw1, dw0), l2rel(db1, db0))


def test_dual_conv_and_deferred_shortcut_are_the_same_csp_layer(golden, monkeypatch):
    """functional._DualConvBnAct (conv1 / conv2 of a CSP layer as one GEMM + one BatchNorm launch over adjacent parameters, the two
    incoming gradients read in place) and functional._defer_finish (a bottleneck's shortcut gradient added by ONE pass after cv1's dgrad
    instead of scale_add_dot + an ATen add): output, input gradient, every parameter gradient and the running statistics of a CSP layer
    laid out by FlatState equal the separate-layer path's; the merged path really ran; a whole train step of the tiny model stays on
    the same trajectory."""
    from super_gradients_b200 import functional as SF
    from super_gradients_b200 import kernels as Kmod
    from super_gradients_b200.modules import Conv, QARepVGGBlock
    from super_gradients_b200.training.flat_state import FlatState
    from super_gradients_b200.training.models.detection_models.yolo_nas.yolo_stages import YoloNASCSPLayer

    cpu_backend.install_training(monkeypatch)
    calls = {"fwd": 0, "bwd2": 0, "sad_acc": 0, "scale_add": 0, "qfwd_res": 0}
    bn_fwd, bn_bwd, sad, sadd, qfwd = Kmod.bn_act_fwd, Kmod.bn_act_bwd, Kmod.scale_add_dot, Kmod.scale_add, Kmod.qarep_fwd

    def count_sadd(*a, **k):
        calls["scale_add"] += 1
        return sadd(*a, **k)

    def count_qfwd(*a, **k):
        calls["qfwd_res"] += k.get("residual") is not None
        return qfwd(*a, **k)

    monkeypatch.setattr(Kmod, "scale_add", count_sadd)
    monkeypatch.setattr(Kmod, "qarep_fwd", count_qfwd)

    def count_fwd(x, *a, **k):
        calls["fwd"] += 1
        return bn_fwd(x, *a, **k)

    def count_bwd(*a, **k):
        calls["bwd2"] += k.get("dy2") is not None
        return bn_bwd(*a, **k)

    def count_sad(x1, a_dev, xd, x2=None, out=None):
        calls["sad_acc"] += x2 is not None
        return sad(x1, a_dev, xd, x2, out=out)

    monkeypatch.setattr(Kmod, "bn_act_fwd", count_fwd)
    monkeypatch.setattr(Kmod, "bn_act_bwd", count_bwd)
    monkeypatch.setattr(Kmod, "scale_add_dot", count_sad)

    def run(dual, defer):
        monkeypatch.setattr(SF, "DUAL_CONV", [dual])
        monkeypatch.setattr(SF, "DEFER_SHORTCUT", [defer])
        torch.manual_seed(3)
        net = torch.nn.Sequential(Conv(16, 32, 1, stride=1, activation_type=torch.nn.ReLU), YoloNASCSPLayer(32, 32, 2, QARepVGGBlock, torch.nn.ReLU, True, True, hidden_channels=16)).train()
        with torch.no_grad():
            for p in net.parameters():
                p.add_(0.05 * torch.randn_like(p))
        flat = FlatState(net)
        csp = net[1]
        assert SF._follows(csp.conv1.bn.weight, csp.conv2.bn.weight) and SF._follows(csp.conv1.bn.running_var, csp.conv2.bn.running_var)
        assert SF._follows(csp.conv1.bn.bias.main_grad, csp.conv2.bn.bias.main_grad)
        x = torch.randn(2, 16, 12, 12).bfloat16().contiguous(memory_format=torch.channels_last).requires_grad_(True)
        for k in calls:
            calls[k] = 0
        y = net(x)
        (y.float() * torch.linspace(-1, 1, y.numel()).reshape(y.shape)).sum().backward()
        grads = {n: flat.grad_of(n).clone() for n, _ in flat.order}
        return y.detach().float(), x.grad.float(), grads, flat.buffers.clone(), dict(calls)

    y0, dx0, g0, b0, c0 = run(False, False)
    y1, dx1, g1, b1, c1 = run(True, True)
    # separate layers: pre, conv1, conv2, conv3 = 4 BatchNorm forwards; merged: 3, one two-source backward, one in-place shortcut pass per bottleneck
    assert (c0["fwd"], c0["bwd2"], c0["sad_acc"]) == (4, 0, 0) and (c1["fwd"], c1["bwd2"], c1["sad_acc"]) == (3, 1, 2), (c0, c1)
    # the shortcut alpha * x + cv2(...) joins cv2's apply pass (bit-identical: the block's output is rounded before the add): no scale_add launch
    assert (c0["scale_add"], c0["qfwd_res"]) == (2, 0) and (c1["scale_add"], c1["qfwd_res"]) == (0, 2), (c0, c1)
    assert torch.equal(y0, y1)  # per-channel arithmetic: the merged forward is the same computation
    torch.testing.assert_close(b1, b0, rtol=1e-6, atol=1e-7)
    assert l2rel(dx1, dx0) < 8e-3, l2rel(dx1, dx0)  # one bf16 rounding of the merged dgrad's sum instead of two + an add
    scale = max(float(v.norm()) for v in g0.values())
    for k in g0:
        if float(g0[k].norm()) < 1e-4 * scale:
            assert float(g1[k].norm()) < 1e-4 * scale, k
            continue
        assert l2rel(g1[k], g0[k]) < 2e-2, (k, l2rel(g1[k], g0[k]))
    # each switch alone
    for dual, defer in ((True, False), (False, True)):
        y2, dx2, g2, _, _ = run(dual, defer)
        assert torch.equal(y2, y0) and l2rel(dx2, dx0) < 8e-3
        for k in g0:
            assert float(g0[k].norm()) < 1e-4 * scale or l2rel(g2[k], g0[k]) < 2e-2, (dual, defer, k)

    g = golden("tiny_yolo_nas")
    x, t = g["x"], _padded_targets(g)
    res = {}
    for on in (False, True):
        monkeypatch.setattr(SF, "DUAL_CONV", [on])
        monkeypatch.setattr(SF, "DEFER_SHORTCUT", [on])
        _, st = _train_step(g, monkeypatch)
        res[on] = _run(st, x, t, 2)
    assert abs(res[True][0][0] - res[False][0][0]) < 2e-2 * abs(res[False][0][0])
    assert l2rel(res[True][1][3], res[False][1][3]) < 1e-3  # parameters after two steps
