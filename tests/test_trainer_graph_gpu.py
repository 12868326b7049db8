"""Trainer.train() with cuda_graph on detection and pose losses, whose host targets are padded into a pinned staging ring and copied
into the captured step's static target buffer (TrainStep.run_padded): the captured runs follow the eager ones, the losses do not
depend on n_max, a batch over n_max or of another size runs eagerly and the step is captured again at the next epoch, accumulation
mixes replays and eager micro-batches, and packed GPU-augmentation batches are written straight into the static input."""
import copy
import warnings

import numpy as np
import pytest
import torch

from super_gradients_b200.training.sg_trainer import Trainer, TrainStep

pytestmark = pytest.mark.gpu
DEV = "cuda"


def rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-20))


class _Loader(list):
    batch_size = 4


def _tiny_yolo_nas(g):
    from super_gradients_b200.training.models.detection_models.yolo_nas import YoloNAS

    ap = copy.deepcopy(g["arch"])
    m = YoloNAS(backbone=ap["backbone"], neck=ap["neck"], heads=ap["heads"], num_classes=4, bn_eps=1e-3, bn_momentum=0.03, inplace_act=True, in_channels=3)
    m.load_state_dict({k: v.clone() for k, v in g["sd0"].items()}, strict=False)
    return m.to(DEV).train()


def _tiny_pose(g0):
    from super_gradients_b200.training.models.pose_estimation_models import YoloNASPose

    ap = copy.deepcopy(g0["arch"])
    m = YoloNASPose(backbone=ap["backbone"], neck=ap["neck"], heads=ap["heads"], num_classes=5, bn_eps=1e-3, bn_momentum=0.03, inplace_act=True, in_channels=3)
    m.load_state_dict({k: v.clone() for k, v in g0["sd0"].items()}, strict=False)
    return m.to(DEV).train()


def _det_targets(g, counts, seed):
    """[N, 6] targets with counts[b] boxes in image b: the fixture's boxes, jittered, cycled."""
    base = g["targets"]
    gen = torch.Generator().manual_seed(seed)
    rows = []
    for b, n in enumerate(counts):
        for k in range(n):
            r = base[k % base.shape[0]].clone()
            r[0] = b
            r[2:4] += torch.randn(2, generator=gen) * 4
            r[4:6] *= 1 + 0.2 * torch.rand(2, generator=gen)
            rows.append(r)
    return torch.stack(rows) if rows else torch.zeros(0, 6)


def _pose_targets(g, counts, seed):
    boxes, joints, crowd = g["targets"]
    gen = torch.Generator().manual_seed(seed)
    out = ([], [], [])
    for b, n in enumerate(counts):
        for k in range(n):
            i = k % boxes.shape[0]
            d = torch.randn(2, generator=gen) * 2
            bx, jt, cr = boxes[i].clone(), joints[i].clone(), crowd[i].clone()
            bx[0], jt[:, 0], cr[0] = b, b, b
            bx[1:3] += d
            bx[3:5] += d
            jt[:, 1:3] += d
            out[0].append(bx)
            out[1].append(jt)
            out[2].append(cr)
    return tuple(torch.stack(v) for v in out)


def _det_loader(g, counts_per_batch, n_images=None):
    return _Loader([(g["x"][: n_images or 4] * (1 + 0.05 * i), _det_targets(g, c, i)) for i, c in enumerate(counts_per_batch)])


def _train(model, tp, loader, tmp_path, name):
    tr = Trainer(name, ckpt_root_dir=str(tmp_path))
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        tr.train(model, tp, loader)
    return tr, [str(x.message) for x in w if "n_max" in str(x.message)]


def _twins(make_model, make_loss, loader, tmp_path, epochs=2, **extra):
    """The same run eagerly and under cuda_graph -> (eager trainer, graph trainer, graph-run n_max warnings)."""
    out = []
    for graph in (False, True):
        torch.manual_seed(0)
        tp = dict(max_epochs=epochs, initial_lr=1e-3, lr_mode="constant", optimizer="SGD", optimizer_params={"weight_decay": 1e-5, "momentum": 0.9}, ema=True,
                  ema_params={"decay": 0.99, "decay_type": "constant"}, loss=make_loss(), cuda_graph=graph, save_model=False, **extra)  # fmt: skip
        out.append(_train(make_model(), tp, loader, tmp_path, f"g{int(graph)}"))
    (ea, _), (gr, warned) = out
    return ea, gr, warned


def _assert_follows(ea, gr):
    """The tolerances of test_trainer_gpu.py::test_cuda_graph_replay_matches_eager."""
    for a, b in zip(ea.history["train_loss"], gr.history["train_loss"]):
        assert abs(a - b) <= 2e-2 * abs(a), (ea.history["train_loss"], gr.history["train_loss"])
    assert rel(gr.step.flat.params, ea.step.flat.params) < 1e-3
    assert rel(gr.step.ema_params, ea.step.ema_params) < 1e-3


@pytest.fixture
def captures(monkeypatch):
    n = []
    real = TrainStep._capture

    def counted(self, *a, **kw):
        n.append(None)
        return real(self, *a, **kw)

    monkeypatch.setattr(TrainStep, "_capture", counted)
    return n


@pytest.mark.parametrize("static", [False, True], ids=["tal", "atss"])
def test_detection_graph_matches_eager(golden, tmp_path, captures, static):
    from super_gradients_b200.training.losses import PPYoloELoss

    g = golden("tiny_yolo_nas")
    loader = _det_loader(g, [(3, 1, 0, 2), (1, 0, 2, 1), (0, 3, 1, 1), (2, 2, 2, 0)])
    ea, gr, warned = _twins(lambda: _tiny_yolo_nas(g), lambda: PPYoloELoss(num_classes=4, use_static_assigner=static), loader, tmp_path)
    st = gr.step
    assert st.graph is not None and st.n_max == 3 and len(captures) == 1 and not warned
    assert st.fallbacks == 0 and st.replays == 8 - st.fallbacks
    assert ea.step.replays == 0 and ea.step.graph is None
    _assert_follows(ea, gr)


def test_pose_graph_matches_eager(golden, tmp_path, captures):
    from super_gradients_b200.training.losses import YoloNASPoseLoss

    g0, g = golden("tiny_yolo_nas_pose"), golden("tiny_yolo_nas_pose_train")
    loader = _Loader([(g["x"] * (1 + 0.05 * i), _pose_targets(g, c, i)) for i, c in enumerate([(2, 1, 0, 3), (1, 3, 2, 0), (0, 1, 1, 1)])])
    # one epoch: after an update a discrete assignment flip can separate two correct runs of the tiny pose model
    ea, gr, warned = _twins(lambda: _tiny_pose(g0), lambda: YoloNASPoseLoss(oks_sigmas=g["sigmas"], **g["kw"]), loader, tmp_path, epochs=1)
    st = gr.step
    assert st.graph is not None and st.n_max == 3 and len(captures) == 1 and not warned
    assert st.fallbacks == 0 and st.replays == 3
    _assert_follows(ea, gr)


def _head_grads(loss, preds, x, targets, pad_to):
    """(loss items, gradients of the head outputs) of one batch padded to `pad_to` targets per image."""
    n_diff = 4 if len(preds) == 8 else 2  # pose: cls, reg, pose coords, pose logits; detection: cls, reg
    leaves = [p.detach().float().clone().requires_grad_(True) for p in preds[:n_diff]]
    padded = tuple(t.to(DEV) for t in loss.pad_targets(targets, x.shape[0], pad_to))
    total, items = loss((None, (*leaves, *preds[n_diff:])), padded)
    total.backward()
    return items.detach().clone(), [p.grad.clone() for p in leaves]


@pytest.mark.parametrize("task", ["tal", "atss", "pose"])
def test_losses_do_not_depend_on_n_max(golden, task):
    from super_gradients_b200.training.losses import PPYoloELoss, YoloNASPoseLoss

    if task == "pose":
        g0, g = golden("tiny_yolo_nas_pose"), golden("tiny_yolo_nas_pose_train")
        model, loss, targets = _tiny_pose(g0), YoloNASPoseLoss(oks_sigmas=g["sigmas"], **g["kw"]), _pose_targets(g, (3, 0, 1, 2), 0)
    else:
        g = golden("tiny_yolo_nas")
        model, loss, targets = _tiny_yolo_nas(g), PPYoloELoss(num_classes=4, use_static_assigner=task == "atss"), _det_targets(g, (3, 0, 1, 2), 0)
    x = g["x"].to(DEV)
    need = loss.max_targets(targets)
    assert need == 3
    with torch.no_grad():
        _, preds = model(x)
    items_a, grads_a = _head_grads(loss, preds, x, targets, need)
    items_b, grads_b = _head_grads(loss, preds, x, targets, need + 37)
    assert bool(torch.isfinite(items_a).all()) and float(items_a[-1]) > 0
    torch.testing.assert_close(items_b, items_a, rtol=1e-5, atol=1e-7)
    for a, b in zip(grads_a, grads_b):
        torch.testing.assert_close(b, a, rtol=1e-4, atol=1e-6 * float(a.abs().max()))


def test_overflow_runs_eagerly_then_regrows(golden, tmp_path, captures):
    """Epoch 1's second batch needs 5 > n_max 2: it runs eagerly with one warning, the rest of the epoch replays, and epoch 2 replays a
    graph captured again with n_max 5."""
    from super_gradients_b200.training.losses import PPYoloELoss

    g = golden("tiny_yolo_nas")
    loader = _det_loader(g, [(2, 1, 0, 1), (1, 5, 0, 2), (2, 2, 1, 0), (0, 1, 2, 1)])
    ea, gr, warned = _twins(lambda: _tiny_yolo_nas(g), lambda: PPYoloELoss(num_classes=4, use_static_assigner=False), loader, tmp_path)
    st = gr.step
    assert len(warned) == 1 and "5 targets" in warned[0] and "n_max=2" in warned[0]
    assert len(captures) == 2 and st.n_max == 5 and st.fallbacks == 1 and st.replays == 8 - 1
    _assert_follows(ea, gr)


def test_short_last_batch_runs_eagerly_without_regrowing(golden, tmp_path, captures):
    from super_gradients_b200.training.losses import PPYoloELoss

    g = golden("tiny_yolo_nas")
    loader = _Loader([(g["x"] * (1 + 0.05 * i), _det_targets(g, c, i)) for i, c in enumerate([(2, 1, 0, 1), (1, 2, 0, 2), (2, 1, 1, 0)])])
    loader.append((g["x"][:2] * 0.9, _det_targets(g, (1, 2), 7)))  # drop_last=False: two images
    ea, gr, warned = _twins(lambda: _tiny_yolo_nas(g), lambda: PPYoloELoss(num_classes=4, use_static_assigner=False), loader, tmp_path)
    st = gr.step
    assert not warned and len(captures) == 1 and st.n_max == 2 and st.fallbacks == 2 and st.replays == 8 - 2
    _assert_follows(ea, gr)


def test_accumulation_with_a_fallback_inside_the_window(golden, tmp_path, captures):
    """batch_accumulate 2 (the split graph): the first micro-batch of the second window overflows and runs eagerly, its gradients
    add up with the replayed second micro-batch's."""
    from super_gradients_b200.training.losses import PPYoloELoss

    g = golden("tiny_yolo_nas")
    loader = _det_loader(g, [(2, 1, 0, 1), (1, 2, 0, 2), (0, 4, 1, 1), (2, 1, 2, 1)])
    ea, gr, warned = _twins(lambda: _tiny_yolo_nas(g), lambda: PPYoloELoss(num_classes=4, use_static_assigner=False), loader, tmp_path, batch_accumulate=2)
    st = gr.step
    assert len(warned) == 1 and len(captures) == 2 and st.fallbacks == 1 and st.replays == 8 - 1 and st.opt_steps == ea.step.opt_steps == 4
    _assert_follows(ea, gr)


def _packed_batches():
    """One packed batch of each GPU-augmentation loader."""
    from pose_augment_cases import golden as pose_golden
    from pose_augment_cases import replay as pose_replay
    from test_detection_augment_replay import replay as det_replay
    from test_imagenet_augment_replay import GOLDEN as IN_GOLDEN
    from test_imagenet_augment_replay import replay as in_replay

    from super_gradients_b200.training.datasets.detection_augment_dataset import DetectionAugmentCollateFN
    from super_gradients_b200.training.datasets.pose_estimation_datasets.pose_augment_dataset import PoseAugmentCollateFN

    ds, items = det_replay("recipe", 0)
    det = DetectionAugmentCollateFN.for_dataset(ds)(items).pin_memory()
    ds, items = pose_replay(*sorted(pose_golden()["cases"])[0])
    pose = PoseAugmentCollateFN.for_dataset(ds)(items).pin_memory()
    _, _, imagenet = in_replay(sorted(IN_GOLDEN["cases"])[0])
    return {"detection": det, "pose": pose, "imagenet": imagenet.pin_memory()}


def test_packed_batches_write_into_out():
    from super_gradients_b200 import kernels as K
    from super_gradients_b200 import lib as L

    for name, b in _packed_batches().items():
        want = b.to_model_input(DEV)[0]
        assert tuple(want.shape) == b.input_shape, name
        out = torch.full_like(want, 3.0)  # dirty, channels_last like the static input cloned from a first batch
        got = b.to_model_input(DEV, out=out)[0]
        assert got is out and torch.equal(out, want), name
        for bad in (torch.empty(b.input_shape, dtype=torch.bfloat16, device=DEV), want.float(), K.empty_nhwc(b.input_shape[0] + 1, 16, *b.input_shape[2:], DEV)):
            with pytest.raises(L.SgbError):
                b.to_model_input(DEV, out=bad)


def test_trainer_writes_packed_batches_into_the_static_input(golden, tmp_path, monkeypatch):
    """After the capture, every step's input IS the graph's static input (the augmentation launch wrote it) and nothing copies a batch
    into it."""
    from test_detection_augment_replay import replay

    from super_gradients_b200.training.datasets.detection_augment_dataset import DetectionAugmentCollateFN
    from super_gradients_b200.training.losses import PPYoloELoss

    ds, items = replay("recipe", 0)
    collate = DetectionAugmentCollateFN.for_dataset(ds)
    loader = _Loader([collate(items[:4]).pin_memory(), collate(items[4:]).pin_memory(), collate(items[:4]).pin_memory()])
    copies = []
    real = TrainStep._copy_static

    def recording(dst, src):
        if torch.is_tensor(dst) and dst is not src:
            copies.append(tuple(dst.shape))
        return real(dst, src)

    monkeypatch.setattr(TrainStep, "_copy_static", staticmethod(recording))
    seen = []

    class Record:
        def on_train_batch_start(self, context):
            seen.append(context.inputs)

    torch.manual_seed(0)
    # max_targets_per_image above every batch's need (the fixture's batches need 4 and 5): no step falls back
    tp = dict(max_epochs=2, initial_lr=1e-3, lr_mode="constant", optimizer="SGD", loss=PPYoloELoss(num_classes=4, use_static_assigner=False, max_targets_per_image=8),
              cuda_graph=True, save_model=False, phase_callbacks=[Record()])  # fmt: skip
    tr = Trainer("static_in", ckpt_root_dir=str(tmp_path))
    tr.train(_tiny_yolo_nas(golden("tiny_yolo_nas")), tp, loader)
    st = tr.step
    assert st.graph is not None and st.n_max == 8 and st.fallbacks == 0 and st.replays == 6
    static = st.static_in[0]
    assert seen[0] is not static and all(x is static for x in seen[1:])
    assert not [c for c in copies if c == tuple(static.shape)]  # the batch is never copied into the static input
    assert np.isfinite(tr.history["train_loss"]).all()



def test_fallback_after_replays_sees_the_moved_weights(golden):
    """batch_accumulate 2: the first micro-batches of two windows overflow and run eagerly, with a full replay (which moves the
    weights on the device only) between them.  The second eager micro-batch's loss equals a fresh model's loss on the same weights."""
    from super_gradients_b200.training.losses import PPYoloELoss

    g = golden("tiny_yolo_nas")
    x = g["x"].to(DEV)
    fits, over = _det_targets(g, (2, 1, 0, 2), 0), _det_targets(g, (1, 4, 2, 0), 1)
    st = TrainStep(_tiny_yolo_nas(g), PPYoloELoss(num_classes=4, use_static_assigner=False), "SGD", {"momentum": 0.9}, zero_wd_on_bias_and_bn=True, batch_accumulate=2)
    losses = []
    for targets, do_step in ((fits, False), (fits, True), (over, False), (fits, True), (over, False)):
        st.set_hyper_params(5e-2)
        losses.append(float(st.run_padded(x, targets, do_step)[0]))
    assert st.n_max == 2 and st.fallbacks == 2 and st.replays == 3
    assert abs(losses[4] - losses[2]) > 1e-3 * abs(losses[2])  # the replay between the two fallbacks did move the weights
    torch.cuda.synchronize()
    fresh = _tiny_yolo_nas(g)
    fresh.load_state_dict({k: v.detach().clone() for k, v in st.model.state_dict().items()})
    ref = TrainStep(fresh, PPYoloELoss(num_classes=4, use_static_assigner=False), "SGD", {"momentum": 0.9}, zero_wd_on_bias_and_bn=True)
    want = float(ref.forward_backward(x, over)[0])
    assert abs(losses[4] - want) <= 1e-4 * abs(want), (losses, want)


class _PredictionRecord:
    """A train metric that records, per step, the batch size and the score sum of the predictions it is given."""

    def __init__(self):
        self.seen = []

    def reset(self):
        pass

    def update(self, preds, target):
        scores = preds[0][1]
        self.seen.append((int(scores.shape[0]), float(scores.float().sum())))

    def compute(self):
        return {"record": float(len(self.seen))}


def test_train_metrics_after_fallbacks_get_the_step_predictions(golden, tmp_path):
    """A short last batch falls back in every epoch; the replays after it still hand the train metrics their own predictions."""
    from super_gradients_b200.training.losses import PPYoloELoss

    g = golden("tiny_yolo_nas")
    loader = _Loader([(g["x"] * (1 + 0.05 * i), _det_targets(g, c, i)) for i, c in enumerate([(2, 1, 0, 1), (1, 2, 0, 2), (2, 1, 1, 0)])])
    loader.append((g["x"][:2] * 0.9, _det_targets(g, (1, 2), 7)))
    records = []
    for graph in (False, True):
        torch.manual_seed(0)
        rec = _PredictionRecord()
        tp = dict(max_epochs=2, initial_lr=1e-3, lr_mode="constant", optimizer="SGD", optimizer_params={"momentum": 0.9}, loss=PPYoloELoss(num_classes=4, use_static_assigner=False),
                  cuda_graph=graph, save_model=False, train_metrics_list=[rec])  # fmt: skip
        tr, _ = _train(_tiny_yolo_nas(g), tp, loader, tmp_path, f"m{int(graph)}")
        records.append(rec.seen)
    assert tr.step.fallbacks == 2 and tr.step.replays == 6
    eager, captured = records
    assert [n for n, _ in captured] == [n for n, _ in eager] == [4, 4, 4, 2] * 2
    for (_, a), (_, b) in zip(eager, captured):
        assert abs(a - b) <= 2e-2 * abs(a), (eager, captured)
