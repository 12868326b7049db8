"""Classification without a GPU: (1) the numpy restatement of Pillow's bilinear resize == the installed Pillow, and the restated
ImageNet chain == the unmodified reference's recorded outputs; (2) the product's ComposeProcessing, Accuracy / Top5 and predict()
running on the HOST BUILD of the kernels' arithmetic (csrc/resample_math.cuh, csrc/classify_math.cuh) == the same recordings, bit
for bit; (3) metric semantics, two gloo ranks, Trainer.train() with train / valid metric lists, and C-ABI validation.  The kernels'
launches are covered by tests/test_classification_gpu.py."""
import hashlib
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

import cpu_backend
import host_classification as H
import pil_resize_oracle as R
from super_gradients_b200 import kernels as K
from super_gradients_b200 import lib as L

HERE = os.path.dirname(os.path.abspath(__file__))
needs_gxx = pytest.mark.skipif(shutil.which("g++") is None, reason="g++ not available")


def _image(case):
    h, w = case["image_shape"]
    return np.random.RandomState(case["image_seed"]).randint(0, 256, (h, w, 3)).astype(np.uint8)


def _sha(t_bf16):
    return hashlib.sha256(t_bf16.contiguous().view(torch.int16).numpy().tobytes()).hexdigest()


def _chain(kw):
    from super_gradients_b200.training import processing as P

    steps = [P.ReverseImageChannels()] if kw["reverse"] else []
    steps += [P.Resize(size=kw["resize"]), P.CenterCrop(size=kw["crop"]), P.StandardizeImage(max_value=255.0)]
    if kw["mean"] is not None:
        steps.append(P.NormalizeImage(mean=kw["mean"], std=kw["std"]))
    return P.ComposeProcessing(steps + [P.ImagePermute()])


def test_resize_restatement_matches_installed_pillow():
    Image = pytest.importorskip("PIL.Image")
    rng = np.random.RandomState(4)
    for (h, w, oh, ow) in [(375, 500, 256, 341), (480, 640, 256, 341), (100, 60, 426, 256), (1000, 1333, 256, 341), (256, 300, 256, 299), (300, 256, 299, 256),
                           (37, 41, 256, 283), (1, 5, 3, 7), (5, 1, 2, 1), (1, 1, 4, 4), (7, 9, 1, 1), (64, 48, 17, 13)]:  # fmt: skip
        img = rng.randint(0, 256, (h, w, 3)).astype(np.uint8)
        np.testing.assert_array_equal(R.resize_bilinear_u8(img, oh, ow), np.array(Image.fromarray(img).resize((ow, oh), Image.BILINEAR)), err_msg=str((h, w, oh, ow)))


@pytest.mark.parametrize("chain", ["imagenet", "small_reversed"])
def test_oracle_chain_matches_reference(golden, chain):
    g = golden("classification")["images"][chain]
    kw = g["kw"]
    for case in g["cases"]:
        t = torch.from_numpy(R.classification_chain(_image(case), kw["resize"], kw["crop"], kw["reverse"], 255.0, kw["mean"], kw["std"])).to(torch.bfloat16)
        assert tuple(t.shape) == tuple(case["pre_shape"])
        assert _sha(t) == case["pre_sha256"], case["image_shape"]


def test_default_imagenet_chain_is_the_recorded_one(golden):
    from super_gradients_b200.training import processing as P

    cp = P.default_imagenet_processing_params()["image_processor"]
    assert [type(p).__name__ for p in cp.processings] == ["Resize", "CenterCrop", "StandardizeImage", "NormalizeImage", "ImagePermute"]
    assert cp.resize.size == 256 and cp.crop.size == 224 and cp.standardize.max_value == 255.0
    np.testing.assert_array_equal(cp.normalize.mean, np.float32(golden("classification")["images"]["imagenet"]["kw"]["mean"]))


@needs_gxx
@pytest.mark.parametrize("chain", ["imagenet", "small_reversed"])
def test_product_processing_on_the_kernel_arithmetic_matches_reference(golden, monkeypatch, chain):
    """All images of a chain in ONE batch through ComposeProcessing.preprocess_crop_batch on the host build: every image's model input
    has the reference's sha256, the resized shapes are the reference's, and the padding channels are zero."""
    cpu_backend.install(monkeypatch)
    H.install(monkeypatch)
    g = golden("classification")["images"][chain]
    cp = _chain(g["kw"])
    images = [_image(c) for c in g["cases"]]
    batch = cp.preprocess_crop_batch(images, "cpu")
    assert tuple(batch.shape) == (len(images), 16) + tuple(g["cases"][0]["pre_shape"][1:]) and batch.dtype == torch.bfloat16
    assert float(batch[:, 3:].abs().max()) == 0.0
    for b, case in enumerate(g["cases"]):
        assert cp.crop_geometry(*case["image_shape"])[0] == tuple(case["resized_shape"])
        t = batch[b, :3].contiguous()
        torch.testing.assert_close(t[:, ::13, ::17].float(), case["pre_sample"].float(), rtol=0, atol=0)
        assert _sha(t) == case["pre_sha256"], case["image_shape"]


@needs_gxx
def test_kernel_arithmetic_resizes_one_axis_and_extreme_shapes_like_pillow(monkeypatch):
    """Tables the Resize step never produces (one axis resized, a 1-pixel side, an upscale without crop) straight into the host
    build: the uint8 resize equals Pillow."""
    Image = pytest.importorskip("PIL.Image")
    rng = np.random.RandomState(9)
    for (h, w, rh, rw) in [(256, 300, 256, 299), (300, 256, 299, 256), (1, 40, 7, 20), (37, 41, 256, 283), (48, 48, 48, 48)]:
        img = rng.randint(0, 256, (h, w, 3)).astype(np.uint8)
        table = torch.tensor([[0, h, w, w * 3, rh, rw, 0, 0]], dtype=torch.int64)
        out = K.empty_nhwc(1, 8, rh, rw, "cpu")
        H.resample_crop_u8(table, table, torch.from_numpy(img.reshape(-1).copy()), out, max_value=0.0)
        np.testing.assert_array_equal(out[0, :3].permute(1, 2, 0).float().numpy().astype(np.uint8), np.array(Image.fromarray(img).resize((rw, rh), Image.BILINEAR)))


@needs_gxx
@pytest.mark.parametrize("name", ["imagenet", "cifar", "five"])
def test_row_decode_arithmetic_matches_reference(golden, name):
    g = golden("classification")["logits"][name]
    n = g["logits"].shape[0]
    for target in (g["target"], g["soft"]):
        counters = torch.zeros(4, dtype=torch.int64)
        label, conf = torch.empty(n, dtype=torch.int32), torch.empty(n)
        H.classify_rows(g["logits"], target, k=5, counters=counters, label=label, confidence=conf)
        assert counters.tolist()[2:] == [n, 0]
        assert counters[0] * 100.0 / n == pytest.approx(g["top1_percent"], rel=1e-6) and counters[1] * 100.0 / n == pytest.approx(g["top5_percent"], rel=1e-6)
        assert torch.equal(label.long(), g["labels"])
        torch.testing.assert_close(conf.double(), g["confidence"], rtol=1e-6, atol=0)


@needs_gxx
def test_row_decode_ranks_ties_and_nan_like_torch():
    """Exact ties go to the lower index, NaN ranks above every number (torch.argmax and a stable descending sort)."""
    x = torch.tensor([[1.0, 3.0, 3.0, 0.5, 3.0, 2.0, 2.0], [float("nan"), 1.0, float("nan"), 9.0, 0.0, 0.0, 0.0], [0.0] * 7])
    target = torch.tensor([4, 2, 6])
    counters, label = torch.zeros(4, dtype=torch.int64), torch.empty(3, dtype=torch.int32)
    H.classify_rows(x, target, k=3, counters=counters, label=label)
    assert label.tolist() == torch.argmax(x, 1).tolist() == [1, 0, 0]
    rank = torch.sort(x, dim=1, descending=True, stable=True)[1]
    in_top3 = (rank[:, :3] == target[:, None]).any(1)
    assert in_top3.tolist() == [True, True, False]
    assert counters.tolist() == [0, 2, 3, 0]


@needs_gxx
def test_metric_classes(monkeypatch):
    from super_gradients_b200.common.factories import MetricsFactory
    from super_gradients_b200.training.metrics import Accuracy, Top5

    cpu_backend.install(monkeypatch)
    H.install(monkeypatch)
    gen = torch.Generator().manual_seed(2)
    x = torch.randn(50, 12, generator=gen)
    y = torch.randint(0, 12, (50,), generator=gen)
    acc, top5 = MetricsFactory().get("Accuracy"), MetricsFactory().get({"Top5": {"dist_sync_on_step": False}})
    assert isinstance(acc, Accuracy) and isinstance(top5, Top5) and acc.greater_is_better and top5.greater_is_better
    for m in (acc, top5):
        m.update(x[:20], y[:20])
        m.update(x[20:], torch.nn.functional.one_hot(y[20:], 12).float() * 0.8 + 0.01)  # soft labels: argmax is the target
    want1 = float((x.argmax(1) == y).double().mean())
    want5 = float((torch.sort(x, dim=1, descending=True, stable=True)[1][:, :5] == y[:, None]).any(1).double().mean())
    assert acc.compute() == pytest.approx(want1, abs=1e-12) and top5.compute() == pytest.approx(want5, abs=1e-12)
    acc.reset()
    acc.update(x[:4], y[:4])
    assert acc.compute() == pytest.approx(float((x[:4].argmax(1) == y[:4]).double().mean()))
    few = torch.randn(6, 3, generator=gen)  # fewer than five classes: Accuracy works, Top5 refuses like torch.topk(5)
    acc.reset()
    acc.update(few, torch.tensor([0, 1, 2, 0, 1, 2]))
    assert 0.0 <= acc.compute() <= 1.0
    with pytest.raises(ValueError):
        Top5().update(few, torch.zeros(6, dtype=torch.int64))
    bad = Accuracy()
    bad.update(x[:3], torch.tensor([0, 12, -1]))  # update() never inspects the values (no sync); compute() refuses
    with pytest.raises(ValueError, match="2 target"):
        bad.compute()


_DP_SCRIPT = r"""
import os, sys
root = sys.argv[1]
sys.path[:0] = [root, os.path.join(root, "tests")]
import torch
import torch.distributed as dist
from _pytest.monkeypatch import MonkeyPatch
import cpu_backend, host_classification
from super_gradients_b200.training.metrics import Accuracy, Top5

dist.init_process_group("gloo", init_method="env://")
rank = dist.get_rank()
mp = MonkeyPatch()
cpu_backend.install(mp)
host_classification.install(mp)
gen = torch.Generator().manual_seed(11)
x, y = torch.randn(40, 9, generator=gen), torch.randint(0, 9, (40,), generator=gen)
shard = slice(0, 30) if rank == 0 else slice(30, 40)   # unequal shards
acc, top5 = Accuracy(), Top5()
acc.update(x[shard], y[shard])
top5.update(x[shard], y[shard])
a, t = acc.compute(), top5.compute()
want_a = float((x.argmax(1) == y).double().mean())
want_t = float((torch.sort(x, dim=1, descending=True, stable=True)[1][:, :5] == y[:, None]).any(1).double().mean())
assert abs(a - want_a) < 1e-12 and abs(t - want_t) < 1e-12, (a, want_a, t, want_t)
print("rank", rank, "ok")
"""


@needs_gxx
def test_metrics_sum_counters_across_ranks_world2_gloo(tmp_path):
    script = tmp_path / "dp_cls_metric.py"
    script.write_text(_DP_SCRIPT)
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1", "--master-port", "29553", str(script), os.path.dirname(HERE)],
                         capture_output=True, text=True, timeout=600, env=dict(os.environ, OMP_NUM_THREADS="2"))  # fmt: skip
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    assert out.stdout.count("ok") == 2


@needs_gxx
def test_trainer_train_and_test_with_classification_metrics(monkeypatch, tmp_path):
    """The ResNet recipes' metric parameters through Trainer.train() of resnet18_cifar on the CPU stand-in: train metrics are fed
    every train batch's outputs and reported as train_<name>, the validation metrics equal a recomputation from the model's
    outputs, the checkpoint's acc is the watched validation Accuracy, and Trainer.test() reports them too."""
    from super_gradients_b200.training import models, sg_trainer
    from super_gradients_b200.training.losses import CrossEntropyLoss
    from super_gradients_b200.training.metrics import Accuracy
    from super_gradients_b200.training.sg_trainer import Trainer

    cpu_backend.install_training(monkeypatch)
    H.install(monkeypatch)
    monkeypatch.setattr(sg_trainer, "setup_device", lambda device=None: torch.device("cpu"))
    torch.manual_seed(0)
    m = models.get("resnet18_cifar", num_classes=10)
    gen = torch.Generator().manual_seed(8)
    X, Y = torch.randn(48, 3, 32, 32, generator=gen), torch.randint(0, 10, (48,), generator=gen)
    train = [(X[i : i + 16], Y[i : i + 16]) for i in range(0, 32, 16)]
    valid = [(X[32:], Y[32:])]
    seen = []
    orig = Accuracy.update
    monkeypatch.setattr(Accuracy, "update", lambda self, preds, target: (seen.append((preds.clone(), target.clone())), orig(self, preds, target))[1])
    tp = dict(max_epochs=2, initial_lr=0.05, lr_mode="constant", optimizer="SGD", loss=CrossEntropyLoss(), train_metrics_list=["Accuracy", "Top5"], valid_metrics_list=["Accuracy", "Top5"],
              metric_to_watch="Accuracy", greater_metric_to_watch_is_better=True, save_model=True)  # fmt: skip
    trainer = Trainer("cls_metrics", ckpt_root_dir=str(tmp_path))
    trainer.train(m, tp, train, valid_loader=valid)
    assert len(seen) == 2 * (2 + 1)  # two train batches and one validation batch per epoch
    ck = torch.load(tmp_path / "cls_metrics" / "ckpt_latest.pth", weights_only=False)
    met = ck["metrics"]
    assert {"train_loss", "train_Accuracy", "train_Top5", "valid_loss", "Accuracy", "Top5"} <= set(met)
    p_train = torch.cat([p for p, _ in seen[3:5]])
    assert met["train_Accuracy"] == pytest.approx(float((p_train.argmax(1) == Y[:32]).double().mean()))
    p_valid = seen[5][0]
    assert met["Accuracy"] == pytest.approx(float((p_valid.argmax(1) == Y[32:]).double().mean()))
    assert ck["acc"] == pytest.approx(max(float((seen[2][0].argmax(1) == Y[32:]).double().mean()), met["Accuracy"]))
    res = trainer.test(model=m, test_loader=valid, loss=CrossEntropyLoss(), test_metrics_list=["Accuracy", "Top5"], silent_mode=True)
    assert set(res) >= {"Accuracy", "Top5"} and 0.0 <= res["Top5"] <= 1.0


@needs_gxx
def test_predict_on_the_kernel_arithmetic(monkeypatch):
    """resnet18_cifar.predict() on raw images of several sizes (Resize(36) -> CenterCrop(32) chain) on the host builds: labels and
    confidences equal torch.max(softmax(model(batch))) on the batch the chain produced."""
    from super_gradients_b200.training import models
    from super_gradients_b200.training import processing as P

    cpu_backend.install_training(monkeypatch)  # the training subset carries the global average pool
    H.install(monkeypatch)
    torch.manual_seed(0)
    m = models.get("resnet18_cifar", num_classes=10).eval()
    with pytest.raises(RuntimeError, match="set_dataset_processing_params"):
        m.predict(np.zeros((40, 40, 3), np.uint8))
    cp = P.ComposeProcessing([P.Resize(36), P.CenterCrop(32), P.StandardizeImage(), P.NormalizeImage([0.5, 0.5, 0.5], [0.25, 0.25, 0.25]), P.ImagePermute()])
    m.set_dataset_processing_params(class_names=[f"c{i}" for i in range(10)], image_processor=cp)
    rng = np.random.RandomState(1)
    images = [rng.randint(0, 256, s).astype(np.uint8) for s in [(40, 50, 3), (36, 36, 3), (20, 30, 3), (64, 48, 3), (33, 80, 3)]]
    preds = m.predict(images, batch_size=3)
    assert len(preds) == 5 and [p.image_shape for p in preds] == [im.shape for im in images]
    with torch.no_grad():
        ref = torch.cat([torch.softmax(m(cp.preprocess_crop_batch(images[i : i + 3], "cpu")), 1) for i in (0, 3)])
    conf, lab = torch.max(ref, 1)
    assert [p.label for p in preds] == lab.tolist() and preds[0].class_name == f"c{lab[0]}"
    np.testing.assert_allclose([p.confidence for p in preds], conf.numpy(), rtol=1e-6)
    same = m.predict([im[:32, :32] for im in images[:2] if im.shape[0] >= 32 and im.shape[1] >= 32], skip_image_resizing=True)
    assert len(same) == 2


def test_processing_chain_errors():
    from super_gradients_b200.training import processing as P

    with pytest.raises(NotImplementedError):
        P.ComposeProcessing([P.CenterCrop(8), P.Resize(16)])  # wrong order
    with pytest.raises(NotImplementedError):
        P.ComposeProcessing([P.DetectionRescale((8, 8)), P.CenterCrop(8)])  # detection and classification steps mixed
    P.ComposeProcessing([P.CenterCrop(8), P.StandardizeImage()])  # CenterCrop alone is a valid chain
    cp = P.ComposeProcessing([P.Resize(16), P.CenterCrop(24)])
    with pytest.raises(ValueError):  # a crop larger than the resized image
        cp.preprocess_crop_batch([np.zeros((16, 20, 3), np.uint8)], "cpu")
    with pytest.raises(NotImplementedError):
        P.ComposeProcessing([P.Resize(16)]).preprocess_crop_batch([np.zeros((16, 20, 4), np.uint8)], "cpu")  # RGBA
    with pytest.raises(ValueError):  # without a crop the images of a batch must map to one shape
        P.ComposeProcessing([P.Resize(16)]).preprocess_crop_batch([np.zeros((16, 20, 3), np.uint8), np.zeros((16, 24, 3), np.uint8)], "cpu")


def test_abi_validation(monkeypatch):
    """sgb_resample_crop_u8 / sgb_classify_rows through the product wrappers with host tensors and directly: bad arguments raise
    SgbError in the wrapper or return SGB_E_INVALID from the entry point; a valid call gets as far as the first CUDA call (SGB_E_CUDA
    here); an empty batch is a no-op."""
    monkeypatch.setattr(K, "require_cuda", lambda t, name="tensor": None)
    monkeypatch.setattr(K, "_stream", lambda: None)
    lib = L.load()
    p = lambda t: t.data_ptr()  # noqa: E731
    # ---- resample
    src = torch.zeros(40 * 50 * 3, dtype=torch.uint8)
    out = K.empty_nhwc(1, 16, 24, 24, "cpu")

    def table(**over):
        row = dict(offset=0, h=40, w=50, pitch=150, rh=30, rw=37, top=3, left=6)
        row.update(over)
        return torch.tensor([list(row.values())], dtype=torch.int64)

    def rs(t, **kw):
        a = dict(src=src, batch=1, channels=3, out_h=24, out_w=24, pitch=16, mean=None, std=None, out=out)
        a.update(kw)
        return lib.sgb_resample_crop_u8(p(t), p(t), p(a["src"]) if a["src"] is not None else None, 6000, a["batch"], a["channels"], a["out_h"], a["out_w"], a["pitch"], 0, 255.0,
                                        a["mean"], a["std"], p(a["out"]) if a["out"] is not None else None, None)  # fmt: skip

    assert rs(table()) == -3
    assert rs(table(), batch=0, out=None) == 0
    assert rs(table(), src=None) == -1 and rs(table(), out=None) == -1
    assert rs(table(), channels=4) == -1 and rs(table(), channels=1) == -1
    assert rs(table(), pitch=2) == -1 and rs(table(), pitch=12) == -1
    assert rs(table(top=7)) == -1 and rs(table(left=-1)) == -1 and rs(table(rw=29)) == -1
    assert b"crop window" in lib.sgb_last_error()
    assert rs(table(h=41)) == -1 and rs(table(pitch=100)) == -1
    mean = (torch.ones(3)).numpy().ctypes.data
    assert rs(table(), mean=mean) == -1
    assert rs(table(h=40, rh=1, top=0), out_h=1, out_w=24, out=K.empty_nhwc(1, 16, 1, 24, "cpu")) == -3
    big = torch.zeros(40000 * 4 * 3, dtype=torch.uint8)
    t = torch.tensor([[0, 40000, 4, 12, 24, 24, 0, 0]], dtype=torch.int64)  # a ~1670x downscale: the rows of one output row exceed shared memory
    assert lib.sgb_resample_crop_u8(p(t), p(t), p(big), big.numel(), 1, 3, 24, 24, 16, 0, 255.0, None, None, p(out), None) == -1
    assert b"shared memory" in lib.sgb_last_error()
    with pytest.raises(L.SgbError):
        K.resample_crop_u8(table().int(), table(), src, out)
    with pytest.raises(L.SgbError):
        K.resample_crop_u8(table(), table(), src, K.empty_nhwc(2, 16, 24, 24, "cpu"))
    # ---- classify
    x = torch.zeros(6, 10)
    y = torch.zeros(6, dtype=torch.int64)
    c = torch.zeros(4, dtype=torch.int64)

    def cl(**kw):
        a = dict(logits=x, N=6, C=10, stride=10, target=y, soft=None, k=5, counters=c, label=None)
        a.update(kw)
        q = lambda t: p(t) if t is not None else None  # noqa: E731
        return lib.sgb_classify_rows(q(a["logits"]), a["N"], a["C"], a["stride"], 0, q(a["target"]), q(a["soft"]), 10, 0, a["k"], q(a["counters"]), q(a["label"]), None, None)

    assert cl() == -3
    assert cl(N=0, logits=None) == 0
    assert cl(k=11) == -1 and cl(k=0) == -1
    assert cl(logits=None) == -1 and cl(counters=None) == -1 and cl(target=None) == -1 and cl(soft=x) == -1
    assert cl(counters=None, target=None, label=torch.zeros(6, dtype=torch.int32)) == -3
    assert cl(stride=9) == -1 and cl(N=-1) == -1
    with pytest.raises(L.SgbError):
        K.classify_rows(x.double(), y, counters=c)
    with pytest.raises(L.SgbError):
        K.classify_rows(x, y[:5], counters=c)
    with pytest.raises(L.SgbError):
        K.classify_rows(x, y, counters=c.int())
    with pytest.raises(L.SgbError):
        K.classify_rows(x.t(), None, label=torch.zeros(10, dtype=torch.int32))
