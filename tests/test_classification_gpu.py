"""Classification on the H100: the batched resize + crop kernel against the host build of its arithmetic and the reference's
recorded outputs, the row-wise decode kernel against torch, ResNet-50 predict() on raw images, Trainer.train() with the train /
valid metric lists under a CUDA graph, and a train step plus the metric update without host synchronisation."""
import hashlib

import numpy as np
import pytest
import torch

import host_classification as H

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _sha(t_bf16):
    return hashlib.sha256(t_bf16.contiguous().view(torch.int16).cpu().numpy().tobytes()).hexdigest()


def _imagenet():
    from super_gradients_b200.training import processing as P

    return P.default_imagenet_processing_params()["image_processor"]


def _image(case):
    h, w = case["image_shape"]
    return np.random.RandomState(case["image_seed"]).randint(0, 256, (h, w, 3)).astype(np.uint8)


def _host_batch(cp, images, monkeypatch):
    with monkeypatch.context() as mp:
        H.install(mp)
        return cp.preprocess_crop_batch(images, "cpu")


def test_resample_kernel_matches_reference_and_host_build(golden, monkeypatch):
    from super_gradients_b200.training import processing as P

    for chain, cp in (("imagenet", _imagenet()), ("small_reversed", P.ComposeProcessing([P.ReverseImageChannels(), P.Resize(160), P.CenterCrop(128), P.StandardizeImage(), P.ImagePermute()]))):
        cases = golden("classification")["images"][chain]["cases"]
        batch = cp.preprocess_crop_batch([_image(c) for c in cases], DEV)
        torch.cuda.synchronize()
        assert float(batch[:, 3:].abs().max()) == 0.0
        for b, c in enumerate(cases):
            assert _sha(batch[b, :3]) == c["pre_sha256"], (chain, c["image_shape"])


def test_resample_kernel_one_launch_over_64_mixed_images(monkeypatch):
    """64 images of 64 sizes (downscales up to 4000 px, upscales, exactly-256 sides) in ONE launch == the host build, bit for bit."""
    from super_gradients_b200 import lib as L

    rng = np.random.RandomState(7)
    sizes = [(int(rng.randint(60, 1200)), int(rng.randint(60, 1200))) for _ in range(58)] + [(256, 256), (256, 900), (4000, 3000), (60, 90), (224, 224), (2000, 257)]
    images = [rng.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in sizes]
    cp = _imagenet()
    n0 = L.LAUNCHES[0]
    batch = cp.preprocess_crop_batch(images, DEV)
    assert L.LAUNCHES[0] - n0 == 1
    want = _host_batch(cp, images, monkeypatch)
    got = batch.cpu()
    for b in range(len(images)):
        assert _sha(got[b]) == _sha(want[b]), sizes[b]


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_classify_kernel_matches_torch(dtype):
    from super_gradients_b200 import kernels as K

    g = torch.Generator().manual_seed(3)
    x = (torch.randn(256, 1000, generator=g) * 4).round() / 4  # quarter steps: many exact ties, also at the top and at the 5th place
    x[::7, 13] = x[::7].max(1).values  # ties for the maximum
    x = x.to(dtype)
    y = torch.randint(0, 1000, (256,), generator=g)
    y[::3] = torch.sort(x[::3].float(), dim=1, descending=True, stable=True)[1][:, 4]  # targets at the 5th place
    xd, yd = x.to(DEV), y.to(DEV)
    counters = torch.zeros(4, dtype=torch.int64, device=DEV)
    label = torch.empty(256, dtype=torch.int32, device=DEV)
    conf = torch.empty(256, dtype=torch.float32, device=DEV)
    K.classify_rows(xd, yd, k=5, counters=counters, label=label, confidence=conf)
    xf = x.float()
    rank = torch.sort(xf, dim=1, descending=True, stable=True)[1]
    assert torch.equal(label.cpu().long(), torch.argmax(xf, 1))
    assert counters.cpu().tolist() == [int((torch.argmax(xf, 1) == y).sum()), int((rank[:, :5] == y[:, None]).any(1).sum()), 256, 0]
    torch.testing.assert_close(conf.cpu().double(), torch.softmax(xf.double(), 1).max(1).values, rtol=1e-6, atol=0)
    c2, l2, f2 = torch.zeros(4, dtype=torch.int64), torch.empty(256, dtype=torch.int32), torch.empty(256)
    H.classify_rows(x, y, k=5, counters=c2, label=l2, confidence=f2)  # the host build of the same arithmetic
    assert torch.equal(c2, counters.cpu()) and torch.equal(l2, label.cpu())
    torch.testing.assert_close(f2, conf.cpu(), rtol=1e-6, atol=0)
    soft = torch.nn.functional.one_hot(y, 1000).float().to(DEV) * 0.7 + 0.0003
    c3 = torch.zeros(4, dtype=torch.int64, device=DEV)
    K.classify_rows(xd, soft, k=5, counters=c3)
    assert torch.equal(c3, counters)


def test_resnet50_predict_on_raw_images(monkeypatch):
    from super_gradients_b200 import lib as L
    from super_gradients_b200.training import models

    torch.manual_seed(0)
    m = models.get("resnet50", num_classes=1000).to(DEV).eval()
    cp = _imagenet()
    m.set_dataset_processing_params(image_processor=cp)
    rng = np.random.RandomState(5)
    images = [rng.randint(0, 256, (int(rng.randint(200, 700)), int(rng.randint(200, 700)), 3)).astype(np.uint8) for _ in range(64)]
    m.predict(images[:2])  # the first call prepares the filters
    n0 = L.LAUNCHES[0]
    preds = m.predict(images, batch_size=64)
    assert len(preds) == 64
    per_batch = L.LAUNCHES[0] - n0
    with torch.no_grad():
        logits = m(_host_batch(cp, images, monkeypatch).to(DEV))
        n1 = L.LAUNCHES[0]
        m(_host_batch(cp, images, monkeypatch).to(DEV))
        model_launches = L.LAUNCHES[0] - n1
    assert per_batch == model_launches + 2  # one pre-processing launch + the model + one decode launch
    conf, lab = torch.max(torch.softmax(logits.float(), 1), 1)
    assert [p.label for p in preds] == lab.cpu().tolist()
    np.testing.assert_allclose([p.confidence for p in preds], conf.cpu().numpy(), rtol=1e-6)


def _cifar_loaders(n_train=4, bs=32):
    g = torch.Generator().manual_seed(9)
    X, Y = torch.randn(bs * (n_train + 1), 3, 32, 32, generator=g), torch.randint(0, 10, (bs * (n_train + 1),), generator=g)
    train = [(X[i * bs : (i + 1) * bs], Y[i * bs : (i + 1) * bs]) for i in range(n_train)]
    return train, [(X[n_train * bs :], Y[n_train * bs :])]


def test_trainer_cuda_graph_with_classification_metrics(tmp_path):
    from super_gradients_b200.training import models
    from super_gradients_b200.training.losses import CrossEntropyLoss
    from super_gradients_b200.training.sg_trainer import Trainer

    torch.manual_seed(0)
    m = models.get("resnet18_cifar", num_classes=10)
    train, valid = _cifar_loaders()
    tp = dict(max_epochs=2, initial_lr=0.05, lr_mode="cosine", optimizer="SGD", loss=CrossEntropyLoss(), cuda_graph=True, train_metrics_list=["Accuracy", "Top5"],
              valid_metrics_list=["Accuracy", "Top5"], metric_to_watch="Accuracy", greater_metric_to_watch_is_better=True, save_model=True)  # fmt: skip
    trainer = Trainer("cls_graph", ckpt_root_dir=str(tmp_path))
    trainer.train(m, tp, train, valid_loader=valid)
    assert trainer.step.graph is not None
    ck = torch.load(tmp_path / "cls_graph" / "ckpt_latest.pth", weights_only=False)
    met = ck["metrics"]
    assert all(0.0 <= met[k] <= 1.0 for k in ("train_Accuracy", "train_Top5", "Accuracy", "Top5")) and met["train_Top5"] >= met["train_Accuracy"]
    with torch.no_grad():
        m.eval()
        p = m(valid[0][0].to(DEV)).float().cpu()
    assert met["Accuracy"] == pytest.approx(float((p.argmax(1) == valid[0][1]).double().mean()))
    assert ck["acc"] >= met["Accuracy"]


def test_train_step_and_metric_update_do_not_synchronise():
    """After warm-up, one captured step's replay plus the train metrics' update() on TrainStep.last_outputs runs under
    set_sync_debug_mode("error"); the counters then equal a recomputation from those outputs."""
    from super_gradients_b200.training import models
    from super_gradients_b200.training.losses import CrossEntropyLoss
    from super_gradients_b200.training.metrics import Accuracy, Top5
    from super_gradients_b200.training.sg_trainer import TrainStep

    torch.manual_seed(0)
    m = models.get("resnet18_cifar", num_classes=10).to(DEV).train()
    st = TrainStep(m, CrossEntropyLoss(), "SGD", {"momentum": 0.9}, zero_wd_on_bias_and_bn=True, keep_outputs=True)
    x, y = _cifar_loaders(1)[0][0]
    x, y = x.to(DEV), y.to(DEV)
    st.set_hyper_params(0.01)
    st.capture(x, y, warmup=2)
    metrics = [Accuracy(), Top5()]
    st.set_hyper_params(0.01)
    st.run(x, y)
    for mt in metrics:
        mt.update(st.last_outputs, y)  # allocates the counters outside the checked region
        mt.reset()
    torch.cuda.synchronize()
    st.set_hyper_params(0.01)
    torch.cuda.set_sync_debug_mode("error")
    try:
        st.run(x, y)
        for mt in metrics:
            mt.update(st.last_outputs, y)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    out = st.last_outputs.float().cpu()
    yc = y.cpu()
    assert metrics[0].compute() == pytest.approx(float((out.argmax(1) == yc).double().mean()))
    assert metrics[1].compute() == pytest.approx(float((torch.sort(out, dim=1, descending=True, stable=True)[1][:, :5] == yc[:, None]).any(1).double().mean()))
