"""GPU checks of the CIFAR-10 augmentation kernel (csrc/cifar_augment.cu): the bf16 NHWC batch is, bit for bit, the reference
chains' float32 output rounded to bf16, from packed batches and from a device-resident data set, for every crop corner and flip;
bad tables are refused; Trainer.train() of resnet18_cifar runs from the packed and the device loaders, eagerly and under a CUDA
graph, and one batch's model input and loss equal those of the torchvision chain's output with the same draws."""
import numpy as np
import pytest
import torch

from cifar_augment_cases import MEAN, STD, golden, images, torchvision_chain
from super_gradients_b200 import kernels as K
from super_gradients_b200 import lib as L
from super_gradients_b200.training.datasets.cifar_augment_dataset import (Cifar10AugmentCollateFN, Cifar10DeviceLoader, PackedCifarBatch, pack)  # fmt: skip

pytestmark = pytest.mark.gpu


def _bits(x: torch.Tensor) -> torch.Tensor:
    """float32 NCHW -> the bf16 bits of the model input's first three channels, NCHW."""
    return x.bfloat16().view(torch.int16)


def _out_bits(images: torch.Tensor) -> torch.Tensor:
    assert images.shape[1:] == (16, 32, 32) and images.dtype == torch.bfloat16
    assert bool((images[:, 3:] == 0).all())
    return images[:, :3].contiguous().view(torch.int16).cpu()


def _golden_batch(B):
    g = golden()["train"]
    k = torch.arange(B) % len(g["draws"])
    return g["images"][k].numpy(), g["draws"][k], g["output"][k], g["images"]


@pytest.mark.parametrize("B", [1, 3, 80, 256])
def test_packed_and_resident_sources_match_the_golden(B):
    ims, draws, want, resident = _golden_batch(B)
    packed = Cifar10AugmentCollateFN(MEAN, STD)([(ims[b], b, tuple(draws[b].tolist())) for b in range(B)]).pin_memory()
    got, labels = packed.to_model_input("cuda")
    assert torch.equal(_out_bits(got), _bits(want)) and labels.tolist() == list(range(B))
    table = np.concatenate([(np.arange(B) % len(resident))[:, None], draws.numpy()], 1).astype(np.int32)
    dev = resident.cuda()
    batch = PackedCifarBatch(pack(table, np.arange(B), pin=True), B, MEAN, STD, images=dev)
    got, _ = batch.to_model_input("cuda")
    assert torch.equal(_out_bits(got), _bits(want))


def test_every_corner_and_flip_matches_torchvision():
    ims = images(162, seed=4)
    table = np.array([(k, (k // 2) // 9, (k // 2) % 9, k % 2) for k in range(162)], np.int32)
    want = torch.stack([torchvision_chain(ims[k], *table[k, 1:3].tolist(), bool(table[k, 3])) for k in range(162)])
    out = K.empty_nhwc(162, 16, 32, 32, "cuda")
    t = torch.from_numpy(table)
    K.cifar_augment(t, t.cuda(), torch.from_numpy(ims).cuda(), out, MEAN, STD)
    assert torch.equal(_out_bits(out), _bits(want))


def test_validation_chain_matches_the_golden():
    g = golden()["val"]
    n = len(g["images"])
    dl = Cifar10DeviceLoader(g["images"], torch.arange(n), batch_size=5, shuffle=False, augment=False)
    got = torch.cat([_out_bits(b.to_model_input("cuda")[0]) for b in dl])
    assert torch.equal(got, _bits(g["output"]))


def test_refusals():
    src = torch.zeros(4, 32, 32, 3, dtype=torch.uint8, device="cuda")

    def run(table, out_c=16, mean=MEAN, std=STD):
        t = torch.tensor(table, dtype=torch.int32).reshape(-1, K.CF_FIELDS)
        out = K.empty_nhwc(t.shape[0], out_c, 32, 32, "cuda")
        K.cifar_augment(t, t.cuda(), src, out, mean, std)

    run([[0, 0, 0, 0], [3, 8, 8, 1]])
    torch.cuda.synchronize()
    for bad in ([[4, 0, 0, 0]], [[-1, 0, 0, 0]], [[0, 9, 0, 0]], [[0, 0, -1, 0]], [[0, 0, 0, 2]], []):
        with pytest.raises(L.SgbError):
            run(bad)
    with pytest.raises(L.SgbError):
        run([[0, 0, 0, 0]], std=(0.2, 0.0, 0.2))
    with pytest.raises(L.SgbError):
        run([[0, 0, 0, 0]], mean=(float("nan"), 0.0, 0.0))
    torch.cuda.synchronize()


def _loaders(n, bs, device_loader):
    ims = images(n, seed=6)
    labels = np.arange(n) % 10
    if device_loader:
        return Cifar10DeviceLoader(ims, labels, bs, shuffle=True, drop_last=False, seed=0)
    from test_cifar_augment_replay import _Plain
    from super_gradients_b200.training.datasets.cifar_augment_dataset import Cifar10AugmentDataset

    ds = Cifar10AugmentDataset(_Plain(ims))
    return torch.utils.data.DataLoader(ds, batch_size=bs, shuffle=True, num_workers=2, collate_fn=Cifar10AugmentCollateFN.for_dataset(ds), pin_memory=True)


@pytest.mark.parametrize("device_loader", [False, True], ids=["packed", "device"])
@pytest.mark.parametrize("cuda_graph", [False, True])
def test_trainer_trains_resnet18_cifar(tmp_path, device_loader, cuda_graph):
    """The recipe's training_hyperparams (SGD momentum 0.9, weight decay 1e-4, StepLRScheduler, Accuracy / Top5), one short epoch
    with a short last batch (600 = 2 x 256 + 88), validated by the device loader's validation chain.  The packed loader runs in
    worker processes with pin_memory, as the recipe's loader does: its pin-memory thread works while the step is captured."""
    from super_gradients_b200.training import models
    from super_gradients_b200.training.sg_trainer import Trainer

    torch.manual_seed(0)
    train = _loaders(600, 256, device_loader)
    g = golden()["val"]
    valid = Cifar10DeviceLoader(g["images"], torch.arange(len(g["images"])) % 10, batch_size=8, shuffle=False, augment=False)
    tp = dict(max_epochs=1, initial_lr=0.1, lr_mode="StepLRScheduler", lr_updates=[100, 150, 200], lr_decay_factor=0.1, lr_warmup_epochs=0,
              optimizer="SGD", optimizer_params={"weight_decay": 1e-4, "momentum": 0.9}, loss="CrossEntropyLoss", train_metrics_list=["Accuracy", "Top5"],
              valid_metrics_list=["Accuracy", "Top5"], metric_to_watch="Accuracy", greater_metric_to_watch_is_better=True, save_model=False, cuda_graph=cuda_graph)  # fmt: skip
    tr = Trainer("cifar_aug", ckpt_root_dir=str(tmp_path))
    tr.train(models.get("resnet18_cifar", num_classes=10).cuda().train(), tp, train, valid)
    assert len(tr.history["train_loss"]) == 1 and np.isfinite(tr.history["train_loss"][0])
    if cuda_graph:
        assert tr.step.replays == 2 and tr.step.fallbacks == 1  # the two 256-sample batches replay, the 88-sample batch runs eagerly


def test_one_batch_equals_the_torchvision_chain():
    from super_gradients_b200.training import models
    from super_gradients_b200.training.losses import CrossEntropyLoss

    ims, draws, _, _ = _golden_batch(64)
    labels = torch.arange(64) % 10
    packed = Cifar10AugmentCollateFN(MEAN, STD)([(ims[b], int(labels[b]), tuple(draws[b].tolist())) for b in range(64)]).pin_memory()
    x, y = packed.to_model_input("cuda")
    ref = torch.stack([torchvision_chain(ims[b], *draws[b].tolist()) for b in range(64)]).cuda()
    torch.manual_seed(0)
    model = models.get("resnet18_cifar", num_classes=10).cuda().eval()
    assert torch.equal(_out_bits(x), _bits(ref.cpu()))
    with torch.no_grad():
        a, _ = CrossEntropyLoss()(model(x), y)
        b, _ = CrossEntropyLoss()(model(ref), labels.cuda())
    assert torch.isfinite(a) and torch.equal(a, b)
