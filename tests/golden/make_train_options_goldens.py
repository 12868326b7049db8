"""Generates tests/golden/train_options.pt: resnet18_cifar trained by the unmodified reference (CPU, fp32, through
oracle/ref_shim.py) with clip_grad_norm, batch_accumulate 2, precise_bn with a precise_bn_batch_size, and EMA.

The reference's own pieces run in the order of its train loop: forward + loss + backward on every micro-batch; at every
accumulation boundary (global_step % batch_accumulate == 0) clip_grad_norm_, the SGD step, zero_grad and the EMA update
(sg_trainer.py:611-644); after the epoch compute_precise_bn_stats on the live model, then on the EMA model (:1552-1563).  Recorded:
per-micro-batch losses, each step's total norm and clip coefficient, the final weights and the live and EMA BatchNorm statistics.
Usage: python tests/golden/make_train_options_goldens.py"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import ref_shim  # noqa: E402

# the run, as Trainer.train() training_params (tests/test_train_options_gpu.py trains the product with exactly these)
CONFIG = dict(batch_size=16, n_batches=6, data_seed=6, init_seed=0, lr=0.05, momentum=0.9, weight_decay=1e-4, batch_accumulate=2, clip_grad_norm=0.5,
              precise_bn_batch_size=48, ema_decay=0.9)  # fmt: skip


def data(cfg=CONFIG):
    g = torch.Generator().manual_seed(cfg["data_seed"])
    n = cfg["batch_size"] * cfg["n_batches"]
    return torch.randn(n, 3, 32, 32, generator=g), torch.randint(0, 10, (n,), generator=g)


def loader(cfg=CONFIG):
    x, y = data(cfg)
    return torch.utils.data.DataLoader(torch.utils.data.TensorDataset(x, y), batch_size=cfg["batch_size"], shuffle=False)


def main():
    ref_shim.install()
    from super_gradients.training import models
    from super_gradients.training.losses.label_smoothing_cross_entropy_loss import CrossEntropyLoss
    from super_gradients.training.utils.distributed_training_utils import compute_precise_bn_stats
    from super_gradients.training.utils.ema import ModelEMA
    from super_gradients.training.utils.ema_decay_schedules import ConstantDecay

    cfg = CONFIG
    torch.manual_seed(cfg["init_seed"])
    m = models.get("resnet18_cifar", num_classes=10)
    sd0 = {k: v.clone() for k, v in m.state_dict().items()}
    ld = loader(cfg)
    crit = CrossEntropyLoss()
    opt = torch.optim.SGD(m.parameters(), lr=cfg["lr"], momentum=cfg["momentum"], weight_decay=cfg["weight_decay"])
    ema = ModelEMA(m, cfg["ema_decay"], ConstantDecay())
    losses, norms, coefs = [], [], []
    m.train()
    total_steps = len(ld)
    for batch_idx, (xb, yb) in enumerate(ld):
        loss = crit(m(xb), yb)
        loss = loss[0] if isinstance(loss, tuple) else loss
        loss.backward()
        losses.append(float(loss))
        global_step = batch_idx + 1
        if global_step % cfg["batch_accumulate"] == 0:
            total = torch.nn.utils.clip_grad_norm_(m.parameters(), cfg["clip_grad_norm"])
            norms.append(float(total))
            coefs.append(float(torch.clamp(cfg["clip_grad_norm"] / (total + 1e-6), max=1.0)))
            opt.step()
            opt.zero_grad()
            ema.update(m, step=global_step, total_steps=total_steps)
    real_cuda = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self  # compute_precise_bn_stats moves its inputs with .cuda(); this run is on the CPU
    try:
        before = {k: v.clone() for k, v in m.state_dict().items() if "running_" in k}
        compute_precise_bn_stats(model=m, loader=ld, precise_bn_batch_size=cfg["precise_bn_batch_size"], num_gpus=1)
        compute_precise_bn_stats(model=ema.ema, loader=ld, precise_bn_batch_size=cfg["precise_bn_batch_size"], num_gpus=1)
    finally:
        torch.Tensor.cuda = real_cuda
    sd, esd = m.state_dict(), ema.ema.state_dict()
    assert all(c < 1 for c in coefs), coefs  # the bound clips every step
    assert not torch.equal(before["layer1.0.bn1.running_mean"], sd["layer1.0.bn1.running_mean"])
    # weights as float64 per-tensor sums and norms (the full tensors are 45 MB), the BatchNorm statistics in full
    summary = lambda d: {k: (float(v.double().sum()), float(v.double().norm())) for k, v in d.items() if v.dtype.is_floating_point and "running_" not in k}  # noqa: E731
    stats = lambda d: {k: v.clone() for k, v in d.items() if "running_" in k}  # noqa: E731
    torch.save(
        dict(config=cfg, init_sums={k: float(v.double().sum()) for k, v in sd0.items() if v.dtype.is_floating_point}, losses=losses, norms=norms, coefs=coefs,
             final=summary(sd), ema_final=summary(esd), bn=stats(sd), ema_bn=stats(esd), num_batches_tracked={k: int(v) for k, v in sd.items() if k.endswith("num_batches_tracked")}),
        os.path.join(HERE, "train_options.pt"),
    )  # fmt: skip
    print("losses", losses, "\nnorms", norms, "\ncoefs", coefs)


if __name__ == "__main__":
    main()
