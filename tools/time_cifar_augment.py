"""Times the CIFAR-10 augmentation and the cifar10_resnet train loop it feeds, in one process:

- the kernel per batch of 256 and 512 from the device-resident data set (CUDA events over --iters launches);
- the host half per sample (Cifar10AugmentDataset's draws plus Cifar10AugmentCollateFN's packing) against the reference's
  torchvision chain (RandomCrop(32, padding=4), RandomHorizontalFlip, ToTensor, Normalize on a PIL image, plus default_collate),
  both as process time on one CPU thread;
- Trainer.train() images/s of resnet18_cifar at batch 256 under cuda_graph (SGD momentum 0.9, weight decay 1e-4), fed three ways:
  the reference-style torchvision DataLoader (8 workers, shuffle, pin_memory, drop_last False), the packed loader (same DataLoader
  settings, Cifar10AugmentDataset + Cifar10AugmentCollateFN) and Cifar10DeviceLoader.  The rate is that of the second epoch (the
  first captures the graph), host clock between device synchronisations at the epoch's start and end.

The images are --images seeded random uint8 32 x 32 x 3 arrays (CIFAR-10's train set size by default).  Prints one JSON line with
the card name, its power limit and the host's CPU count.  Usage: python tools/time_cifar_augment.py [--images N] [--iters N]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import torchvision.transforms as TT  # noqa: E402
from PIL import Image  # noqa: E402

from super_gradients_b200 import kernels as K  # noqa: E402
from super_gradients_b200.training.datasets.cifar_augment_dataset import (CIFAR10_MEAN, CIFAR10_STD, Cifar10AugmentCollateFN, Cifar10AugmentDataset,  # noqa: E402
                                                                          Cifar10DeviceLoader)  # fmt: skip
from super_gradients_b200.training.utils.callbacks import Callback  # noqa: E402


class Images(torch.utils.data.Dataset):
    """(PIL RGB image, label) as torchvision's CIFAR10 returns them, optionally through a transform."""

    def __init__(self, arrays, labels, transform=None):
        self.arrays, self.labels, self.transform = arrays, labels, transform

    def __len__(self):
        return len(self.arrays)

    def __getitem__(self, i):
        img = Image.fromarray(self.arrays[i])
        return (self.transform(img) if self.transform else img), int(self.labels[i])


class EpochClock(Callback):
    def __init__(self):
        self.times = []

    def on_train_loader_start(self, context):
        torch.cuda.synchronize()
        self.t0 = time.perf_counter()

    def on_train_loader_end(self, context):
        torch.cuda.synchronize()
        self.times.append(time.perf_counter() - self.t0)


def launch_ms(images_dev, B, iters):
    g = torch.Generator().manual_seed(B)
    t = torch.zeros(B, K.CF_FIELDS, dtype=torch.int32)
    t[:, 0] = torch.randint(0, images_dev.shape[0], (B,), generator=g, dtype=torch.int32)
    t[:, 1:3] = torch.randint(0, 9, (B, 2), generator=g, dtype=torch.int32)
    t[:, 3] = torch.randint(0, 2, (B,), generator=g, dtype=torch.int32)
    td, out = t.cuda(), K.empty_nhwc(B, 16, 32, 32, "cuda")
    for _ in range(20):
        K.cifar_augment(t, td, images_dev, out, CIFAR10_MEAN, CIFAR10_STD)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        K.cifar_augment(t, td, images_dev, out, CIFAR10_MEAN, CIFAR10_STD)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def host_ms_per_sample(arrays, labels, n):
    chain = TT.Compose([TT.RandomCrop(32, padding=4), TT.RandomHorizontalFlip(), TT.ToTensor(), TT.Normalize(CIFAR10_MEAN, CIFAR10_STD)])
    ref, ours = Images(arrays, labels, chain), Cifar10AugmentDataset(Images(arrays, labels))
    collate = Cifar10AugmentCollateFN.for_dataset(ours)
    out = {}
    for name, ds, fn in (("torchvision", ref, torch.utils.data.default_collate), ("gpu_loader_host_half", ours, collate)):
        t0 = time.process_time()
        for s in range(0, n, 256):
            fn([ds[i] for i in range(s, min(n, s + 256))])
        out[name] = (time.process_time() - t0) * 1e3 / n
    return out


def train_rate(loader, n):
    from super_gradients_b200.training import models
    from super_gradients_b200.training.sg_trainer import Trainer

    clock = EpochClock()
    tp = dict(max_epochs=2, initial_lr=0.1, lr_mode="StepLRScheduler", lr_updates=[100, 150, 200], lr_decay_factor=0.1, optimizer="SGD",
              optimizer_params={"weight_decay": 1e-4, "momentum": 0.9}, loss="CrossEntropyLoss", save_model=False, cuda_graph=True, phase_callbacks=[clock],
              silent_mode=True)  # fmt: skip
    torch.manual_seed(0)
    tr = Trainer("time_cifar", ckpt_root_dir=os.path.join("/tmp", f"time_cifar_{os.getpid()}"))
    tr.train(models.get("resnet18_cifar", num_classes=10).cuda().train(), tp, loader)
    assert all(np.isfinite(v) for v in tr.history["train_loss"]), tr.history["train_loss"]
    return dict(images_per_s=n / clock.times[1], epoch_s=[round(t, 3) for t in clock.times], train_loss=[round(v, 4) for v in tr.history["train_loss"]])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=50000)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--host-samples", type=int, default=5120)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to time")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    rng = np.random.default_rng(0)
    arrays = rng.integers(0, 256, (args.images, 32, 32, 3), dtype=np.uint8)
    labels = rng.integers(0, 10, args.images)
    res = dict(gpu=q[0] if q else None, cpus=os.cpu_count(), cpus_usable=len(os.sched_getaffinity(0)), images=args.images)
    dev = torch.from_numpy(arrays).cuda()
    res["launch_ms"] = {B: round(launch_ms(dev, B, args.iters), 4) for B in (256, 512)}
    del dev
    res["host_ms_per_sample"] = {k: round(v, 4) for k, v in host_ms_per_sample(arrays, labels, args.host_samples).items()}
    chain = TT.Compose([TT.RandomCrop(32, padding=4), TT.RandomHorizontalFlip(), TT.ToTensor(), TT.Normalize(CIFAR10_MEAN, CIFAR10_STD)])
    dl = dict(batch_size=256, shuffle=True, num_workers=8, drop_last=False, pin_memory=True)
    ours = Cifar10AugmentDataset(Images(arrays, labels))
    feeds = {
        "torchvision_dataloader_8_workers": lambda: torch.utils.data.DataLoader(Images(arrays, labels, chain), **dl),
        "packed_loader_8_workers": lambda: torch.utils.data.DataLoader(ours, collate_fn=Cifar10AugmentCollateFN.for_dataset(ours), **dl),
        "device_loader": lambda: Cifar10DeviceLoader(arrays, labels, 256, shuffle=True, drop_last=False, seed=0),
    }
    res["train"] = {}
    for name, make in feeds.items():
        res["train"][name] = train_rate(make(), args.images)
        print(name, res["train"][name], flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
