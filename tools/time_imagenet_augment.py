"""Times the ImageNet train augmentation at 224 x 224: the GPU kernel per batch (CUDA events), the host pack + host-to-device copy
per batch, the loader's host half per sample (ImageNetAugmentDataset's draws and the window copy) and the PIL chain the reference
runs per sample (torchvision's RandomResizedCrop / resized_crop, the flip, the two RandAugment ops through Pillow, ToTensor and
Normalize, from the same draws), both as process time on one CPU thread, in one process.  Sources are ImageNet-like sizes (shorter
side 300 to 500, aspect 3:4 to 4:3).  Prints one JSON line with the card name and power limit.
Usage: python tools/time_imagenet_augment.py [--batch B] [--iters N] [--samples N]"""
import argparse
import json
import os
import random
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import torchvision.transforms as TT  # noqa: E402
import torchvision.transforms.functional as TF  # noqa: E402
from PIL import Image  # noqa: E402

from imagenet_augment_cases import IMG_MEAN, IMG_STD, image, pil_op  # noqa: E402
from super_gradients_b200.training.datasets.imagenet_augment_dataset import ImageNetAugmentCollateFN, ImageNetAugmentDataset  # noqa: E402
from super_gradients_b200.training.transforms import imagenet_augment as IA  # noqa: E402


class Sources:
    def __init__(self, n, seed=0):
        rng = np.random.default_rng(seed)
        self.items = []
        for _ in range(n):
            short = int(rng.integers(300, 501))
            long_ = int(short * rng.uniform(1.0, 4.0 / 3.0))
            h, w = (short, long_) if rng.random() < 0.5 else (long_, short)
            self.items.append((image(rng, h, w), int(rng.integers(0, 1000))))

    def __len__(self):
        return len(self.items)

    def __getitem__(self, i):
        return self.items[i]


def pil_chain(arr, normalize):
    """The reference's per-sample PIL work on one source, with draws of its own (same distribution as the recipe's)."""
    img = Image.fromarray(arr)
    i, j, h, w = TT.RandomResizedCrop.get_params(img, (0.08, 1.0), (3.0 / 4.0, 4.0 / 3.0))
    img = TF.resized_crop(img, i, j, h, w, [224, 224], random.choice((TT.InterpolationMode.BILINEAR, TT.InterpolationMode.BICUBIC)))
    if torch.rand(1) < 0.5:
        img = TF.hflip(img)
    for k in np.random.choice(len(IA.RAND_TRANSFORMS), 2):
        if random.random() > 0.5:
            continue
        img = pil_op(img, IA.RAND_TRANSFORMS[k], min(10.0, max(0.0, random.gauss(7, 0.5))), random.random() > 0.5)
    return normalize(TF.to_tensor(img))


def cpu_ms(fn, n):
    t0 = time.process_time()
    for i in range(n):
        fn(i)
    return (time.process_time() - t0) * 1e3 / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--samples", type=int, default=512)
    a = ap.parse_args()
    torch.set_num_threads(1)
    random.seed(0)
    np.random.seed(0)
    torch.manual_seed(0)
    src = Sources(max(a.batch, a.samples))
    ds = ImageNetAugmentDataset(src)
    collate = ImageNetAugmentCollateFN.for_dataset(ds, mixup_alpha=0.2, cutmix_alpha=1.0, label_smoothing=0.1)
    normalize = TT.Normalize(IMG_MEAN, IMG_STD)

    res = {"batch": a.batch}
    try:
        res["cpu"] = [ln.split(":", 1)[1].strip() for ln in open("/proc/cpuinfo") if ln.startswith("model name")][0]
    except (OSError, IndexError):
        res["cpu"] = "unknown"
    res["host_half_cpu_ms_per_sample"] = cpu_ms(lambda i: ds[i % len(ds)], a.samples)
    res["pil_chain_cpu_ms_per_sample"] = cpu_ms(lambda i: pil_chain(src[i % len(src)][0], normalize), a.samples)
    plans = [ds[i] for i in range(a.batch)]
    t0 = time.process_time()
    for _ in range(5):
        batch = collate(plans)
    res["collate_pack_cpu_ms_per_batch"] = (time.process_time() - t0) * 1e3 / 5
    res["window_mb_per_batch"] = batch.buffer.numel() / 1e6

    if not torch.cuda.is_available():
        res["gpu"] = "not measured (no CUDA device)"
        print(json.dumps(res))
        return
    pinned = batch.pin_memory()
    res["mix_mode"] = pinned.mix_mode
    for _ in range(3):
        pinned.to_model_input("cuda")
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    # launch alone: the table and windows already on the device
    from super_gradients_b200 import kernels as K

    head = pinned.batch * K.IN_FIELDS * 8
    dev = pinned.buffer.cuda()
    ws = torch.empty(pinned.workspace_bytes, dtype=torch.uint8, device="cuda")
    out = K.empty_nhwc(pinned.batch, 16, 224, 224, "cuda")
    th = pinned.buffer[:head].view(torch.int64).view(pinned.batch, K.IN_FIELDS)
    td = dev[:head].view(torch.int64).view(pinned.batch, K.IN_FIELDS)
    per_mode = {}
    for mode in (0, 1, 2):
        launch = lambda: K.imagenet_augment(th, td, dev[head:], ws, out, ds.fill, ds.img_mean, ds.img_std, mix_mode=mode, lam=0.7, box=(20, 180, 40, 200))  # noqa: E731
        for _ in range(5):
            launch()
        e0.record()
        for _ in range(a.iters):
            launch()
        e1.record()
        torch.cuda.synchronize()
        per_mode[mode] = e0.elapsed_time(e1) / a.iters
    res["launch_ms_per_batch"] = {"nomix": per_mode[0], "mixup": per_mode[1], "cutmix": per_mode[2]}
    e0.record()
    for _ in range(a.iters):
        pinned.buffer.to("cuda", non_blocking=True)
    e1.record()
    torch.cuda.synchronize()
    res["h2d_copy_ms_per_batch"] = e0.elapsed_time(e1) / a.iters
    t0 = time.perf_counter()
    for _ in range(a.iters):
        pinned.to_model_input("cuda")
    torch.cuda.synchronize()
    res["to_model_input_wall_ms_per_batch"] = (time.perf_counter() - t0) * 1e3 / a.iters
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res["gpu"] = q.splitlines()[0] if q else torch.cuda.get_device_name()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
