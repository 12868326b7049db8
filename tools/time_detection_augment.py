"""Times the detection train augmentation at 640 x 640: the GPU kernel per batch (CUDA events), the host pack + host-to-device
copy per batch, the host half of the transforms per sample (draws, boxes, packing) and the same pixel chain with cv2 / numpy per
sample, both as process time on one CPU thread, in one process.  --recipe coco (default): the COCO recipe chain's draws at
B = --batch.  --recipe roboflow: the Roboflow fine-tuning list (DetectionMosaic first, four source images per sample) at B = 16
and B = 32, once on sources fitted into 640 (mosaic tiles read as they are) and once on larger and smaller ones (tiles resized).  Prints one JSON line with the card name and power limit.
Usage: python tools/time_detection_augment.py [--recipe coco|roboflow] [--batch B] [--iters N]"""
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

import cv2  # noqa: E402
from augment_cases import RECIPE, StubRawDataset, _image, make_plan, oracle_u8  # noqa: E402
from mosaic_cases import ROBOFLOW, oracle_mosaic_u8  # noqa: E402
from super_gradients_b200.common.registry import TRANSFORMS  # noqa: E402
from super_gradients_b200.training.datasets.detection_augment_dataset import DetectionAugmentCollateFN, DetectionAugmentDataset  # noqa: E402
from super_gradients_b200 import kernels as K  # noqa: E402
from super_gradients_b200.training.transforms import detection_augment as DA  # noqa: E402


def recipe_batch(rng, B):
    """Images fitted into 640 (longest side 640, both orientations), affine on, half of each coin flip, mixup with probability 0.5."""
    plans = []
    for _ in range(B):
        short = int(rng.integers(360, 641))
        h, w = (640, short) if rng.random() < 0.5 else (short, 640)
        mix = None
        if rng.random() < 0.5:
            s2 = int(rng.integers(360, 641))
            mix = (640, s2) if rng.random() < 0.5 else (s2, 640)
        plans.append(make_plan(rng, h, w, mixup=mix))
    return plans


class SizedStub:
    """n raw samples with a few boxes each, in get_sample() form: longest side in [longest[0], longest[1]] (640, 640: fitted into
    the mosaic's input_dim, so every tile keeps its size), the other side 0.56-1 times it, both orientations."""

    def __init__(self, rng, n, longest=(640, 640)):
        self.samples = []
        for _ in range(n):
            long_side = int(rng.integers(longest[0], longest[1] + 1))
            short = int(rng.integers(long_side * 9 // 16, long_side + 1))
            h, w = (long_side, short) if rng.random() < 0.5 else (short, long_side)
            x1, y1 = rng.uniform(0, w * 0.7, 4), rng.uniform(0, h * 0.7, 4)
            boxes = np.stack([x1, y1, x1 + rng.uniform(8, w * 0.3, 4), y1 + rng.uniform(8, h * 0.3, 4), rng.integers(0, 4, 4)], -1).astype(np.float32)
            self.samples.append({"image": _image(rng, h, w), "target": boxes})

    def __len__(self):
        return len(self.samples)

    def get_sample(self, index, ignore_empty_annotations=False):
        return {k: v.copy() for k, v in self.samples[index].items()}


def time_gpu(plans, iters):
    """(kernel ms per batch over `iters` launches, pack + copy ms per batch) of one batch of plans."""
    B = len(plans)
    aug = DA.BatchAugmenter()
    for _ in range(5):
        aug(plans, "cuda")
    torch.cuda.synchronize()
    staging, used = aug.pack(plans, pin=True)
    head = B * K.AUG_FIELDS * 8
    dev = staging[:used].cuda()
    th, td = staging[:head].view(torch.int64).view(B, K.AUG_FIELDS), dev[:head].view(torch.int64).view(B, K.AUG_FIELDS)
    out = K.empty_nhwc(B, 16, 640, 640, "cuda")
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        K.detection_augment(th, td, dev[head:], out)
    e1.record()
    torch.cuda.synchronize()
    kernel_ms = e0.elapsed_time(e1) / iters
    t0 = time.perf_counter()
    for _ in range(50):
        s, u = aug.pack(plans, pin=True)
        s[:u].to("cuda", non_blocking=True)
        torch.cuda.synchronize()
    return kernel_ms, (time.perf_counter() - t0) * 1e3 / 50


def cpu_chain_ms(plans, oracle):
    """The same pixel chain with cv2 / numpy on one CPU thread: process time per sample after a warm-up pass."""
    cv2.setNumThreads(1)
    for p in plans[:4]:
        oracle(p)
    t0 = time.process_time()
    for p in plans:
        (oracle(p) / 255.0).astype(np.float32)
    return (time.process_time() - t0) * 1e3 / len(plans)


def host_half_ms(ds, n):
    """The host half on one thread: draws, extra samples, box arithmetic and packing (DetectionAugmentDataset + collate)."""
    collate = DetectionAugmentCollateFN.for_dataset(ds)
    t0 = time.process_time()
    for _ in range(4):
        collate([ds[i] for i in range(n)])
    return (time.process_time() - t0) * 1e3 / (4 * n)


def gpu_name():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def roboflow(iters):
    """Both kinds of source: fitted into 640 (every tile is read without a resize) and of longest side 400-1000 (every tile is
    resized, up or down, in the kernel)."""
    out = {"recipe": "roboflow"}
    for name, longest in (("fitted_640", (640, 640)), ("longest_400_1000", (400, 1000))):
        ds = DetectionAugmentDataset(SizedStub(np.random.default_rng(0), 64, longest), [TRANSFORMS[n](**kw) for n, kw in ROBOFLOW])
        random.seed(0)
        np.random.seed(0)
        plans = [ds[i][0] for i in range(32)]
        per_batch = {}
        for B in (16, 32):
            kernel_ms, pack_copy_ms = time_gpu(plans[:B], iters)
            per_batch[str(B)] = {"gpu_kernel_ms_per_batch": round(kernel_ms, 3), "host_pack_copy_ms_per_batch": round(pack_copy_ms, 3)}
        out[name] = {"per_batch": per_batch, "cpu_cv2_pixel_chain_ms_per_sample_1_thread": round(cpu_chain_ms(plans, oracle_mosaic_u8), 2),
                     "host_draws_boxes_pack_ms_per_sample_1_thread": round(host_half_ms(ds, 32), 3)}  # fmt: skip
    out["gpu"] = gpu_name()
    print(json.dumps(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--iters", type=int, default=400)
    ap.add_argument("--recipe", choices=("coco", "roboflow"), default="coco")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures the GPU")
    if a.recipe == "roboflow":
        return roboflow(a.iters)
    rng = np.random.default_rng(0)
    plans = recipe_batch(rng, a.batch)
    kernel_ms, pack_copy_ms = time_gpu(plans, a.iters)
    cpu_ms = cpu_chain_ms(plans, oracle_u8)
    host_ms = host_half_ms(DetectionAugmentDataset(StubRawDataset(), [TRANSFORMS[n](**kw) for n, kw in RECIPE]), len(StubRawDataset.SIZES))
    print(json.dumps({"batch": a.batch, "gpu_kernel_ms_per_batch": round(kernel_ms, 3), "host_pack_copy_ms_per_batch": round(pack_copy_ms, 3),
                      "cpu_cv2_pixel_chain_ms_per_sample_1_thread": round(cpu_ms, 2), "host_draws_boxes_pack_ms_per_sample_1_thread": round(host_ms, 3), "gpu": gpu_name()}))  # fmt: skip

if __name__ == "__main__":
    main()
