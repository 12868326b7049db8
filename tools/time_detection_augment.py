"""Times the detection train augmentation for B = 32 at 640 x 640 on the recipe chain's draws: the GPU kernel per batch (CUDA
events), the host pack + host-to-device copy per batch, the host half of the transforms per sample (draws, boxes, packing) and the
same pixel chain with cv2 / numpy per sample, both as process time on one CPU thread, in one process.  Prints one JSON line with the card name and power limit.  Usage: python tools/time_detection_augment.py [--iters N]"""
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

import cv2  # noqa: E402
from augment_cases import RECIPE, StubRawDataset, make_plan, oracle_u8  # noqa: E402
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--iters", type=int, default=400)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures the GPU")
    rng = np.random.default_rng(0)
    plans = recipe_batch(rng, a.batch)
    aug = DA.BatchAugmenter()
    for _ in range(5):
        aug(plans, "cuda")
    torch.cuda.synchronize()

    staging, used = aug.pack(plans, pin=True)
    head = a.batch * K.AUG_FIELDS * 8
    dev = staging[:used].cuda()
    th, td = staging[:head].view(torch.int64).view(a.batch, K.AUG_FIELDS), dev[:head].view(torch.int64).view(a.batch, K.AUG_FIELDS)
    out = K.empty_nhwc(a.batch, 16, 640, 640, "cuda")
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.iters):
        K.detection_augment(th, td, dev[head:], out)
    e1.record()
    torch.cuda.synchronize()
    kernel_ms = e0.elapsed_time(e1) / a.iters

    t0 = time.perf_counter()
    for _ in range(50):
        s, u = aug.pack(plans, pin=True)
        s[:u].to("cuda", non_blocking=True)
        torch.cuda.synchronize()
    pack_copy_ms = (time.perf_counter() - t0) * 1e3 / 50

    # the same pixel chain with cv2 / numpy on one CPU thread: process time per sample after one warm-up pass
    cv2.setNumThreads(1)
    for p in plans[:4]:
        oracle_u8(p)
    t0 = time.process_time()
    for p in plans:
        (oracle_u8(p) / 255.0).astype(np.float32)
    cpu_ms = (time.process_time() - t0) * 1e3 / len(plans)
    # the host half on the same thread: draws, mixup partner, box arithmetic and packing (DetectionAugmentDataset + collate)
    ds = DetectionAugmentDataset(StubRawDataset(), [TRANSFORMS[n](**kw) for n, kw in RECIPE])
    collate = DetectionAugmentCollateFN.for_dataset(ds)
    t0 = time.process_time()
    for _ in range(4):
        collate([ds[i] for i in range(len(ds))])
    host_ms = (time.process_time() - t0) * 1e3 / (4 * len(ds))

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    print(json.dumps({"batch": a.batch, "gpu_kernel_ms_per_batch": round(kernel_ms, 3), "host_pack_copy_ms_per_batch": round(pack_copy_ms, 3),
                      "cpu_cv2_pixel_chain_ms_per_sample_1_thread": round(cpu_ms, 2), "host_draws_boxes_pack_ms_per_sample_1_thread": round(host_ms, 3), "gpu": q[0] if q else "unknown"}))  # fmt: skip


if __name__ == "__main__":
    main()
