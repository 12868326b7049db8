"""Times the pose train augmentation at 640 x 640 for batches of 24 and 48 drawn by the mosaic (N / S) and the mosaic-heavy (M / L)
YOLO-NAS-POSE recipe lists over seeded 480 x 640-class images: the two kernel launches per batch (CUDA events over many calls), the
host pack + host-to-device copy per batch, and on one CPU thread (process time) the loader's host half per sample (draws, joint /
box arithmetic, packing), the brightness-contrast channel mean inside it, and the cv2 / numpy pixel chain per sample.  Prints one
JSON line with the card name and power limit.  Usage: python tools/time_pose_augment.py [--iters N]"""
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
from pose_augment_cases import GOLDEN_LISTS, StubPoseDataset, build, oracle_u8  # noqa: E402
from super_gradients_b200 import kernels as K  # noqa: E402
from super_gradients_b200.training.datasets.pose_estimation_datasets.pose_augment_dataset import PoseAugmentCollateFN, PoseAugmentDataset  # noqa: E402
from super_gradients_b200.training.transforms import keypoints as KP  # noqa: E402


def items(name, B):
    ds = PoseAugmentDataset(StubPoseDataset(), build(GOLDEN_LISTS[name], KP))
    random.seed(0)
    np.random.seed(0)
    return ds, [ds[i % len(ds)] for i in range(B)]


def kernel_ms(batch, iters):
    used = batch.buffer.numel()
    head = batch.batch * K.POSE_FIELDS * 8
    host = batch.buffer.pin_memory()
    dev = host.cuda()
    th, td = host[:head].view(torch.int64).view(batch.batch, K.POSE_FIELDS), dev[:head].view(torch.int64).view(batch.batch, K.POSE_FIELDS)
    ws = torch.empty(used - head, dtype=torch.uint8, device="cuda")
    out = K.empty_nhwc(batch.batch, 16, 640, 640, "cuda")
    for _ in range(5):
        K.pose_augment(th, td, dev[head:], ws, out)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        K.pose_augment(th, td, dev[head:], ws, out)
    e1.record()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(20):
        batch.buffer.pin_memory().to("cuda", non_blocking=True)
        torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters, (time.perf_counter() - t0) * 1e3 / 20


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures the GPU")
    cv2.setNumThreads(1)
    res = {}
    for name in ("mosaic", "heavy"):
        for B in (24, 48):
            ds, it = items(name, B)
            batch = PoseAugmentCollateFN.for_dataset(ds)(it)
            k, pc = kernel_ms(batch, a.iters)
            res[f"{name}_b{B}_gpu_kernel_ms_per_batch"] = round(k, 3)
            res[f"{name}_b{B}_host_pack_copy_ms_per_batch"] = round(pc, 3)
        ds, it = items(name, 48)
        plans = [p for p, _ in it]
        t0 = time.process_time()
        for p in plans:
            np.divide(oracle_u8(p), 255.0, dtype=np.float32)
        res[f"{name}_cpu_cv2_pixel_chain_ms_per_sample_1_thread"] = round((time.process_time() - t0) * 1e3 / len(plans), 2)
        collate = PoseAugmentCollateFN.for_dataset(ds)
        t0 = time.process_time()
        collate([ds[i % len(ds)] for i in range(48)])
        res[f"{name}_host_half_ms_per_sample_1_thread"] = round((time.process_time() - t0) * 1e3 / 48, 3)
    img = StubPoseDataset().samples[0]["image"]
    t0 = time.process_time()
    for _ in range(20):
        np.mean(np.ascontiguousarray(np.fliplr(img)).astype(np.float32), axis=(0, 1))
    res["bc_mean_ms_per_480x640_image_1_thread"] = round((time.process_time() - t0) * 1e3 / 20, 3)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    res["gpu"] = q[0] if q else "unknown"
    print(json.dumps(res))


if __name__ == "__main__":
    main()
