#!/usr/bin/env python
"""Times the best-snapshot average of Trainer.train(average_best_models=True) at k = 10 slots for the float32 state of YOLO-NAS-S,
YOLO-NAS-L and YOLO-NAS-POSE-L:

  - kernel: sgb_average_snapshots alone (CUDA events, median of the timed launches), with the bytes it must move (k * n * 4 read,
    n * 4 written) over that time and over the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s);
  - average: what ModelWeightAveraging.get_average_model does per validated epoch -- the launch plus one device-to-host copy into
    pinned memory (host clock around a synchronise, median);
  - CPU loop: the reference's running mean in torch on this host's CPU (weight_averaging_utils.py:89-95), over the same n floats.

Prints the card's name and power limit with the numbers.  Usage: python tools/time_weight_averaging.py [--iters 20] [--cpu-iters 3]"""
import argparse
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

MODELS = (("yolo_nas_s", 80), ("yolo_nas_l", 80), ("yolo_nas_pose_l", 17))
HBM_TBPS = 3.35


def float_state_numel(name, num_classes):
    from super_gradients_b200.training import models

    sd = models.get(name, num_classes=num_classes).state_dict()
    return sum(v.numel() for v in sd.values() if v.dtype == torch.float32)


def time_kernel(n, k, iters):
    from super_gradients_b200 import kernels as K

    slots = torch.randn(k, n, device="cuda")
    table = torch.tensor([slots[j].data_ptr() for j in range(k)], dtype=torch.int64, device="cuda")
    out = torch.empty(n, device="cuda")
    host = torch.empty(n, pin_memory=True)
    for _ in range(3):
        K.average_snapshots(table, k, out)
    torch.cuda.synchronize()
    kernel = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        K.average_snapshots(table, k, out)
        b.record()
        b.synchronize()
        kernel.append(a.elapsed_time(b))
    average = []
    for _ in range(iters):
        t0 = time.perf_counter()
        K.average_snapshots(table, k, out)
        host.copy_(out)
        torch.cuda.synchronize()
        average.append((time.perf_counter() - t0) * 1e3)
    del slots
    return statistics.median(kernel), statistics.median(average)


def time_cpu_loop(n, k, iters):
    slots = [torch.randn(n) for _ in range(k)]
    times = []
    for _ in range(iters):
        t0 = time.perf_counter()
        a = slots[0].clone()
        for m in range(1, k):
            a = torch.true_divide(a * m + slots[m], (m + 1))
        times.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--cpu-iters", type=int, default=3)
    ap.add_argument("--k", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device: this tool times the sm_90a kernel")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()[0]
    print(f"card: {card}; k = {args.k}; torch {torch.__version__}, {torch.get_num_threads()} CPU threads")
    print("| model | float32 entries | slots (GB) | kernel (ms) | kernel GB/s | of 3.35 TB/s | kernel + D2H (ms) | CPU loop (ms) |")
    print("|---|---|---|---|---|---|---|---|")
    for name, ncls in MODELS:
        n = float_state_numel(name, ncls)
        kernel, average = time_kernel(n, args.k, args.iters)
        cpu = time_cpu_loop(n, args.k, args.cpu_iters)
        moved = (args.k + 1) * n * 4
        gbps = moved / kernel / 1e6
        print(f"| {name} | {n / 1e6:.2f} M | {args.k * n * 4 / 1e9:.2f} | {kernel:.3f} | {gbps:.0f} | {gbps / (HBM_TBPS * 1e3):.0%} | {average:.1f} | {cpu:.0f} |")


if __name__ == "__main__":
    main()
