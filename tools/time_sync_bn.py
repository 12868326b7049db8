#!/usr/bin/env python
"""Times the config-2 training step (YOLO-NAS-S 640 x 640, 32 images per GPU, AdamW + EMA, CUDA graph; bench.py's workload) with
sync_bn off and on, in one process.  Per mode: ms/step as the median of device-event-timed graph replays after warm-up, our kernel
launches in one eager step (lib.LAUNCHES, as bench.py counts them) and the BatchNorm reductions of one step (functional.SYNC_CALLS;
at world size 1 they are identities and no collective is issued).  Prints one JSON line per mode, from rank 0.

    python tools/time_sync_bn.py [--steps 30 --warmup 5]                      # one GPU
    torchrun --nproc-per-node N tools/time_sync_bn.py [--steps 30 --warmup 5]  # N GPUs over NCCL
"""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def run_mode(sync_bn, steps, warmup, dev, rank, world):
    import bench
    from super_gradients_b200 import functional as SF
    from super_gradients_b200 import lib
    from super_gradients_b200.training.sg_trainer import TrainStep

    cfg = bench.CONFIGS[2]
    model, step, host = bench.build_train_workload(cfg, dev, rank, cfg["batch"])
    if sync_bn:
        model = nn.SyncBatchNorm.convert_sync_batchnorm(model)
        step = TrainStep(model, step.criterion, "AdamW", {"weight_decay": 1e-5}, zero_wd_on_bias_and_bn=True, ema=True)
    xs = [x.to(dev) for x, _ in host]
    ts = [tuple(t.to(dev) for t in tt) for _, tt in host]
    step.set_hyper_params(2e-4, 0.9997)
    lib.LAUNCHES[0], calls0 = 0, SF.SYNC_CALLS[0]
    step.run(xs[0], ts[0])
    torch.cuda.synchronize()
    launches, reductions = lib.LAUNCHES[0], SF.SYNC_CALLS[0] - calls0
    step.capture(xs[0], ts[0], warmup=2)
    times = []
    for i in range(warmup + steps):
        step.set_hyper_params(2e-4, 0.9997)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        step.run(xs[i % len(xs)], ts[i % len(ts)])
        b.record()
        b.synchronize()
        if i >= warmup:
            times.append(a.elapsed_time(b))
    times.sort()
    med = times[len(times) // 2] if len(times) % 2 else (times[len(times) // 2 - 1] + times[len(times) // 2]) / 2
    n_bn = sum(isinstance(m, nn.modules.batchnorm._BatchNorm) for m in model.modules())
    return {"sync_bn": sync_bn, "world": world, "ms_per_step_median": round(med, 3), "ms_min": round(times[0], 3), "ms_max": round(times[-1], 3), "timed_steps": steps,
            "our_launches_per_step": launches, "bn_reductions_per_step": reductions, "bn_collectives_issued_per_step": reductions if world > 1 else 0, "batchnorm_modules": n_bn,
            "graph": type(step.graph).__name__}  # fmt: skip


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    from super_gradients_b200.training.sg_trainer import setup_device

    dev = setup_device()
    rank = dist.get_rank() if dist.is_initialized() else 0
    world = dist.get_world_size() if dist.is_initialized() else 1
    if not dist.is_initialized():  # world size 1: a one-rank NCCL group, so that SyncBatchNorm layers take the synced path
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29591")
        dist.init_process_group("nccl", init_method="env://", rank=0, world_size=1, device_id=dev)
    gpu = torch.cuda.get_device_name()
    try:
        for sync_bn in (False, True):
            r = run_mode(sync_bn, args.steps, args.warmup, dev, rank, world)
            if rank == 0:
                print(json.dumps({**r, "gpu": gpu}), flush=True)
    finally:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
