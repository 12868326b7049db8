"""The train-mode QARepVGG stem with [y3 | u] stored (functional.STEM_RECOMPUTE off) and recomputed (on): per-pass timings.

    python tools/time_stem.py [--batch 32] [--size 640] [--rounds 5] [--iters 20]

Runs the YOLO-NAS-S stem block (QARepVGG 3 -> 48, 3 x 3 stride 2) forward + backward at the benchmark's size, the two arms alternated
round by round.  Prints the card, its power limit and SM clock, then per arm the median over rounds of the forward + backward wall time
(CUDA events around `iters` repetitions) and, from a second pass with per-launch CUDA events, the median us of each launch of the block
with the bytes it must move (computed from the shapes) over its time, against the H100 SXM data-sheet 3.35 TB/s.
"""
import argparse
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from super_gradients_b200 import functional as SF  # noqa: E402
from super_gradients_b200 import kernels as K  # noqa: E402
from super_gradients_b200.modules import QARepVGGBlock  # noqa: E402

HBM = 3.35e12


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, check=True)
        return q.stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return torch.cuda.get_device_name()


def pass_bytes(m, k):
    """Bytes each launch must move at m output pixels and k stem channels (bf16; xp has 32 patch channels)."""
    xp, y, cat = 64 * m, 2 * k * m, 4 * k * m
    return {
        "sgb_conv_fprop": xp + cat,  # the patch GEMM writes [y3 | u]
        "sgb_qarep_fwd_fused": 2 * cat + y,  # moments half reads [y3 | u], apply half reads it again and writes out
        "sgb_qarep_bwd_fused": 2 * (y + cat) + cat,  # reduce and apply halves read dout and [y3 | u]; apply writes [dy3 | du]
        "sgb_stem_qarep_moments": xp,
        "sgb_stem_qarep_fwd": xp + y,
        "sgb_stem_qarep_bwd_reduce": xp + y,
        "sgb_stem_qarep_bwd_apply": xp + y + cat,
        "sgb_conv_wgrad": cat + xp,
        "sgb_stem_patches_f32": 4 * 3 * 4 * m + xp,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", type=int, default=640)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    dev = torch.device("cuda")
    print(f"card: {card()}")
    torch.manual_seed(0)
    x = torch.randn(args.batch, 3, args.size, args.size, device=dev)
    blk = QARepVGGBlock(3, 48, stride=2, use_residual_connection=False).to(dev).train()
    m = args.batch * (args.size // 2) ** 2
    gy = torch.randn(args.batch, 48, args.size // 2, args.size // 2, device=dev).bfloat16().contiguous(memory_format=torch.channels_last)

    def step():
        blk(x).backward(gy)

    arms = {"stored": False, "recompute": True}
    wall = {a: [] for a in arms}
    per = {a: {} for a in arms}
    for a, on in arms.items():  # warm-up of every shape
        SF.STEM_RECOMPUTE[0] = on
        for _ in range(3):
            step()
    torch.cuda.synchronize()
    for _ in range(args.rounds):
        for a, on in arms.items():
            SF.STEM_RECOMPUTE[0] = on
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.iters):
                step()
            e1.record()
            torch.cuda.synchronize()
            wall[a].append(e0.elapsed_time(e1) * 1e3 / args.iters)
            K.PROFILE.clear()
            K.PROFILE_ON[0] = True
            step()
            K.PROFILE_ON[0] = False
            torch.cuda.synchronize()
            for name, b0, b1, _tag in K.PROFILE:
                per[a].setdefault(name, []).append(b0.elapsed_time(b1) * 1e3)
            K.PROFILE.clear()
    nb = pass_bytes(m, 48)
    for a in arms:
        print(f"{a}: forward + backward median {statistics.median(wall[a]):.1f} us (rounds: {' '.join(f'{v:.0f}' for v in wall[a])})")
        for name, ts in per[a].items():
            us = statistics.median(ts)
            bw = f"{nb[name] / 1e6:.0f} MB, {nb[name] / us / 1e6:.2f} TB/s = {nb[name] / us / 1e6 / (HBM / 1e12) * 100:.0f} % of 3.35 TB/s" if name in nb else ""
            print(f"  {name:28s} {us:9.1f} us  {bw}")
    print(f"speed-up of forward + backward: {statistics.median(wall['stored']) / statistics.median(wall['recompute']):.3f}x")


if __name__ == "__main__":
    main()
