#!/usr/bin/env python
"""Times one optimizer update over the live float32 parameters of YOLO-NAS-S and YOLO-NAS-L (the flat buffers of
training/flat_state.py with zero_weight_decay_on_bias_and_bn, so two weight-decay ranges) with each of SGD, AdamW, Adam, RMSprop,
RMSpropTF, Lion and Lamb through FlatOptimizer.  CUDA events around the launches of one step, median of --iters steps.  Reports the
bytes each update must move (every state and parameter read and written once, the gradient read once) over that time, against the H100 SXM
data-sheet HBM3 bandwidth (3.35 TB/s).  Lamb's first launch (the global gradient sum of squares) is also timed on its own.

Prints the card's name and power limit with the numbers.  Usage: python tools/time_optimizers.py [--iters 20]"""
import argparse
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

MODELS = ("yolo_nas_s", "yolo_nas_l")
HBM_TBPS = 3.35
# bytes per element of one update: (reads + writes) * 4
BYTES = {"SGD": 5 * 4, "AdamW": 7 * 4, "Adam": 7 * 4, "RMSprop": 7 * 4, "RMSpropTF": 7 * 4, "Lion": 5 * 4, "Lamb": 11 * 4}
OPTIMIZERS = (("SGD", {}), ("AdamW", {}), ("Adam", {}), ("RMSprop", {}), ("RMSpropTF", {}), ("Lion", {}), ("Lamb", {}))


def median_ms(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return statistics.median(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device: this tool times the sm_90a kernels")
    from super_gradients_b200 import kernels as K
    from super_gradients_b200.training import fused_optimizers as FO
    from super_gradients_b200.training import models
    from super_gradients_b200.training.flat_state import FlatState

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()[0]
    print(f"card: {card}; median of {args.iters} steps; torch {torch.__version__}")
    print("| model | live params | optimizer | launches | step (us) | bytes moved (MB) | GB/s | of 3.35 TB/s | Lamb gradient-norm pass (us) |")
    print("|---|---|---|---|---|---|---|---|---|")
    for name in MODELS:
        model = models.get(name, num_classes=80).cuda()
        flat = FlatState(model, True)
        flat.grads.normal_()
        n = flat.n_live
        for opt, params in OPTIMIZERS:
            op, wd = FO.resolve(opt, params, True)
            fo = FO.FlatOptimizer(opt, op, wd, flat)
            hp = torch.tensor(fo.rows(1e-4, 10, 1.0), dtype=torch.float32, device="cuda")

            def step():
                fo.step(flat, hp)

            launches = 3 if opt == "Lamb" else 2
            extra = ""
            if opt == "Lamb":
                extra = f"{median_ms(lambda: K.lamb_grad_sqnorm(flat.grads, fo.chunks, hp, fo.partials), args.iters) * 1e3:.1f}"
            ms = median_ms(step, args.iters)
            moved = BYTES[opt] * n
            gbps = moved / ms / 1e6
            print(f"| {name} | {n / 1e6:.2f} M | {opt} | {launches} | {ms * 1e3:.1f} | {moved / 1e6:.1f} | {gbps:.0f} | {gbps / (HBM_TBPS * 1e3):.0%} | {extra} |")
            del step
        del model, flat
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
