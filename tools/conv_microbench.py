#!/usr/bin/env python
"""Per-shape timing of the convolution kernels (CUDA events, L2 flushed between iterations)."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from super_gradients_b200 import kernels as K  # noqa: E402
from super_gradients_b200 import lib  # noqa: E402

SHAPES = [
    # (n, c, h, w, k, r, stride)  YOLO-NAS-S, batch 32 (SURVEY.md appendix A)
    (32, 96, 160, 160, 96, 1, 1),
    (32, 32, 160, 160, 32, 3, 1),
    (32, 48, 320, 320, 96, 3, 2),
    (32, 64, 80, 80, 64, 3, 1),
    (32, 96, 160, 160, 192, 3, 2),
    (32, 96, 40, 40, 96, 3, 1),
    (32, 192, 80, 80, 384, 3, 2),
    (32, 384, 40, 40, 768, 3, 2),
    (32, 192, 20, 20, 192, 3, 1),
    (32, 1536, 20, 20, 768, 1, 1),
    (32, 128, 40, 40, 128, 3, 1),
]


def bench(fn, flush, iters=5):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return min(ts) * 1e3


def main():
    which = sys.argv[1] if len(sys.argv) > 1 else "fprop"
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    print(f"mode={which}")
    shapes = SHAPES[: int(os.environ.get('NSHAPES', len(SHAPES)))]
    if os.environ.get("SHAPES"):
        shapes = [tuple(int(v) for v in t.split(",")) for t in os.environ["SHAPES"].split(";")]
    for n, c, h, w, k, r, s in shapes:
        pad = r // 2
        x = torch.randn(n, c, h, w, device="cuda").bfloat16().contiguous(memory_format=torch.channels_last)
        wt = torch.randn(k, c, r, r, device="cuda") * 0.05
        krsc, crsk = K.weight_prepare(wt)
        P, Q = (h + 2 * pad - r) // s + 1, (w + 2 * pad - r) // s + 1
        y = K.empty_nhwc(n, k, P, Q, "cuda")
        stats = K.new_stats(k, "cuda")
        flops = 2.0 * n * P * Q * k * c * r * r
        bytes_ = 2.0 * (x.numel() + y.numel())
        n0 = lib.load().sgb_sm100_launches()
        if which == "fprop":
            us = bench(lambda: K.conv_fprop(x, krsc, k, r, r, s, pad, stats=None if os.environ.get('NOSTATS') else stats, out=y), flush)
        elif which == "dgrad":
            dx = torch.empty_like(x)
            us = bench(lambda: K.conv_dgrad(y, crsk, x.shape, r, r, s, pad, out=dx), flush)
        else:
            dw = torch.zeros(k, r, r, c, device="cuda")
            us = bench(lambda: K.conv_wgrad(x, y, r, r, s, pad, dw_krsc=dw), flush)
        used = lib.load().sgb_sm100_launches() > n0
        print(f"{which} C={c:4d} {h}x{w} K={k:4d} r={r} s={s}: {us:8.1f} us  {flops / us / 1e6:7.1f} TFLOP/s  {bytes_ / us / 1e3:7.1f} GB/s(min traffic)  wgmma={used}")


if __name__ == "__main__":
    main()
