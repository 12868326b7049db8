"""Skipping the zero taps of folded QARepVGG filters (SgbConvDesc.centre_from): per-shape timings of fprop, dgrad and wgrad.

    python tools/time_zero_taps.py [--configs 2 3] [--rounds 7] [--iters 40]

Prints the card and its power limit, then one line per folded convolution shape of the configurations' training steps (shapes
taken from one batch-1 eager step, N scaled to the configuration's batch) and per pass: the engine, median us per call with
centre_from on and off (the two arms alternated round by round, CUDA events over `iters` launches), and the MMA FLOP each arm
issues, counted from the shapes and the kernels' tiles (padding included).
"""
import argparse
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

import bench  # noqa: E402
from super_gradients_b200 import kernels as K  # noqa: E402
from super_gradients_b200 import lib  # noqa: E402
from super_gradients_b200.training.sg_trainer import setup_device  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, check=True)
        return q.stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return torch.cuda.get_device_name()


def collect_shapes(cfg_id, dev):
    """{(N, H, W, C, 2K)} of the folded convolutions (calls with centre_from) of one batch-1 step, N scaled to the batch."""
    cfg = bench.CONFIGS[cfg_id]
    seen = set()
    orig = K.conv_fprop

    def spy(x, w, kout, *a, centre_from=0, **kw):
        if centre_from:
            n, c, h, wd = x.shape
            seen.add((n * cfg["batch"], h, wd, c, kout))
        return orig(x, w, kout, *a, centre_from=centre_from, **kw)

    K.conv_fprop = spy
    try:
        _model, step, host = bench.build_train_workload(cfg, dev, 0, 1)
        x, t = bench._to_dev(host[0], dev)
        step.set_hyper_params(2e-4, 0.9997)
        step._step_eager(x, t)
        torch.cuda.synchronize()
    finally:
        K.conv_fprop = orig
    return seen


def pick_bn(n):  # conv_sm100.cu pick_bn
    for bn in (16, 32, 48, 64, 96, 128):
        if n <= bn:
            return bn
    best, waste = 128, -n % 128
    for bn in (96, 64):
        if -n % bn < waste:
            best, waste = bn, -n % bn
    return best


def issued_flop(op, engine, n, h, w, c, k2, cf):
    """MMA FLOP the kernels issue (M, N and K padded to their tiles) with centre_from = cf (0: every tap)."""
    if op == "wgrad":  # M = dy rows in 64-row blocks, N = C, K = pixels
        rows_all = -(-k2 // 64) * 64
        rows_off = -(-cf // 64) * 64 if cf else rows_all
        return 2.0 * n * h * w * c * (rows_all + 8 * rows_off)
    gather, nout = (c, k2) if op == "fprop" else (k2, c)
    m = n * -(-h // 8) * -(-w // 8) * 64 if engine == "halo" else -(-n * h * w // 128) * 128
    kc = 16 if engine == "halo" else (64 if gather > 32 else (32 if gather % 32 == 0 else 16))
    depth = -(-gather // kc) * kc
    bn = pick_bn(nout)
    total = 0
    for n0 in range(0, nout, bn):
        off_depth = depth  # a tile that straddles cf runs every tap
        if cf and op == "fprop" and n0 >= cf and engine != "halo":  # the halo kernel runs every tap of fprop
            off_depth = 0
        if cf and op == "dgrad":
            off_depth = -(-cf // kc) * kc
        total += bn * depth + 8 * bn * off_depth
    return 2.0 * m * total


def make_call(op, n, h, w, c, k2, dev):
    g = torch.Generator(device=dev).manual_seed(0)
    wt = torch.zeros(k2, c, 3, 3, device=dev)
    wt[: k2 // 2] = torch.randn(k2 // 2, c, 3, 3, generator=g, device=dev) * 0.05
    wt[k2 // 2 :, :, 1, 1] = torch.randn(k2 - k2 // 2, c, generator=g, device=dev) * 0.2
    krsc, crsk = K.weight_prepare(wt)
    x = torch.randn(n, h, w, c, generator=g, device=dev).to(torch.bfloat16).permute(0, 3, 1, 2)
    dy = torch.randn(n, h, w, k2, generator=g, device=dev).to(torch.bfloat16).permute(0, 3, 1, 2)
    if op == "fprop":
        y, st = K.empty_nhwc(n, k2, h, w, dev), K.new_stats(k2, dev)
        return lambda cf: K.conv_fprop(x, krsc, k2, 3, 3, 1, 1, out=y, stats=st, centre_from=cf)
    if op == "dgrad":
        dx = K.empty_nhwc(n, c, h, w, dev)
        return lambda cf: K.conv_dgrad(dy, crsk, (n, c, h, w), 3, 3, 1, 1, out=dx, centre_from=cf)
    dw = torch.zeros(k2, 3, 3, c, dtype=torch.float32, device=dev)
    return lambda cf: K.conv_wgrad(x, dy, 3, 3, 1, 1, dw_krsc=dw, centre_from=cf)


def time_calls(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) * 1e3 / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", type=int, nargs="+", default=[2, 3])
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=40)
    args = ap.parse_args()
    dev = setup_device()
    lib.call("sgb_check_device")
    L = lib.load()
    print(f"card: {card()}")
    shapes = {}
    for c in args.configs:
        for s in collect_shapes(c, dev):
            shapes.setdefault(s, []).append(c)
    print(f"{'op':5s} {'N':>4s} {'HxW':>9s} {'C':>4s} {'2K':>4s} {'cfg':>5s} {'engine':>6s} {'all us':>8s} {'skip us':>8s} {'gain':>6s}"
          f" {'all GFLOP':>9s} {'skip GFLOP':>10s} {'issued':>6s}")
    tot = {}
    for (n, h, w, c, k2), cfgs in sorted(shapes.items(), key=lambda kv: (-kv[0][1], kv[0][3], kv[0][4], kv[0][0])):
        for op in ("fprop", "dgrad", "wgrad"):
            fn = make_call(op, n, h, w, c, k2, dev)
            h0 = L.sgb_conv_halo_launches()
            fn(k2 // 2)
            engine = "halo" if L.sgb_conv_halo_launches() > h0 else ("im2col" if op != "wgrad" else "wgrad")
            fn(0)
            t_all, t_skip = [], []
            for _ in range(args.rounds):
                t_all.append(time_calls(lambda: fn(0), args.iters))
                t_skip.append(time_calls(lambda: fn(k2 // 2), args.iters))
            ta, ts = statistics.median(t_all), statistics.median(t_skip)
            fa, fs = issued_flop(op, engine, n, h, w, c, k2, 0), issued_flop(op, engine, n, h, w, c, k2, k2 // 2)
            for cfg in cfgs:
                acc = tot.setdefault((cfg, op), [0.0, 0.0])
                acc[0] += ta
                acc[1] += ts
            print(f"{op:5s} {n:4d} {h:4d}x{w:<4d} {c:4d} {k2:4d} {','.join(map(str, cfgs)):>5s} {engine:>6s} {ta:8.1f} {ts:8.1f} {ta / ts:6.3f}"
                  f" {fa / 1e9:9.1f} {fs / 1e9:10.1f} {fs / fa:6.3f}", flush=True)
    print("per configuration, one call of each distinct shape (not weighted by how often a step runs it):")
    for (cfg, op), (ta, ts) in sorted(tot.items()):
        print(f"  config {cfg} {op}: all taps {ta:8.1f} us, skipping {ts:8.1f} us, ratio {ta / ts:.3f}")


if __name__ == "__main__":
    main()
