"""Per-shape table of the convolution calls of one eager training step (CUDA events around every C-ABI call, side-stream weight
gradients off so nothing overlaps): count, total ms, average us, algorithmic activation bytes -> GB/s, FLOP -> TF/s.
Tells which shapes of which engine are furthest from the HBM / tensor rooflines.

    python tools/conv_table.py [--model yolo_nas_s] [--batch 32] [--top 60] > conv_table.txt
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

import bench  # noqa: E402
from super_gradients_b200 import kernels as K  # noqa: E402
from super_gradients_b200.training import models  # noqa: E402
from super_gradients_b200.training.losses import PPYoloELoss, pad_targets_host  # noqa: E402
from super_gradients_b200.training.sg_trainer import TrainStep, setup_device  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--model", default="yolo_nas_s")
    ap.add_argument("--top", type=int, default=70)
    ap.add_argument("--all", action="store_true", help="every C-ABI call, not only the convolutions")
    ap.add_argument("--config", type=int, default=0, help="a bench.py training configuration (3: YOLO-NAS-M, 4: ResNet-50) instead of --model / --batch")
    args = ap.parse_args()
    dev = setup_device()
    torch.manual_seed(0)
    if args.config:
        cfg = bench.CONFIGS[args.config]
        args.model, args.batch = cfg["model"], cfg["batch"]
        model, step, host = bench.build_train_workload(cfg, dev, 0, args.batch)
        x, t = bench._to_dev(host[0], dev)
    else:
        model = models.get(args.model, num_classes=bench.NCLS).to(dev).train()
        crit = PPYoloELoss(num_classes=bench.NCLS, use_static_assigner=False)
        step = TrainStep(model, crit, "AdamW", {"weight_decay": 1e-5}, zero_wd_on_bias_and_bn=True, ema=True)
        x, t = bench.synth_batch(args.batch, 0)
        x = x.to(dev)
        t = tuple(a.to(dev) for a in pad_targets_host(t, args.batch, bench.NBOX))
    step.ctx.side_stream = None  # weight gradients on the main stream: no call overlaps another's events
    for _ in range(3):
        step.set_hyper_params(2e-4, 0.9997)
        step._step_eager(x, t)
    torch.cuda.synchronize()
    # which engine served each convolution call: the library counts launches of the wgmma / TMA kernels
    lib = K.L.load()
    engines = []
    orig_call = K.L.call

    def call(name, *a):
        if not name.startswith("sgb_conv_"):
            return orig_call(name, *a)
        u0 = lib.sgb_sm100_launches()
        rc = orig_call(name, *a)
        u1 = lib.sgb_sm100_launches()
        engines.append("wgmma" if u1 > u0 else "mma.sync")
        return rc

    K.L.call = call
    K.PROFILE.clear()
    K.PROFILE_ON[0] = True
    n = 3
    for _ in range(n):
        step.set_hyper_params(2e-4, 0.9997)
        step._step_eager(x, t)
    torch.cuda.synchronize()
    K.PROFILE_ON[0] = False
    K.L.call = orig_call
    agg = {}
    eng = iter(engines)
    for name, a, b, tag in K.PROFILE:
        if name.startswith("sgb_conv_"):
            name = name + ":" + next(eng)
        elif not args.all:
            continue
        d = agg.setdefault((name, tag), [0, 0.0])
        d[0] += 1
        d[1] += a.elapsed_time(b)
    rows = []
    for (name, tag), (cnt, ms) in agg.items():
        us = ms / cnt * 1e3
        gbs = tfs = 0.0
        desc = ""
        if len(tag) == 7:
            N, H, W, C, Kc, R, s = tag
            P, Q = (H + s - 1) // s, (W + s - 1) // s
            byts = 2.0 * N * (H * W * C + P * Q * Kc)
            flop = 2.0 * N * P * Q * Kc * C * R * R
            gbs, tfs = byts / us / 1e3, flop / us / 1e6
            desc = f"C={C:4d} K={Kc:4d} {R}x{R} s{s} {H:3d}x{W:3d}"
        rows.append((ms / n, cnt // n, us, name, desc, gbs, tfs))
    rows.sort(reverse=True)
    tot = sum(r[0] for r in rows)
    by_engine = {}
    for ms, cnt, us, name, desc, gbs, tfs in rows:
        if ":" in name:
            e = by_engine.setdefault(name.split("_", 1)[1], [0, 0.0])
            e[0] += cnt
            e[1] += ms
    for k, (cnt, ms) in sorted(by_engine.items(), key=lambda kv: -kv[1][1]):
        print(f"  {k:24s} {cnt:4d} calls  {ms:7.3f} ms/step")
    print(f"{args.model} batch {args.batch}: {tot:.3f} ms/step in the listed calls (eager, events per call, no side stream)")
    print(f"{'ms/step':>8s} {'n':>3s} {'avg us':>8s}  {'call':24s} {'shape':32s} {'GB/s':>7s} {'TF/s':>7s}")
    for ms, cnt, us, name, desc, gbs, tfs in rows[: args.top]:
        print(f"{ms:8.3f} {cnt:3d} {us:8.1f}  {name[4:]:24s} {desc:32s} {gbs:7.0f} {tfs:7.1f}")


if __name__ == "__main__":
    main()
