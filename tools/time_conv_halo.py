"""Halo-tile kernels against the im2col / per-tap wgmma kernels on the 3x3 / stride-1 convolutions of the bench.py configurations.

    python tools/time_conv_halo.py [--configs 2 3 4 5] [--rounds 5] [--iters 30] [--step-rounds 5] [--step-iters 20]

Prints the card and its power limit, then
  1. a per-shape table: every 3x3 / stride-1 fprop, dgrad and wgrad shape of the configurations at their batch sizes (shapes
     taken from one batch-1 step of each model; cf: the centre_from of a folded QARepVGG weight gradient), the two kernels
     alternated round by round and timed by CUDA events over many launches: median us per call, the algorithmic HBM bytes
     (input + output + filter, once each; wgrad: x + dy + the fp32 dW) and FLOP (the full 3x3 filter), and the rates against the
     H100 SXM data-sheet figures (3.35 TB/s, 989 dense BF16 TFLOP/s); for the fprop / dgrad halo kernel also the bytes it moves
     L2 -> shared memory (10 x 10 halo per 8 x 8 tile) as a rate;
  2. the config-2 TrainStep CUDA graph captured twice (im2col forced, and the automatic choice), replays alternated: median ms
     per step and the spread (max - min) of each arm.
The engine switches are the library's test-only sgb_conv_force_im2col (fprop / dgrad) and sgb_conv_wgrad_force_im2col (wgrad).
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
from super_gradients_b200.training import models  # noqa: E402
from super_gradients_b200.training.sg_trainer import setup_device  # noqa: E402

PEAK_BW, PEAK_TF = 3.35e12, 989e12


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, check=True)
        return q.stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return torch.cuda.get_device_name()


def collect_shapes(cfg_id, dev):
    """{(op, N, H, W, C, K, cf)} of the 3x3 / stride-1 convolutions of one batch-1 step, N scaled to the configuration's batch."""
    cfg = bench.CONFIGS[cfg_id]
    K.PROFILE.clear()
    shapes = set()
    orig_wgrad = K.conv_wgrad

    def spy(x, dy, R, S, stride, pad, dw_krsc=None, centre_from=0):
        if R == 3 and stride == 1:
            n, c, h, w = x.shape
            shapes.add(("wgrad", n * cfg["batch"], h, w, c, dy.shape[1], centre_from))
        return orig_wgrad(x, dy, R, S, stride, pad, dw_krsc, centre_from)

    K.conv_wgrad = spy
    if cfg["kind"] == "predict_pose":
        model = models.get(cfg["model"], num_classes=17).to(dev).eval()
        from super_gradients_b200.training.processing import default_yolo_nas_pose_coco_processing_params

        proc = default_yolo_nas_pose_coco_processing_params()["image_processor"]
        x = proc.preprocess_batch(bench.synth_images_u8(1, 0, cfg["img"]), dev)[0]
        K.PROFILE_ON[0] = True
        with torch.no_grad():
            model(x)
    else:
        _model, step, host = bench.build_train_workload(cfg, dev, 0, 1)
        x, t = bench._to_dev(host[0], dev)
        step.set_hyper_params(2e-4, 0.9997)
        K.PROFILE_ON[0] = True
        step._step_eager(x, t)
    K.conv_wgrad = orig_wgrad
    torch.cuda.synchronize()
    K.PROFILE_ON[0] = False
    for name, _a, _b, tag in K.PROFILE:
        if name in ("sgb_conv_fprop", "sgb_conv_dgrad") and len(tag) == 7 and tag[5] == 3 and tag[6] == 1:
            n, h, w, c, k = tag[:5]
            shapes.add((name[9:], n * cfg["batch"], h, w, c, k, 0))
    K.PROFILE.clear()
    return shapes


def make_call(op, n, h, w, c, k, cf, dev):
    g = torch.Generator(device=dev).manual_seed(0)
    if op == "wgrad":
        x = torch.randn(n, h, w, c, generator=g, device=dev).to(torch.bfloat16).permute(0, 3, 1, 2)
        dy = torch.randn(n, h, w, k, generator=g, device=dev).to(torch.bfloat16).permute(0, 3, 1, 2)
        dw = torch.zeros(k, 3, 3, c, device=dev)
        return lambda: K.conv_wgrad(x, dy, 3, 3, 1, 1, dw_krsc=dw, centre_from=cf)
    if op == "fprop":
        x = torch.randn(n, h, w, c, generator=g, device=dev).to(torch.bfloat16).permute(0, 3, 1, 2)
        krsc, _ = K.weight_prepare(torch.randn(k, c, 3, 3, generator=g, device=dev) * 0.05)
        y = K.empty_nhwc(n, k, h, w, dev)
        return lambda: K.conv_fprop(x, krsc, k, 3, 3, 1, 1, out=y)
    dy = torch.randn(n, h, w, k, generator=g, device=dev).to(torch.bfloat16).permute(0, 3, 1, 2)
    _, crsk = K.weight_prepare(torch.randn(k, c, 3, 3, generator=g, device=dev) * 0.05)
    dx = K.empty_nhwc(n, c, h, w, dev)
    return lambda: K.conv_dgrad(dy, crsk, (n, c, h, w), 3, 3, 1, 1, out=dx)


def time_calls(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) * 1e3 / iters


def shape_table(cfg_ids, rounds, iters, dev):
    L = lib.load()
    shapes = {}
    for c in cfg_ids:
        for s in collect_shapes(c, dev):
            shapes.setdefault(s, []).append(c)
    print(f"{'op':5s} {'N':>4s} {'HxW':>9s} {'C':>4s} {'K':>4s} {'cf':>4s} {'cfg':>7s} {'engine':>6s} {'im2col us':>9s} {'halo us':>8s} {'speedup':>7s}"
          f" {'MB':>6s} {'GFLOP':>6s} {'halo TB/s':>9s} {'halo TF/s':>9s} {'%peak':>6s} {'halo L2->SM GB/s':>16s}")
    for (op, n, h, w, c, k, cf), cfgs in sorted(shapes.items(), key=lambda kv: (kv[0][0], -kv[0][2], kv[0][4], kv[0][5], kv[0][6])):
        fn = make_call(op, n, h, w, c, k, cf, dev)
        force, launches = (L.sgb_conv_wgrad_force_im2col, L.sgb_conv_wgrad_halo_launches) if op == "wgrad" else (L.sgb_conv_force_im2col, L.sgb_conv_halo_launches)
        h0 = launches()
        fn()
        engine = "halo" if launches() > h0 else "im2col"
        t_i, t_h = [], []
        for _ in range(rounds):
            force(1)
            fn()
            t_i.append(time_calls(fn, iters))
            force(0)
            fn()
            t_h.append(time_calls(fn, iters))
        ti, th = statistics.median(t_i), statistics.median(t_h)
        cin, cout = (c, k) if op != "dgrad" else (k, c)
        byts = 2.0 * n * h * w * (cin + cout) + (4.0 if op == "wgrad" else 2.0) * 9 * c * k
        flop = 2.0 * n * h * w * cin * cout * 9
        tb = byts / (th * 1e-6)
        tf = flop / (th * 1e-6)
        floor_us = max(byts / PEAK_BW, flop / PEAK_TF) * 1e6
        halo_bytes = n * ((h + 7) // 8) * ((w + 7) // 8) * cin * 100 * 2.0 if engine == "halo" else 0.0
        l2 = f"{halo_bytes / (th * 1e-6) / 1e9:16.0f}" if engine == "halo" and op != "wgrad" else f"{'-':>16s}"
        print(f"{op:5s} {n:4d} {h:4d}x{w:<4d} {cin:4d} {cout:4d} {cf:4d} {','.join(map(str, cfgs)):>7s} {engine:>6s} {ti:9.1f} {th:8.1f} {ti / th:7.2f}"
              f" {byts / 1e6:6.1f} {flop / 1e9:6.1f} {tb / 1e12:9.2f} {tf / 1e12:9.1f} {floor_us / th * 100:5.1f}% {l2}", flush=True)
    L.sgb_conv_force_im2col(0)
    L.sgb_conv_wgrad_force_im2col(0)


def step_ab(rounds, iters, dev):
    L = lib.load()
    cfg = bench.CONFIGS[2]
    arms = {}
    for name, force in (("im2col", 1), ("auto", 0)):
        L.sgb_conv_force_im2col(force)
        _model, step, host = bench.build_train_workload(cfg, dev, 0, cfg["batch"])
        x, t = bench._to_dev(host[0], dev)
        step.set_hyper_params(2e-4, 0.9997)
        step.run(x, t)
        step.capture(x, t, warmup=2)
        arms[name] = (step, x, t)
    L.sgb_conv_force_im2col(0)
    res = {k: [] for k in arms}
    for _ in range(rounds):
        for name, (step, x, t) in arms.items():
            for _ in range(3):
                step.run(x, t)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(iters):
                step.set_hyper_params(2e-4, 0.9997)
                step.run(x, t)
            b.record()
            b.synchronize()
            res[name].append(a.elapsed_time(b) / iters)
    for name, v in res.items():
        print(f"config 2 step, {name:6s}: median {statistics.median(v):.3f} ms  spread {max(v) - min(v):.3f} ms  rounds {['%.3f' % x for x in v]}")
    print(f"auto / im2col: {statistics.median(res['auto']) / statistics.median(res['im2col']):.4f}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", type=int, nargs="+", default=[2, 3, 4, 5])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--step-rounds", type=int, default=5)
    ap.add_argument("--step-iters", type=int, default=20)
    ap.add_argument("--no-step", action="store_true")
    args = ap.parse_args()
    dev = setup_device()
    lib.call("sgb_check_device")
    print(f"card: {card()}")
    shape_table(args.configs, args.rounds, args.iters, dev)
    if not args.no_step:
        step_ab(args.step_rounds, args.step_iters, dev)


if __name__ == "__main__":
    main()
