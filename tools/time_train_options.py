#!/usr/bin/env python
"""Times clip_grad_norm and precise_bn on bench.py's train workloads (config 2: YOLO-NAS-S, 640x640, 32 images, AdamW + EMA;
config 4: ResNet-50, 224x224, 256 images, SGD).

- The whole step captured twice, without and with clip_grad_norm, replayed alternately over --rounds rounds of --iters steps:
  median ms per step of each.
- The two clip kernels alone (sgb_clip_grad_norm: the per-chunk float64 sums, then the one-CTA finalize) over the live float32
  gradients: CUDA events, median of --iters calls; the bytes they must read (every live gradient once) over that time, against
  the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s).
- Config 4: one precise_bn pass at the end of an epoch (Trainer._precise_bn, --pbn-batches eager train-mode forwards).

Prints the card's name and power limit with the numbers.  Usage: python tools/time_train_options.py [--iters 20] [--rounds 5]"""
import argparse
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

HBM_TBPS = 3.35


def events_ms(fn, iters):
    out = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--clip", type=float, default=1.0)
    ap.add_argument("--pbn-batches", type=int, default=4)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device: this tool times the sm_90a kernels")
    import bench

    from super_gradients_b200 import kernels as K
    from super_gradients_b200.training import fused_optimizers as FO
    from super_gradients_b200.training.sg_trainer import Trainer

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()[0]
    print(f"card: {card}; torch {torch.__version__}; {args.rounds} rounds x {args.iters} replays, medians")
    print("| config | live params | step, no clip (ms) | step, clip (ms) | difference (ms) | clip kernels (us) | gradient bytes (MB) | GB/s | of 3.35 TB/s |")
    print("|---|---|---|---|---|---|---|---|---|")
    dev = torch.device("cuda")
    for cid in (2, 4):
        cfg = bench.CONFIGS[cid]
        batch = 32 if cid == 2 else 256
        model, step, host = bench.build_train_workload(cfg, dev, 0, batch)
        x, t = bench._to_dev(host[0], dev)
        f = step.flat
        graphs = {}
        for clip in (None, args.clip):
            step.clip_grad_norm = clip
            if clip is not None:
                step.clip_partials = torch.zeros(f.chunks.shape[0], dtype=torch.float64, device=dev)
                step.clip_norm_coef = torch.zeros(2, dtype=torch.float32, device=dev)
            step.set_hyper_params(1e-4, 0.999)
            step.graph = None
            graphs[clip] = (step.capture(x, t, warmup=2), step.static_in, step.static_out)  # static buffers stay alive with their graph
        times = {c: [] for c in graphs}
        for _ in range(args.rounds):
            for c, (g, *_keep) in graphs.items():
                step.set_hyper_params(1e-4, 0.999)
                g.replay()
                torch.cuda.synchronize()
                times[c] += events_ms(g.replay, args.iters)
        off, on = statistics.median(times[None]), statistics.median(times[args.clip])
        hp = step.hp
        col = FO.GRAD_SCALE_COLUMN[step.opt_name]
        clip_us = statistics.median(events_ms(lambda: K.clip_grad_norm(f.grads, f.chunks, hp, col, args.clip, step.clip_partials, step.clip_norm_coef), args.iters * args.rounds)) * 1e3
        moved = f.n_live * 4
        gbps = moved / clip_us / 1e3
        print(f"| {cid} ({cfg['model']}) | {f.n_live / 1e6:.2f} M | {off:.3f} | {on:.3f} | {on - off:+.3f} | {clip_us:.1f} | {moved / 1e6:.1f} | {gbps:.0f} | {gbps / (HBM_TBPS * 1e3):.0%} |")
        if cid == 4:
            tr = Trainer("time_train_options", ckpt_root_dir=os.path.join(os.environ.get("TMPDIR", "/tmp"), "time_train_options"))
            tr.net, tr.step, tr.criterion = model, step, step.criterion

            class Loader(list):
                batch_size = batch

            loader = Loader([bench._to_dev(h, dev) for h in host[: args.pbn_batches]])
            tp = {"precise_bn_batch_size": batch * args.pbn_batches}
            tr._precise_bn(loader, tp)  # warm-up
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            tr._precise_bn(loader, tp)
            torch.cuda.synchronize()
            print(f"\nconfig 4 precise_bn pass at epoch end: {len(loader)} forwards of {batch} images, {(time.perf_counter() - t0) * 1e3:.1f} ms")
        del graphs, step, model, host
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
