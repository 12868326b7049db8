#!/usr/bin/env python
"""Times Trainer.train() with cuda_graph False against True on detection and pose, whose host targets the captured step pads into a
pinned staging ring (TrainStep.run_padded):

- YOLO-NAS-S, 32 x 640^2, PPYoloELoss (task-aligned assigner), AdamW + EMA (bench.py config 2's step), fed DetectionAugmentCollateFN
  batches of seeded stub images with COCO-like box counts, collated and pinned before the run, so the loader is not what is timed;
  the same for YOLO-NAS-POSE-N with PoseAugmentCollateFN.  Each round trains one epoch of --warmup + --iters steps eagerly, then
  one captured, on a fresh model: ms per step from a host clock around the last --iters steps, between two device synchronisations;
  medians over --rounds rounds.
- The captured detection step at n_max 32 / 64 / 128 / 256: CUDA events around --iters replays, median over the rounds.
- The per-step device-to-device copy of the model input into the static input that writing it in place (to_model_input(out=))
  saves, and the augmentation launch with and without `out`: CUDA events, medians.

Prints the card's name and power limit with the numbers.  Usage: python tools/time_trainer_graph.py [--iters 20] [--rounds 5]"""
import argparse
import os
import random
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

COCO_SIGMAS = [0.026, 0.025, 0.025, 0.035, 0.035, 0.079, 0.079, 0.072, 0.072, 0.062, 0.062, 0.107, 0.107, 0.087, 0.087, 0.089, 0.089]


class StubDetection:
    """n seeded raw samples in get_sample() form: longest side 640, the other 360-640, both orientations; per image a COCO-like number
    of boxes (geometric with mean 7.3, at most 60: COCO train2017 has 7.3 boxes per image and a long tail)."""

    def __init__(self, n, seed=0):
        from augment_cases import _image

        rng = np.random.default_rng(seed)
        self.samples = []
        for _ in range(n):
            short = int(rng.integers(360, 641))
            h, w = (640, short) if rng.random() < 0.5 else (short, 640)
            k = int(min(rng.geometric(1 / 7.3), 60))
            x1, y1 = rng.uniform(0, w * 0.8, k), rng.uniform(0, h * 0.8, k)
            boxes = np.stack([x1, y1, x1 + rng.uniform(8, w * 0.2, k), y1 + rng.uniform(8, h * 0.2, k), rng.integers(0, 80, k)], -1).astype(np.float32)
            self.samples.append({"image": _image(rng, h, w), "target": boxes})

    def __len__(self):
        return len(self.samples)

    def get_sample(self, index, ignore_empty_annotations=False):
        return {k: v.copy() for k, v in self.samples[index].items()}


class Loader(list):
    batch_size = 32


def packed_batches(task, batch, n_unique):
    """n_unique packed, pinned batches of the GPU augmentation loader."""
    random.seed(0)
    np.random.seed(0)
    if task == "detection":
        from augment_cases import RECIPE

        from super_gradients_b200.common.registry import TRANSFORMS
        from super_gradients_b200.training.datasets.detection_augment_dataset import DetectionAugmentCollateFN, DetectionAugmentDataset

        ds = DetectionAugmentDataset(StubDetection(2 * batch), [TRANSFORMS[n](**kw) for n, kw in RECIPE])
        collate = DetectionAugmentCollateFN.for_dataset(ds)
    else:
        from pose_augment_cases import GOLDEN_LISTS, StubPoseDataset, build

        from super_gradients_b200.training.datasets.pose_estimation_datasets.pose_augment_dataset import PoseAugmentCollateFN, PoseAugmentDataset
        from super_gradients_b200.training.transforms import keypoints as KP

        ds = PoseAugmentDataset(StubPoseDataset(), build(GOLDEN_LISTS["base"], KP))
        collate = PoseAugmentCollateFN.for_dataset(ds)
    return [collate([ds[(i * batch + j) % len(ds)] for j in range(batch)]).pin_memory() for i in range(n_unique)]


def model_and_loss(task, floor=0):
    """floor: the loss's max_targets_per_image."""
    from super_gradients_b200.training import models
    from super_gradients_b200.training.losses import PPYoloELoss, YoloNASPoseLoss

    torch.manual_seed(0)
    if task == "detection":
        return models.get("yolo_nas_s", num_classes=80), PPYoloELoss(num_classes=80, use_static_assigner=False, max_targets_per_image=floor)
    return models.get("yolo_nas_pose_n", num_classes=17), YoloNASPoseLoss(oks_sigmas=COCO_SIGMAS, max_targets_per_image=floor)


def loss_need(task, batch):
    from super_gradients_b200.training.losses import max_pose_targets_host, max_targets_host

    return max_targets_host(batch.targets) if task == "detection" else max_pose_targets_host(batch.targets)


class Clock:
    """Host clock between a device synchronisation before step `start` and one after the last step of the epoch."""

    def __init__(self, start):
        self.start, self.t0, self.t1 = start, None, None

    def on_train_batch_start(self, context):
        if context.batch_idx == self.start:
            torch.cuda.synchronize()
            self.t0 = time.perf_counter()

    def on_train_loader_end(self, context):
        torch.cuda.synchronize()
        self.t1 = time.perf_counter()


def train_ms(task, batches, graph, warmup, iters, tmp):
    """One epoch; max_targets_per_image is the batches' largest need, so no captured step falls back (a run without that floor falls
    back in its first epoch only, see DESIGN.md)."""
    from super_gradients_b200.training.sg_trainer import Trainer

    model, loss = model_and_loss(task, max(loss_need(task, b) for b in batches))
    clock = Clock(warmup)
    tp = dict(max_epochs=1, initial_lr=1e-4, lr_mode="constant", optimizer="AdamW", optimizer_params={"weight_decay": 1e-5}, zero_weight_decay_on_bias_and_bn=True,
              ema=True, ema_params={"decay": 0.9997, "decay_type": "threshold"}, loss=loss, cuda_graph=graph, save_model=False, phase_callbacks=[clock])  # fmt: skip
    tr = Trainer(f"time_{task}", ckpt_root_dir=tmp)
    tr.train(model, tp, Loader([batches[i % len(batches)] for i in range(warmup + iters)]))
    st = tr.step
    info = (st.n_max, st.replays, st.fallbacks)
    del tr, model, st
    torch.cuda.empty_cache()
    return (clock.t1 - clock.t0) * 1e3 / iters, info


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


def at_most(targets, n):
    """The rows of flat [N, 6] targets that are among the first n of their image."""
    img = targets[:, 0].long()
    rank = torch.tensor([int((img[:i] == img[i]).sum()) for i in range(img.numel())], dtype=torch.long)
    return targets[rank < n]


def n_max_costs(batches, iters, rounds):
    """Replays of the captured detection step with the first batch's targets padded to each n_max."""
    from super_gradients_b200.training.sg_trainer import TrainStep

    dev = torch.device("cuda")
    out = {}
    for n_max in (32, 64, 128, 256):
        model, loss = model_and_loss("detection")
        step = TrainStep(model.to(dev).train(), loss, "AdamW", {"weight_decay": 1e-5}, zero_wd_on_bias_and_bn=True, ema=True)
        x, t = batches[0].to_model_input(dev)
        padded = tuple(v.to(dev) for v in loss.pad_targets(at_most(t, 32), x.shape[0], n_max))  # the same targets at every n_max
        step.set_hyper_params(1e-4, 0.9997)
        g = step.capture(x, padded)
        times = []
        for _ in range(rounds):
            step.set_hyper_params(1e-4, 0.9997)
            g.replay()
            torch.cuda.synchronize()
            times += events_ms(g.replay, iters)
        out[n_max] = statistics.median(times)
        step.release_graph()
        del step, model, g
        torch.cuda.empty_cache()
    return out


def copy_costs(batches, iters):
    dev = torch.device("cuda")
    b = batches[0]
    x = b.to_model_input(dev)[0]
    static = x.clone()
    copy = statistics.median(events_ms(lambda: static.copy_(x, non_blocking=True), iters))
    fresh = statistics.median(events_ms(lambda: b.to_model_input(dev), iters))
    into = statistics.median(events_ms(lambda: b.to_model_input(dev, out=static), iters))
    assert torch.equal(static, x)
    return x.numel() * x.element_size(), copy, fresh, into


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=32)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device: this tool times the sm_90a training step")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()[0]
    print(f"card: {card}; torch {torch.__version__}; batch {args.batch} x 640^2; {args.rounds} rounds of {args.iters} steps after {args.warmup} warm-up steps, medians")
    Loader.batch_size = args.batch
    with tempfile.TemporaryDirectory() as tmp:
        det = None
        print("| workload | eager Trainer step (ms) | captured Trainer step (ms) | saved (ms) | captured n_max | replays | fallbacks |")
        print("|---|---|---|---|---|---|---|")
        for task, name in (("detection", "YOLO-NAS-S, PPYoloELoss (TAL)"), ("pose", "YOLO-NAS-POSE-N, YoloNASPoseLoss")):
            batches = packed_batches(task, args.batch, 4)
            if task == "detection":
                det = batches
            times = {False: [], True: []}
            for _ in range(args.rounds):
                for graph in (False, True):
                    ms, info = train_ms(task, batches, graph, args.warmup, args.iters, tmp)
                    times[graph].append(ms)
                    if graph:
                        n_max, replays, fallbacks = info
            e, c = statistics.median(times[False]), statistics.median(times[True])
            print(f"| {name} | {e:.2f} | {c:.2f} | {e - c:.2f} | {n_max} | {replays} | {fallbacks} |")
            print(f"  per-round eager {[round(v, 2) for v in times[False]]}, captured {[round(v, 2) for v in times[True]]}")
        costs = n_max_costs(det, args.iters, args.rounds)
        print("\n| n_max | captured YOLO-NAS-S step, replay (ms) |\n|---|---|")
        for n_max, ms in costs.items():
            print(f"| {n_max} | {ms:.3f} |")
        nbytes, copy, fresh, into = copy_costs(det, args.iters * args.rounds)
        print(f"\ninput batch {nbytes / 1e6:.0f} MB: device-to-device copy into the static input {copy:.3f} ms ({2 * nbytes / copy / 1e6:.0f} GB/s read + write); "
              f"augmentation launch into a new tensor {fresh:.3f} ms, into the static input {into:.3f} ms")


if __name__ == "__main__":
    main()
