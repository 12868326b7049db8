#!/usr/bin/env python
"""Times the classification paths on the GPU, reading the card's name and power limit in the same run:
  (1) ResNet-50 predict(batch_size=256) on 256 seeded 375 x 500 uint8 images with the ImageNet chain: pre-processing ms per batch
      (CUDA events around the one resize + crop launch and its staging copy), model ms (forward + decode), end-to-end images/s;
  (2) the config-4 train step (ResNet-50, 224 x 224, CrossEntropyLoss, SGD) as a CUDA-graph replay, without and with the
      Accuracy / Top5 train-metric updates, alternated.
Usage: python tools/time_classification.py [--batch 256] [--train-batch 64] [--iters 20]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name()


def events_ms(fn, iters):
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
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--train-batch", type=int, default=64)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures the GPU and has no CPU fallback")
    from super_gradients_b200.training import models
    from super_gradients_b200.training.losses import CrossEntropyLoss
    from super_gradients_b200.training.metrics import Accuracy, Top5
    from super_gradients_b200.training.processing import default_imagenet_processing_params
    from super_gradients_b200.training.sg_trainer import TrainStep

    res = {"card": card()}
    torch.manual_seed(0)
    m = models.get("resnet50", num_classes=1000).cuda().eval()
    cp = default_imagenet_processing_params()["image_processor"]
    m.set_dataset_processing_params(image_processor=cp)
    rng = np.random.RandomState(0)
    images = [rng.randint(0, 256, (375, 500, 3)).astype(np.uint8) for _ in range(args.batch)]
    for _ in range(3):
        m.predict(images, batch_size=args.batch)
    torch.cuda.synchronize()
    res["preprocess_ms_per_batch"] = events_ms(lambda: cp.preprocess_crop_batch(images, "cuda"), args.iters)
    batch = cp.preprocess_crop_batch(images, "cuda")
    with torch.no_grad():
        res["model_ms_per_batch"] = events_ms(lambda: m(batch), args.iters)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(args.iters):
        m.predict(images, batch_size=args.batch)  # ends in a device -> host copy
    res["predict_images_per_s"] = args.batch * args.iters / (time.perf_counter() - t0)

    torch.manual_seed(0)
    net = models.get("resnet50", num_classes=1000).cuda().train()
    st = TrainStep(net, CrossEntropyLoss(), "SGD", {"momentum": 0.9, "weight_decay": 5e-5}, zero_wd_on_bias_and_bn=True, keep_outputs=True)
    x = torch.randn(args.train_batch, 3, 224, 224, device="cuda")
    y = torch.randint(0, 1000, (args.train_batch,), device="cuda")
    st.set_hyper_params(0.1)
    st.capture(x, y)
    metrics = [Accuracy(), Top5()]

    def step(with_metrics):
        st.set_hyper_params(0.1)
        st.run(x, y)
        if with_metrics:
            for mt in metrics:
                mt.update(st.last_outputs, y)

    for _ in range(3):
        step(True)
    off, on = [], []
    for _ in range(5):  # alternated
        off.append(events_ms(lambda: step(False), args.iters))
        on.append(events_ms(lambda: step(True), args.iters))
    res["train_step_ms_metrics_off"] = statistics.median(off)
    res["train_step_ms_metrics_on"] = statistics.median(on)
    res["train_batch"] = args.train_batch
    print(json.dumps({k: (round(v, 3) if isinstance(v, float) else v) for k, v in res.items()}))


if __name__ == "__main__":
    main()
