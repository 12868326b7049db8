"""Times SlidingWindowInferenceDetectionWrapper.predict() on YOLO-NAS-S: 16 seeded 1500 x 2520 uint8 images, tile 640, step 160,
skip_image_resizing=True (160 tiles per image), end to end and per stage (CUDA events), against the reference's schedule (one
batch-1 model call and one callback per tile, host lists, torchvision batched_nms per image) with the same model.  Prints one JSON
line with the card name and power limit.

    python tools/time_sliding_window.py [--images 16] [--batch-size 4] [--conf 0.005] [--ref-images 2]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
import torchvision

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from super_gradients_b200 import kernels as K  # noqa: E402
from super_gradients_b200.training import models  # noqa: E402
from super_gradients_b200.training.models.detection_models import sliding_window_detection_forward_wrapper as SW  # noqa: E402
from super_gradients_b200.training.processing import DetectionAutoPadding, default_yolo_nas_coco_processing_params  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout.strip()
        return q.splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=16)
    ap.add_argument("--batch-size", type=int, default=4)
    ap.add_argument("--conf", type=float, default=0.005)  # the seeded random-init model scores ~0.01: a low threshold loads the merge
    ap.add_argument("--ref-images", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_sliding_window.py needs a CUDA device")
    torch.manual_seed(0)
    model = models.get("yolo_nas_s", num_classes=80).cuda().eval()
    wrapper = SW.SlidingWindowInferenceDetectionWrapper(tile_size=640, tile_step=160, model=model)
    rng = np.random.RandomState(0)
    images = [rng.randint(0, 256, (1500, 2520, 3), dtype=np.uint8) for _ in range(a.images)]
    kw = dict(conf=a.conf, skip_image_resizing=True, batch_size=a.batch_size)
    wrapper.predict(images[: a.batch_size], **kw)  # warm-up
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    out = wrapper.predict(images, **kw)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    peak = torch.cuda.max_memory_allocated()

    # per-stage CUDA events over one batch, same schedule as predict()
    processor = default_yolo_nas_coco_processing_params()["image_processor"].get_equivalent_compose_without_resizing(DetectionAutoPadding((32, 32), 0))
    cb = wrapper._callback(None, a.conf, None, None, None, None)
    ev = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731
    stages = {k: 0.0 for k in ("preprocess", "gather", "model", "tile_nms", "merge", "copy")}
    cands = []
    for i in range(0, a.images, a.batch_size):
        e = [ev() for _ in range(2)]
        e[0].record()
        canvas, geos = processor.preprocess_batch(images[i : i + a.batch_size], "cuda")
        e[1].record()
        torch.cuda.synchronize()
        stages["preprocess"] += e[0].elapsed_time(e[1])
        B, _, H, W = canvas.shape
        origins = SW.tile_origins(H, W, 640, 160, 30)
        T, per = B * len(origins), len(origins)
        th = torch.tensor([(b, y, x) for b in range(B) for (y, x) in origins], dtype=torch.int32)
        ith = torch.arange(0, T + 1, per, dtype=torch.int32)
        td, itd = th.cuda(), ith.cuda()
        P = cb.max_rows()
        rows = torch.empty((T, P, 6), device="cuda")
        idx = torch.empty((T, P), dtype=torch.int32, device="cuda")
        cnt = torch.empty((T,), dtype=torch.int32, device="cuda")
        step = SW.chunk_tiles(640)
        for c0 in range(0, T, step):
            c1 = min(T, c0 + step)
            e = [ev() for _ in range(4)]
            e[0].record()
            batch = K.sliding_window_gather(canvas, th[c0:c1], td[c0:c1], 640)
            e[1].record()
            o = model(batch)
            e[2].record()
            cb.forward_batched(o, out=rows[c0:c1], out_idx=idx[c0:c1], out_count=cnt[c0:c1])
            e[3].record()
            torch.cuda.synchronize()
            stages["gather"] += e[0].elapsed_time(e[1])
            stages["model"] += e[1].elapsed_time(e[2])
            stages["tile_nms"] += e[2].elapsed_time(e[3])
        cands += cnt.view(B, per).sum(1).tolist()
        e = [ev() for _ in range(3)]
        e[0].record()
        merged, mc = K.sliding_window_merge(rows, cnt, td, ith, itd, 80, cb.nms_threshold)
        e[1].record()
        host = torch.cat([merged.reshape(-1), mc.view(torch.float32)]).cpu()
        e[2].record()
        torch.cuda.synchronize()
        stages["merge"] += e[0].elapsed_time(e[1])
        stages["copy"] += e[1].elapsed_time(e[2])

    # the reference's schedule on the same model, for a few images
    t1 = time.perf_counter()
    for im in images[: a.ref_images]:
        canvas, _ = processor.preprocess_batch([im], "cuda")
        _, _, H, W = canvas.shape
        padded = torch.zeros(1, 16, H + 640, W + 640, dtype=torch.bfloat16, device="cuda")
        padded[:, :, :H, :W] = canvas
        dets = []
        for y, x in SW.tile_origins(H, W, 640, 160, 30):
            r = cb(model(K.as_nhwc(padded[:, :, y : y + 640, x : x + 640])))[0]
            if len(r):
                r = r.clone()
                r[:, :4] += torch.tensor([x, y, x, y], dtype=torch.float32, device="cuda")
                dets.append(r)
        if dets:
            d = torch.cat(dets).cpu()
            d[torchvision.ops.batched_nms(d[:, :4], d[:, 4], d[:, 5], cb.nms_threshold)]
    torch.cuda.synchronize()
    dt_ref = (time.perf_counter() - t1) / a.ref_images
    tiles_per_image = len(SW.tile_origins(*processor.geometry(1500, 2520)[1], 640, 160, 30))
    print(json.dumps(dict(card=card(), images=a.images, batch_size=a.batch_size, conf=a.conf, seconds=round(dt, 4), images_per_s=round(a.images / dt, 2),
                          tiles_per_s=round(a.images * tiles_per_image / dt, 1), stage_ms_total=({k: round(v, 2) for k, v in stages.items()}),
                          merge_candidates_per_image=dict(min=min(cands), max=max(cands), mean=round(sum(cands) / len(cands), 1)),
                          kept_per_image_mean=round(sum(r.shape[0] for r in out) / len(out), 1), peak_mem_gb=round(peak / 2**30, 2),
                          reference_schedule_s_per_image=round(dt_ref, 4), ours_s_per_image=round(dt / a.images, 4))))  # fmt: skip


if __name__ == "__main__":
    main()
