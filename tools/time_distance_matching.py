"""Times the DetectionMetricsDistanceBased matching kernel at COCO validation size -- B = 32 images, 300 NMS rows per image, up to
100 targets, 1 and 10 distance thresholds, Euclidean and Manhattan -- from CUDA events over many launches, next to the CPU process
time of the reference-style per-image torch loop (DistanceMatching.compute_targets / compute_crowd_targets restated with the same
tensor operations) on the same inputs.  Prints one JSON line per configuration with the card name and power limit read in the
same run.

    python tools/time_distance_matching.py [--iters 200]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from super_gradients_b200 import kernels as K  # noqa: E402
from super_gradients_b200.training.utils import detection_utils as DU  # noqa: E402


def scene(gen, B, P, M, n_cls, H, W):
    out, tg = [], []
    for b in range(B):
        nt = int(torch.randint(M // 2, M + 1, (1,), generator=gen))
        c = torch.rand(nt, 2, generator=gen) * torch.tensor([W, H])
        wh = torch.rand(nt, 2, generator=gen) * 60 + 4
        tg.append(torch.cat([torch.full((nt, 1), float(b)), torch.randint(0, n_cls, (nt, 1), generator=gen).float(), c, wh], 1))
        src = torch.randint(0, nt, (P,), generator=gen)
        cc = c[src] + (torch.rand(P, 2, generator=gen) - 0.5) * 20
        w = wh[src] * (0.7 + 0.6 * torch.rand(P, 2, generator=gen))
        sc = torch.rand(P, generator=gen).sort(descending=True).values
        cls = torch.where(torch.rand(P, generator=gen) < 0.8, tg[-1][src, 1], torch.randint(0, n_cls, (P,), generator=gen).float())
        out.append(torch.cat([cc - w / 2, cc + w / 2, sc[:, None], cls[:, None]], 1))
    return out, torch.cat(tg)


def reference_loop(out, targets, H, W, thresholds, dist, top_k=100):
    """Per image: top-k per class, clipping, centre distances, stable sort and the greedy (prediction, target) loop of
    DistanceMatching.compute_targets, as the reference runs it on the CPU."""
    thr_t = torch.tensor(thresholds)
    for b, preds in enumerate(out):
        preds = preds.clone()
        t = targets[targets[:, 0] == b, 1:].clone()
        T = len(thresholds)
        pm = torch.zeros(len(preds), T, dtype=torch.bool)
        tm = torch.zeros(len(t), T, dtype=torch.bool)
        cls, scores = preds[:, -1], preds[:, 4]
        n_cls = int(cls.max())
        mask = cls.view(-1, 1) == torch.arange(n_cls + 1).view(1, -1)
        s, idx = (scores.view(-1, 1) * mask).sort(0, descending=True)
        use = idx[s[:top_k, :].nonzero(as_tuple=False).split(1, dim=1)].view(-1)
        preds[:, [0, 2]] = preds[:, [0, 2]].clip(0, W)
        preds[:, [1, 3]] = preds[:, [1, 3]].clip(0, H)
        tb = t[:, 1:5]
        tb[:, 1] = tb[:, 1] - tb[:, 3] * 0.5
        tb[:, 0] = tb[:, 0] - tb[:, 2] * 0.5
        tb[:, 3] = tb[:, 3] + tb[:, 1]
        tb[:, 2] = tb[:, 2] + tb[:, 0]
        d = dist.calculate_distance(preds[use, :4], tb)
        d[cls[use].view(-1, 1) != t[:, 0].view(1, -1)] = float("inf")
        sd, ts = d.sort(stable=True)
        for pi, ti in (sd < max(thresholds)).nonzero(as_tuple=False):
            p, tt = use[pi], ts[pi, ti]
            good = (sd[pi, ti] < thr_t) & ~pm[p] & ~tm[tt]
            tm[tt, good] = True
            pm[p, good] = True
            if tm.all():
                break


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in q.split(",")]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--cpu-batches", type=int, default=1)
    args = ap.parse_args()
    name, power = gpu_info()
    B, P, M, H, W = 32, 300, 100, 640, 640
    gen = torch.Generator().manual_seed(0)
    out, targets = scene(gen, B, P, M, 80, H, W)
    rows, counts = DU.pad_predictions(out, "cuda")
    t_pad, t_cnt = DU.pad_matching_targets_host(targets, B)
    t_pad, t_cnt = t_pad.cuda(), t_cnt.cuda()
    for metric, dist in (("euclidean", DU.EuclideanDistance()), ("manhattan", DU.ManhattanDistance())):
        for thresholds in ([5.0], [float(v) for v in torch.linspace(2.0, 20.0, 10)]):
            for _ in range(10):
                K.detection_distance_matching(rows, counts, t_pad, t_cnt, None, None, thresholds, metric, H, W)
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.iters):
                K.detection_distance_matching(rows, counts, t_pad, t_cnt, None, None, thresholds, metric, H, W)
            b.record()
            torch.cuda.synchronize()
            gpu_ms = a.elapsed_time(b) / args.iters
            t0 = time.process_time()
            for _ in range(args.cpu_batches):
                reference_loop(out, targets, H, W, thresholds, dist)
            cpu_ms = (time.process_time() - t0) * 1e3 / args.cpu_batches
            print(json.dumps({"metric": metric, "B": B, "preds_per_image": P, "max_targets": M, "T": len(thresholds), "kernel_ms_per_batch_incl_launch": round(gpu_ms, 4),
                              "reference_loop_cpu_process_ms_per_batch": round(cpu_ms, 1), "gpu": name, "power_limit": power, "iters": args.iters}), flush=True)  # fmt: skip


if __name__ == "__main__":
    main()
