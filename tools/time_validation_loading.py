"""Times the packed validation chains (YOLO-NAS COCO, YOLO-NAS-POSE, ResNet-50 ImageNet) against the same chains run on the CPU
with cv2 / numpy / PIL / torchvision, on seeded images, and prints one JSON line per measurement after the card's name, power limit
and maximum SM clock (read in the same run):

  (a) process CPU time per sample on one thread: the CPU chain + the reference's collate arithmetic, against the packed path's
      host half + packing;
  (b) time per batch of the packed path's copy + launch, CUDA events over many batches, at the batch sizes given;
  (c) images/s of a full validation pass with each loader at the same worker count, ending in a device synchronise.

    python tools/time_validation_loading.py [--images 512] [--workers 8]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from super_gradients_b200.training.datasets.detection_augment_dataset import CrowdDetectionAugmentCollateFN, DetectionAugmentDataset  # noqa: E402
from super_gradients_b200.training.datasets.imagenet_augment_dataset import ImageNetValidationCollateFN, ImageNetValidationDataset  # noqa: E402
from super_gradients_b200.training.datasets.pose_estimation_datasets.pose_augment_dataset import PoseAugmentDataset, YoloNASPoseAugmentCollateFN  # noqa: E402
from super_gradients_b200.training.transforms import keypoints as KP  # noqa: E402
from super_gradients_b200.training.transforms import transforms as T  # noqa: E402

MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


def _image(rng, h, w):
    return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)


class Det:
    """COCO validation samples after the dataset's load-time resize to 636."""

    def __init__(self, n, seed=0):
        rng = np.random.default_rng(seed)
        shapes = [(636, 477), (477, 636), (636, 636), (424, 636)]
        self.s = []
        for i in range(n):
            h, w = shapes[i % len(shapes)]
            k = int(rng.integers(1, 12))
            x1, y1 = rng.uniform(0, w * 0.7, k), rng.uniform(0, h * 0.7, k)
            t = np.stack([x1, y1, x1 + rng.uniform(4, w * 0.3, k), y1 + rng.uniform(4, h * 0.3, k), rng.integers(0, 80, k)], -1).astype(np.float32)
            self.s.append({"image": _image(rng, h, w), "target": t, "crowd_target": t[:1].copy()})

    def __len__(self):
        return len(self.s)

    def get_sample(self, i, ignore_empty_annotations=False):
        return {k: v.copy() for k, v in self.s[i].items()}

    def __getitem__(self, i):  # the CPU chain: RGB2BGR -> center pad to 640 (114) -> /255 -> CHW, then the collate's torch.stack
        s = self.get_sample(i)
        im = s["image"][..., ::-1]
        h, w = im.shape[:2]
        top, left = (640 - h) // 2, (640 - w) // 2
        im = np.pad(im, ((top, 640 - h - top), (left, 640 - w - left), (0, 0)), constant_values=114)
        return torch.from_numpy(np.ascontiguousarray((im / 255.0).astype(np.float32).transpose(2, 0, 1)))


class Pose:
    def __init__(self, n, seed=0):
        import types

        rng = np.random.default_rng(seed)
        shapes = [(480, 640), (640, 427), (425, 640), (640, 480)]
        self.s, self.ns = [], types.SimpleNamespace
        for i in range(n):
            h, w = shapes[i % len(shapes)]
            k = int(rng.integers(1, 6))
            joints = np.concatenate([rng.uniform(0, min(h, w), (k, 17, 2)), rng.integers(0, 3, (k, 17, 1))], -1).astype(np.float32)
            self.s.append(dict(image=_image(rng, h, w), joints=joints, areas=np.full(k, 500.0, np.float32), bboxes_xywh=np.tile([10.0, 10, 100, 100], (k, 1)).astype(np.float32),
                               is_crowd=np.zeros(k, np.int64)))  # fmt: skip

    def __len__(self):
        return len(self.s)

    def load_sample(self, i):
        s = {k: v.copy() for k, v in self.s[i].items()}
        return self.ns(mask=np.ones(s["image"].shape[:2], np.float32), additional_samples=None, **s)

    def __getitem__(self, i):  # the CPU chain: LongestMaxSize(640) (cv2 INTER_LINEAR) -> bottom-right pad 127 -> /255 -> CHW
        import cv2

        im = self.s[i]["image"]
        h, w = im.shape[:2]
        r = 640 / max(h, w)
        nh, nw = int(round(h * r)), int(round(w * r))
        im = cv2.resize(im, (nw, nh), interpolation=cv2.INTER_LINEAR) if (nh, nw) != (h, w) else im
        im = np.pad(im, ((0, 640 - nh), (0, 640 - nw), (0, 0)), constant_values=127)
        return torch.from_numpy(np.ascontiguousarray((im / 255.0).astype(np.float32).transpose(2, 0, 1)))


class Cls:
    def __init__(self, n, seed=0):
        from PIL import Image

        rng = np.random.default_rng(seed)
        shapes = [(375, 500), (500, 375), (333, 500), (480, 640)]
        self.s = [(Image.fromarray(_image(rng, *shapes[i % len(shapes)])), int(rng.integers(0, 1000))) for i in range(n)]
        self.chain = None

    def __len__(self):
        return len(self.s)

    def __getitem__(self, i):
        return self.s[i]

    def cpu_item(self, i):
        from torchvision import transforms as TV

        if self.chain is None:
            self.chain = TV.Compose([TV.Resize(236), TV.CenterCrop(224), TV.ToTensor(), TV.Normalize(MEAN, STD)])
        return self.chain(self.s[i][0])


class CpuView(torch.utils.data.Dataset):
    def __init__(self, get, n):
        self.get, self.n = get, n

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        return self.get(i)


def chains(n):
    det, pose, cls = Det(n), Pose(n), Cls(n)
    dds = DetectionAugmentDataset(det, [T.DetectionRGB2BGR(1), T.DetectionPadToSize(640, 114), T.DetectionStandardize(255.0), T.DetectionImagePermute(),
                                        T.DetectionTargetsFormatTransform(input_dim=640)], with_crowd=True)  # fmt: skip
    pds = PoseAugmentDataset(pose, [KP.KeypointsLongestMaxSize(640, 640), KP.KeypointsPadIfNeeded(640, 640, 127, 1, "bottom_right"), KP.KeypointsImageStandardize(255)],
                             with_gt_samples=True)  # fmt: skip
    cds = ImageNetValidationDataset(cls)
    return {
        "yolo_nas_coco": (dds, CrowdDetectionAugmentCollateFN.for_dataset(dds), CpuView(det.__getitem__, n), 25),
        "yolo_nas_pose": (pds, YoloNASPoseAugmentCollateFN.for_dataset(pds), CpuView(pose.__getitem__, n), 32),
        "resnet50_imagenet": (cds, ImageNetValidationCollateFN.for_dataset(cds), CpuView(cls.cpu_item, n), 200),
    }


def cpu_per_sample(ds, collate, cpu, bs, reps=2):
    n = len(ds)
    torch.set_num_threads(1)
    cpu[0], collate([ds[0]])  # first calls: imports and the transforms' construction stay out of the timed window
    t0 = time.process_time()
    for _ in range(reps):
        for s in range(0, n, bs):
            torch.stack([cpu[i] for i in range(s, min(n, s + bs))])
    t_cpu = (time.process_time() - t0) / (reps * n)
    t0 = time.process_time()
    for _ in range(reps):
        for s in range(0, n, bs):
            collate([ds[i] for i in range(s, min(n, s + bs))])
    t_gpu_host = (time.process_time() - t0) / (reps * n)
    return t_cpu, t_gpu_host


def launch_ms(ds, collate, bs, iters=50):
    batch = collate([ds[i % len(ds)] for i in range(bs)]).pin_memory()
    for _ in range(5):
        batch.to_model_input("cuda")
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        batch.to_model_input("cuda")
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def pass_rate(dataset, collate, bs, workers, packed):
    loader = torch.utils.data.DataLoader(dataset, batch_size=bs, num_workers=workers, collate_fn=collate, pin_memory=True, persistent_workers=False)
    t0 = time.perf_counter()
    n = 0
    for batch in loader:
        x = batch.to_model_input("cuda")[0] if packed else batch.to("cuda", non_blocking=True)
        n += x.shape[0]
    torch.cuda.synchronize()
    return n / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=512)
    ap.add_argument("--workers", type=int, default=8)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: these are GPU measurements")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"card": card, "torch": torch.__version__, "images": args.images, "workers": args.workers}))
    threads = torch.get_num_threads()
    for name, (ds, collate, cpu, bs) in chains(args.images).items():
        t_cpu, t_host = cpu_per_sample(ds, collate, cpu, bs)
        torch.set_num_threads(threads)
        ms = launch_ms(ds, collate, bs)
        rate_cpu = pass_rate(cpu, None, bs, args.workers, packed=False)
        rate_gpu = pass_rate(ds, collate, bs, args.workers, packed=True)
        print(json.dumps({"chain": name, "batch": bs, "cpu_chain_ms_per_sample": round(t_cpu * 1e3, 3), "packed_host_ms_per_sample": round(t_host * 1e3, 3),
                          "packed_copy_launch_ms_per_batch": round(ms, 3), "cpu_loader_images_per_s": round(rate_cpu, 1), "packed_loader_images_per_s": round(rate_gpu, 1)}))  # fmt: skip


if __name__ == "__main__":
    main()
