"""Seeded merge-NMS inputs shared by the CPU and GPU sliding-window tests, and a g++ build of tests/host_kernels/merge_nms_host.cpp
(the serial merge over the product header nms_math.cuh)."""
import ctypes
import os
import subprocess
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_LIB = {}


def merge_case(n: int, ncls: int, seed: int, tied: bool = False):
    """n candidate rows (boxes [n, 4] f32 in canvas pixels, scores [n] f32, labels [n] f32) in clusters, so that NMS suppresses.
    Scores are distinct unless `tied` (then drawn from 8 values)."""
    g = torch.Generator().manual_seed(seed)
    centers = torch.rand(max(1, n // 6), 2, generator=g) * 900
    which = torch.randint(0, centers.shape[0], (n,), generator=g)
    c = centers[which] + torch.randn(n, 2, generator=g) * 6
    wh = 12 + torch.rand(n, 2, generator=g) * 40
    boxes = torch.cat([c - wh / 2, c + wh / 2], dim=1).float()
    if tied:
        scores = (torch.randint(1, 9, (n,), generator=g).float() / 8).float()
    else:
        scores = ((torch.randperm(n, generator=g) + 1).double() / (n + 1)).float()
    labels = torch.randint(0, ncls, (n,), generator=g).float()
    return boxes, scores, labels


def _handle():
    if "h" not in _LIB:
        d = tempfile.mkdtemp(prefix="sgb_merge_host_")
        so = os.path.join(d, "merge_nms_host.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", os.path.join(ROOT, "tests", "host_kernels", "merge_nms_host.cpp"),
                        "-I", os.path.join(ROOT, "super_gradients_b200", "csrc"), "-o", so], check=True)  # fmt: skip
        h = ctypes.CDLL(so)
        P = ctypes.c_void_p
        h.merge_nms_host.argtypes = [P, P, P, ctypes.c_int, ctypes.c_double, P]
        h.merge_nms_host.restype = ctypes.c_int
        _LIB["h"] = h
    return _LIB["h"]


def merge_nms_host(boxes, scores, labels, iou: float) -> torch.Tensor:
    """-> kept list indices in output order (int64), as the merge kernel orders them."""
    n = boxes.shape[0]
    b, s = boxes.float().contiguous(), scores.float().contiguous()
    lab = labels.to(torch.int32).contiguous()
    keep = torch.empty(max(n, 1), dtype=torch.int64)
    nk = _handle().merge_nms_host(b.data_ptr(), s.data_ptr(), lab.data_ptr(), n, float(iou), keep.data_ptr())
    return keep[:nk]


class StubDetector(torch.nn.Module):
    """Seeded stand-in detector for the sliding-window goldens.  Every call returns, per tile of its batch, decoded predictions
    (boxes [L, 4] in tile pixels, scores [L, ncls]) drawn from a CPU generator seeded by (seed, running tile index, number of exactly
    zero values in the tile's channel 0): the tile order, and the zero fill beyond the canvas, both decide the output.  It runs
    unchanged under the reference wrapper (fp32 NCHW tiles) and under ours (bf16 NHWC tiles); `callback_cls` is the
    PPYoloEPostPredictionCallback of either side."""

    def __init__(self, callback_cls, seed: int, anchors: int = 200, ncls: int = 4, tied: bool = False, nms=None):
        super().__init__()
        self.callback_cls, self.seed, self.anchors, self.ncls, self.tied = callback_cls, seed, anchors, ncls, tied
        self.nms = dict(iou=0.3, conf=0.2, nms_top_k=77, max_predictions=11, multi_label_per_box=False, class_agnostic_nms=True) if nms is None else nms
        self.calls = []  # (tile index, zero count) of every tile seen
        self._dummy = torch.nn.Parameter(torch.zeros(1))

    def tile_output(self, k: int, zeros: int, size: int):
        g = torch.Generator().manual_seed(self.seed * 1000003 + k * 7919 + zeros)
        L = self.anchors
        centers = torch.rand(max(1, L // 5), 2, generator=g) * size
        c = centers[torch.randint(0, centers.shape[0], (L,), generator=g)] + torch.randn(L, 2, generator=g) * 4
        wh = 8 + torch.rand(L, 2, generator=g) * 50
        boxes = torch.cat([c - wh / 2, c + wh / 2], 1).float()
        scores = torch.rand(L, self.ncls, generator=g)
        if self.tied:
            scores = torch.floor(scores * 8) / 8
        return boxes, scores.float()

    def forward(self, x):
        out_b, out_s = [], []
        for i in range(x.shape[0]):
            zeros = int((x[i, 0] == 0).sum())
            k = len(self.calls)
            self.calls.append((k, zeros))
            b, s = self.tile_output(k, zeros, x.shape[-1])
            out_b.append(b)
            out_s.append(s)
        return torch.stack(out_b).to(x.device), torch.stack(out_s).to(x.device)

    def get_dataset_processing_params(self):
        return dict(class_names=[f"c{i}" for i in range(self.ncls)], image_processor=None, **self.nms)

    def get_post_prediction_callback(self, *, conf, iou, nms_top_k, max_predictions, multi_label_per_box, class_agnostic_nms):
        return self.callback_cls(score_threshold=conf, nms_threshold=iou, nms_top_k=nms_top_k, max_predictions=max_predictions, multi_label_per_box=multi_label_per_box,
                                 class_agnostic_nms=class_agnostic_nms)  # fmt: skip

    def get_input_channels(self) -> int:
        return 3


def golden_inputs(seed: int, B: int, H: int, W: int) -> torch.Tensor:
    """fp32 NCHW batch of bf16-representable values with no exact zero (so the zeros a tile holds are the fill beyond the canvas)."""
    g = torch.Generator().manual_seed(seed)
    return (0.01 + torch.rand(B, 3, H, W, generator=g)).bfloat16().float()


# name -> (input seed, B, H, W, tile, step, wrapper kwargs, stub kwargs).  Exact fit; a dropped right strip; an image smaller than a
# tile with tiles past the canvas, and one with none; step > tile; the single-label and class-agnostic tile callbacks; merges on both
# sides of n = 1000; one class holding every candidate; tied scores.
GOLDEN_CASES = {
    "exact_fit": (1, 2, 640, 640, 320, 160, dict(tile_nms_conf=0.5), dict(seed=1)),
    "dropped_strip": (2, 1, 800, 985, 320, 160, dict(tile_nms_conf=0.6), dict(seed=2)),
    "small_covered": (3, 1, 200, 250, 320, 160, dict(tile_nms_conf=0.5), dict(seed=3)),
    "small_no_tiles": (4, 2, 170, 400, 320, 160, dict(tile_nms_conf=0.5), dict(seed=4)),
    "step_gt_tile": (5, 1, 700, 900, 200, 250, dict(tile_nms_conf=0.5), dict(seed=5)),
    "single_label": (6, 1, 480, 640, 320, 160, dict(tile_nms_conf=0.3, tile_nms_multi_label_per_box=False), dict(seed=6)),
    "agnostic_tiles": (7, 1, 480, 640, 320, 160, dict(tile_nms_conf=0.4, tile_nms_class_agnostic_nms=True, tile_nms_iou=0.5), dict(seed=7)),
    "merge_below_1000": (8, 1, 480, 480, 320, 160, dict(tile_nms_conf=0.3, tile_nms_iou=0.8, tile_nms_max_predictions=240), dict(seed=8)),
    "merge_above_1000": (9, 1, 800, 1000, 320, 160, dict(tile_nms_conf=0.2, tile_nms_iou=0.8), dict(seed=9)),
    "one_class": (10, 1, 800, 1000, 320, 160, dict(tile_nms_conf=0.05, tile_nms_iou=0.8), dict(seed=10, ncls=1)),
    "tied_scores": (11, 1, 480, 480, 320, 160, dict(tile_nms_conf=0.3, tile_nms_iou=0.6, tile_nms_max_predictions=200), dict(seed=11, tied=True)),
}
