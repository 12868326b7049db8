"""Edge cases of the batched NMS kernel (csrc/nms.cu over csrc/nms_math.cuh), shared by tests/golden/make_nms_edge_goldens.py, the
CPU test (the oracle against the reference's outputs) and the GPU test (the kernel against the oracle, bit for bit).

Every case is rebuilt from its seed; only the reference's outputs are stored (tests/golden/nms_edges.pt).  A case is a dict:
  kind    "ppyoloe" (PPYoloEPostPredictionCallback), "yolox" (detection_utils.non_max_suppression) or "pose"
          (YoloNASPosePostPredictionCallback);
  boxes [B, L, 4], scores [B, L, C] float32 (ppyoloe), pred [B, A, 5 + C] (yolox), or boxes / conf / coords / jscores (pose);
  params  the callback's keyword arguments.

The families:
  * path matrix -- every reachable combination of the host's launch choices (pre-filter or direct scan, split or one launch,
    coordinate trick / per-class / class-agnostic NMS, radix select or take everything), with the candidate count planted at
    exactly top_k and at top_k + 1 per image, top_k at 512 / 513, 1000 / 1001 and 1024, and pre-filtered rows that are not a
    multiple of 4 floats long (odd images start unaligned, the last slice is short);
  * ties and thresholds -- scores on multiples of 2^-6 whose runs straddle warp segments and pre-filter slices, all scores equal,
    scores at fp32(0.3) and one ulp either side under `>` and `>=`, +inf scores;
  * boxes -- fp32 IoU exactly 0.5 at threshold 0.5, IoU one ulp either side of double(0.65), zero-area and inverted boxes,
    identical boxes in different classes, coordinates around 1e6;
  * non-finite inputs and batch shapes -- NaN / +-inf coordinates on the trick and per-class paths, NaN class scores, +-0.0 scores
    at score_threshold 0.0, an image without candidates next to one with more than top_k, max_out 1 / below the survivors / 1024.
"""
import functools

import numpy as np
import torch

PF_SLICE = 24576  # floats per pre-filter slice (nms.cu); rows longer than 4 slices are pre-filtered
KMAX = 1024


def _boxes(g, B, L, span=600.0, size=(30.0, 40.0), cluster=4):
    """[B, L, 4] xyxy boxes in at most 150 clusters (of about `cluster` anchors when L is small), so that NMS suppresses also among
    a sparse subset of the anchors."""
    n_c = max(1, min(150, L // cluster))
    centers = torch.rand(B, n_c, 2, generator=g) * span
    which = torch.randint(0, n_c, (B, L), generator=g)
    c = torch.gather(centers, 1, which[..., None].expand(B, L, 2)) + torch.randn(B, L, 2, generator=g) * size[0] * 0.3
    wh = size[0] + torch.rand(B, L, 2, generator=g) * (size[1] - size[0])
    return torch.cat([c - wh / 2, c + wh / 2], -1).float()


def _planted(g, B, L, C, thr, counts, per_anchor=False, quant=None):
    """Scores [B, L, C] with exactly counts[b] entries above `thr` in image b (per_anchor: counts[b] anchors whose best class is
    above `thr`); everything else at most thr / 2.  `quant`: round the passing scores down to multiples of 2^-quant (ties)."""
    s = torch.rand(B, L, C, generator=g) * (thr / 2)
    for b, n in enumerate(counts):
        if per_anchor:
            a = torch.randperm(L, generator=g)[:n]
            v = thr + (1 - thr) * (0.02 + 0.98 * torch.rand(n, generator=g))
            c = torch.randint(0, C, (n,), generator=g)
            if quant is not None:
                v = torch.clamp(torch.floor(v * 2**quant) / 2**quant, min=thr + 2.0**-quant)
            s[b, a, c] = v
        else:
            f = torch.randperm(L * C, generator=g)[:n]
            v = thr + (1 - thr) * (0.02 + 0.98 * torch.rand(n, generator=g))
            if quant is not None:
                v = torch.clamp(torch.floor(v * 2**quant) / 2**quant, min=thr + 2.0**-quant)
            s[b].view(-1)[f] = v
    return s.float()


def _pp(boxes, scores, thr, iou, top_k, max_out, multi=True, agnostic=False):
    return dict(kind="ppyoloe", boxes=boxes, scores=scores,
                params=dict(score_threshold=thr, nms_threshold=iou, nms_top_k=top_k, max_predictions=max_out, multi_label_per_box=multi, class_agnostic_nms=agnostic))  # fmt: skip


def _matrix(seed, B, L, C, top_k, counts, multi=True, agnostic=False, max_out=300, thr=0.5):
    g = torch.Generator().manual_seed(seed)
    boxes = _boxes(g, B, L)
    scores = _planted(g, B, L, C, thr, counts, per_anchor=not multi)
    return _pp(boxes, scores, thr, 0.65, top_k, max_out, multi, agnostic)


# ------------------------------------------------------------------------------------------------------------------ ties
def _tied_prefilter(seed):
    # 8400 x 80: 2^-6-quantised scores; each slice's own top_k cut and the image's cut fall inside runs of equal scores that cross
    # warp segments and slices
    g = torch.Generator().manual_seed(seed)
    B, L, C = 2, 8400, 80
    s = torch.floor(torch.rand(B, L, C, generator=g) ** 40 * 64) / 64  # ~1 400 of each slice's ~24 600 pass; ~280 share the cut
    return _pp(_boxes(g, B, L), s.float(), 0.1, 0.65, 1000, 300)


def _tied_direct(seed):
    # 3000 x 4 = 12 000 items: warp segments of 384 items, one run of 2^-6 values through all of them
    g = torch.Generator().manual_seed(seed)
    B, L, C = 2, 3000, 4
    s = torch.floor(torch.rand(B, L, C, generator=g) * 16) / 64 + 0.5
    return _pp(_boxes(g, B, L), s.float(), 0.5, 0.65, 1024, 500)


def _all_equal(seed, multi=True):
    g = torch.Generator().manual_seed(seed)
    B, L, C = 2, 2000, 3
    s = torch.full((B, L, C), 0.625)
    return _pp(_boxes(g, B, L), s, 0.5, 0.65, 700, 300, multi)


def _thr_ulps(seed, multi):
    # fp32(0.3) and one ulp either side; 0.3 has no exact fp32 value
    g = torch.Generator().manual_seed(seed)
    B, L, C = 2, 600, 3
    t = np.float32(0.3)
    vals = torch.tensor([np.nextafter(t, np.float32(0)), t, np.nextafter(t, np.float32(1))], dtype=torch.float32)
    s = torch.rand(B, L, C, generator=g) * 0.25
    pick = torch.randint(0, 3, (B, L, C), generator=g)
    on = torch.rand(B, L, C, generator=g) < (0.3 if multi else 0.6)
    s = torch.where(on, vals[pick], s)
    return _pp(_boxes(g, B, L), s.float(), 0.3, 0.65, 1000, 300, multi)


def _inf_scores(seed):
    g = torch.Generator().manual_seed(seed)
    B, L, C = 2, 500, 4
    s = torch.rand(B, L, C, generator=g)
    s[torch.rand(B, L, C, generator=g) < 0.01] = float("inf")
    return _pp(_boxes(g, B, L), s.float(), 0.5, 0.65, 300, 300)


# ------------------------------------------------------------------------------------------------------------------ boxes
def _ovr32(a, b):
    """nms_math.cuh's IoU of two boxes in fp32 with one rounding per operation (numpy float32 scalars)."""
    f = np.float32
    area = lambda x: f(f(x[2] - x[0]) * f(x[3] - x[1]))  # noqa: E731
    w = max(f(0), f(min(a[2], b[2]) - max(a[0], b[0])))
    h = max(f(0), f(min(a[3], b[3]) - max(a[1], b[1])))
    inter = f(w * h)
    return f(inter / f(f(area(a) + area(b)) - inter))


def iou_pairs(target: float, n_each: int = 6):
    """Pairs of boxes (a, b) whose fp32 IoU is the fp32 value nearest `target` and each of its two neighbours, searched on the host with
    nms_math's arithmetic: b = [0, 0, x, 1] inside a = [0, 0, w, 1].  Returns {"below"/"at"/"above": [(a, b), ...]}."""
    f = np.float32
    t = f(target)
    goal = {"below": np.nextafter(t, f(0)), "at": t, "above": np.nextafter(t, f(1))}
    found = {k: [] for k in goal}
    for w in (f(37.0), f(41.5), f(53.25), f(64.0), f(97.75), f(120.5), f(211.0), f(333.0)):
        x = f(w * t)
        for _ in range(40):
            x = np.nextafter(x, f(0))
        for _ in range(80):
            a, b = (f(0), f(0), w, f(1)), (f(0), f(0), x, f(1))
            o = _ovr32(a, b)
            for k, v in goal.items():
                if o == v and len(found[k]) < n_each:
                    found[k].append((a, b))
            x = np.nextafter(x, f(1000))
    assert all(len(v) > 0 for v in found.values()), {k: len(v) for k, v in found.items()}
    return found


def _iou_edges(seed, target, iou):
    # pairs at exactly the threshold's fp32 value and one ulp either side, in class 0 (offset 0 on the trick path, so the boxes are
    # compared as built); pair k lies in the band y in [2k, 2k + 1], which no other pair overlaps.  The first box of a pair has the
    # higher score, so it decides over the second.
    g = torch.Generator().manual_seed(seed)
    pairs = [p for v in iou_pairs(target).values() for p in v]
    B, C = 1, 2
    L = 2 * len(pairs) + 40
    boxes = _boxes(g, B, L, span=50.0) + 5000.0
    scores = torch.rand(B, L, C, generator=g) * 0.4
    scores[0, 2 * len(pairs) :, 1] += 0.5  # the clutter far away, in class 1
    for k, (a, b) in enumerate(pairs):
        y = float(2 * k)
        boxes[0, 2 * k] = torch.tensor([float(a[0]), y, float(a[2]), y + 1.0])
        boxes[0, 2 * k + 1] = torch.tensor([float(b[0]), y, float(b[2]), y + 1.0])
        scores[0, 2 * k, 0] = 0.9 - 0.001 * k
        scores[0, 2 * k + 1, 0] = 0.8 - 0.001 * k
    return _pp(boxes, scores.float(), 0.5, iou, 1000, 300)


def _degenerate(seed):
    g = torch.Generator().manual_seed(seed)
    B, L, C = 2, 400, 3
    boxes = _boxes(g, B, L, span=200.0)
    z = torch.rand(B, L, generator=g)
    boxes[..., 2] = torch.where(z < 0.15, boxes[..., 0], boxes[..., 2])  # zero width
    boxes[..., 3] = torch.where((z >= 0.15) & (z < 0.3), boxes[..., 1], boxes[..., 3])  # zero height
    inv = (z >= 0.3) & (z < 0.5)
    boxes[inv] = boxes[inv][:, [2, 3, 0, 1]]  # inverted: negative width and height, positive area
    boxes[(z >= 0.5) & (z < 0.55)] = boxes[(z >= 0.5) & (z < 0.55)][:, [2, 1, 0, 3]]  # inverted in x only: negative area
    return _pp(boxes, torch.rand(B, L, C, generator=g), 0.4, 0.5, 1000, 300)


def _same_box_classes(seed, per_class):
    # each anchor's box is shared by all its classes; classes only suppress within themselves
    g = torch.Generator().manual_seed(seed)
    B, L, C = 2, (700 if per_class else 200), 5
    s = torch.rand(B, L, C, generator=g) * 0.5 + 0.45
    return _pp(_boxes(g, B, L, cluster=2), s.float(), 0.5, 0.5, 1024, 1024)


def _large_coords(seed, per_class):
    g = torch.Generator().manual_seed(seed)
    B, L, C = 2, (900 if per_class else 300), 6
    boxes = _boxes(g, B, L, span=4000.0, size=(30.0, 300.0)) + 1.0e6
    s = torch.rand(B, L, C, generator=g)
    return _pp(boxes, s.float(), 0.6 if not per_class else 0.35, 0.6, 1024, 1024)


# ------------------------------------------------------------------------------------------------------- non-finite / batch
def _nonfinite_boxes(seed, what, per_class):
    g = torch.Generator().manual_seed(seed)
    B, L, C = 2, (1500 if per_class else 300), 4
    boxes = _boxes(g, B, L, span=300.0)
    s = torch.rand(B, L, C, generator=g)
    thr = 0.45 if per_class else 0.6
    m = torch.rand(B, L, 4, generator=g) < 0.02
    if what == "nan":
        boxes[m] = float("nan")
    elif what == "inf":
        boxes[..., 2:][m[..., 2:]] = float("inf")
        boxes[..., :2][m[..., :2]] = float("-inf")
    else:  # -inf only: the maximum stays finite
        boxes[m] = float("-inf")
    return _pp(boxes, s.float(), thr, 0.5, 1024, 1024)


def _nan_scores(seed, multi):
    g = torch.Generator().manual_seed(seed)
    B, L, C = 2, 500, 5
    s = torch.rand(B, L, C, generator=g)
    s[torch.rand(B, L, C, generator=g) < 0.05] = float("nan")
    s[0, :40, 1] = float("nan")  # NaN after column 0, next to large scores
    s[0, :40, 2] = 0.99
    s[1, :20, 0] = float("nan")  # NaN in column 0
    return _pp(_boxes(g, B, L), s.float(), 0.5, 0.65, 300, 300, multi)


def _signed_zero(seed, top_k):
    # single-label at score_threshold 0.0 admits +0.0 and -0.0 (`>=`); they tie in the reference's sort
    g = torch.Generator().manual_seed(seed)
    B, L, C = 2, 300, 3
    s = torch.rand(B, L, C, generator=g) * 0.5 - 0.6  # negative: fails the threshold
    z = torch.rand(B, L, generator=g)
    s[..., 0] = torch.where(z < 0.3, torch.tensor(-0.0), torch.where(z < 0.6, torch.tensor(0.0), s[..., 0]))
    s[:, :5, 1] = 0.25  # a few positive scores ahead of the zeros
    return _pp(_boxes(g, B, L, span=150.0), s.float(), 0.0, 0.5, top_k, 300, False)


def _mixed_batch(seed):
    g = torch.Generator().manual_seed(seed)
    B, L, C = 3, 3000, 4
    return _pp(_boxes(g, B, L), _planted(g, B, L, C, 0.5, [0, 1300, 17]), 0.5, 0.65, 1000, 300)


def _max_out(seed, max_out):
    g = torch.Generator().manual_seed(seed)
    B, L, C = 2, 1200, 2
    return _pp(_boxes(g, B, L), _planted(g, B, L, C, 0.5, [1100, 1050]), 0.5, 0.65, 1024, max_out)


# ----------------------------------------------------------------------------------------------------------- public callers
def _yolox(seed, A, C, counts, multi=True, agnostic=False, conf=0.4):
    """YoloX-format predictions [B, A, 5 + C] (cx, cy, w, h, objectness, class scores) with exactly counts[b] candidates in image b
    (multi-label: (anchor, class) pairs above conf; single-label: anchors), objectness above conf everywhere, with_confidence off."""
    g = torch.Generator().manual_seed(seed)
    B = len(counts)
    cls = _planted(g, B, A, C, conf, counts, per_anchor=not multi)
    cxy = _boxes(g, B, A)[..., :2] + 20.0
    wh = 8.0 + torch.rand(B, A, 2, generator=g) * 50
    obj = conf + (1 - conf) * (0.05 + 0.95 * torch.rand(B, A, 1, generator=g))
    pred = torch.cat([cxy, wh, obj, cls], -1).float()
    return dict(kind="yolox", pred=pred, params=dict(conf_thres=conf, iou_thres=0.6, multi_label_per_box=multi, with_confidence=False, class_agnostic_nms=agnostic))


def _yolox_single_ulps(seed):
    # single-label with `>` (thr_inclusive off) at fp32(0.3) and its neighbours
    c = _thr_ulps(seed, False)
    s = c["scores"]
    g = torch.Generator().manual_seed(seed + 1)
    B, L, C = s.shape
    cxy = torch.rand(B, L, 2, generator=g) * 200 + 20
    wh = 8.0 + torch.rand(B, L, 2, generator=g) * 50
    obj = torch.full((B, L, 1), 0.9)
    return dict(kind="yolox", pred=torch.cat([cxy, wh, obj, s], -1).float(), params=dict(conf_thres=0.3, iou_thres=0.6, multi_label_per_box=False, with_confidence=False, class_agnostic_nms=False))


def _pose(seed, L, quant, thr, pre, post):
    g = torch.Generator().manual_seed(seed)
    B, J = 2, 5
    boxes = _boxes(g, B, L, span=300.0)
    conf = torch.rand(B, L, 1, generator=g)
    if quant == "ulps":
        t = np.float32(thr)
        vals = torch.tensor([np.nextafter(t, np.float32(0)), t, np.nextafter(t, np.float32(1))], dtype=torch.float32)
        on = torch.rand(B, L, 1, generator=g) < 0.5
        conf = torch.where(on, vals[torch.randint(0, 3, (B, L, 1), generator=g)], conf)
    elif quant is not None:
        conf = torch.floor(conf * 2**quant) / 2**quant
    coords = torch.rand(B, L, J, 2, generator=g) * 300
    jscores = torch.rand(B, L, J, generator=g)
    return dict(kind="pose", boxes=boxes, conf=conf.float(), coords=coords, jscores=jscores,
                params=dict(pose_confidence_threshold=thr, nms_iou_threshold=0.6, pre_nms_max_predictions=pre, post_nms_max_predictions=post))  # fmt: skip


CASES = {
    # ---- path matrix: direct scan (rows of at most 4 slices)
    "direct_k512": lambda: _matrix(101, 2, 600, 4, 512, [512, 513]),
    "direct_k513": lambda: _matrix(102, 2, 600, 4, 513, [513, 514]),
    "direct_k1000": lambda: _matrix(103, 2, 800, 4, 1000, [1000, 1001]),
    "direct_k1001": lambda: _matrix(104, 2, 800, 4, 1001, [1001, 1002]),
    "direct_k1024": lambda: _matrix(105, 2, 900, 4, 1024, [1024, 1025], max_out=1024),
    "direct_agnostic_k512": lambda: _matrix(106, 2, 600, 4, 512, [512, 513], agnostic=True),
    "direct_agnostic_k1024": lambda: _matrix(107, 2, 900, 4, 1024, [1024, 1025], agnostic=True),
    "single_k512": lambda: _matrix(108, 2, 1200, 4, 512, [512, 513], multi=False),
    "single_k1000": lambda: _matrix(109, 2, 1500, 4, 1000, [1000, 1001], multi=False),
    "single_k1024": lambda: _matrix(110, 2, 1500, 4, 1024, [1024, 1025], multi=False, max_out=1024),
    "single_agnostic_k1001": lambda: _matrix(111, 2, 1500, 4, 1001, [1001, 1002], multi=False, agnostic=True),
    # ---- path matrix: pre-filter (8400 x 80, and 8401 x 13 whose odd images start unaligned and whose last slice is short)
    "prefilter_k512": lambda: _matrix(121, 2, 8400, 80, 512, [512, 513]),
    "prefilter_agnostic_k512": lambda: _matrix(122, 2, 8400, 80, 512, [512, 513], agnostic=True),
    "prefilter_k1000": lambda: _matrix(123, 2, 8400, 80, 1000, [1000, 1001]),
    "prefilter_k1001": lambda: _matrix(124, 2, 8400, 80, 1001, [1001, 1002]),
    "prefilter_k1024": lambda: _matrix(125, 2, 8400, 80, 1024, [1024, 1025], max_out=1024),
    "prefilter_agnostic_k1024": lambda: _matrix(126, 2, 8400, 80, 1024, [1024, 5000], agnostic=True),
    "prefilter_unaligned_k1010": lambda: _matrix(127, 3, 8401, 13, 1010, [1010, 1011, 30000]),
    "prefilter_unaligned_k513": lambda: _matrix(128, 3, 8401, 13, 513, [513, 514, 400]),
    # ---- ties and thresholds
    "tied_prefilter": lambda: _tied_prefilter(131),
    "tied_direct": lambda: _tied_direct(132),
    "all_equal_multi": lambda: _all_equal(133, True),
    "all_equal_single": lambda: _all_equal(134, False),
    "thr_ulps_multi": lambda: _thr_ulps(135, True),
    "thr_ulps_single": lambda: _thr_ulps(136, False),
    "inf_scores": lambda: _inf_scores(137),
    # ---- boxes
    "iou_exact_half": lambda: _iou_edges(141, 0.5, 0.5),
    "iou_ulps_065": lambda: _iou_edges(142, 0.65, 0.65),
    "degenerate_boxes": lambda: _degenerate(143),
    "same_box_classes_trick": lambda: _same_box_classes(144, False),
    "same_box_classes_per_class": lambda: _same_box_classes(145, True),
    "large_coords_trick": lambda: _large_coords(146, False),
    "large_coords_per_class": lambda: _large_coords(147, True),
    # ---- non-finite inputs and batch shapes
    "nan_box_trick": lambda: _nonfinite_boxes(151, "nan", False),
    "nan_box_per_class": lambda: _nonfinite_boxes(152, "nan", True),
    "inf_box_trick": lambda: _nonfinite_boxes(153, "inf", False),
    "inf_box_per_class": lambda: _nonfinite_boxes(154, "inf", True),
    "neg_inf_box_trick": lambda: _nonfinite_boxes(155, "-inf", False),
    "nan_score_single": lambda: _nan_scores(156, False),
    "nan_score_multi": lambda: _nan_scores(157, True),
    "signed_zero_single": lambda: _signed_zero(158, 1000),
    "signed_zero_topk": lambda: _signed_zero(163, 120),
    "mixed_batch": lambda: _mixed_batch(159),
    "max_out_1": lambda: _max_out(160, 1),
    "max_out_small": lambda: _max_out(161, 37),
    "max_out_1024": lambda: _max_out(162, 1024),
    # ---- public callers
    "yolox_prefilter_1024": lambda: _yolox(171, 8400, 80, [1024, 10]),
    "yolox_direct_1024": lambda: _yolox(172, 2000, 4, [1024, 3]),
    "yolox_single_1024": lambda: _yolox(173, 3000, 6, [1024, 5], multi=False),
    "yolox_single_ulps": lambda: _yolox_single_ulps(174),
    "pose_ulps": lambda: _pose(181, 900, "ulps", 0.3, 1000, 100),
    "pose_tied_topk": lambda: _pose(182, 2000, 6, 0.2, 700, 100),
}

# cases that the reference and the parent kernel disagreed on (the kernel's NaN maximum, NaN arg-max and signed-zero sort key)
FIXED_BY_KERNEL_CHANGE = ("nan_box_trick", "nan_score_single", "signed_zero_single", "signed_zero_topk")


@functools.lru_cache(maxsize=None)
def build(name: str) -> dict:
    """The case's inputs and parameters (cached: callers must not modify them)."""
    return CASES[name]()


def nms_mode(case: dict, nsel: int) -> str:
    """How torchvision's batched_nms (CPU) runs on nsel candidates, and so which branch of the kernel serves them."""
    p = case["params"]
    if case["kind"] == "pose" or p.get("class_agnostic_nms"):
        return "agnostic"
    return "trick" if 4 * nsel <= 4000 else "per_class"


def order_defined(case: dict):
    """Per image: True when the reference's output order is fully determined, so that the oracle must match it row for row.  It is
    not when equal scores were selected by torch.topk (their order is implementation defined) or reach the per-class path (whose
    final sort is not stable)."""
    k = top_k_of(case)
    res = []
    for s, tied in zip(candidate_scores(case), tied_selection(case)):
        res.append(not tied or (s.size <= k and nms_mode(case, s.size) != "per_class"))
    return res


# ----------------------------------------------------------------------------------------------------- per-image selection
def candidate_scores(case: dict):
    """Per image: the scores that pass the threshold, in candidate-list order, as the kernel and the reference enumerate them."""
    p = case["params"]
    out = []
    if case["kind"] == "ppyoloe":
        for ss in case["scores"]:
            if p["multi_label_per_box"]:
                out.append(ss[ss > p["score_threshold"]].numpy())
            else:
                m = ss.max(1).values
                out.append(m[m >= p["score_threshold"]].numpy())
    elif case["kind"] == "yolox":
        for pr in case["pred"]:
            cls = pr[:, 5:][pr[:, 4] > p["conf_thres"]]
            out.append(cls[cls > p["conf_thres"]].numpy() if p["multi_label_per_box"] else cls.max(1).values[cls.max(1).values > p["conf_thres"]].numpy())
    else:
        for cc in case["conf"]:
            cc = cc.reshape(-1)
            out.append(cc[cc >= p["pose_confidence_threshold"]].numpy())
    return out


def top_k_of(case: dict) -> int:
    p = case["params"]
    return {"ppyoloe": lambda: p["nms_top_k"], "yolox": lambda: KMAX, "pose": lambda: p["pre_nms_max_predictions"]}[case["kind"]]()


def tied_cut(case: dict):
    """Per image: True when more than top_k pass and the top_k-th largest score equals the next one.  torch.topk's choice among the
    tied entries is implementation defined there, so only the count and the score multiset of the selection are determined."""
    k = top_k_of(case)
    res = []
    for s in candidate_scores(case):
        srt = np.sort(s)[::-1]
        res.append(bool(srt.size > k and srt[k - 1] == srt[k]))
    return res


def tied_selection(case: dict):
    """Per image: True when the top_k selection (or, below top_k, the candidate list) holds equal scores.  The order of equal scores
    in the reference's output then depends on torch.topk's order (selection) or on torchvision's per-class sort, which is not
    stable; the kept set and the score order are still determined when the cut itself is not tied."""
    k = top_k_of(case)
    res = []
    for s in candidate_scores(case):
        sel = np.sort(s)[::-1][:k]
        res.append(bool(np.unique(sel).size < sel.size))
    return res


def merge_candidates(name: str, b: int):
    """Image b of a ppyoloe case as a sliding-window merge input: the candidates passing the threshold (boxes [n, 4], scores [n],
    labels [n] float) in candidate-list order."""
    c = build(name)
    p, s = c["params"], c["scores"][b]
    if p["multi_label_per_box"]:
        a, j = (s > p["score_threshold"]).nonzero().T
        conf = s[a, j]
    else:
        conf, j = s.max(1)
        m = conf >= p["score_threshold"]
        a, conf, j = m.nonzero().flatten(), conf[m], j[m]
    return c["boxes"][b][a], conf, j.float()


# the merge's edge cases: NaN / +-inf boxes under the coordinate trick (n <= 1000) and per class, +-0.0 scores
MERGE_EDGE_CASES = ("nan_box_trick", "nan_box_per_class", "inf_box_trick", "signed_zero_single")


# ----------------------------------------------------------------------------------------------------- stored reference rows
def reference_outputs(case: dict, g: dict):
    """The stored reference outputs of a case (tests/golden/nms_edges.pt entry `g`), per image: ppyoloe rows [N, 6], yolox rows or
    None, pose (poses, scores, boxes); and per image the sorted pre-NMS scores of a tied cut, or None."""
    out, o = [], 0
    for b, n in enumerate(g["count"]):
        out.append(None if n < 0 else rows_from_idx(case, b, g["idx"][o : o + n]))
        o += max(n, 0)
    pre, o = [], 0
    for t in tied_cut(case):
        k = min(top_k_of(case), 10**9)
        pre.append(g["pre_nms"][o : o + k] if t else None)
        o += k if t else 0
    return out, pre


def _bits(t):
    return t.contiguous().view(torch.int32)


def _xyxy(pred):
    """(cx, cy, w, h) -> (x1, y1, x2, y2) of YoloX rows, as the reference's convert_cxcywh_bbox_to_xyxy rounds it."""
    return torch.stack([pred[:, 0] - pred[:, 2] / 2, pred[:, 1] - pred[:, 3] / 2, pred[:, 0] + pred[:, 2] / 2, pred[:, 1] + pred[:, 3] / 2], 1)


def rows_from_idx(case: dict, b: int, idx):
    """The output of image b as a gather of the inputs: ppyoloe / yolox rows [N, 6] = (box of anchor idx // C, score idx, class
    idx % C) for flat indices idx = anchor * C + class; pose (poses [N, J, 3], scores [N], boxes [N, 4]) for anchor indices idx."""
    idx = torch.as_tensor(idx, dtype=torch.int64)
    if case["kind"] == "yolox":
        pr = case["pred"][b]
        C = pr.shape[-1] - 5
        a, c = idx // C, idx % C
        return torch.cat([_xyxy(pr)[a], pr[a, 5 + c][:, None], c[:, None].float()], 1)
    if case["kind"] == "ppyoloe":
        C = case["scores"].shape[-1]
        a, c = idx // C, idx % C
        return torch.cat([case["boxes"][b][a], case["scores"][b].reshape(-1)[idx, None], c[:, None].float()], 1)
    poses = torch.cat([case["coords"][b][idx], case["jscores"][b][idx][..., None]], -1)
    return poses, case["conf"][b].reshape(-1)[idx], case["boxes"][b][idx]


def idx_of_rows(case: dict, b: int, rows):
    """Inverse of rows_from_idx for the reference's output: the flat (ppyoloe) or anchor (pose) index of every row, found by the
    bit pattern of its box (every case's boxes are distinct within an image, NaN payloads included)."""
    boxes = _xyxy(case["pred"][b]) if case["kind"] == "yolox" else case["boxes"][b]
    where = {}
    for a, key in enumerate(map(tuple, _bits(boxes).tolist())):
        where.setdefault(key, []).append(a)
    out_boxes = rows[2] if case["kind"] == "pose" else rows[:, :4]
    C = case["pred"].shape[-1] - 5 if case["kind"] == "yolox" else case.get("scores", torch.zeros(1)).shape[-1]
    idx = []
    for r, key in enumerate(map(tuple, _bits(out_boxes).tolist())):
        (a,) = where[key]
        idx.append(a if case["kind"] == "pose" else a * C + int(rows[r, 5]))
    return torch.tensor(idx, dtype=torch.int32)
