"""YoloX-format post-processing (row N3; reference: training/utils/detection_utils.py:63-86, 279-334): objectness filter,
objectness x class score, multi- or single-label candidates, class-aware or class-agnostic NMS -- on the same one-CTA-per-image
kernel as the PP-YOLOE / YOLO-NAS callback (csrc/nms.cu), i.e. for the whole batch in one launch instead of a Python loop over
images around torchvision.  The kernel keeps its IoU bit-matrix in shared memory, so an image may have at most 1024 candidates
above the confidence threshold; more raise (the reference has no such limit).

Second half (row (f)-N4): the DetectionMetrics helpers -- IouThreshold, target / prediction padding, the matching strategies
(IoUMatching, DistanceMatching with EuclideanDistance / ManhattanDistance), the batched matching kernels' wrappers with the
reference's `compute_detection_matching` signature on top, and the precision / recall / AP summary."""
import enum
from abc import ABC, abstractmethod
from typing import List, Optional, Sequence, Tuple, Union

import numpy as np
import torch
from torch import Tensor

from ... import kernels as K
from ...lib import SgbError

MAX_CANDIDATES = 1024


def convert_cxcywh_bbox_to_xyxy(input_bbox: Tensor) -> Tensor:
    """[..., (cx, cy, w, h)] -> [..., (x1, y1, x2, y2)], 2-d (one image) or 3-d (a batch) like the reference."""
    cx, cy, w, h = input_bbox[..., 0], input_bbox[..., 1], input_bbox[..., 2], input_bbox[..., 3]
    return torch.stack([cx - w / 2, cy - h / 2, cx + w / 2, cy + h / 2], -1)


@torch.no_grad()
def non_max_suppression(prediction: Tensor, conf_thres: float = 0.1, iou_thres: float = 0.6, multi_label_per_box: bool = True, with_confidence: bool = False,
                        class_agnostic_nms: bool = False) -> List[Optional[Tensor]]:  # fmt: skip
    """prediction [B, A, 5 + C] = (cx, cy, w, h, objectness, class scores).  Returns, per image, [n, 6] rows
    (x1, y1, x2, y2, confidence, class) in descending confidence, or None when nothing survives (as the reference does)."""
    K.require_cuda(prediction, "prediction")
    pred = prediction.float()
    obj = pred[..., 4]
    cls = pred[..., 5:] * obj.unsqueeze(-1) if with_confidence else pred[..., 5:]
    # anchors whose objectness fails the filter can never become candidates: their class scores drop below any threshold
    scores = torch.where((obj > conf_thres).unsqueeze(-1), cls, torch.full_like(cls, -1.0)).contiguous()
    passing = scores > conf_thres
    n_cand = (passing.sum((1, 2)) if multi_label_per_box else passing.any(-1).sum(1)).max()
    if int(n_cand) > MAX_CANDIDATES:  # one host read; this is the predict / validation path
        raise SgbError(f"non_max_suppression: {int(n_cand)} candidates above conf_thres={conf_thres} in one image; the NMS kernel holds at most {MAX_CANDIDATES}")
    boxes = convert_cxcywh_bbox_to_xyxy(pred[..., :4]).contiguous()
    rows, _idx, count = K.batched_nms(boxes, scores, conf_thres, iou_thres, MAX_CANDIDATES, MAX_CANDIDATES, multi_label=multi_label_per_box, class_agnostic=class_agnostic_nms,
                                      thr_inclusive=False)  # fmt: skip
    counts = count.tolist()
    return [rows[b, : counts[b]] if counts[b] else None for b in range(rows.shape[0])]


# ------------------------------------------------------------------------------------------------ validation metrics (row (f)-N4)

class IouThreshold(tuple, enum.Enum):
    """detection_utils.py:231-254."""

    MAP_05 = (0.5, 0.5)
    MAP_05_TO_095 = (0.5, 0.95)

    def is_range(self):
        return self[0] != self[1]

    def to_tensor(self):
        return self.from_bounds(self[0], self[1], step=0.05) if self.is_range() else torch.tensor([self[0]])

    @classmethod
    def from_bounds(cls, low: float, high: float, step: float = 0.05) -> Tensor:
        return torch.linspace(low, high, int(round((high - low) / step)) + 1)


def pad_matching_targets_host(targets: Tensor, batch_size: int) -> Tuple[Tensor, Tensor]:
    """flat [N, 6] (image, class, cx, cy, w, h) -> ([B, M, 5] float32 rows (class, cx, cy, w, h), counts [B] int32) on the host, M =
    the largest per-image count (>= 1), rows kept in their original order -- the layout sgb_detection_matching reads."""
    t = targets.detach().float().cpu().numpy().reshape(-1, 6)
    img = t[:, 0].astype(np.int64)
    keep = (img >= 0) & (img < batch_size)
    t, img = t[keep], img[keep]
    order = np.argsort(img, kind="stable")
    t, img = t[order], img[order]
    counts = np.bincount(img, minlength=batch_size).astype(np.int32)
    padded = np.zeros((batch_size, max(int(counts.max()) if len(counts) else 0, 1), 5), np.float32)
    if len(t):
        first = np.searchsorted(img, np.arange(batch_size))
        padded[img, np.arange(len(t)) - first[img]] = t[:, 1:]
    return torch.from_numpy(padded), torch.from_numpy(counts)


def pad_predictions(output: List[Optional[Tensor]], device) -> Tuple[Tensor, Tensor]:
    """Per-image list of [n, 6] NMS rows (None: no prediction) -> the padded ([B, P, 6], counts [B]) layout of batched_nms."""
    counts = [0 if o is None else int(o.shape[0]) for o in output]
    rows = torch.zeros((len(output), max(max(counts, default=0), 1), 6), dtype=torch.float32, device=device)
    for b, o in enumerate(output):
        if counts[b]:
            rows[b, : counts[b]] = o.to(device=device, dtype=torch.float32)
    return rows, torch.tensor(counts, dtype=torch.int32, device=device)


class IoUMatching:
    """IoUMatching (detection_utils.py:880-904): the matching strategy object of the reference's API; here it only carries the IoU
    thresholds -- compute_targets / compute_crowd_targets are the matching kernel."""

    def __init__(self, iou_thresholds: Tensor):
        self.iou_thresholds = iou_thresholds

    def get_thresholds(self) -> Tensor:
        return self.iou_thresholds


class DistanceMetric(ABC):
    """detection_utils.py:1293-1296.  Only the two metrics below have a kernel (csrc/detection_match.cu); calculate_distance is the
    reference's torch expression, kept as the definition the kernel is tested against."""

    @abstractmethod
    def calculate_distance(self, predicted: Tensor, target: Tensor) -> Tensor:
        pass


class EuclideanDistance(DistanceMetric):
    """detection_utils.py:1299-1318: L2 distance between box centres, [N, 4] x [M, 4] XYXY -> [N, M]."""

    def calculate_distance(self, predicted: Tensor, target: Tensor) -> Tensor:
        centers1 = (predicted[:, :2] + predicted[:, 2:]) / 2
        centers2 = (target[:, :2] + target[:, 2:]) / 2
        diff = centers1.view(-1, 1, 2) - centers2.view(1, -1, 2)
        return torch.sqrt((diff**2).sum(dim=2))


class ManhattanDistance(DistanceMetric):
    """detection_utils.py:1321-1339: L1 distance between box centres, [N, 4] x [M, 4] XYXY -> [N, M]."""

    def calculate_distance(self, predicted: Tensor, target: Tensor) -> Tensor:
        centers1 = (predicted[:, :2] + predicted[:, 2:]) / 2
        centers2 = (target[:, :2] + target[:, 2:]) / 2
        diff = centers1.view(-1, 1, 2) - centers2.view(1, -1, 2)
        return torch.abs(diff).sum(dim=2)


# the kernel's name of each metric it implements (exact types: a subclass may redefine the distance)
_KERNEL_DISTANCE = {EuclideanDistance: "euclidean", ManhattanDistance: "manhattan"}


class DistanceMatching:
    """DistanceMatching (detection_utils.py:1008-1030): a prediction matches the nearest free same-class target whose box centre is
    nearer than the threshold (pixels, strict); compute_targets / compute_crowd_targets are the distance matching kernel."""

    def __init__(self, distance_metric: DistanceMetric, distance_thresholds: Union[Sequence[float], Tensor]):
        self.distance_metric = distance_metric
        self.distance_thresholds = distance_thresholds

    def get_thresholds(self) -> Tensor:
        return torch.tensor(self.distance_thresholds)

    def kernel_metric(self) -> str:
        """The kernel's name of the distance metric; any other DistanceMetric raises."""
        name = _KERNEL_DISTANCE.get(type(self.distance_metric))
        if name is None:
            raise NotImplementedError(f"only EuclideanDistance and ManhattanDistance have a kernel, got {type(self.distance_metric).__name__}")
        return name


@torch.no_grad()
def compute_detection_matching(output: List[Optional[Tensor]], targets: Tensor, height: int, width: int, denormalize_targets: bool, device: str = None,
                               iou_thresholds: Tensor = None, crowd_targets: Optional[Tensor] = None, top_k: int = 100, return_on_cpu: bool = True,
                               matching_strategy: Union[IoUMatching, DistanceMatching] = None) -> List[Tuple]:  # fmt: skip
    """The reference's signature and return value (detection_utils.py:1120-1193): per image (preds_matched [n, T] bool,
    preds_to_ignore [n, T] bool, scores [n], classes [n], target classes).  One kernel launch for the batch
    (compute_detection_matching_with), then one device->host copy to split the flags per image."""
    if matching_strategy is None:
        raise ValueError("matching_strategy must not be None")
    if not isinstance(matching_strategy, (IoUMatching, DistanceMatching)):
        raise NotImplementedError(f"only IoUMatching and DistanceMatching have a kernel, got {type(matching_strategy).__name__}")
    output = list(output)
    dev = next((o.device for o in output if o is not None), torch.device(device) if device is not None else targets.device)
    rows, counts = pad_predictions(output, dev)
    matched, ignore = compute_detection_matching_with(matching_strategy, rows, counts, targets, height, width, denormalize_targets, crowd_targets, top_k)
    if return_on_cpu:
        rows, matched, ignore = rows.cpu(), matched.cpu(), ignore.cpu()
    t = targets.detach().float().to(rows.device)
    res = []
    for b, o in enumerate(output):
        n = 0 if o is None else int(o.shape[0])
        res.append((matched[b, :n].bool(), ignore[b, :n].bool(), rows[b, :n, 4], rows[b, :n, 5], t[t[:, 0] == b, 1]))
    return res


def _padded_targets(dev, B: int, targets: Tensor, crowd_targets: Optional[Tensor]):
    """The reference's flat [N, 6] targets / crowd targets -> the kernels' padded per-image layout on `dev` (crowd: None, None when
    there is none)."""
    t_pad, t_cnt = pad_matching_targets_host(targets, B)
    c_pad = c_cnt = None
    if crowd_targets is not None and crowd_targets.numel():
        c_pad, c_cnt = pad_matching_targets_host(crowd_targets, B)
        c_pad, c_cnt = c_pad.to(dev, non_blocking=True), c_cnt.to(dev, non_blocking=True)
    return t_pad.to(dev, non_blocking=True), t_cnt.to(dev, non_blocking=True), c_pad, c_cnt


@torch.no_grad()
def compute_detection_matching_batched(rows: Tensor, counts: Tensor, targets: Tensor, height: int, width: int, iou_thresholds: Tensor, denormalize_targets: bool,
                                       crowd_targets: Optional[Tensor] = None, top_k: int = 100) -> Tuple[Tensor, Tensor]:  # fmt: skip
    """compute_detection_matching + IoUMatching (detection_utils.py:1120-1290, :880-1005) for a whole batch in one kernel launch.
    rows / counts: the padded NMS output ([B, P, 6], [B]) on the device; targets / crowd_targets: the reference's flat [N, 6]
    (image, class, cx, cy, w, h) tensors (read on the host, where the data loader left them).  Returns uint8 [B, P, T] tensors
    (preds_matched, preds_to_ignore); prediction rows past counts[b] are zero."""
    dev = rows.device
    t_pad, t_cnt, c_pad, c_cnt = _padded_targets(dev, rows.shape[0], targets, crowd_targets)
    return K.detection_matching(rows.contiguous().float(), counts.to(torch.int32), t_pad, t_cnt, c_pad, c_cnt, iou_thresholds.to(device=dev, dtype=torch.float32).contiguous(),
                                height, width, top_k, denormalize_targets)  # fmt: skip


@torch.no_grad()
def compute_detection_matching_with(matching_strategy: Union[IoUMatching, DistanceMatching], rows: Tensor, counts: Tensor, targets: Tensor, height: int, width: int,
                                    denormalize_targets: bool, crowd_targets: Optional[Tensor] = None, top_k: int = 100) -> Tuple[Tensor, Tensor]:  # fmt: skip
    """compute_detection_matching_batched for either strategy: IoUMatching runs the IoU kernel, DistanceMatching
    (detection_utils.py:1008-1118) the centre-distance kernel -- one launch for the batch either way, same inputs and outputs.  The
    distance thresholds are read on the host (they are launch parameters), so no device synchronisation happens here."""
    if isinstance(matching_strategy, IoUMatching):
        return compute_detection_matching_batched(rows, counts, targets, height, width, matching_strategy.get_thresholds(), denormalize_targets, crowd_targets, top_k)
    if not isinstance(matching_strategy, DistanceMatching):
        raise NotImplementedError(f"only IoUMatching and DistanceMatching have a kernel, got {type(matching_strategy).__name__}")
    metric = matching_strategy.kernel_metric()
    t_pad, t_cnt, c_pad, c_cnt = _padded_targets(rows.device, rows.shape[0], targets, crowd_targets)
    return K.detection_distance_matching(rows.contiguous().float(), counts.to(torch.int32), t_pad, t_cnt, c_pad, c_cnt, matching_strategy.get_thresholds(), metric, height, width,
                                         top_k, denormalize_targets)  # fmt: skip


def compute_detection_metrics_per_cls(preds_matched: Tensor, preds_to_ignore: Tensor, preds_scores: Tensor, n_targets, recall_thresholds: Tensor, score_threshold: float, device="cpu"):
    """Precision / recall at `score_threshold`, the F1-optimal confidence and the 101-point interpolated AP of one class for
    every IoU threshold (detection_utils.py:1449-1580).  Host-side summary arithmetic on the accumulated matching flags, once per
    validation run; same torch operations, in the same order, as the reference."""
    nb_iou, nb_score = preds_matched.shape[-1], len(recall_thresholds)
    zeros = torch.zeros(nb_iou, device=device)
    if len(preds_matched) == 0:
        return zeros, zeros.clone(), zeros.clone(), torch.zeros(nb_score, device=device), torch.tensor(0.0, device=device)
    tps = preds_matched
    fps = torch.logical_and(torch.logical_not(preds_matched), torch.logical_not(preds_to_ignore))
    sort_ind = torch.argsort(preds_scores, descending=True)
    tps, fps, preds_scores = tps[sort_ind, :], fps[sort_ind, :], preds_scores[sort_ind].contiguous()
    rolling_tps, rolling_fps = torch.cumsum(tps, 0, dtype=torch.float), torch.cumsum(fps, 0, dtype=torch.float)
    rolling_recalls = rolling_tps / n_targets
    rolling_precisions = rolling_tps / (rolling_tps + rolling_fps + torch.finfo(torch.float64).eps)
    rolling_precisions = rolling_precisions.flip(0).cummax(0).values.flip(0)

    k = int(torch.searchsorted(-preds_scores, torch.tensor(-score_threshold, dtype=preds_scores.dtype, device=device), right=True))
    recall, precision = (zeros, zeros.clone()) if k == 0 else (rolling_recalls[k - 1], rolling_precisions[k - 1])

    all_score_thresholds = torch.linspace(0, 1, nb_score, device=device)
    ks = torch.searchsorted(-preds_scores, -all_score_thresholds, right=True)
    pad = torch.zeros(1, nb_iou, device=device)
    recalls_t = torch.cat((pad, rolling_recalls), 0).index_select(0, ks)
    precisions_t = torch.cat((pad, rolling_precisions), 0).index_select(0, ks)
    f1_t = 2 * recalls_t * precisions_t / (recalls_t + precisions_t + 1e-16)
    mean_f1_per_threshold = f1_t.mean(1)
    best_score_threshold = all_score_thresholds[torch.argmax(mean_f1_per_threshold)]

    rt = recall_thresholds.to(device).view(1, -1).repeat(nb_iou, 1)
    idx = torch.searchsorted(rolling_recalls.T.contiguous(), rt, right=False).T
    ap = torch.gather(torch.cat((rolling_precisions, pad), 0), 0, idx).mean(0)
    return ap, precision, recall, mean_f1_per_threshold, best_score_threshold


def compute_detection_metrics(preds_matched: Tensor, preds_to_ignore: Tensor, preds_scores: Tensor, preds_cls: Tensor, targets_cls: Tensor, device="cpu",
                              recall_thresholds: Optional[Tensor] = None, score_threshold: float = 0.1):  # fmt: skip
    """detection_utils.py:1361-1446: (ap, precision, recall, f1) [n_present_classes, T], the present classes, the overall best
    confidence threshold and the per-class ones."""
    preds_matched, preds_to_ignore = preds_matched.to(device).bool(), preds_to_ignore.to(device).bool()
    preds_scores, preds_cls, targets_cls = preds_scores.to(device), preds_cls.to(device), targets_cls.to(device)
    recall_thresholds = torch.linspace(0, 1, 101, device=device) if recall_thresholds is None else recall_thresholds.to(device)
    unique_classes = torch.unique(targets_cls).long()
    n_class, nb_iou, nb_score = len(unique_classes), preds_matched.shape[-1], len(recall_thresholds)
    ap, precision, recall = (torch.zeros((n_class, nb_iou), device=device) for _ in range(3))
    f1_per_class_per_threshold = torch.zeros((n_class, nb_score), device=device)
    best_score_threshold_per_cls = torch.zeros(n_class, device=device)
    for i, c in enumerate(unique_classes):
        sel = preds_cls == c
        ap[i], precision[i], recall[i], f1_per_class_per_threshold[i], best_score_threshold_per_cls[i] = compute_detection_metrics_per_cls(
            preds_matched[sel], preds_to_ignore[sel], preds_scores[sel], (targets_cls == c).sum(), recall_thresholds, score_threshold, device
        )
    f1 = 2 * precision * recall / (precision + recall + 1e-16)
    best_score_threshold = torch.linspace(0, 1, nb_score, device=device)[torch.argmax(f1_per_class_per_threshold.mean(0))]
    return ap, precision, recall, f1, unique_classes, best_score_threshold, best_score_threshold_per_cls
