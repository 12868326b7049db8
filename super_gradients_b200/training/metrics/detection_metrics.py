"""DetectionMetrics (row (f)-N4; reference: training/metrics/detection_metrics.py:27-468): precision / recall / F1 / mAP of a
detector over a validation run.

`update()` is the per-batch part: NMS (the callback's batched kernel) followed by ONE matching kernel for the whole batch
(csrc/detection_match.cu) -- no Python loop over images or (prediction, target) pairs and no device->host synchronisation; the
flags stay on the device until `compute()`, which copies them once and runs the reference's summary arithmetic
(utils/detection_utils.compute_detection_metrics).  The class keeps the reference's constructor, `update(preds, target, device,
inputs, crowd_targets)`, `compute()` keys and `greater_component_is_better` so `valid_metrics_list` / `metric_to_watch` entries
written for the reference work unchanged.  It is a plain object (torchmetrics is not a dependency): `reset()` clears the state,
and in a distributed run `compute()` gathers every rank's flags (all_gather_object, as the reference's _sync_dist does)."""
import collections
from typing import Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch
from torch import Tensor

from ...common.registry import register_metric
from ..utils.detection_utils import (DistanceMatching, DistanceMetric, EuclideanDistance, IouThreshold, compute_detection_matching_batched, compute_detection_matching_with,
                                     compute_detection_metrics, pad_predictions)  # fmt: skip


@register_metric("DetectionMetrics")
class DetectionMetrics:
    def __init__(self, num_cls: int, post_prediction_callback=None, normalize_targets: bool = False,
                 iou_thres: Union[IouThreshold, Tuple[float, float], float] = IouThreshold.MAP_05_TO_095, recall_thres: Tensor = None, score_thres: float = 0.1,
                 top_k_predictions: int = 100, dist_sync_on_step: bool = False, accumulate_on_cpu: bool = True, calc_best_score_thresholds: bool = True,
                 include_classwise_ap: bool = False, class_names: List[str] = None, state_dict_prefix: str = ""):  # fmt: skip
        class_names = ["class_" + str(i) for i in range(num_cls)] if class_names is None else list(class_names)
        if len(class_names) != num_cls:
            raise ValueError(f"Number of class names ({len(class_names)}) does not match number of classes ({num_cls})")
        self.num_cls, self.iou_thres, self.class_names = num_cls, iou_thres, class_names
        if isinstance(iou_thres, tuple):  # IouThreshold members are tuples too
            self.iou_thresholds = IouThreshold.from_bounds(*iou_thres)
        else:
            self.iou_thresholds = torch.tensor([iou_thres], dtype=torch.float32)
        rng = self._get_range_str()
        self.map_str = "mAP" + rng
        self.include_classwise_ap = include_classwise_ap
        self.precision_metric_key, self.recall_metric_key = f"{state_dict_prefix}Precision{rng}", f"{state_dict_prefix}Recall{rng}"
        self.f1_metric_key, self.map_metric_key = f"{state_dict_prefix}F1{rng}", f"{state_dict_prefix}mAP{rng}"
        better = [(self.precision_metric_key, True), (self.recall_metric_key, True), (self.map_metric_key, True), (self.f1_metric_key, True)]
        if include_classwise_ap:
            self.per_class_ap_names = [f"{state_dict_prefix}AP{rng}_{n}" for n in class_names]
            better += [(k, True) for k in self.per_class_ap_names]
        self.greater_component_is_better = collections.OrderedDict(better)
        self.component_names = list(self.greater_component_is_better.keys())
        self.calc_best_score_thresholds = calc_best_score_thresholds
        self.best_threshold_per_class_names = [f"Best_score_threshold_{n}" for n in class_names]
        if calc_best_score_thresholds:
            self.component_names.append("Best_score_threshold")
        if calc_best_score_thresholds and include_classwise_ap:
            self.component_names += self.best_threshold_per_class_names
        self.components = len(self.component_names)
        self.post_prediction_callback = post_prediction_callback
        self.denormalize_targets = not normalize_targets
        self.recall_thresholds = torch.linspace(0, 1, 101) if recall_thres is None else torch.as_tensor(recall_thres, dtype=torch.float32)
        self.score_threshold, self.top_k_predictions = score_thres, top_k_predictions
        self.accumulate_on_cpu = accumulate_on_cpu
        self.state_key = f"{state_dict_prefix}matching_info{rng}"
        self._thr_dev = None
        self.reset()

    def _get_range_str(self):
        t = self.iou_thresholds
        return "@%.2f" % t[0] if not len(t) > 1 else "@%.2f:%.2f" % (t[0], t[-1])

    def reset(self):
        self._batches = []  # (rows [B, P, 6], counts [B], matched, ignore [B, P, T], target classes) -- device tensors, no sync

    def to(self, device):
        return self

    @torch.no_grad()
    def update(self, preds, target: Tensor, device=None, inputs: Tensor = None, crowd_targets: Optional[Tensor] = None) -> None:
        """preds: raw model output (run through post_prediction_callback) or, with no callback, the per-image list of NMS rows;
        target / crowd_targets [N, 6] (image, class, cx, cy, w, h); inputs: the batch (only its H x W is read)."""
        height, width = inputs.shape[-2:]
        cb = self.post_prediction_callback
        if cb is not None and hasattr(cb, "forward_batched"):
            rows, _idx, counts = cb.forward_batched(preds)
        else:
            out = cb(preds, device=device) if cb is not None else preds
            dev = next((o.device for o in out if o is not None), inputs.device)
            rows, counts = pad_predictions(out, dev)
        matched, ignore = self._match(rows, counts, target, height, width, crowd_targets)
        self._batches.append((rows[..., 4:6], counts, matched, ignore, target.detach()[:, 1].float().cpu().clone()))

    def _match(self, rows, counts, target, height, width, crowd_targets):
        """The batch's one matching launch: (matched, ignore) uint8 [B, P, T] on the device."""
        if self._thr_dev is None or self._thr_dev.device != rows.device:
            self._thr_dev = self.iou_thresholds.to(rows.device)
        return compute_detection_matching_batched(rows, counts, target, height, width, self._thr_dev, self.denormalize_targets, crowd_targets, self.top_k_predictions)

    def _n_thresholds(self) -> int:
        return len(self.iou_thresholds)

    def _matching_info(self):
        """Device state -> the reference's five flat tensors (preds_matched, preds_to_ignore, scores, classes, target classes)."""
        T = self._n_thresholds()
        m, g, s, c, t = [torch.zeros((0, T), dtype=torch.bool)], [torch.zeros((0, T), dtype=torch.bool)], [torch.zeros(0)], [torch.zeros(0)], [torch.zeros(0)]
        for sc_cls, counts, matched, ignore, tcls in self._batches:
            counts = counts.cpu()
            valid = torch.arange(sc_cls.shape[1]).unsqueeze(0) < counts.unsqueeze(1)
            sc_cls, matched, ignore = sc_cls.cpu(), matched.cpu(), ignore.cpu()
            m.append(matched[valid].bool())
            g.append(ignore[valid].bool())
            s.append(sc_cls[..., 0][valid])
            c.append(sc_cls[..., 1][valid])
            t.append(tcls)
        return [torch.cat(x, 0) for x in (m, g, s, c, t)]

    def compute(self) -> Dict[str, Union[float, Tensor]]:
        mean_ap, mean_precision, mean_recall, mean_f1, best_score_threshold = -1.0, -1.0, -1.0, -1.0, -1.0
        best_score_threshold_per_cls, mean_ap_per_class = np.zeros(self.num_cls), np.zeros(self.num_cls)
        info = self._matching_info()
        if torch.distributed.is_available() and torch.distributed.is_initialized() and torch.distributed.get_world_size() > 1:
            gathered = [None] * torch.distributed.get_world_size()
            torch.distributed.all_gather_object(gathered, info)
            info = [torch.cat([g[i] for g in gathered], 0) for i in range(5)]
        if len(self._batches):
            ap, precision, recall, f1, present, best_score_threshold, best_per_cls = compute_detection_metrics(
                *info, device="cpu", recall_thresholds=self.recall_thresholds, score_threshold=self.score_threshold
            )
            mean_precision, mean_recall, mean_f1, mean_ap = precision.mean(), recall.mean(), f1.mean(), ap.mean()
            ap_per_class = ap.mean(1)
            for i, ci in enumerate(present):
                mean_ap_per_class[ci] = float(ap_per_class[i])
                best_score_threshold_per_cls[ci] = float(best_per_cls[i])
        out = {self.precision_metric_key: float(mean_precision), self.recall_metric_key: float(mean_recall), self.map_metric_key: float(mean_ap), self.f1_metric_key: float(mean_f1)}
        if self.include_classwise_ap:
            for i, v in enumerate(mean_ap_per_class):
                out[self.per_class_ap_names[i]] = float(v)
        if self.calc_best_score_thresholds:
            out["Best_score_threshold"] = float(best_score_threshold)
        if self.include_classwise_ap and self.calc_best_score_thresholds:
            for n, v in zip(self.best_threshold_per_class_names, best_score_threshold_per_cls):
                out[n] = float(v)
        return out


@register_metric("DetectionMetricsDistanceBased")
class DetectionMetricsDistanceBased(DetectionMetrics):
    """DetectionMetricsDistanceBased (detection_metrics.py:295-374): DetectionMetrics with a true positive defined by the distance
    between box centres (EuclideanDistance or ManhattanDistance, in pixels, strictly below the threshold) instead of IoU -- for
    point-like or tiny objects and crowded scenes.  update() is the batched NMS plus ONE distance-matching launch
    (csrc/detection_match.cu), with no device->host synchronisation; compute(), reset() and the distributed gather are
    DetectionMetrics'.  Keys carry the prefix "distance_based_" and the range "@DIST5.00" / "@DIST5.00:10.00"."""

    def __init__(self, num_cls: int, post_prediction_callback, normalize_targets: bool = False, distance_thresholds: Sequence[float] = (5.0,),
                 distance_metric: DistanceMetric = EuclideanDistance(), recall_thres: Tensor = None, score_thres: float = 0.1, top_k_predictions: int = 100,
                 dist_sync_on_step: bool = False, accumulate_on_cpu: bool = True, calc_best_score_thresholds: bool = True, include_classwise_ap: bool = False,
                 class_names: List[str] = None):  # fmt: skip
        # the range string -- and so every component name -- is built from these inside DetectionMetrics.__init__
        self.distance_thresholds = distance_thresholds
        self.distance_metric = distance_metric
        self._matcher = DistanceMatching(distance_metric, distance_thresholds)
        self._matcher.kernel_metric()  # a metric without a kernel fails here, not at the first validation batch
        DetectionMetrics.__init__(self, num_cls=num_cls, post_prediction_callback=post_prediction_callback, normalize_targets=normalize_targets, recall_thres=recall_thres,
                                  score_thres=score_thres, top_k_predictions=top_k_predictions, dist_sync_on_step=dist_sync_on_step, accumulate_on_cpu=accumulate_on_cpu,
                                  calc_best_score_thresholds=calc_best_score_thresholds, include_classwise_ap=include_classwise_ap, class_names=class_names,
                                  state_dict_prefix="distance_based_")  # fmt: skip

    def _get_range_str(self):
        t = self.distance_thresholds
        return "@DIST%.2f" % t[0] if not len(t) > 1 else "@DIST%.2f:%.2f" % (t[0], t[-1])

    def _match(self, rows, counts, target, height, width, crowd_targets):
        return compute_detection_matching_with(self._matcher, rows, counts, target, height, width, self.denormalize_targets, crowd_targets, self.top_k_predictions)

    def _n_thresholds(self) -> int:
        return len(self.distance_thresholds)


def _fixed(name, iou_thres):
    def __init__(self, num_cls: int, post_prediction_callback=None, normalize_targets: bool = False, recall_thres: Tensor = None, score_thres: float = 0.1,
                 top_k_predictions: int = 100, dist_sync_on_step: bool = False, accumulate_on_cpu: bool = True, calc_best_score_thresholds: bool = True,
                 include_classwise_ap: bool = False, class_names: List[str] = None):  # fmt: skip
        DetectionMetrics.__init__(self, num_cls, post_prediction_callback, normalize_targets, iou_thres, recall_thres, score_thres, top_k_predictions, dist_sync_on_step,
                                  accumulate_on_cpu, calc_best_score_thresholds, include_classwise_ap, class_names)  # fmt: skip

    return register_metric(name)(type(name, (DetectionMetrics,), {"__init__": __init__, "__doc__": f"DetectionMetrics at IoU {iou_thres} (detection_metrics.py:375-468)."}))


DetectionMetrics_050 = _fixed("DetectionMetrics_050", IouThreshold.MAP_05)
DetectionMetrics_075 = _fixed("DetectionMetrics_075", 0.75)
DetectionMetrics_050_095 = _fixed("DetectionMetrics_050_095", IouThreshold.MAP_05_TO_095)
