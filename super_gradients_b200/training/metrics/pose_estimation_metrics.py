"""PoseEstimationMetrics (reference: training/metrics/pose_estimation_metrics.py:24-381, pose_estimation_utils.py:35-263): COCO
keypoint AP / AR of a single-class pose model, with object keypoint similarity (OKS) in place of box IoU.

`update()` is the per-batch part: the callback's batched NMS (or the per-image prediction list, padded on the device), the batch's
ground truth packed into one pinned host buffer and sent with one non-blocking copy, and ONE matching kernel for the whole batch
(csrc/pose_match.cu) -- no Python loop over (target, prediction) pairs and no device->host synchronisation.  The flags stay on the
device until `compute()`, which copies them once and runs the reference's summary (compute_detection_metrics_per_cls at score
threshold 0, then the mean over thresholds).  The class keeps the reference's constructor, `update()` / `update_single_image()`
signatures, `compute()` keys and `greater_component_is_better`, so the pose recipe's `valid_metrics_list` entry and
`metric_to_watch: AP` work unchanged.  It is a plain object (torchmetrics is not a dependency): `reset()` clears the state, and in a
distributed run `compute()` gathers every rank's flags with all_gather_object, as the reference's _sync_dist does."""
import logging
from typing import Any, Dict, Iterable, List, Optional, Union

import numpy as np
import torch
from torch import Tensor

from ... import kernels as K
from ...common.registry import register_metric
from ..utils.detection_utils import compute_detection_metrics_per_cls

logger = logging.getLogger(__name__)

__all__ = ["PoseEstimationMetrics"]

COCO_OKS_SIGMAS = [0.026, 0.025, 0.025, 0.035, 0.035, 0.079, 0.079, 0.072, 0.072, 0.062, 0.062, 0.107, 0.107, 0.087, 0.087, 0.089, 0.089]

# bits of the per-target flag byte read by sgb_pose_keypoint_matching
FLAG_CROWD, FLAG_HAS_BOX, FLAG_HAS_AREA = 1, 2, 4


@register_metric("PoseEstimationMetrics")
class PoseEstimationMetrics:
    def __init__(self, post_prediction_callback, num_joints: int, max_objects_per_image: int = 20, oks_sigmas: Optional[Iterable] = None, iou_thresholds: Optional[Iterable] = None,
                 recall_thresholds: Optional[Iterable] = None, iou_thresholds_to_report: Optional[Iterable] = None):  # fmt: skip
        """pose_estimation_metrics.py:45-129: COCO defaults (10 OKS thresholds 0.50:0.95, 101 recall points, the COCO sigmas for 17
        joints); `iou_thresholds_to_report` adds AP_t / AR_t keys for thresholds among `iou_thresholds`."""
        self.num_joints = num_joints
        self.max_objects_per_image = max_objects_per_image
        self.stats_names = ["AP", "AR"]
        if recall_thresholds is None:
            recall_thresholds = np.linspace(0.0, 1.00, int(np.round((1.00 - 0.0) / 0.01)) + 1, endpoint=True, dtype=np.float32)
        self.recall_thresholds = torch.tensor(recall_thresholds, dtype=torch.float32)
        if iou_thresholds is None:
            iou_thresholds = np.linspace(0.5, 0.95, int(np.round((0.95 - 0.5) / 0.05)) + 1, endpoint=True, dtype=np.float32)
        self.iou_thresholds = torch.tensor(iou_thresholds, dtype=torch.float32)
        if iou_thresholds_to_report is not None:
            self.iou_thresholds_to_report = np.array([float(t) for t in iou_thresholds_to_report], dtype=np.float32)
            missing = ~np.isin(self.iou_thresholds_to_report, self.iou_thresholds.numpy())
            if missing.any():
                raise RuntimeError(f"One or many IoU thresholds to report are not present in IoU thresholds. Missing thresholds: {self.iou_thresholds_to_report[missing]}")
            self.stats_names += [f"AP_{t:.2f}" for t in self.iou_thresholds_to_report]
            self.stats_names += [f"AR_{t:.2f}" for t in self.iou_thresholds_to_report]
        else:
            self.iou_thresholds_to_report = None
        self.greater_component_is_better = dict((k, True) for k in self.stats_names)
        if oks_sigmas is None:
            if num_joints == 17:
                oks_sigmas = np.array(COCO_OKS_SIGMAS)
            else:
                oks_sigmas = np.array([0.1] * num_joints)
                logger.warning(f"Using default OKS sigmas of `0.1` for a custom dataset with {num_joints} joints. "
                               f"To silence this warning, you may want to specify OKS sigmas explicitly as it has direct impact on the AP score.")  # fmt: skip
        if len(oks_sigmas) != num_joints:
            raise ValueError(f"Length of oks_sigmas ({len(oks_sigmas)}) should be equal to num_joints {num_joints}")
        self.oks_sigmas = torch.tensor(oks_sigmas).float()
        self.component_names = list(self.greater_component_is_better.keys())
        self.components = len(self.component_names)
        self.post_prediction_callback = post_prediction_callback
        self.reset()

    def reset(self) -> None:
        # per batch: (matched, ignore [B, K, T] u8, used scores [B, K], used count [B], regular targets [B]) on the device, and the
        # host-side ground-truth counts [B] (an image with neither predictions nor targets is skipped, as in the reference)
        self._batches = []

    def to(self, device):
        return self

    @torch.no_grad()
    def update(self, preds: Any, target: Any, gt_joints: List[np.ndarray] = None, gt_iscrowd: List[np.ndarray] = None, gt_bboxes: List[np.ndarray] = None,
               gt_areas: List[np.ndarray] = None, gt_samples: List[Any] = None) -> None:  # fmt: skip
        """pose_estimation_metrics.py:134-235.  preds: the raw model output, decoded by post_prediction_callback (without a callback:
        the list of PoseEstimationPredictions itself); target is not used.  Ground truth either as `gt_samples` (objects with
        joints [N, J, 3], bboxes_xywh [N, 4] or None, areas [N] or None, is_crowd [N] or None -- what YoloNASPoseCollateFN hands to
        the trainer) or as the per-image lists gt_joints / gt_bboxes / gt_areas / gt_iscrowd (None: derived / all regular)."""
        cb = self.post_prediction_callback
        if cb is not None and hasattr(cb, "forward_batched"):
            rows, poses, _idx, count = cb.forward_batched(preds)
            n_img = poses.shape[0]
        else:
            predictions = cb(preds) if cb is not None else preds
            n_img = len(predictions)
        if gt_samples is not None:
            gt = [(s.joints, s.bboxes_xywh, getattr(s, "areas", None), s.is_crowd) for s in gt_samples]
        else:
            if any(lst is not None and len(lst) != n_img for lst in (gt_joints, gt_bboxes, gt_areas, gt_iscrowd)):
                raise ValueError(f"{n_img} images of predictions but ground-truth lists of another length")
            pick = lambda lst, i: None if lst is None else lst[i]  # noqa: E731
            gt = [(gt_joints[i], pick(gt_bboxes, i), pick(gt_areas, i), pick(gt_iscrowd, i)) for i in range(n_img)]
        if len(gt) != n_img:
            raise ValueError(f"{n_img} images of predictions but ground truth for {len(gt)}")
        if cb is not None and hasattr(cb, "forward_batched"):
            self._match(poses.float().contiguous(), rows[..., 4].contiguous(), count.to(torch.int32), gt, None)
        else:
            self._match_lists([(p.poses, p.scores) for p in predictions], gt)

    @torch.no_grad()
    def update_single_image(self, predicted_poses: Union[Tensor, np.ndarray], predicted_scores: Union[Tensor, np.ndarray], gt_joints: np.ndarray, gt_bboxes: Optional[np.ndarray],
                            gt_areas: Optional[np.ndarray], gt_iscrowd: Optional[np.ndarray]) -> None:  # fmt: skip
        """pose_estimation_metrics.py:237-314: one image -- the same kernel with a batch of one."""
        self._match_lists([(predicted_poses, predicted_scores)], [(gt_joints, gt_bboxes, gt_areas, gt_iscrowd)])

    def _match_lists(self, predictions, gt) -> None:
        """Per-image (poses [n, J, 3], scores [n]) tensors or arrays -> the padded device layout, then _match."""
        counts = [len(p) for p, _ in predictions]
        for (p, s), n in zip(predictions, counts):
            if n != len(s):
                raise ValueError("Length of predicted poses and scores should be equal. Got {} and {}".format(n, len(s)))
        dev = next((t.device for p, s in predictions for t in (p, s) if torch.is_tensor(t)), None)
        if dev is None:
            dev = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu")
        P, J = max(max(counts, default=0), 1), self.num_joints
        poses = torch.zeros((len(predictions), P, J, 3), dtype=torch.float32, device=dev)
        scores = torch.zeros((len(predictions), P), dtype=torch.float32, device=dev)
        for b, ((p, s), n) in enumerate(zip(predictions, counts)):
            if n:
                poses[b, :n] = torch.as_tensor(p).to(device=dev, dtype=torch.float32).reshape(n, J, 3)
                scores[b, :n] = torch.as_tensor(s).to(device=dev, dtype=torch.float32).reshape(n)
        self._match(poses, scores, None, gt, counts)

    def _match(self, poses: Tensor, scores: Tensor, pred_count: Optional[Tensor], gt, host_pred_count: Optional[List[int]]) -> None:
        """One kernel launch for the batch.  The ground truth (and the prediction counts when they are known on the host), sigmas and
        thresholds go to the device in one pinned buffer with one non-blocking copy."""
        dev, B, J, T = poses.device, poses.shape[0], self.num_joints, len(self.iou_thresholds)
        if poses.shape[2] != J:
            raise ValueError(f"predicted poses have {poses.shape[2]} joints, the metric was built for {J}")
        gt = [(np.zeros((0, J, 3), np.float32) if j is None else np.asarray(j), bx, ar, cr) for j, bx, ar, cr in gt]
        n_gt = np.array([len(j) for j, _, _, _ in gt], np.int32)
        M = max(int(n_gt.max(initial=0)), 1)
        sizes = dict(joints=(np.float32, B * M * J * 3), boxes=(np.float32, B * M * 4), areas=(np.float32, B * M), sigmas=(np.float32, J), thr=(np.float32, T),
                     gt_count=(np.int32, B), pred_count=(np.int32, B), flags=(np.uint8, B * M))  # fmt: skip
        offsets, total = {}, 0
        for k, (dt, n) in sizes.items():
            offsets[k] = total
            total += (n * np.dtype(dt).itemsize + 15) // 16 * 16
        buf = torch.empty(total, dtype=torch.uint8, pin_memory=dev.type == "cuda")
        raw = buf.numpy()
        host = {k: raw[offsets[k] : offsets[k] + n * np.dtype(dt).itemsize].view(dt) for k, (dt, n) in sizes.items()}
        joints, boxes, areas, flags = host["joints"].reshape(B, M, J, 3), host["boxes"].reshape(B, M, 4), host["areas"].reshape(B, M), host["flags"].reshape(B, M)
        joints[:], boxes[:], areas[:], flags[:] = 0, 0, 0, 0
        for b, (j, bx, ar, cr) in enumerate(gt):
            n = int(n_gt[b])
            if n == 0:
                continue
            if j.reshape(n, -1).shape[1] != J * 3:
                raise ValueError(f"ground-truth joints of image {b} have shape {j.shape}, expected [N, {J}, 3]")
            joints[b, :n] = j.reshape(n, J, 3)
            f = np.zeros(n, np.uint8)
            if bx is not None:
                bx = np.asarray(bx).reshape(n, 4)
                boxes[b, :n] = bx
                f |= FLAG_HAS_BOX
                if ar is None:  # pose_estimation_metrics.py:267-268, in the boxes' own dtype
                    ar = bx[:, 2] * bx[:, 3]
            if ar is not None:
                areas[b, :n] = np.asarray(ar).reshape(n)
                f |= FLAG_HAS_AREA
            if cr is not None:
                f |= np.where(np.asarray(cr).astype(bool).reshape(n), FLAG_CROWD, 0).astype(np.uint8)
            flags[b, :n] = f
        host["sigmas"][:] = self.oks_sigmas.numpy()
        host["thr"][:] = self.iou_thresholds.numpy()
        host["gt_count"][:] = n_gt
        host["pred_count"][:] = host_pred_count if host_pred_count is not None else 0
        d = buf.to(dev, non_blocking=True)
        view = lambda k, shape, dt: d[offsets[k] : offsets[k] + sizes[k][1] * np.dtype(sizes[k][0]).itemsize].view(dt).view(shape)  # noqa: E731
        if pred_count is None:
            pred_count = view("pred_count", (B,), torch.int32)
        out = K.pose_keypoint_matching(poses, scores, pred_count, view("joints", (B, M, J, 3), torch.float32), view("boxes", (B, M, 4), torch.float32), view("areas", (B, M), torch.float32),
                                       view("flags", (B, M), torch.uint8), view("gt_count", (B,), torch.int32), view("sigmas", (J,), torch.float32), view("thr", (T,), torch.float32),
                                       self.max_objects_per_image)  # fmt: skip
        self._batches.append((*out, n_gt))

    def _matching_info(self):
        """Device state -> (preds_matched [N, T] bool, preds_to_ignore [N, T] bool, preds_scores [N], num_targets, images recorded),
        with one device->host copy per kind of flag."""
        T = len(self.iou_thresholds)
        if not self._batches:
            return torch.zeros((0, T), dtype=torch.bool), torch.zeros((0, T), dtype=torch.bool), torch.zeros(0), 0, 0
        flags = torch.cat([torch.cat([m.reshape(-1), g.reshape(-1)]) for m, g, *_ in self._batches]).cpu()
        scores = torch.cat([s.reshape(-1) for _, _, s, *_ in self._batches]).cpu()
        counts = torch.cat([torch.stack([u, n]) for _, _, _, u, n, _ in self._batches], 1).cpu()
        m_all, g_all, s_all, n_targets, n_images, fo, so, co = [], [], [], 0, 0, 0, 0, 0
        for matched, _ignore, _scores, _u, _n, n_gt in self._batches:
            B, Kb = matched.shape[:2]
            m = flags[fo : fo + B * Kb * T].view(B, Kb, T)
            g = flags[fo + B * Kb * T : fo + 2 * B * Kb * T].view(B, Kb, T)
            s = scores[so : so + B * Kb].view(B, Kb)
            used, reg = counts[0, co : co + B], counts[1, co : co + B]
            fo, so, co = fo + 2 * B * Kb * T, so + B * Kb, co + B
            for b in range(B):
                n = int(used[b])
                if n == 0 and n_gt[b] == 0:
                    continue
                m_all.append(m[b, :n].bool())
                g_all.append(g[b, :n].bool())
                s_all.append(s[b, :n])
                n_targets += int(reg[b])
                n_images += 1
        if not n_images:
            return torch.zeros((0, T), dtype=torch.bool), torch.zeros((0, T), dtype=torch.bool), torch.zeros(0), 0, 0
        return torch.cat(m_all), torch.cat(g_all), torch.cat(s_all), n_targets, n_images

    def compute(self) -> Dict[str, Union[float, Tensor]]:
        """pose_estimation_metrics.py:335-381: {"AP", "AR"} (+ AP_t / AR_t), -1 when no image was recorded."""
        T = len(self.iou_thresholds)
        precision, recall = -np.ones((T, 1)), -np.ones((T, 1))
        matched, ignore, scores, n_targets, n_images = self._matching_info()
        if torch.distributed.is_available() and torch.distributed.is_initialized() and torch.distributed.get_world_size() > 1:
            gathered = [None] * torch.distributed.get_world_size()
            torch.distributed.all_gather_object(gathered, (matched, ignore, scores, n_targets, n_images))
            matched, ignore, scores = (torch.cat([g[i] for g in gathered], 0) for i in range(3))
            n_targets, n_images = sum(g[3] for g in gathered), sum(g[4] for g in gathered)
        if n_images > 0:
            cls_precision, _, cls_recall, _, _ = compute_detection_metrics_per_cls(preds_matched=matched, preds_to_ignore=ignore, preds_scores=scores, n_targets=n_targets,
                                                                                   recall_thresholds=self.recall_thresholds.cpu(), score_threshold=0, device="cpu")  # fmt: skip
            precision[:, 0] = cls_precision.cpu().numpy()
            recall[:, 0] = cls_recall.cpu().numpy()

        def summarize(s):
            return -1 if len(s[s > -1]) == 0 else float(np.mean(s[s > -1]))

        metrics = {"AP": summarize(precision), "AR": summarize(recall)}
        if self.iou_thresholds_to_report is not None and len(self.iou_thresholds_to_report):
            thr = self.iou_thresholds.numpy()
            for t in self.iou_thresholds_to_report:
                mask = np.where(t == thr)[0]
                metrics[f"AP_{t:.2f}"] = summarize(precision[mask])
                metrics[f"AR_{t:.2f}"] = summarize(recall[mask])
        return metrics
