"""Test infrastructure: numpy restatement of the reference's PoseEstimationMetrics matching and summary
(training/metrics/pose_estimation_metrics.py:237-381, training/metrics/pose_estimation_utils.py:8-263), each function citing the
reference lines.  Pinned against outputs of the unmodified reference (tests/golden/pose_metrics.pt, made by
tests/golden/make_pose_goldens.py); the product never imports it."""
import numpy as np

from oracle.sg_oracle import detection_metrics_per_cls

COCO_OKS_SIGMAS = np.array([0.026, 0.025, 0.025, 0.035, 0.035, 0.079, 0.079, 0.072, 0.072, 0.062, 0.062, 0.107, 0.107, 0.087, 0.087, 0.089, 0.089])


def visible_bbox_xywh(joints: np.ndarray) -> np.ndarray:
    """compute_visible_bbox_xywh (pose_estimation_utils.py:8-32) with the numpy semantics it was written for (np.min / np.max with
    where= and initial=): joints [M, J, 3] -> float32 XYWH [M, 4]."""
    joints = np.asarray(joints, np.float32)
    joints = joints.reshape(len(joints), -1, 3) if joints.size else joints.reshape(0, 1, 3)
    vis = joints[:, :, 2] > 0
    init = np.float32(1_000_000)
    x1 = np.min(joints[:, :, 0], where=vis, initial=init, axis=-1)
    y1 = np.min(joints[:, :, 1], where=vis, initial=init, axis=-1)
    x1[x1 == init] = 0
    y1[y1 == init] = 0
    x2 = np.max(joints[:, :, 0], where=vis, initial=np.float32(0), axis=-1)
    y2 = np.max(joints[:, :, 1], where=vis, initial=np.float32(0), axis=-1)
    return np.stack([x1, y1, x2 - x1, y2 - y1], -1).astype(np.float32)


def keypoint_oks_matrix(pred_xy: np.ndarray, gt_joints: np.ndarray, sigmas: np.ndarray, areas: np.ndarray, bboxes: np.ndarray) -> np.ndarray:
    """compute_oks (pose_estimation_utils.py:35-96): OKS [K, M] of K predicted poses (x, y first) against M targets (x, y,
    visibility), float32 in the reference's operation order; exp and the per-pair sum in float64, rounded to float32 once."""
    f32 = np.float32
    pred_xy = np.asarray(pred_xy, f32)
    gt = np.asarray(gt_joints, f32).reshape(len(gt_joints), len(sigmas), 3)
    out = np.zeros((len(pred_xy), len(gt)), f32)
    s2 = np.asarray(sigmas, f32) * f32(2)
    var = s2 * s2
    areas, bboxes = np.asarray(areas, f32), np.asarray(bboxes, f32).reshape(-1, 4)
    for t in range(len(gt)):
        vis = gt[t, :, 2] > 0
        k1 = int(vis.sum())
        x, y, w, h = bboxes[t]
        x0, x1, y0, y1 = x - w, x + w * f32(2), y - h, y + h * f32(2)
        a = areas[t] + f32(np.finfo(np.float64).eps)
        for k in range(len(pred_xy)):
            xd, yd = pred_xy[k, :, 0], pred_xy[k, :, 1]
            if k1 > 0:
                dx, dy = xd - gt[t, :, 0], yd - gt[t, :, 1]
            else:
                dx = np.maximum(x0 - xd, f32(0)) + np.maximum(xd - x1, f32(0))
                dy = np.maximum(y0 - yd, f32(0)) + np.maximum(yd - y1, f32(0))
            e = (dx * dx + dy * dy) / var / a / f32(2)
            if k1 > 0:
                e = e[vis]
            out[k, t] = f32(np.exp(-e.astype(np.float64)).sum() / len(e))
    return out


def pose_keypoint_matching_image(poses, scores, gt_joints, gt_bboxes, gt_areas, gt_iscrowd, iou_thresholds, sigmas, top_k):
    """PoseEstimationMetrics.update_single_image + compute_img_keypoint_matching (pose_estimation_metrics.py:237-314,
    pose_estimation_utils.py:107-263) for one image.  Returns None when the image has neither predictions nor targets (the reference
    records nothing for it), else a dict: matched / ignore [k, T] bool and scores [k] in confidence order (k = min(top_k, P); equal
    scores by prediction index), num_targets, and the OKS matrices of the used predictions against the regular / ignored targets."""
    f32 = np.float32
    poses = np.asarray(poses, f32).reshape(len(poses), -1, 3) if len(poses) else np.zeros((0, len(sigmas), 3), f32)
    scores = np.asarray(scores, f32).reshape(-1)
    gt = np.asarray(gt_joints, f32).reshape(len(gt_joints), -1, 3) if len(gt_joints) else np.zeros((0, len(sigmas), 3), f32)
    if len(poses) == 0 and len(gt) == 0:
        return None
    thr = np.asarray(iou_thresholds, f32)
    T = len(thr)
    boxes = visible_bbox_xywh(gt) if gt_bboxes is None else np.asarray(gt_bboxes).reshape(-1, 4)
    areas = (boxes[:, 2] * boxes[:, 3]) if gt_areas is None else np.asarray(gt_areas)
    boxes, areas = boxes.astype(f32), np.asarray(areas).astype(f32).reshape(-1)
    crowd = np.zeros(len(gt), bool) if gt_iscrowd is None else np.asarray(gt_iscrowd).astype(bool).reshape(-1)
    ignored = (gt[:, :, 2] == 0).all(1) | crowd
    reg, ign = np.nonzero(~ignored)[0], np.nonzero(ignored)[0]
    k = min(top_k, len(scores))
    use = np.argsort(-scores, kind="stable")[:k]
    matched = np.zeros((k, T), bool)
    ignore = np.zeros((k, T), bool)
    oks_reg = keypoint_oks_matrix(poses[use][:, :, :2], gt[reg], sigmas, areas[reg], boxes[reg])
    oks_ign = keypoint_oks_matrix(poses[use][:, :, :2], gt[ign], sigmas, areas[ign], boxes[ign])
    t_matched = np.zeros((len(reg), T), bool)
    for i in range(k):  # :196-233, targets_ignored is all False here (see pose_match_math.cuh)
        row = oks_reg[i]
        for t in np.argsort(-np.where(np.isnan(row), np.inf, row), kind="stable"):
            v = row[t]
            if not v > thr[0]:
                continue
            good = (v > thr) & ~matched[i] & ~t_matched[t]
            t_matched[t] |= good
            matched[i] |= good
    if len(ign):  # :237-256
        best = np.where(np.isnan(oks_ign).any(1), np.nan, np.nan_to_num(oks_ign, nan=0.0).max(1))
        ignore |= best[:, None] > thr[None, :]
    return dict(matched=matched, ignore=ignore, scores=scores[use], num_targets=int(len(reg)), oks=oks_reg, oks_crowd=oks_ign)


def pose_keypoint_matching(predictions, gt_joints, gt_bboxes, gt_areas, gt_iscrowd, iou_thresholds, sigmas, top_k):
    """Batch form: per-image lists (predictions = [(poses, scores)], gt_* = per-image arrays or None lists)."""
    n = len(predictions)
    pick = lambda lst, i: None if lst is None else lst[i]  # noqa: E731
    return [pose_keypoint_matching_image(predictions[i][0], predictions[i][1], gt_joints[i], pick(gt_bboxes, i), pick(gt_areas, i), pick(gt_iscrowd, i), iou_thresholds, sigmas, top_k)
            for i in range(n)]  # fmt: skip


def pose_metrics(results, iou_thresholds, recall_thresholds=None, iou_thresholds_to_report=None):
    """PoseEstimationMetrics.compute (pose_estimation_metrics.py:335-381) over per-image results of pose_keypoint_matching_image."""
    f32 = np.float32
    thr = np.asarray(iou_thresholds, f32)
    rt = np.linspace(0.0, 1.00, 101, endpoint=True, dtype=f32) if recall_thresholds is None else np.asarray(recall_thresholds, f32)
    T = len(thr)
    precision, recall = -np.ones((T, 1)), -np.ones((T, 1))
    results = [r for r in results if r is not None]
    if results:
        m = np.concatenate([r["matched"] for r in results], 0)
        g = np.concatenate([r["ignore"] for r in results], 0)
        s = np.concatenate([r["scores"] for r in results], 0)
        ap, _p, rec, _f1, _best = detection_metrics_per_cls(m, g, s, sum(r["num_targets"] for r in results), rt, 0)
        precision[:, 0], recall[:, 0] = ap, rec

    def summarize(v):
        return -1 if len(v[v > -1]) == 0 else float(np.mean(v[v > -1]))

    out = {"AP": summarize(precision), "AR": summarize(recall)}
    for t in np.asarray(iou_thresholds_to_report if iou_thresholds_to_report is not None else [], f32):
        mask = np.where(t == thr)[0]
        out[f"AP_{t:.2f}"], out[f"AR_{t:.2f}"] = summarize(precision[mask]), summarize(recall[mask])
    return out
