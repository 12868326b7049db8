#!/usr/bin/env python
"""Times one PoseEstimationMetrics.update() on a validation-size batch: 64 images, 30 post-NMS poses each (the pose recipe's
callback), up to 30 targets per image including crowd ones, 17 joints, 10 OKS thresholds.  CUDA events around the call, median
of 20 after warm-up; prints one JSON line.  Usage: python tools/time_pose_metrics.py"""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def validation_batch(B=64, n_anchor=600, J=17, seed=0):
    """Decoded YOLO-NAS-POSE outputs of a validation-size batch (anchors are jittered copies of the targets plus clutter) and the
    per-image ground truth: up to 30 targets per image, some crowd, some with every joint invisible."""
    gen = torch.Generator().manual_seed(seed)
    boxes, conf, coords, jsc, samples = [], [], [], [], []
    for b in range(B):
        nt = int(torch.randint(5, 31, (1,), generator=gen))
        xy = torch.rand(nt, 2, generator=gen) * 500 + 20
        wh = torch.rand(nt, 2, generator=gen) * 100 + 20
        joints = torch.cat([xy[:, None] + torch.rand(nt, J, 2, generator=gen) * wh[:, None], torch.randint(0, 3, (nt, J, 1), generator=gen).float()], -1)
        joints[torch.rand(nt, generator=gen) < 0.08, :, 2] = 0
        crowd = (torch.rand(nt, generator=gen) < 0.1).numpy()
        src = torch.randint(0, nt, (n_anchor,), generator=gen)
        scale = torch.rand(n_anchor, 1, 1, generator=gen) * 12
        c = joints[src, :, :2] + torch.randn(n_anchor, J, 2, generator=gen) * scale
        bx = torch.cat([xy[src], xy[src] + wh[src]], 1) + torch.randn(n_anchor, 4, generator=gen) * 8
        boxes.append(bx)
        conf.append(torch.rand(n_anchor, 1, generator=gen))
        coords.append(c)
        jsc.append(torch.rand(n_anchor, J, generator=gen))
        samples.append(type("Sample", (), dict(joints=joints.numpy(), bboxes_xywh=torch.cat([xy, wh], 1).numpy(), areas=(wh.prod(1) * 0.6).numpy(), is_crowd=crowd))())
    preds = ((torch.stack(boxes).cuda(), torch.stack(conf).cuda(), torch.stack(coords).cuda(), torch.stack(jsc).cuda()), None)
    return preds, samples


def recipe_callback():
    from super_gradients_b200.training.models.pose_estimation_models.yolo_nas_pose.yolo_nas_pose_post_prediction_callback import YoloNASPosePostPredictionCallback

    # recipes/training_hyperparams/coco2017_yolo_nas_pose_train_params.yaml:48-58
    return YoloNASPosePostPredictionCallback(pose_confidence_threshold=0.01, nms_iou_threshold=0.7, pre_nms_max_predictions=300, post_nms_max_predictions=30)



def main():
    from super_gradients_b200.training.metrics import PoseEstimationMetrics

    preds, samples = validation_batch()
    metric = PoseEstimationMetrics(post_prediction_callback=recipe_callback(), num_joints=17, max_objects_per_image=30)
    for _ in range(5):
        metric.update(preds, None, gt_samples=samples)
    torch.cuda.synchronize()
    times = []
    for _ in range(20):
        metric.reset()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        metric.update(preds, None, gt_samples=samples)
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    times.sort()
    print(json.dumps({"update_ms_median": (times[9] + times[10]) / 2, "update_ms_min": times[0], "update_ms_max": times[-1], "images": 64, "gpu": torch.cuda.get_device_name()}))


if __name__ == "__main__":
    main()
