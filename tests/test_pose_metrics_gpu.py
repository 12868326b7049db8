"""PoseEstimationMetrics on the H100: sgb_pose_keypoint_matching through the C ABI against the reference's goldens, a
validation-size batch against the numpy restatement without a device->host synchronisation in update(), and the Trainer's
validation of the tiny YOLO-NAS-POSE mirror on the device."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import host_pose_match as H  # noqa: E402
import pose_metrics_oracle as O  # noqa: E402
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tools"))
from time_pose_metrics import recipe_callback, validation_batch  # noqa: E402
from super_gradients_b200 import kernels as K  # noqa: E402
from super_gradients_b200.training.metrics import PoseEstimationMetrics  # noqa: E402

GOLD = torch.load(os.path.join(HERE, "golden", "pose_metrics.pt"), weights_only=False)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(GOLD))
def test_pose_matching_kernel_vs_reference_golden(name):
    """Flags, scores and target counts equal the reference's; OKS within 2e-6 of its compute_oks."""
    case = GOLD[name]
    J = len(case["sigmas"])
    for batch in case["batches"]:
        args = [t.cuda() for t in H.pad_golden_batch(batch["images"], J, case["no_areas"])]
        out = K.pose_keypoint_matching(*args, case["sigmas"].cuda(), case["iou_thresholds"].cuda(), case["kw"].get("max_objects_per_image", 20), oks_out=True)
        torch.cuda.synchronize()
        H.assert_matches_golden(case, batch, out)


@pytest.mark.gpu
def test_validation_size_batch_vs_oracle_without_sync():
    """64 images x 30 post-NMS poses, up to 30 targets, 17 joints, 10 thresholds: update() makes no device->host synchronisation
    (sync debug mode "error"), the flags equal the oracle's per image and compute() equals the oracle's summary."""
    preds, samples = validation_batch()
    cb = recipe_callback()
    metric = PoseEstimationMetrics(post_prediction_callback=cb, num_joints=17, max_objects_per_image=30, iou_thresholds_to_report=[0.5, 0.75])
    metric.update(preds, None, gt_samples=samples)  # warm-up: library load, first allocations
    metric.reset()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        metric.update(preds, None, gt_samples=samples)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    rows, poses, _idx, count = (t.cpu() for t in cb.forward_batched(preds))
    assert int(count.min()) == 30, "the batch should fill every image's 30 post-NMS slots"
    matched, ignore, used_scores, used_count, n_targets, _n_gt = metric._batches[0]
    matched, ignore, used_scores, used_count, n_targets = (t.cpu() for t in (matched, ignore, used_scores, used_count, n_targets))
    thr, sig = metric.iou_thresholds.numpy(), metric.oks_sigmas.numpy()
    res = []
    for b, s in enumerate(samples):
        ref = O.pose_keypoint_matching_image(poses[b].numpy(), rows[b, :, 4].numpy(), s.joints, s.bboxes_xywh, s.areas, s.is_crowd, thr, sig, 30)
        res.append(ref)
        assert int(used_count[b]) == 30 and int(n_targets[b]) == ref["num_targets"]
        assert np.array_equal(matched[b].bool().numpy(), ref["matched"]), b
        assert np.array_equal(ignore[b].bool().numpy(), ref["ignore"]), b
        assert np.array_equal(used_scores[b].numpy(), ref["scores"]), b
    assert sum(int(r["matched"][:, 0].sum()) for r in res) > 100 and sum(int(r["ignore"][:, 0].sum()) for r in res) > 0
    got, want = metric.compute(), O.pose_metrics(res, thr, iou_thresholds_to_report=[0.5, 0.75])
    assert list(got) == list(want)
    for k in want:
        assert got[k] == pytest.approx(want[k], abs=1e-6), k


@pytest.mark.gpu
def test_trainer_validates_pose_model_with_pose_metrics_on_device(golden, tmp_path):
    """The end-to-end validation of tests/test_pose_metrics_host.py on the device: AP / AR every epoch equal the oracle on the
    callback's outputs, and the checkpoint's acc holds the best AP."""
    from test_pose_metrics_host import oracle_ap, pose_validation_setup

    from super_gradients_b200.training.sg_trainer import Trainer

    m, g, valid, cb = pose_validation_setup(golden)
    aps = []
    orig = PoseEstimationMetrics.compute

    def compute(self):
        r = orig(self)
        aps.append(r)
        return r

    PoseEstimationMetrics.compute = compute
    try:
        tp = dict(max_epochs=2, initial_lr=1e-3, lr_mode="constant", optimizer="AdamW", optimizer_params={"weight_decay": 1e-5}, zero_weight_decay_on_bias_and_bn=True, ema=False,
                  loss="yolo_nas_pose_loss", criterion_params=dict(oks_sigmas=g["sigmas"], **g["kw"]), save_model=True, metric_to_watch="AP", greater_metric_to_watch_is_better=True,
                  valid_metrics_list=[{"PoseEstimationMetrics": {"num_joints": 5, "oks_sigmas": g["sigmas"], "max_objects_per_image": 30, "post_prediction_callback": cb}}])  # fmt: skip
        trainer = Trainer("pose_metric_gpu", ckpt_root_dir=str(tmp_path))
        hist = trainer.train(m, tp, [(g["x"], g["targets"]), (g["x"] * 0.9, g["targets"])], valid_loader=valid)
    finally:
        PoseEstimationMetrics.compute = orig
    assert len(hist["valid_loss"]) == 2 and len(aps) == 2 and len(cb.seen) == 4
    assert sum(int(s[3].sum()) for s in cb.seen) > 0
    for e in range(2):
        want = oracle_ap(cb.seen[2 * e : 2 * e + 2], valid, g["sigmas"])
        assert aps[e]["AP"] == pytest.approx(want["AP"], abs=1e-6) and aps[e]["AR"] == pytest.approx(want["AR"], abs=1e-6)
    ck = torch.load(tmp_path / "pose_metric_gpu" / "ckpt_latest.pth", weights_only=False)
    assert ck["acc"] == pytest.approx(max(a["AP"] for a in aps))
