"""DetectionMetricsDistanceBased on the H100: the distance matching kernel (csrc/detection_match.cu) against the reference's
flags and compute() dictionary in tests/golden/distance_matching.pt, the IoU kernel's flags on the same scenes unchanged, the
entry point's argument checks, and Trainer.test() with the metric on the tiny YOLO-NAS fixture."""
import copy
import ctypes
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import distance_matching_cases as DC  # noqa: E402
import host_detection_match  # noqa: E402
from super_gradients_b200 import kernels as K  # noqa: E402
from super_gradients_b200 import lib as L  # noqa: E402
from super_gradients_b200.training.metrics import DetectionMetricsDistanceBased  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name,metric", DC.CASES)
def test_kernel_flags_match_reference(name, metric):
    case = DC.GOLD[name]
    H_, W_ = case["hw"]
    for i, batch in enumerate(case["batches"]):
        rows, counts, t_pad, t_cnt, c_pad, c_cnt = DC.padded(batch, "cuda")
        matched, ignore = K.detection_distance_matching(rows, counts, t_pad, t_cnt, c_pad, c_cnt, case["thresholds"], metric, H_, W_, case["top_k"], case["normalized"])
        DC.assert_flags_equal(matched, ignore, counts, case[metric]["matching"][i], (name, metric, i))


@pytest.mark.parametrize("name,metric", DC.CASES)
def test_compute_equals_reference(name, metric):
    case = DC.GOLD[name]
    m = DetectionMetricsDistanceBased(num_cls=case["n_cls"], post_prediction_callback=None, normalize_targets=not case["normalized"], distance_thresholds=list(case["thresholds"]),
                                      distance_metric=DC.METRICS[metric](), recall_thres=case["recall_thresholds"], score_thres=case["score_thres"],
                                      top_k_predictions=case["top_k"], include_classwise_ap=True)  # fmt: skip
    n0 = L.LAUNCHES[0]
    for batch in case["batches"]:
        out = [None if o is None else o.cuda() for o in batch["output"]]
        m.update(out, batch["targets"], device="cuda", inputs=torch.zeros(len(out), 3, *case["hw"], device="cuda"), crowd_targets=batch["crowd_targets"])
    assert L.LAUNCHES[0] - n0 == len(case["batches"])  # one matching launch per batch
    DC.assert_compute_equal(m.compute(), case[metric]["compute"])


@pytest.mark.parametrize("name", sorted(DC.GOLD))
def test_iou_kernel_unchanged_on_the_same_scenes(name):
    """sgb_detection_matching shares the kernel body: its flags on these scenes equal the serial host driver of the IoU arithmetic
    (which tests/test_detection_match_host.py pins to the reference)."""
    case = DC.GOLD[name]
    H_, W_ = case["hw"]
    thr = torch.linspace(0.5, 0.95, 10)
    for batch in case["batches"]:
        rows, counts, t_pad, t_cnt, c_pad, c_cnt = DC.padded(batch, "cuda")
        matched, ignore = K.detection_matching(rows, counts, t_pad, t_cnt, c_pad, c_cnt, thr.cuda(), H_, W_, case["top_k"], case["normalized"])
        h_rows, h_counts, h_t, h_tc, h_c, h_cc = DC.padded(batch)
        want_m, want_g = host_detection_match.detection_matching(h_rows, h_counts, h_t, h_tc, h_c, h_cc, thr, H_, W_, case["top_k"], case["normalized"])
        assert torch.equal(matched.cpu(), want_m) and torch.equal(ignore.cpu(), want_g)


def test_invalid_arguments_are_refused():
    """Ordinary host-side argument checks: SGB_E_INVALID (-1) and nothing launched."""
    case = DC.GOLD["edges_pixels_thr5"]
    rows, counts, t_pad, t_cnt, c_pad, c_cnt = DC.padded(case["batches"][0], "cuda")
    lib = L.load()
    out = torch.zeros(rows.shape[0], rows.shape[1], 40, dtype=torch.uint8, device="cuda")

    def call(thr, metric=0, max_preds=None):
        d = K.match_desc(rows, t_pad, c_pad, len(thr), 100, 120, 100, False)
        if max_preds is not None:
            d.max_preds = max_preds
        host = (ctypes.c_float * len(thr))(*thr)
        p = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
        return lib.sgb_detection_distance_matching(ctypes.byref(d), metric, p(rows), p(counts), p(t_pad), p(t_cnt), p(c_pad), p(c_cnt), ctypes.cast(host, ctypes.c_void_p), p(out),
                                                   p(out), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))  # fmt: skip

    assert call([5.0], metric=2) == -1 and call([5.0], metric=-1) == -1
    assert call([5.0, float("nan")]) == -1 and call([float("inf")]) == -1 and call([-1.0]) == -1
    assert call([1.0] * 33) == -1 and call([]) == -1
    assert call([5.0], max_preds=8000) == -1  # 8000 predictions of one image exceed the 200 KB of shared memory
    assert call([5.0, 0.0]) == 0 and call([5.0], metric=1) == 0
    torch.cuda.synchronize()
    with pytest.raises(L.SgbError, match="code -1"):
        K.detection_distance_matching(rows, counts, t_pad, t_cnt, c_pad, c_cnt, [-2.0], "euclidean", 100, 120)
    with pytest.raises(L.SgbError, match="distance metric"):
        K.detection_distance_matching(rows, counts, t_pad, t_cnt, c_pad, c_cnt, [2.0], "chebyshev", 100, 120)


def test_trainer_test_with_distance_metric(golden, tmp_path):
    from super_gradients_b200.training.losses import PPYoloELoss
    from super_gradients_b200.training.models.detection_models.pp_yolo_e.post_prediction_callback import PPYoloEPostPredictionCallback
    from super_gradients_b200.training.models.detection_models.yolo_nas import YoloNAS
    from super_gradients_b200.training.sg_trainer import Trainer
    from super_gradients_b200.training.utils.detection_utils import ManhattanDistance

    g = golden("tiny_yolo_nas")
    ap = copy.deepcopy(g["arch"])
    model = YoloNAS(backbone=ap["backbone"], neck=ap["neck"], heads=ap["heads"], num_classes=4, bn_eps=1e-3, bn_momentum=0.03, inplace_act=True, in_channels=3)
    model.load_state_dict({k: v.clone() for k, v in g["sd0"].items()}, strict=False)
    callback = PPYoloEPostPredictionCallback(score_threshold=0.01, nms_threshold=0.7, nms_top_k=200, max_predictions=50)
    metric = DetectionMetricsDistanceBased(num_cls=4, post_prediction_callback=callback, normalize_targets=True, score_thres=0.01, distance_thresholds=[8.0, 16.0, 32.0],
                                           distance_metric=ManhattanDistance(), include_classwise_ap=True)  # fmt: skip
    loader = [(g["x"], g["targets"]), (g["x"].flip(0), g["targets"])]
    res = Trainer("distance_test", ckpt_root_dir=str(tmp_path)).test(model=model.cuda(), test_loader=loader, loss=PPYoloELoss(num_classes=4, use_static_assigner=False),
                                                                      test_metrics_list=[metric], silent_mode=True)  # fmt: skip
    keys = ["distance_based_Precision@DIST8.00:32.00", "distance_based_Recall@DIST8.00:32.00", "distance_based_mAP@DIST8.00:32.00", "distance_based_F1@DIST8.00:32.00"]
    assert set(keys) <= set(res) and "distance_based_AP@DIST8.00:32.00_class_0" in res and "Best_score_threshold" in res
    assert all(0.0 <= res[k] <= 1.0 for k in keys), res
