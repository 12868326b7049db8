"""DetectionMetricsDistanceBased glue on the CPU stand-in of the kernel wrappers (the distance kernel's arithmetic behind a serial
host driver): compute() equals the reference's dictionary in tests/golden/distance_matching.pt, compute_detection_matching with
a DistanceMatching strategy returns the reference's tuples, and the metric resolves by name through MetricsFactory and Trainer."""
import copy
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import cpu_backend  # noqa: E402
import distance_matching_cases as DC  # noqa: E402
import host_distance_match as H  # noqa: E402
from super_gradients_b200 import kernels as K  # noqa: E402
from super_gradients_b200.training.metrics import DetectionMetricsDistanceBased  # noqa: E402
from super_gradients_b200.training.utils import detection_utils as DU  # noqa: E402


def _install(monkeypatch, training=False):
    (cpu_backend.install_training if training else cpu_backend.install)(monkeypatch)
    monkeypatch.setattr(K, "detection_distance_matching", H.detection_distance_matching)


def _metric(case, metric, **kw):
    return DetectionMetricsDistanceBased(num_cls=case["n_cls"], post_prediction_callback=None, normalize_targets=not case["normalized"], distance_thresholds=list(case["thresholds"]),
                                         distance_metric=DC.METRICS[metric](), recall_thres=case["recall_thresholds"], score_thres=case["score_thres"],
                                         top_k_predictions=case["top_k"], include_classwise_ap=True, **kw)  # fmt: skip


@pytest.mark.parametrize("name,metric", DC.CASES)
def test_compute_equals_reference(monkeypatch, name, metric):
    _install(monkeypatch)
    case = DC.GOLD[name]
    m = _metric(case, metric)
    for batch in case["batches"]:
        m.update(batch["output"], batch["targets"], device="cpu", inputs=torch.zeros(len(batch["output"]), 3, *case["hw"]), crowd_targets=batch["crowd_targets"])
    DC.assert_compute_equal(m.compute(), case[metric]["compute"])
    m.reset()
    assert m.compute()[m.map_metric_key] == -1.0


@pytest.mark.parametrize("name,metric", DC.CASES)
def test_compute_detection_matching_with_distance_strategy(monkeypatch, name, metric):
    """The reference's call: compute_detection_matching(..., matching_strategy=DistanceMatching(metric, thresholds))."""
    _install(monkeypatch)
    case = DC.GOLD[name]
    for i, batch in enumerate(case["batches"]):
        res = DU.compute_detection_matching(batch["output"], batch["targets"], case["hw"][0], case["hw"][1], denormalize_targets=case["normalized"], device="cpu",
                                            crowd_targets=batch["crowd_targets"], top_k=case["top_k"], matching_strategy=DU.DistanceMatching(DC.METRICS[metric](), case["thresholds"]))  # fmt: skip
        ref = case[metric]["matching"][i]
        assert len(res) == len(ref)
        for b, (mine, (ref_m, ref_g)) in enumerate(zip(res, ref)):
            assert mine[0].dtype == torch.bool and torch.equal(mine[0], ref_m) and torch.equal(mine[1], ref_g), (name, metric, i, b)
            out = batch["output"][b]
            assert torch.equal(mine[2], out[:, 4] if out is not None else torch.zeros(0)) and torch.equal(mine[3], out[:, 5] if out is not None else torch.zeros(0))
            t = batch["targets"]
            assert torch.equal(mine[4], t[t[:, 0] == b, 1])


def test_names_strategies_and_refusals():
    from super_gradients_b200.common.factories import MetricsFactory

    m = MetricsFactory().get({"DetectionMetricsDistanceBased": {"num_cls": 3, "post_prediction_callback": None}})
    assert isinstance(m, DetectionMetricsDistanceBased) and m.distance_thresholds == (5.0,) and isinstance(m.distance_metric, DU.EuclideanDistance)
    assert m.component_names == ["distance_based_Precision@DIST5.00", "distance_based_Recall@DIST5.00", "distance_based_mAP@DIST5.00", "distance_based_F1@DIST5.00", "Best_score_threshold"]
    m = DetectionMetricsDistanceBased(num_cls=2, post_prediction_callback=None, distance_thresholds=[4.0, 8.0], distance_metric=DU.ManhattanDistance())
    assert m.map_metric_key == "distance_based_mAP@DIST4.00:8.00" and m.state_key == "distance_based_matching_info@DIST4.00:8.00"
    assert DU.DistanceMatching(DU.ManhattanDistance(), [4.0, 8.0]).get_thresholds().tolist() == [4.0, 8.0]

    class Chebyshev(DU.DistanceMetric):
        def calculate_distance(self, predicted, target):
            return torch.zeros(len(predicted), len(target))

    with pytest.raises(NotImplementedError):
        DetectionMetricsDistanceBased(num_cls=2, post_prediction_callback=None, distance_metric=Chebyshev())
    with pytest.raises(NotImplementedError):
        DU.compute_detection_matching([None], torch.zeros(0, 6), 8, 8, True, "cpu", matching_strategy=DU.DistanceMatching(Chebyshev(), [1.0]))
    with pytest.raises(NotImplementedError):
        DU.compute_detection_matching([None], torch.zeros(0, 6), 8, 8, True, "cpu", matching_strategy=object())
    with pytest.raises(ValueError):
        DU.compute_detection_matching([None], torch.zeros(0, 6), 8, 8, True, "cpu")


def test_trainer_watches_a_distance_metric(golden, monkeypatch, tmp_path):
    """valid_metrics_list: [{DetectionMetricsDistanceBased: {...}}] builds the metric by name, the validation reports its keys and a
    fuzzy metric_to_watch ("distance_based_map@dist5.00:10.00") selects the checkpoint."""
    from super_gradients_b200.training import sg_trainer
    from super_gradients_b200.training.losses import PPYoloELoss
    from super_gradients_b200.training.models.detection_models.pp_yolo_e.post_prediction_callback import PPYoloEPostPredictionCallback
    from super_gradients_b200.training.models.detection_models.yolo_nas import YoloNAS
    from super_gradients_b200.training.sg_trainer import Trainer

    _install(monkeypatch, training=True)
    monkeypatch.setattr(sg_trainer, "setup_device", lambda device=None: torch.device("cpu"))
    g = golden("tiny_yolo_nas")
    ap = copy.deepcopy(g["arch"])
    model = YoloNAS(backbone=ap["backbone"], neck=ap["neck"], heads=ap["heads"], num_classes=4, bn_eps=1e-3, bn_momentum=0.03, inplace_act=True, in_channels=3)
    model.load_state_dict({k: v.clone() for k, v in g["sd0"].items()}, strict=False)
    callback = PPYoloEPostPredictionCallback(score_threshold=0.01, nms_threshold=0.7, nms_top_k=200, max_predictions=50)
    loader = [(g["x"], g["targets"])]
    tp = dict(max_epochs=1, initial_lr=1e-3, lr_mode="constant", optimizer="SGD", loss=PPYoloELoss(num_classes=4, use_static_assigner=False), save_model=True,
              valid_metrics_list=[{"DetectionMetricsDistanceBased": {"num_cls": 4, "post_prediction_callback": callback, "normalize_targets": True, "score_thres": 0.01,
                                                                     "distance_thresholds": [5.0, 10.0], "distance_metric": DU.ManhattanDistance()}}],
              metric_to_watch="distance_based_map@dist5.00:10.00", greater_metric_to_watch_is_better=True)  # fmt: skip
    trainer = Trainer("distance", ckpt_root_dir=str(tmp_path))
    trainer.train(model, tp, loader, valid_loader=loader)
    ck = torch.load(tmp_path / "distance" / "ckpt_latest.pth", weights_only=False)
    keys = {"distance_based_Precision@DIST5.00:10.00", "distance_based_Recall@DIST5.00:10.00", "distance_based_mAP@DIST5.00:10.00", "distance_based_F1@DIST5.00:10.00"}
    assert keys <= set(ck["metrics"]), sorted(ck["metrics"])
    assert sg_trainer._match_metric_name("distance_based_map@dist5.00:10.00", list(ck["metrics"])) == "distance_based_mAP@DIST5.00:10.00"
