"""Sliding-window detection on the CPU: the merge NMS arithmetic and schedule (host build of the kernel's algorithm over
nms_math.cuh) against torchvision's CPU batched_nms, and the wrapper's tiling / callback rules."""
import os

import numpy as np
import pytest
import torch
import torchvision

import nms_cases
from sliding_window_cases import GOLDEN_CASES, StubDetector, golden_inputs, merge_case, merge_nms_host
from super_gradients_b200.training.models.detection_models.sliding_window_detection_forward_wrapper import chunk_tiles, tile_origins


@pytest.mark.parametrize("n", [1, 999, 1000, 1001, 5000, 50000])
def test_merge_matches_torchvision_cpu_index_for_index(n):
    ncls = 1 if n == 50000 else 7  # 50,000 candidates of one class: one long blocked greedy pass
    boxes, scores, labels = merge_case(n, ncls, seed=n)
    ref = torchvision.ops.batched_nms(boxes, scores, labels, 0.5)
    got = merge_nms_host(boxes, scores, labels, 0.5)
    assert torch.equal(got, ref), (n, got.numel(), ref.numel())


def test_merge_tied_scores_coordinate_trick_path():
    # n <= 1000: torchvision's nms sorts stably, so ties keep list order in both
    boxes, scores, labels = merge_case(900, 5, seed=3, tied=True)
    assert torch.equal(merge_nms_host(boxes, scores, labels, 0.6), torchvision.ops.batched_nms(boxes, scores, labels, 0.6))


def test_merge_tied_scores_per_class_path_same_set():
    # n > 1000: torchvision's final scores.sort() is not stable on the CPU; the kept set and the score order agree
    boxes, scores, labels = merge_case(3000, 5, seed=4, tied=True)
    ref = torchvision.ops.batched_nms(boxes, scores, labels, 0.6)
    got = merge_nms_host(boxes, scores, labels, 0.6)
    assert torch.equal(got.sort().values, ref.sort().values)
    assert torch.equal(scores[got], scores[ref])


@pytest.mark.parametrize("name", nms_cases.MERGE_EDGE_CASES)
def test_merge_nan_boxes_and_signed_zero(name):
    """NaN / +-inf boxes (a NaN maximum makes every offset box NaN on the coordinate-trick path: nothing is suppressed) and +-0.0
    scores (equal in torchvision's sort: list order decides)."""
    for b in range(2):
        boxes, scores, labels = nms_cases.merge_candidates(name, b)
        ref = torchvision.ops.batched_nms(boxes, scores, labels, 0.5)
        got = merge_nms_host(boxes, scores, labels, 0.5)
        if boxes.shape[0] > 1000:  # the per-class path: torchvision's final sort is not stable
            assert torch.equal(got.sort().values, ref.sort().values) and torch.equal(scores[got], scores[ref])
        else:
            assert torch.equal(got, ref), (name, b)


def test_tile_origin_edge_cases():
    # the 2520 x 1500 example on its 2528 x 1504 canvas: remainders 64 and 128 are covered by tiles reaching past the canvas
    assert tile_origins(1504, 2528, 640, 160, 30) == [(y, x) for y in range(0, 1441, 160) for x in range(0, 2401, 160)]  # 10 x 16
    assert tile_origins(170, 170, 320, 160, 30) == []  # (170 - 320) % 160 = 10 < 30: no tile at all
    assert tile_origins(200, 200, 320, 160, 30) == [(0, 0), (0, 160), (160, 0), (160, 160)]  # (200 - 320) % 160 = 40: the grid reaches 480
    assert tile_origins(800, 1000, 320, 160, 30) == [(y, x) for y in range(0, 481, 160) for x in range(0, 961, 160)]  # 28 tiles
    assert tile_origins(800, 990, 320, 160, 30) == [(y, x) for y in range(0, 481, 160) for x in range(0, 961, 160)]  # remainder 30: covered
    assert tile_origins(800, 985, 320, 160, 30) == [(y, x) for y in range(0, 481, 160) for x in range(0, 641, 160)]  # remainder 25 < 30: strip dropped
    assert chunk_tiles(640) == 64 and chunk_tiles(320) == 256 and chunk_tiles(1280) == 16


def test_tile_callback_rule_forward_vs_predict():
    """forward() uses the constructor's tile_nms_* over the wrapper's defaults; predict() builds its callback from its own
    arguments over the same defaults -- never from the constructor's values nor from the model's NMS defaults."""
    from super_gradients_b200.training.models.detection_models.pp_yolo_e.post_prediction_callback import PPYoloEPostPredictionCallback
    from super_gradients_b200.training.models.detection_models.sliding_window_detection_forward_wrapper import SlidingWindowInferenceDetectionWrapper

    class Stub(torch.nn.Module):
        def get_dataset_processing_params(self):
            return dict(class_names=["a"], image_processor=None, iou=0.1, conf=0.1, nms_top_k=10, max_predictions=5, multi_label_per_box=False, class_agnostic_nms=True)

        def get_post_prediction_callback(self, *, conf, iou, nms_top_k, max_predictions, multi_label_per_box, class_agnostic_nms):
            return PPYoloEPostPredictionCallback(score_threshold=conf, nms_threshold=iou, nms_top_k=nms_top_k, max_predictions=max_predictions,
                                                 multi_label_per_box=multi_label_per_box, class_agnostic_nms=class_agnostic_nms)  # fmt: skip

    w = SlidingWindowInferenceDetectionWrapper(640, 160, Stub(), tile_nms_conf=0.35, tile_nms_max_predictions=50)
    f = w.sliding_window_post_prediction_callback
    assert (f.score_threshold, f.nms_threshold, f.nms_top_k, f.max_predictions, f.multi_label_per_box, f.class_agnostic_nms) == (0.35, 0.7, 1024, 50, True, False)
    p = w._callback(None, None, None, None, None, None)  # what predict() builds with no arguments
    assert (p.score_threshold, p.nms_threshold, p.nms_top_k, p.max_predictions, p.multi_label_per_box, p.class_agnostic_nms) == (0.5, 0.7, 1024, 300, True, False)
    p = w._callback(0.4, 0.2, None, None, None, True)
    assert (p.score_threshold, p.nms_threshold, p.class_agnostic_nms) == (0.2, 0.4, True)
    assert w._class_names == ("a",)
    d = SlidingWindowInferenceDetectionWrapper(640, 160, Stub()).sliding_window_post_prediction_callback
    assert (d.score_threshold, d.nms_threshold, d.max_predictions) == (0.5, 0.7, 300)


def test_skip_resizing_chain_and_canvas():
    from super_gradients_b200.training.processing import DetectionAutoPadding, default_yolo_nas_coco_processing_params

    chain = default_yolo_nas_coco_processing_params()["image_processor"].get_equivalent_compose_without_resizing(DetectionAutoPadding((32, 32), 0))
    assert [type(p).__name__ for p in chain.processings] == ["DetectionAutoPadding", "StandardizeImage", "ImagePermute"]
    g, canvas = chain.geometry(1500, 2520)
    assert canvas == (1504, 2528) and (g.pad_top, g.pad_left, g.scale_factor_h, g.scale_factor_w) == (0, 0, 1.0, 1.0)
    with pytest.raises(ValueError):
        chain.preprocess_batch([np.zeros((1500, 2520, 3), np.uint8), np.zeros((1400, 2520, 3), np.uint8)], "cpu")


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sliding_window.pt")


def assert_rows_match_reference(got, ref, n_merge):
    """Bit-exact; on the per-class path (more than 1000 merge candidates) exactly tied kept scores may be ordered differently
    (DESIGN.md section 4.9): then the kept rows and the score sequence must still be identical."""
    if n_merge <= 1000 or torch.equal(got, ref):
        assert torch.equal(got, ref), (got.shape, ref.shape)
        return
    assert got.shape == ref.shape
    assert torch.equal(got[:, 4], ref[:, 4])
    key = lambda r: sorted(map(tuple, r.tolist()))  # noqa: E731
    assert key(got) == key(ref)


@pytest.mark.parametrize("name", list(GOLDEN_CASES))
@pytest.mark.parametrize("chunk", [64, 1])
def test_wrapper_glue_reproduces_reference_goldens(name, chunk, monkeypatch):
    """The wrapper's glue on CPU stand-ins (cpu_sliding_window) against the unmodified reference wrapper's rows, tile origins, stub call
    log (tile order and zero fill) and callback; chunk 1 makes each model pass hold fewer tiles than one image has."""
    import cpu_sliding_window
    from super_gradients_b200.training.models.detection_models import sliding_window_detection_forward_wrapper as SW
    from super_gradients_b200.training.models.detection_models.pp_yolo_e.post_prediction_callback import PPYoloEPostPredictionCallback

    g = torch.load(GOLDEN, weights_only=False)["cases"][name]
    cpu_sliding_window.install(monkeypatch)
    monkeypatch.setattr(SW, "_CHUNK_TILES_640", chunk)
    iseed, B, H, W, tile, step, wkw, skw = GOLDEN_CASES[name]
    stub = StubDetector(PPYoloEPostPredictionCallback, **skw)
    w = SW.SlidingWindowInferenceDetectionWrapper(tile_size=tile, tile_step=step, model=stub, **wkw)
    cb = w.sliding_window_post_prediction_callback
    assert (cb.score_threshold, cb.nms_threshold, cb.nms_top_k, cb.max_predictions, cb.multi_label_per_box, cb.class_agnostic_nms) == g["callback"]
    assert (w._default_nms_iou, w._default_nms_conf, w._default_nms_top_k, w._default_max_predictions, w._default_multi_label_per_box, w._default_class_agnostic_nms) == g["defaults"]
    assert [tile_origins(H, W, tile, step, 30)] * B == [[(y, x) for x, y in og] for og in g["origins"]]  # the reference records (x, y)
    rows = w(golden_inputs(iseed, B, H, W))
    assert stub.calls == g["calls"]
    assert len(rows) == B
    for b in range(B):
        assert_rows_match_reference(rows[b], g["rows"][b], g["n_merge"][b])


def test_goldens_cover_both_merge_paths():
    g = torch.load(GOLDEN, weights_only=False)["cases"]
    ns = [n for c in g.values() for n in c["n_merge"]]
    assert min(n for n in ns if n) <= 1000 < max(ns) and 0 in ns
    assert g["small_no_tiles"]["origins"] == [[], []] and g["tied_scores"]["n_merge"][0] <= 1000


def test_skip_resizing_chain_matches_reference_model_input(monkeypatch):
    """The product's skip-resizing chain on the host build of the pre-processing kernel vs the reference chain's model input."""
    import hashlib

    import cpu_backend
    from super_gradients_b200 import kernels as K
    import host_preprocess
    from super_gradients_b200.training.processing import DetectionAutoPadding, default_yolo_nas_coco_processing_params

    cpu_backend.install(monkeypatch)
    monkeypatch.setattr(K, "preprocess_u8", host_preprocess.preprocess_u8)
    chain = default_yolo_nas_coco_processing_params()["image_processor"].get_equivalent_compose_without_resizing(DetectionAutoPadding((32, 32), 0))
    rng = np.random.RandomState(17)
    for rec in torch.load(GOLDEN, weights_only=False)["skip_resizing"]:
        h, w = rec["shape"]
        im = rng.randint(0, 256, (h, w, 3), dtype=np.uint8)
        batch, _ = chain.preprocess_batch([im], "cpu")
        assert tuple(batch.shape[2:]) == rec["out_hw"]
        sha = hashlib.sha256(batch[0].permute(1, 2, 0).contiguous().view(torch.int16).numpy().tobytes()).hexdigest()
        assert sha == rec["sha256"], rec["shape"]
