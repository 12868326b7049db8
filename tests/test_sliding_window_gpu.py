"""Sliding-window detection on the H100: tile gather, merge NMS against torchvision's CPU batched_nms, and predict() on YOLO-NAS-S
against the reference algorithm run tile by tile at batch 1."""
import os

import numpy as np
import pytest
import torch
import torchvision

import nms_cases
from sliding_window_cases import GOLDEN_CASES, StubDetector, golden_inputs, merge_case
from super_gradients_b200 import kernels as K
from super_gradients_b200 import lib as L

pytestmark = pytest.mark.gpu


def _merge_single(boxes, scores, labels, iou, P=1000, origin=(0, 0)):
    """Split one image's candidate list into tiles of P rows (all at `origin`), merge on the device."""
    n = boxes.shape[0]
    T = max(1, (n + P - 1) // P)
    rows = torch.zeros(T, P, 6)
    cnt = torch.zeros(T, dtype=torch.int32)
    tile_rows = torch.cat([boxes - torch.tensor([origin[1], origin[0]] * 2, dtype=torch.float32), scores[:, None], labels[:, None]], 1)
    for t in range(T):
        r = tile_rows[t * P : (t + 1) * P]
        rows[t, : r.shape[0]] = r
        cnt[t] = r.shape[0]
    tiles_h = torch.tensor([[0, origin[0], origin[1]]] * T, dtype=torch.int32)
    it_h = torch.tensor([0, T], dtype=torch.int32)
    out, c = K.sliding_window_merge(rows.cuda(), cnt.cuda(), tiles_h.cuda(), it_h, it_h.cuda(), int(labels.max()) + 1, iou)
    return out.cpu()[0, : int(c.cpu()[0])], tile_rows[:, :4] + torch.tensor([origin[1], origin[0]] * 2, dtype=torch.float32)


def test_gather_equals_torch_slicing():
    g = torch.Generator().manual_seed(0)
    canvas = K.empty_nhwc(2, 16, 96, 130, "cuda")
    canvas.copy_(torch.randn(2, 16, 96, 130, generator=g).bfloat16())
    tiles = torch.tensor([[0, 0, 0], [1, 32, 64], [0, 64, 96], [1, 80, 120]], dtype=torch.int32)
    got = K.sliding_window_gather(canvas, tiles, tiles.cuda(), 48).float().cpu()
    padded = torch.zeros(2, 16, 96 + 48, 130 + 48)
    padded[:, :, :96, :130] = canvas.float().cpu()
    for t, (b, y, x) in enumerate(tiles.tolist()):
        assert torch.equal(got[t], padded[b, :, y : y + 48, x : x + 48])


@pytest.mark.parametrize("n,ncls", [(1, 3), (999, 7), (1000, 7), (1001, 7), (5000, 7), (50000, 1)])
def test_merge_bit_exact_against_torchvision_cpu(n, ncls):
    boxes, scores, labels = merge_case(n, ncls, seed=n)
    got, _ = _merge_single(boxes, scores, labels, 0.5)
    keep = torchvision.ops.batched_nms(boxes, scores, labels, 0.5)
    ref = torch.cat([boxes, scores[:, None], labels[:, None]], 1)[keep]
    assert torch.equal(got, ref), (n, got.shape, ref.shape)


def test_merge_tile_origins_and_tied_scores():
    boxes, scores, labels = merge_case(900, 4, seed=11, tied=True)
    got, shifted = _merge_single(boxes, scores, labels, 0.65, P=300, origin=(160, 480))
    keep = torchvision.ops.batched_nms(shifted, scores, labels, 0.65)
    assert torch.equal(got, torch.cat([shifted, scores[:, None], labels[:, None]], 1)[keep])


@pytest.mark.parametrize("name", nms_cases.MERGE_EDGE_CASES)
def test_merge_nan_boxes_and_signed_zero(name):
    for b in range(2):
        boxes, scores, labels = nms_cases.merge_candidates(name, b)
        got, _ = _merge_single(boxes, scores, labels, 0.5)
        keep = torchvision.ops.batched_nms(boxes, scores, labels, 0.5)
        ref = torch.cat([boxes, scores[:, None], labels[:, None]], 1)[keep]
        # bit for bit (-0.0 scores included), NaN as one value: the merge shifts boxes by the tile origin on the device, whose
        # arithmetic returns the canonical NaN 0x7fffffff whatever the input's payload
        bits = lambda t: torch.where(torch.isnan(t), torch.tensor(float("nan")), t).contiguous().view(torch.int32)  # noqa: E731
        if boxes.shape[0] > 1000:  # the per-class path: torchvision's final sort is not stable
            assert got.shape == ref.shape and torch.equal(bits(got[:, 4]), bits(ref[:, 4]))
            canon = lambda r: sorted(map(tuple, bits(r).tolist()))  # noqa: E731
            assert canon(got) == canon(ref), (name, b)
        else:
            assert torch.equal(bits(got), bits(ref)), (name, b)


def _model():
    from super_gradients_b200.training import models

    torch.manual_seed(0)
    return models.get("yolo_nas_s", num_classes=80).cuda().eval()


def _images(n, h=1500, w=2520):
    rng = np.random.RandomState(5)
    return [rng.randint(0, 256, (h, w, 3), dtype=np.uint8) for _ in range(n)]


def _canonical(rows):
    """Rows ordered by (score desc, then coordinates and label): the per-class torchvision path orders exact ties arbitrarily."""
    keys = np.lexsort([rows[:, 5].numpy(), rows[:, 3].numpy(), rows[:, 2].numpy(), rows[:, 1].numpy(), rows[:, 0].numpy(), -rows[:, 4].numpy()])
    return rows[torch.from_numpy(keys)]


def test_predict_equals_reference_schedule_tile_by_tile():
    from super_gradients_b200.training.models.detection_models.sliding_window_detection_forward_wrapper import SlidingWindowInferenceDetectionWrapper, tile_origins

    model = _model()
    wrapper = SlidingWindowInferenceDetectionWrapper(tile_size=640, tile_step=160, model=model)
    images = _images(2)
    conf, iou = 0.005, 0.6
    got = wrapper.predict(images, conf=conf, iou=iou, skip_image_resizing=True, batch_size=2)
    from super_gradients_b200.training.processing import DetectionAutoPadding, default_yolo_nas_coco_processing_params

    processor = default_yolo_nas_coco_processing_params()["image_processor"].get_equivalent_compose_without_resizing(DetectionAutoPadding((32, 32), 0))
    cb = wrapper._callback(iou, conf, None, None, None, None)
    canvas, geos = processor.preprocess_batch(images, "cuda")
    _, _, H, W = canvas.shape
    assert (H, W) == (1504, 2528)
    padded = torch.zeros(2, 16, H + 640, W + 640, dtype=torch.bfloat16, device="cuda")
    padded[:, :, :H, :W] = canvas
    origins = tile_origins(H, W, 640, 160, 30)
    assert len(origins) == 160
    for b in range(2):
        dets = []
        for y, x in origins:  # the reference's schedule: one model call and one callback per tile, host lists, one batched_nms
            tile = K.as_nhwc(padded[b : b + 1, :, y : y + 640, x : x + 640])
            r = cb(model(tile))[0].cpu()
            if len(r):
                r[:, :4] += torch.tensor([x, y, x, y], dtype=torch.float32)
                dets.append(r)
        d = torch.cat(dets)
        ref = d[torchvision.ops.batched_nms(d[:, :4], d[:, 4], d[:, 5], iou)]
        ref = torch.cat([processor.postprocess_boxes(ref, geos[b])[:, :4], ref[:, 4:]], 1)
        print(f"image {b}: {d.shape[0]} merge candidates, {ref.shape[0]} kept")
        assert got[b].shape == ref.shape
        if d.shape[0] <= 1000:
            assert torch.equal(got[b], ref)
        else:
            assert torch.equal(_canonical(got[b]), _canonical(ref))


def test_device_part_has_no_sync_and_launches_scale_with_chunks():
    from super_gradients_b200.training.models.detection_models.sliding_window_detection_forward_wrapper import SlidingWindowInferenceDetectionWrapper

    model = _model()
    wrapper = SlidingWindowInferenceDetectionWrapper(tile_size=320, tile_step=160, model=model, tile_nms_conf=0.01)
    cb = wrapper.sliding_window_post_prediction_callback
    counts = []
    for w in (320 + 160 * 15, 320 + 160 * 19):  # 16 and 20 tiles per row, 8 rows: 128 / 160 tiles, one chunk of 256 either way
        canvas = K.empty_nhwc(1, 16, 320 + 160 * 7, w, "cuda")
        canvas.zero_()
        wrapper._detect(canvas, cb)  # warm-up
        torch.cuda.synchronize()
        n0 = L.LAUNCHES[0]
        torch.cuda.set_sync_debug_mode("error")
        try:
            wrapper._detect(canvas, cb)
        finally:
            torch.cuda.set_sync_debug_mode("default")
        counts.append(L.LAUNCHES[0] - n0)
    assert counts[0] == counts[1], counts


def test_trainer_test_with_wrapper_equals_metric_on_rows(tmp_path):
    from super_gradients_b200.training.metrics import DetectionMetrics
    from super_gradients_b200.training.models.detection_models.sliding_window_detection_forward_wrapper import SlidingWindowInferenceDetectionWrapper
    from super_gradients_b200.training.sg_trainer import Trainer

    model = _model()
    wrapper = SlidingWindowInferenceDetectionWrapper(tile_size=320, tile_step=160, model=model, tile_nms_conf=0.005, tile_nms_max_predictions=20).eval()
    g = torch.Generator().manual_seed(2)
    x = torch.rand(2, 3, 480, 640, generator=g)
    rows = wrapper(x.cuda())
    # targets made from the wrapper's own eval-mode rows (cx, cy, w, h in pixels): every image has matches, so the metrics are not 0
    tg = []
    for b, r in enumerate(rows):
        r = r.cpu().clone()
        r[:, [0, 2]] = r[:, [0, 2]].clamp(0, 640)  # the metric clips predictions to the image
        r[:, [1, 3]] = r[:, [1, 3]].clamp(0, 480)
        r = r[((r[:, 2] - r[:, 0]) > 4) & ((r[:, 3] - r[:, 1]) > 4)][:5]
        cxcywh = torch.stack([(r[:, 0] + r[:, 2]) / 2, (r[:, 1] + r[:, 3]) / 2, r[:, 2] - r[:, 0], r[:, 3] - r[:, 1]], 1)
        tg.append(torch.cat([torch.full((r.shape[0], 1), float(b)), r[:, 5:6], cxcywh], 1))
    targets = torch.cat(tg)
    assert targets.shape[0] > 0
    res = Trainer("sliding_window", ckpt_root_dir=str(tmp_path)).test(model=wrapper, test_loader=[(x, targets)], silent_mode=True,
                                                                     test_metrics_list=[DetectionMetrics(num_cls=80, post_prediction_callback=None, normalize_targets=True)])  # fmt: skip
    wrapper.eval()  # Trainer.test leaves the network in train mode
    m = DetectionMetrics(num_cls=80, post_prediction_callback=None, normalize_targets=True)
    m.update(wrapper(x.cuda()), targets, inputs=x.cuda())
    direct = m.compute()
    assert any(float(v) > 0 for k, v in direct.items() if "mAP" in k), direct
    for k, v in direct.items():
        assert float(res[k]) == float(v), (k, res[k], v)


def test_merge_refuses_bad_count_and_label():
    rows = torch.zeros(3, 4, 6)
    rows[..., 2:4] = 10.0
    rows[..., 4] = 0.5
    cnt = torch.tensor([2, 2, 2], dtype=torch.int32)
    bad_label = rows.clone()
    bad_label[1, 1, 5] = 2.5  # not integral
    tiles = torch.tensor([[0, 0, 0], [1, 0, 0], [2, 0, 0]], dtype=torch.int32)
    it = torch.tensor([0, 1, 2, 3], dtype=torch.int32)
    _, c = K.sliding_window_merge(bad_label.cuda(), cnt.cuda(), tiles.cuda(), it, it.cuda(), 3, 0.5)
    assert c.cpu().tolist() == [1, -2, 1]
    _, c = K.sliding_window_merge(rows.cuda(), torch.tensor([2, 9, 2], dtype=torch.int32).cuda(), tiles.cuda(), it, it.cuda(), 3, 0.5)
    assert c.cpu().tolist() == [1, -1, 1]


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sliding_window.pt")


@pytest.mark.parametrize("name", list(GOLDEN_CASES))
def test_tile_nms_and_merge_reproduce_reference_goldens(name):
    """Gather, per-tile NMS and merge kernels on the seeded stub detector's outputs against the unmodified reference wrapper's rows."""
    from super_gradients_b200.training.models.detection_models.pp_yolo_e.post_prediction_callback import PPYoloEPostPredictionCallback
    from super_gradients_b200.training.models.detection_models.sliding_window_detection_forward_wrapper import SlidingWindowInferenceDetectionWrapper
    from test_sliding_window_host import assert_rows_match_reference

    g = torch.load(GOLDEN, weights_only=False)["cases"][name]
    iseed, B, H, W, tile, step, wkw, skw = GOLDEN_CASES[name]
    stub = StubDetector(PPYoloEPostPredictionCallback, **skw).cuda()
    w = SlidingWindowInferenceDetectionWrapper(tile_size=tile, tile_step=step, model=stub, **wkw)
    rows = w(golden_inputs(iseed, B, H, W).cuda())
    assert stub.calls == g["calls"]
    for b in range(B):
        assert_rows_match_reference(rows[b].cpu(), g["rows"][b], g["n_merge"][b])
