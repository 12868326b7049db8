"""Generates tests/golden/sliding_window.pt by running the UNMODIFIED reference SlidingWindowInferenceDetectionWrapper
(/root/reference, SG 3.7.1) on CPU through oracle/ref_shim.py, with the seeded StubDetector of tests/sliding_window_cases.py as the
model, for every case of GOLDEN_CASES: the stub's call log (tile index, zero count), the tile origins of _generate_tiles, the
forward() callback's parameters and the wrapper's NMS defaults, and the final rows per image.  It also records the reference's
skip-resizing chain (get_equivalent_compose_without_resizing(DetectionAutoPadding((32, 32), 0)) of the YOLO-NAS COCO chain) on
seeded uint8 images: the shape and the sha256 of the model input rounded to bf16.  Run once in the build container:

    python tests/golden/make_sliding_window_goldens.py
"""
import hashlib
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import ref_shim  # noqa: E402
from sliding_window_cases import GOLDEN_CASES, StubDetector, golden_inputs  # noqa: E402

SKIP_SHAPES = [(1500, 2520), (333, 517), (64, 64)]


def main():
    ref_shim.install()
    from super_gradients.training.models.detection_models.pp_yolo_e.post_prediction_callback import PPYoloEPostPredictionCallback
    from super_gradients.training.models.detection_models.sliding_window_detection_forward_wrapper import SlidingWindowInferenceDetectionWrapper
    from super_gradients.training.processing import processing as P

    out = {"cases": {}, "skip_resizing": []}
    for name, (iseed, B, H, W, tile, step, wkw, skw) in GOLDEN_CASES.items():
        stub = StubDetector(PPYoloEPostPredictionCallback, **skw)
        w = SlidingWindowInferenceDetectionWrapper(tile_size=tile, tile_step=step, model=stub, **wkw)
        x = golden_inputs(iseed, B, H, W)
        origins = [[xy for _, xy in w._generate_tiles(x[b : b + 1], tile, step)] for b in range(B)]
        with torch.no_grad():
            rows = w(x)
        cb = w.sliding_window_post_prediction_callback
        n_merge = [0] * B  # candidates each image's merge saw (sum of per-tile rows)
        out["cases"][name] = dict(
            origins=origins,
            calls=list(stub.calls),
            rows=[r.clone() for r in rows],
            callback=(cb.score_threshold, cb.nms_threshold, cb.nms_top_k, cb.max_predictions, cb.multi_label_per_box, cb.class_agnostic_nms),
            defaults=(w._default_nms_iou, w._default_nms_conf, w._default_nms_top_k, w._default_max_predictions, w._default_multi_label_per_box, w._default_class_agnostic_nms),
        )
        # the per-tile rows again, to report which side of n = 1000 each merge is on
        stub2 = StubDetector(PPYoloEPostPredictionCallback, **skw)
        t = 0
        for b in range(B):
            for _ in origins[b]:
                k, zeros = stub.calls[t]
                bx, sc = stub2.tile_output(k, zeros, tile)
                n_merge[b] += cb((bx[None], sc[None]))[0].shape[0]
                t += 1
        out["cases"][name]["n_merge"] = n_merge
        print(f"{name}: tiles {[len(o) for o in origins]}, merge candidates {n_merge}, kept {[r.shape[0] for r in rows]}")
    chain = P.ComposeProcessing([P.DetectionLongestMaxSizeRescale(output_shape=(636, 636)), P.DetectionCenterPadding(output_shape=(640, 640), pad_value=114),
                                 P.StandardizeImage(max_value=255.0), P.ImagePermute(permutation=(2, 0, 1))])  # fmt: skip
    chain = chain.get_equivalent_compose_without_resizing(auto_padding=P.DetectionAutoPadding(shape_multiple=(32, 32), pad_value=0))
    rng = np.random.RandomState(17)
    for h, w_ in SKIP_SHAPES:
        im = rng.randint(0, 256, (h, w_, 3), dtype=np.uint8)
        x, _meta = chain.preprocess_image(im)
        t = torch.from_numpy(np.ascontiguousarray(x)).float()  # CHW
        nhwc = torch.zeros(t.shape[1], t.shape[2], 16)
        nhwc[..., :3] = t.permute(1, 2, 0)
        sha = hashlib.sha256(nhwc.bfloat16().contiguous().view(torch.int16).numpy().tobytes()).hexdigest()
        out["skip_resizing"].append(dict(shape=(h, w_), seed_index=len(out["skip_resizing"]), out_hw=tuple(t.shape[1:]), sha256=sha))
        print("skip-resizing", (h, w_), "->", tuple(t.shape), sha[:16])
    torch.save(out, os.path.join(HERE, "sliding_window.pt"))


if __name__ == "__main__":
    main()
