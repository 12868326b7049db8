"""Generates tests/golden/detection_mosaic.pt by running the UNMODIFIED reference train transforms (/root/reference, through
oracle/ref_shim.py) with the reference's DetectionDataset.apply_transforms over the seeded StubMosaicDataset of
tests/mosaic_cases.py: the Roboflow fine-tuning list verbatim, DetectionMosaic(prob 0.5) before the COCO list, a 384 mosaic
before the COCO list and the Roboflow list with the mosaic closed, each under random.seed / np.random.seed for every seed of
GOLDEN_SEEDS, samples in index order.  Per sample it records the sha256 of the uint8 image DetectionStandardize receives (HWC,
recovered exactly from the float32 output), the sha256 of the model input (the float32 CHW output rounded to bf16, as
DetectionCollateFN + functional.to_nhwc make it) and the final targets.  It also records the reference DetectionMosaic alone on
CANVAS_CASES: the canvas' sha256 and the boxes, labels and crowd flags.  Run once in the build container:

    python tests/golden/make_detection_mosaic_goldens.py
"""
import hashlib
import os
import random
import sys
from unittest import mock

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from mosaic_cases import CANVAS_CASES, GOLDEN_LISTS, GOLDEN_SEEDS, StubMosaicDataset  # noqa: E402
from oracle import ref_shim  # noqa: E402


def main():
    ref_shim.install()
    import cv2
    from super_gradients.training.datasets.detection_datasets.detection_dataset import DetectionDataset
    from super_gradients.training.transforms import transforms as T
    from super_gradients.training.transforms.transforms import LegacyDetectionTransformMixin

    class Ref:  # the reference's transform application on the stub's raw samples
        apply_transforms = DetectionDataset.apply_transforms
        _get_additional_inputs_for_transform = DetectionDataset._get_additional_inputs_for_transform
        get_random_samples = DetectionDataset.get_random_samples
        get_random_sample = DetectionDataset.get_random_sample

        def __init__(self, stub, transforms):
            self.stub, self.transforms, self._n_samples = stub, transforms, len(stub)

        def get_sample(self, index, ignore_empty_annotations=False):
            return self.stub.get_sample(index)

    out = {"cv2": cv2.__version__, "numpy": np.__version__, "cases": {}, "canvases": []}
    stub = StubMosaicDataset()
    for name, spec in GOLDEN_LISTS.items():
        for seed in GOLDEN_SEEDS:
            transforms = [getattr(T, n)(**kw) for n, kw in spec]
            ref = Ref(stub, transforms)
            random.seed(seed)
            np.random.seed(seed)
            rows = []
            for i in range(len(stub)):
                s = ref.apply_transforms(stub.get_sample(i))
                img = s["image"]
                assert img.dtype == np.float32 and img.shape == (3, 640, 640)
                u8 = np.rint(img * 255.0).astype(np.uint8)
                assert np.array_equal((u8 / 255.0).astype(np.float32), img)
                model_in = torch.from_numpy(img).bfloat16().view(torch.int16).numpy()
                rows.append({"u8_sha256": hashlib.sha256(np.ascontiguousarray(u8.transpose(1, 2, 0)).tobytes()).hexdigest(),
                             "input_sha256": hashlib.sha256(model_in.tobytes()).hexdigest(), "target": torch.from_numpy(np.array(s["target"]))})  # fmt: skip
            out["cases"][(name, seed)] = rows

    convert = LegacyDetectionTransformMixin.convert_input_dict_to_detection_sample
    for indices, input_dim, draws in CANVAS_CASES:
        sample = convert(stub.get_sample(indices[0])).sanitize_sample()
        sample.additional_samples = [convert(stub.get_sample(j)) for j in indices[1:]]
        with mock.patch("random.uniform", side_effect=list(draws)):
            m = T.DetectionMosaic(input_dim=input_dim).apply_to_sample(sample)
        out["canvases"].append({"canvas_sha256": hashlib.sha256(np.ascontiguousarray(m.image).tobytes()).hexdigest(), "shape": tuple(m.image.shape),
                                "bboxes": torch.from_numpy(m.bboxes_xyxy.copy()), "labels": torch.from_numpy(np.asarray(m.labels).copy()),
                                "is_crowd": torch.from_numpy(np.asarray(m.is_crowd).copy())})  # fmt: skip
    torch.save(out, os.path.join(HERE, "detection_mosaic.pt"))
    print("cv2", cv2.__version__, {k: len(v) for k, v in out["cases"].items()}, len(out["canvases"]), "canvases")


if __name__ == "__main__":
    main()
