"""Generates tests/golden/pose_augment.pt by running the UNMODIFIED reference keypoint transforms (/root/reference, through
oracle/ref_shim.py) with the reference's KeypointsCompose and AbstractPoseEstimationDataset.load_random_sample over the seeded
StubPoseDataset of tests/pose_augment_cases.py: the three YOLO-NAS-POSE recipe lists verbatim, each under random.seed /
np.random.seed for every seed of GOLDEN_SEEDS, samples in index order.  Per sample it records the sha256 of the uint8 image
KeypointsImageStandardize receives (HWC, recovered exactly from the float32 output), the sha256 of the model input (the float32
CHW image rounded to bf16, as YoloNASPoseCollateFN + functional.to_nhwc make it) and the targets YoloNASPoseCollateFN takes from
the sample (boxes xyxy, joints, crowd flags).  Run once in the build container:

    python tests/golden/make_pose_augment_goldens.py
"""
import hashlib
import os
import random
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import ref_shim  # noqa: E402
from pose_augment_cases import GOLDEN_LISTS, GOLDEN_PATH, GOLDEN_SEEDS, StubPoseDataset, build  # noqa: E402


def main():
    ref_shim.install()
    import cv2
    from super_gradients.training.datasets.pose_estimation_datasets.abstract_pose_estimation_dataset import AbstractPoseEstimationDataset
    from super_gradients.training.samples import PoseEstimationSample
    from super_gradients.training.transforms import keypoints as KP

    class Ref:  # the reference's sample loading and transform application on the stub
        load_random_sample = AbstractPoseEstimationDataset.load_random_sample

        def __init__(self, stub, transforms):
            self.stub = stub
            self.transforms = KP.KeypointsCompose(transforms, load_sample_fn=self.load_random_sample)

        def __len__(self):
            return len(self.stub)

        def load_sample(self, index):
            return self.stub.load_sample(index)

    stub = StubPoseDataset(sample_cls=PoseEstimationSample)
    out = {"cv2": cv2.__version__, "numpy": np.__version__, "cases": {}}
    for name, spec in GOLDEN_LISTS.items():
        for seed in GOLDEN_SEEDS:
            ref = Ref(stub, build(spec, KP))
            random.seed(seed)
            np.random.seed(seed)
            rows = []
            for i in range(len(stub)):
                s = ref.transforms.apply_to_sample(ref.load_sample(i))
                img = s.image
                assert img.dtype == np.float32 and img.shape == (640, 640, 3), (img.dtype, img.shape)
                u8 = np.rint(img * 255.0).astype(np.uint8)
                assert np.array_equal(np.divide(u8, 255.0, dtype=np.float32), img)
                model_in = torch.from_numpy(np.ascontiguousarray(img.transpose(2, 0, 1))).bfloat16().view(torch.int16).numpy()
                xywh = np.asarray(s.bboxes_xywh)
                xyxy = np.concatenate([xywh[..., :2], xywh[..., :2] + xywh[..., 2:4]], axis=-1)
                crowd = np.zeros(len(xyxy)) if s.is_crowd is None else s.is_crowd
                rows.append({"u8_sha256": hashlib.sha256(u8.tobytes()).hexdigest(), "input_sha256": hashlib.sha256(model_in.tobytes()).hexdigest(),
                             "boxes": torch.from_numpy(xyxy), "joints": torch.from_numpy(s.joints), "is_crowd": torch.from_numpy(crowd.astype(int).reshape((-1, 1)))})  # fmt: skip
            out["cases"][(name, seed)] = rows
    torch.save(out, GOLDEN_PATH)
    print("cv2", cv2.__version__, {k: len(v) for k, v in out["cases"].items()}, os.path.getsize(GOLDEN_PATH), "bytes")


if __name__ == "__main__":
    main()
