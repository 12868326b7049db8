"""Generates tests/golden/validation_chains.pt by running the UNMODIFIED reference validation chains (/root/reference, through
oracle/ref_shim.py) over the seeded stubs of tests/validation_cases.py:

- YOLO-NAS COCO: the recipe's val transforms with DetectionDataset.apply_transforms, then CrowdDetectionCollateFN;
- YOLO-NAS-POSE: the recipe's val transforms with KeypointsCompose, then YoloNASPoseCollateFN;
- ResNet-50 ImageNet: torchvision Resize(236) -> CenterCrop(224) -> ToTensor -> Normalize on PIL images, then default_collate.

Per sample it records the sha256 of the model input (the float32 CHW output rounded to bf16, as functional.to_nhwc makes it); per
chain, the collate's targets and extras over all samples in index order.  Run once in the build container:

    python tests/golden/make_validation_goldens.py
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
from validation_cases import (CROP, DETECTION, GOLDEN_PATH, IMAGENET_MEAN, IMAGENET_STD, POSE, RESIZE, StubDetectionDataset, StubImageNetDataset,  # noqa: E402
                              StubValidationPoseDataset, build)  # fmt: skip


def _sha(chw_f32) -> str:
    t = torch.as_tensor(np.ascontiguousarray(chw_f32)).bfloat16().view(torch.int16).numpy()
    return hashlib.sha256(t.tobytes()).hexdigest()


def detection():
    from super_gradients.training.datasets.detection_datasets.detection_dataset import DetectionDataset
    from super_gradients.training.transforms import transforms as T
    from super_gradients.training.utils.collate_fn.crowd_detection_collate_fn import CrowdDetectionCollateFN

    class Ref:  # the reference's transform application on the stub's raw samples
        apply_transforms = DetectionDataset.apply_transforms
        _get_additional_inputs_for_transform = DetectionDataset._get_additional_inputs_for_transform
        get_random_samples = DetectionDataset.get_random_samples

        def __init__(self, stub, transforms):
            self.stub, self.transforms = stub, transforms

    stub = StubDetectionDataset()
    ref = Ref(stub, build(DETECTION, T))
    items, rows = [], []
    for i in range(len(stub)):
        s = ref.apply_transforms(stub.get_sample(i))
        assert s["image"].dtype == np.float32 and s["image"].shape == (3, 640, 640), (s["image"].dtype, s["image"].shape)
        items.append((s["image"], s["target"], s["crowd_target"]))
        rows.append({"input_sha256": _sha(s["image"]), "target": torch.from_numpy(s["target"]), "crowd_target": torch.from_numpy(s["crowd_target"])})
    _, targets, extras = CrowdDetectionCollateFN()(items)
    return {"rows": rows, "targets": targets, "crowd_targets": extras["crowd_targets"]}


def pose():
    from super_gradients.training.datasets.pose_estimation_datasets.yolo_nas_pose_collate_fn import YoloNASPoseCollateFN
    from super_gradients.training.samples import PoseEstimationSample
    from super_gradients.training.transforms import keypoints as KP

    stub = StubValidationPoseDataset(sample_cls=PoseEstimationSample)
    compose = KP.KeypointsCompose(build(POSE, KP), load_sample_fn=None)
    samples, rows = [], []
    for i in range(len(stub)):
        s = compose.apply_to_sample(stub.load_sample(i))
        assert s.image.dtype == np.float32 and s.image.shape == (640, 640, 3), (s.image.dtype, s.image.shape)
        rows.append({"input_sha256": _sha(s.image.transpose(2, 0, 1))})
        samples.append(s)
    _, (boxes, joints, crowd), extras = YoloNASPoseCollateFN()(samples)
    gt = [{k: getattr(s, k) for k in ("joints", "areas", "bboxes_xywh", "is_crowd")} for s in extras["gt_samples"]]
    return {"rows": rows, "targets": (boxes, joints, crowd), "gt_samples": gt}


def imagenet():
    from torch.utils.data import default_collate
    from torchvision import transforms as TV

    chain = TV.Compose([TV.Resize(RESIZE), TV.CenterCrop(CROP), TV.ToTensor(), TV.Normalize(IMAGENET_MEAN, IMAGENET_STD)])
    stub = StubImageNetDataset(pil=True)
    items = [(chain(im), label) for im, label in (stub[i] for i in range(len(stub)))]
    _, labels = default_collate(items)
    return {"rows": [{"input_sha256": _sha(x.numpy())} for x, _ in items], "labels": labels}


def main():
    ref_shim.install()
    import cv2
    import PIL
    import torchvision

    out = {"cv2": cv2.__version__, "numpy": np.__version__, "PIL": PIL.__version__, "torchvision": torchvision.__version__,
           "detection": detection(), "pose": pose(), "imagenet": imagenet()}  # fmt: skip
    torch.save(out, GOLDEN_PATH)
    print({k: len(out[k]["rows"]) for k in ("detection", "pose", "imagenet")}, os.path.getsize(GOLDEN_PATH), "bytes")


if __name__ == "__main__":
    main()
