"""Test infrastructure for the GPU validation chains: seeded stub datasets in the reference's forms for the YOLO-NAS COCO, YOLO-NAS-POSE
and ResNet-50 ImageNet validation lists, the lists themselves, and the loaders of the packed path over the stubs.

Source sizes: landscape, portrait, exactly 636 x 636 (the COCO recipe's input_dim), odd height and width (odd center padding) and,
for ImageNet, a shorter side under 224 (the resize enlarges it) and one of exactly 236 (the crop's left offset rounds half to even).
Targets: crowd and non-crowd boxes, an image without targets, joints outside the image and invisible ones."""
import os

import numpy as np
import torch

from augment_cases import _image
from pose_augment_cases import StubPoseDataset

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN_PATH = os.path.join(ROOT, "tests", "golden", "validation_chains.pt")


class StubDetectionDataset:
    """Raw samples in DetectionDataset.get_sample() form (image, target, crowd_target), every image at most 640 x 640."""

    SIZES = [(480, 636), (636, 477), (636, 636), (333, 517), (640, 640), (101, 203)]

    def __init__(self, seed=0, sizes=None):
        rng = np.random.default_rng(seed)
        self.samples = []
        for i, (h, w) in enumerate(sizes or self.SIZES):
            n = 0 if i == 3 else int(rng.integers(2, 9))
            x1, y1 = rng.uniform(0, w * 0.8, n), rng.uniform(0, h * 0.8, n)
            bw, bh = rng.uniform(2, w * 0.5, n), rng.uniform(2, h * 0.5, n)
            if n:
                bw[0] = 0.7  # dropped by DetectionTargetsFormatTransform's min_bbox_edge_size
            boxes = np.stack([x1, y1, np.minimum(x1 + bw, w), np.minimum(y1 + bh, h), rng.integers(0, 80, n)], -1).astype(np.float32)
            crowd = boxes[:2].copy() if i % 2 == 0 and n else np.zeros((0, 5), np.float32)
            self.samples.append({"image": _image(rng, h, w), "target": boxes, "crowd_target": crowd})

    def __len__(self):
        return len(self.samples)

    def get_sample(self, index, ignore_empty_annotations=False):
        return {k: v.copy() for k, v in self.samples[index].items()}


class StubValidationPoseDataset(StubPoseDataset):
    SIZES = [(480, 640), (640, 480), (636, 636), (333, 517), (200, 300), (427, 640)]


class StubImageNetDataset:
    """(uint8 H x W x 3 RGB array, label) pairs; `pil` returns PIL images instead (what the reference's ImageFolder gives)."""

    SIZES = [(375, 500), (500, 333), (150, 200), (333, 517), (236, 315), (224, 224), (481, 237)]

    def __init__(self, seed=0, pil=False):
        rng = np.random.default_rng(seed)
        self.pil = pil
        self.samples = [(_image(rng, h, w), int(rng.integers(0, 1000))) for h, w in self.SIZES]

    def __len__(self):
        return len(self.samples)

    def __getitem__(self, index):
        image, label = self.samples[index]
        if self.pil:
            from PIL import Image

            return Image.fromarray(image), label
        return image.copy(), label


# recipes/dataset_params/coco_detection_yolo_nas_dataset_params.yaml val_dataset_params.transforms, verbatim
DETECTION = [
    ("DetectionRGB2BGR", dict(prob=1)),
    ("DetectionPadToSize", dict(output_size=[640, 640], pad_value=114)),
    ("DetectionStandardize", dict(max_value=255.0)),
    ("DetectionImagePermute", dict()),
    ("DetectionTargetsFormatTransform", dict(input_dim=[640, 640], output_format="LABEL_CXCYWH")),
]
# recipes/dataset_params/coco_pose_estimation_yolo_nas_dataset_params.yaml val_dataset_params.transforms, verbatim
POSE = [
    ("KeypointsLongestMaxSize", dict(max_height=640, max_width=640)),
    ("KeypointsPadIfNeeded", dict(min_height=640, min_width=640, image_pad_value=127, mask_pad_value=1, padding_mode="bottom_right")),
    ("KeypointsImageStandardize", dict(max_value=255)),
]
# recipes/dataset_params/imagenet_resnet50_dataset_params.yaml: Resize(236) -> CenterCrop(224) -> ToTensor -> Normalize
RESIZE, CROP = 236, 224
IMAGENET_MEAN, IMAGENET_STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


def build(spec, module):
    return [getattr(module, n)(**kw) for n, kw in spec]


def detection_dataset(stub=None):
    from super_gradients_b200.training.datasets.detection_augment_dataset import DetectionAugmentDataset
    from super_gradients_b200.training.transforms import transforms as T

    return DetectionAugmentDataset(stub or StubDetectionDataset(), build(DETECTION, T), with_crowd=True)


def pose_dataset():
    from super_gradients_b200.training.datasets.pose_estimation_datasets.pose_augment_dataset import PoseAugmentDataset
    from super_gradients_b200.training.transforms import keypoints as KP

    return PoseAugmentDataset(StubValidationPoseDataset(), build(POSE, KP), with_gt_samples=True)


def imagenet_dataset(pil=True):
    from super_gradients_b200.training.datasets.imagenet_augment_dataset import ImageNetValidationDataset

    return ImageNetValidationDataset(StubImageNetDataset(pil=pil), RESIZE, CROP, IMAGENET_MEAN, IMAGENET_STD)


def collates():
    """(detection, pose, imagenet) collate functions of the packed path."""
    from super_gradients_b200.training.datasets.detection_augment_dataset import CrowdDetectionAugmentCollateFN
    from super_gradients_b200.training.datasets.imagenet_augment_dataset import ImageNetValidationCollateFN
    from super_gradients_b200.training.datasets.pose_estimation_datasets.pose_augment_dataset import YoloNASPoseAugmentCollateFN

    return (CrowdDetectionAugmentCollateFN((640, 640), 114, 255.0), YoloNASPoseAugmentCollateFN(640, 255.0),
            ImageNetValidationCollateFN(RESIZE, CROP, IMAGENET_MEAN, IMAGENET_STD))  # fmt: skip


def golden():
    return torch.load(GOLDEN_PATH, weights_only=False)
