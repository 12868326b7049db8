from .detection_augment import AugmentPlan, BatchAugmenter, MixupPlan
from .transforms import (
    DetectionHorizontalFlip,
    DetectionHSV,
    DetectionMixup,
    DetectionPaddedRescale,
    DetectionRandomAffine,
    DetectionRGB2BGR,
    DetectionStandardize,
    DetectionTargetsFormatTransform,
)

__all__ = ["AugmentPlan", "BatchAugmenter", "MixupPlan", "DetectionRandomAffine", "DetectionRGB2BGR", "DetectionHSV", "DetectionHorizontalFlip",
           "DetectionMixup", "DetectionPaddedRescale", "DetectionStandardize", "DetectionTargetsFormatTransform"]  # fmt: skip
