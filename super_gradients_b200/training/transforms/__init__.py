from .detection_augment import AugmentPlan, BatchAugmenter, MixupPlan
from .keypoints import (
    KeypointsBrightnessContrast,
    KeypointsHSV,
    KeypointsImageStandardize,
    KeypointsLongestMaxSize,
    KeypointsMosaic,
    KeypointsPadIfNeeded,
    KeypointsRandomAffineTransform,
    KeypointsRandomHorizontalFlip,
    KeypointsRandomRotate90,
    KeypointsRemoveSmallObjects,
    KeypointsReverseImageChannels,
)
from .transforms import (
    DetectionHorizontalFlip,
    DetectionHSV,
    DetectionImagePermute,
    DetectionMixup,
    DetectionPaddedRescale,
    DetectionPadToSize,
    DetectionRandomAffine,
    DetectionRGB2BGR,
    DetectionStandardize,
    DetectionTargetsFormatTransform,
)

__all__ = ["AugmentPlan", "BatchAugmenter", "MixupPlan", "DetectionRandomAffine", "DetectionRGB2BGR", "DetectionHSV", "DetectionHorizontalFlip",
           "DetectionMixup", "DetectionPaddedRescale", "DetectionPadToSize", "DetectionStandardize", "DetectionImagePermute", "DetectionTargetsFormatTransform", "KeypointsRandomHorizontalFlip",
           "KeypointsBrightnessContrast", "KeypointsReverseImageChannels", "KeypointsHSV", "KeypointsRandomRotate90", "KeypointsRandomAffineTransform",
           "KeypointsMosaic", "KeypointsLongestMaxSize", "KeypointsPadIfNeeded", "KeypointsImageStandardize", "KeypointsRemoveSmallObjects"]  # fmt: skip
