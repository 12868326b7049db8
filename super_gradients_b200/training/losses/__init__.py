from .cross_entropy import CrossEntropyLoss  # noqa: F401
from .ppyolo_loss import PPYoloELoss, max_targets_host, pad_targets_host  # noqa: F401
from .yolo_nas_pose_loss import YoloNASPoseLoss, max_pose_targets_host, pad_pose_targets_host  # noqa: F401
