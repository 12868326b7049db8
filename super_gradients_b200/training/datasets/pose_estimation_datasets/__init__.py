from .yolo_nas_pose_collate_fn import YoloNASPoseCollateFN, flat_collate_tensors_with_batch_index, undo_flat_collate_tensors_with_batch_index  # noqa: F401
from .pose_augment_dataset import PackedPoseBatch, PoseAugmentCollateFN, PoseAugmentDataset, PoseGroundTruth, YoloNASPoseAugmentCollateFN  # noqa: F401
