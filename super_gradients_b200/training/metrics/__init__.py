from .detection_metrics import DetectionMetrics, DetectionMetrics_050, DetectionMetrics_050_095, DetectionMetrics_075, DetectionMetricsDistanceBased  # noqa: F401
from .pose_estimation_metrics import PoseEstimationMetrics  # noqa: F401
from .classification_metrics import Accuracy, Top5  # noqa: F401
