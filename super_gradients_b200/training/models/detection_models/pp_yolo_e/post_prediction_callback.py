"""PPYoloEPostPredictionCallback (reference: training/models/detection_models/pp_yolo_e/post_prediction_callback.py:9-123):
threshold -> top-k -> class-aware NMS -> [x1, y1, x2, y2, conf, class] rows, for the whole batch in ONE kernel launch
(csrc/nms.cu) instead of a Python loop over images calling torchvision."""
from typing import Any, List, Tuple

import torch
from torch import Tensor, nn

from ..... import kernels as K


class DetectionPostPredictionCallback(nn.Module):
    def forward(self, x, device: str = None):
        raise NotImplementedError


class PPYoloEPostPredictionCallback(DetectionPostPredictionCallback):
    def __init__(self, *, score_threshold: float, nms_threshold: float, nms_top_k: int, max_predictions: int, multi_label_per_box: bool = True, class_agnostic_nms: bool = False):
        super().__init__()
        self.score_threshold = score_threshold
        self.nms_threshold = nms_threshold
        self.nms_top_k = nms_top_k
        self.max_predictions = max_predictions
        self.multi_label_per_box = multi_label_per_box
        self.class_agnostic_nms = class_agnostic_nms

    @torch.no_grad()
    def forward_batched(self, outputs: Any, out=None, out_idx=None, out_count=None) -> Tuple[Tensor, Tensor, Tensor]:
        """Device-resident result: rows [B, max_predictions, 6], flat candidate index [B, max_predictions], count [B] (written into
        out / out_idx / out_count when given, see kernels.batched_nms)."""
        pred_bboxes, pred_scores = self._get_decoded_predictions_from_model_output(outputs)
        dest = {k: v for k, v in dict(out=out, out_idx=out_idx, out_count=out_count).items() if v is not None}
        return K.batched_nms(
            pred_bboxes, pred_scores, self.score_threshold, self.nms_threshold, self.nms_top_k, self.max_rows(),
            multi_label=self.multi_label_per_box, class_agnostic=self.class_agnostic_nms, **dest,
        )  # fmt: skip

    def max_rows(self) -> int:
        """Row pitch of forward_batched's result."""
        return min(int(self.max_predictions), 1024)

    @torch.no_grad()
    def forward(self, outputs: Any, device: str = None) -> List[Tensor]:
        rows, _idx, count = self.forward_batched(outputs)
        counts = count.tolist()  # the one device->host read of the post-processing
        return [rows[b, : counts[b]] for b in range(rows.shape[0])]

    def _get_decoded_predictions_from_model_output(self, outputs: Any) -> Tuple[Tensor, Tensor]:
        if isinstance(outputs, tuple) and len(outputs) == 2:
            if torch.is_tensor(outputs[0]) and torch.is_tensor(outputs[1]) and outputs[0].shape[1] == outputs[1].shape[1] and outputs[0].shape[2] == 4:
                return outputs
            return outputs[0]
        raise ValueError(f"Unsupported output format: {outputs}")
