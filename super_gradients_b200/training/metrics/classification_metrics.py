"""Accuracy and Top5 (reference: training/metrics/classification_metrics.py:40-78): top-1 and top-5 accuracy of classification logits,
under the reference's registry names, so that the ResNet recipes' `train_metrics_list` / `valid_metrics_list: [Accuracy, Top5]`
and `metric_to_watch: Accuracy` work unchanged.

`update(preds, target)` is one launch of the row-wise decode kernel (csrc/classify.cu) that adds to four int64 counters on the
device -- top-1 correct, top-k correct, rows, targets outside [0, C) -- so it never synchronises with the host.  `target` is int64
[N] class indices, or [N, C] soft / one-hot labels reduced by argmax (the reference's "smooth labels" branch).  `compute()` copies the
counters once, sums them across ranks when torch.distributed is initialised (torchmetrics' dist_reduce_fx="sum"), raises on invalid
targets and returns correct / total as a float.  Plain objects, like the other metrics here (torchmetrics is not a dependency)."""
import torch

from ... import kernels as K
from ...common.registry import register_metric

__all__ = ["Accuracy", "Top5"]


class _TopK:
    k = 1
    slot = 0  # counter holding the correct rows: 0 top-1, 1 top-k

    def __init__(self, dist_sync_on_step: bool = False):
        self.dist_sync_on_step = dist_sync_on_step  # accepted for the reference's signature; the counters are reduced in compute()
        self.greater_is_better = True
        self._counters = None

    def reset(self) -> None:
        if self._counters is not None:
            self._counters.zero_()

    def to(self, device):
        return self

    @torch.no_grad()
    def update(self, preds: torch.Tensor, target: torch.Tensor) -> None:
        if preds.dim() != 2:
            raise ValueError(f"preds must be [N, C] logits, got shape {tuple(preds.shape)}")
        if self.k > preds.shape[1]:
            raise ValueError(f"{type(self).__name__} needs at least {self.k} classes, the logits have {preds.shape[1]}")
        if self._counters is None or self._counters.device != preds.device:
            self._counters = torch.zeros(4, dtype=torch.int64, device=preds.device)
        if preds.dtype not in (torch.float32, torch.bfloat16):
            preds = preds.float()
        if preds.shape[1] > 1 and preds.stride(1) != 1:
            preds = preds.contiguous()
        if target.shape != preds.shape:
            target = target.reshape(-1).long()  # no-op for the int64 targets of a classification loader
        elif target.dtype not in (torch.float32, torch.bfloat16):
            target = target.float()
        K.classify_rows(preds, target.to(preds.device, non_blocking=True), k=self.k, counters=self._counters)

    def compute(self) -> float:
        c = self._counters.detach().clone() if self._counters is not None else torch.zeros(4, dtype=torch.int64)
        if torch.distributed.is_available() and torch.distributed.is_initialized() and torch.distributed.get_world_size() > 1:
            torch.distributed.all_reduce(c)
        c = c.cpu()
        if int(c[3]):
            raise ValueError(f"{type(self).__name__}: {int(c[3])} target(s) outside [0, num_classes)")
        total = int(c[2])
        return int(c[self.slot]) / total if total else float("nan")


@register_metric("Accuracy")
class Accuracy(_TopK):
    """classification_metrics.py:40-49: fraction of rows whose first maximal logit is the target (torch.argmax)."""


@register_metric("Top5")
class Top5(_TopK):
    """classification_metrics.py:52-78: fraction of rows whose target is among the five largest logits."""

    k = 5
    slot = 1
