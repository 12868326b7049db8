"""EarlyStop (reference: training/utils/early_stopping.py:14-147): stops Trainer.train() when a monitored metric stops improving,
reaches a threshold or becomes non-finite.  The decision is the reference's, in its order and with its float32 arithmetic: the value
goes through torch.tensor(float), the best score starts at float32 +-inf, and min_delta takes the sign of the mode."""
import logging
from typing import Optional

import torch

from ...common.registry import register_callback
from .callbacks import Phase, PhaseCallback, PhaseContext, to_phase

logger = logging.getLogger(__name__)


class MissingMonitorKeyException(Exception):
    """The monitored key is not in metrics_dict (raised only with strict=False, and then logged instead of stopping the run)."""


@register_callback("EarlyStop")
class EarlyStop(PhaseCallback):
    mode_dict = {"min": torch.lt, "max": torch.gt}
    supported_phases = (Phase.VALIDATION_EPOCH_END, Phase.TRAIN_EPOCH_END)

    def __init__(self, phase, monitor: str, mode: str = "min", min_delta: float = 0.0, patience: int = 3, check_finite: bool = True, threshold: Optional[float] = None,
                 verbose: bool = False, strict: bool = True):  # fmt: skip
        """
        :param phase:        Phase.VALIDATION_EPOCH_END or Phase.TRAIN_EPOCH_END, its name, or a recipe's {"_target_": ..., "value": ...}
        :param monitor:      key of the monitored metric in context.metrics_dict
        :param mode:         'min' or 'max': whether a smaller or a greater value is an improvement
        :param min_delta:    smallest change that counts as an improvement
        :param patience:     checks without improvement after which training stops
        :param check_finite: stop when the monitored value is NaN or infinite
        :param threshold:    stop as soon as the value is below (min) / above (max) this
        :param verbose:      log the reason of every check
        :param strict:       raise when the monitored key is missing (else log a warning and skip the check)
        """
        phase = to_phase(phase)
        super().__init__(phase)
        if phase not in self.supported_phases:
            raise ValueError(f"EarlyStop doesn't support phase: {phase}, excepted {', '.join(str(x) for x in self.supported_phases)}")
        if mode not in self.mode_dict:
            raise ValueError(f"`mode` can be {', '.join(self.mode_dict)}, got {mode}")
        self.monitor_key = monitor
        self.patience = patience
        self.mode = mode
        self.check_finite = check_finite
        self.threshold = threshold
        self.verbose = verbose
        self.strict = strict
        self.wait_count = 0
        self.should_stop = False
        self.monitor_op = self.mode_dict[mode]
        self.min_delta = min_delta * (1 if self.monitor_op == torch.gt else -1)
        inf = torch.tensor(float("inf"))
        self.best_score = inf if self.monitor_op == torch.lt else -inf

    def _get_metric_value(self, metrics_dict):
        if self.monitor_key not in metrics_dict:
            msg = f"Can't find EarlyStop monitor {self.monitor_key} in metrics_dict: {metrics_dict.keys()}"
            raise (RuntimeError if self.strict else MissingMonitorKeyException)(msg)
        return metrics_dict[self.monitor_key]

    def _check_for_early_stop(self, current: torch.Tensor):
        """-> (reason, should_stop); reference :92-128."""
        if self.check_finite and not torch.isfinite(current):
            return f"Monitored metric {self.monitor_key} = {current} is not finite. Previous best value was {self.best_score:.3f}. Signaling Trainer to stop.", True
        if self.threshold is not None and self.monitor_op(current, self.threshold):
            return f"Stopping threshold reached: {self.monitor_key} = {current} {self.monitor_op} {self.threshold}. Signaling Trainer to stop.", True
        if self.monitor_op(current - self.min_delta, self.best_score.to(current.device)):
            reason = f"Metric {self.monitor_key} improved. New best score: {current:.3f}"
            self.best_score = current
            self.wait_count = 0
            return reason, False
        self.wait_count += 1
        reason = f"Monitored metric {self.monitor_key} did not improve in the last {self.wait_count} records."
        if self.wait_count >= self.patience:
            return reason + f" Best score: {self.best_score:.3f}. Signaling Trainer to stop.", True
        return reason, False

    def __call__(self, context: PhaseContext):
        try:
            current = self._get_metric_value(context.metrics_dict)
        except MissingMonitorKeyException as e:
            logger.warning(e)
            return
        if not isinstance(current, torch.Tensor):
            current = torch.tensor(current)
        reason, self.should_stop = self._check_for_early_stop(current)
        if self.should_stop:
            logger.info(reason)
            context.update_context(stop_training=True)
        elif self.verbose:
            logger.info(reason)
