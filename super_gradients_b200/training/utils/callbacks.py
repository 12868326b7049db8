"""Phase callbacks of Trainer.train() (reference: training/utils/callbacks/base_callbacks.py:13-110 Phase / PhaseContext, :112-900
Callback, :903-970 PhaseCallback).  Same event names and order as the reference's training loop.  One difference is inherent to this
path: forward, loss, backward and the optimizer step of a batch are ONE fused (optionally CUDA-graphed) call, so the per-batch events
between them (on_train_batch_loss_end, on_train_batch_backward_end, on_train_batch_gradient_step_start / _end) all fire right after
that call, in the reference's order; `context.preds` is not populated in training (the step does not hand the raw predictions out)."""
from enum import Enum
from typing import Any, List


class Phase(Enum):
    PRE_TRAINING = "PRE_TRAINING"
    TRAIN_EPOCH_START = "TRAIN_EPOCH_START"
    TRAIN_BATCH_END = "TRAIN_BATCH_END"
    TRAIN_BATCH_STEP = "TRAIN_BATCH_STEP"
    TRAIN_EPOCH_END = "TRAIN_EPOCH_END"
    VALIDATION_BATCH_END = "VALIDATION_BATCH_END"
    VALIDATION_EPOCH_END = "VALIDATION_EPOCH_END"
    VALIDATION_END_BEST_EPOCH = "VALIDATION_END_BEST_EPOCH"
    TEST_BATCH_END = "TEST_BATCH_END"
    TEST_END = "TEST_END"
    AVERAGE_BEST_MODELS_VALIDATION_START = "AVERAGE_BEST_MODELS_VALIDATION_START"
    AVERAGE_BEST_MODELS_VALIDATION_END = "AVERAGE_MODEL_VALIDATION_END"  # the reference's value (base_callbacks.py:25)
    POST_TRAINING = "POST_TRAINING"

    @staticmethod
    def from_string(phase_str: str) -> "Phase":
        try:
            return Phase[phase_str]
        except KeyError:
            raise ValueError(f"Invalid phase string: '{phase_str}'. Must be one of: {[p.name for p in Phase]}")


def to_phase(phase) -> Phase:
    """A Phase, its name, or a recipe's {"_target_": "...Phase", "value": "<name>"} entry (hydra instantiates it as Phase(value))."""
    if isinstance(phase, Phase):
        return phase
    if isinstance(phase, dict):
        if not str(phase.get("_target_", "")).endswith("Phase") or "value" not in phase:
            raise ValueError(f"not a Phase entry: {phase}")
        return Phase(phase["value"])
    return Phase.from_string(phase)


class PhaseContext:
    """Attribute bag handed to every callback and updated in place by the trainer (epoch, batch_idx, inputs, target, preds,
    loss_log_items, metrics_dict, lr, net, criterion, device, experiment_name, ckpt_dir, train_loader, valid_loader,
    training_params, stop_training ...)."""

    def __init__(self, **kwargs: Any):
        self.epoch = self.batch_idx = self.inputs = self.target = self.preds = self.loss_log_items = self.metrics_dict = None
        self.stop_training = False
        self.update_context(**kwargs)

    def update_context(self, **kwargs: Any) -> None:
        for k, v in kwargs.items():
            setattr(self, k, v)


class Callback:
    def on_training_start(self, context: PhaseContext) -> None: ...
    def on_train_loader_start(self, context: PhaseContext) -> None: ...
    def on_train_batch_start(self, context: PhaseContext) -> None: ...
    def on_train_batch_loss_end(self, context: PhaseContext) -> None: ...
    def on_train_batch_backward_end(self, context: PhaseContext) -> None: ...
    def on_train_batch_gradient_step_start(self, context: PhaseContext) -> None: ...
    def on_train_batch_gradient_step_end(self, context: PhaseContext) -> None: ...
    def on_train_batch_end(self, context: PhaseContext) -> None: ...
    def on_train_loader_end(self, context: PhaseContext) -> None: ...
    def on_validation_loader_start(self, context: PhaseContext) -> None: ...
    def on_validation_batch_start(self, context: PhaseContext) -> None: ...
    def on_validation_batch_end(self, context: PhaseContext) -> None: ...
    def on_validation_loader_end(self, context: PhaseContext) -> None: ...
    def on_validation_end_best_epoch(self, context: PhaseContext) -> None: ...
    def on_test_loader_start(self, context: PhaseContext) -> None: ...
    def on_test_batch_start(self, context: PhaseContext) -> None: ...
    def on_test_batch_end(self, context: PhaseContext) -> None: ...
    def on_test_loader_end(self, context: PhaseContext) -> None: ...
    def on_average_best_models_validation_start(self, context: PhaseContext) -> None: ...
    def on_average_best_models_validation_end(self, context: PhaseContext) -> None: ...
    def on_training_end(self, context: PhaseContext) -> None: ...


_PHASE_OF_EVENT = {
    "on_training_start": Phase.PRE_TRAINING, "on_train_loader_start": Phase.TRAIN_EPOCH_START, "on_train_batch_loss_end": Phase.TRAIN_BATCH_END,
    "on_train_batch_gradient_step_end": Phase.TRAIN_BATCH_STEP, "on_train_loader_end": Phase.TRAIN_EPOCH_END, "on_validation_batch_end": Phase.VALIDATION_BATCH_END,
    "on_validation_loader_end": Phase.VALIDATION_EPOCH_END, "on_validation_end_best_epoch": Phase.VALIDATION_END_BEST_EPOCH, "on_test_batch_end": Phase.TEST_BATCH_END,
    "on_test_loader_end": Phase.TEST_END, "on_average_best_models_validation_start": Phase.AVERAGE_BEST_MODELS_VALIDATION_START,
    "on_average_best_models_validation_end": Phase.AVERAGE_BEST_MODELS_VALIDATION_END, "on_training_end": Phase.POST_TRAINING,
}  # fmt: skip


class PhaseCallback(Callback):
    """Callback bound to ONE phase: subclasses implement __call__(context) (base_callbacks.py:903-970)."""

    def __init__(self, phase: Phase):
        self.phase = phase

    def __call__(self, *args, **kwargs):
        raise NotImplementedError


class CallbackHandler:
    """Fires an event on every callback: Callback subclasses get their on_<event> method called, PhaseCallbacks are called when the
    event is the one their phase corresponds to."""

    def __init__(self, callbacks: List[Callback]):
        self.callbacks = list(callbacks or [])

    def fire(self, event: str, context: PhaseContext) -> None:
        for cb in self.callbacks:
            if isinstance(cb, PhaseCallback) or (hasattr(cb, "phase") and callable(cb) and not isinstance(cb, Callback)):
                if _PHASE_OF_EVENT.get(event) == cb.phase:
                    cb(context)
            else:
                getattr(cb, event, lambda c: None)(context)
