"""Trainer with the reference's entry points -- Trainer(experiment_name, ckpt_root_dir).train(model, training_params,
train_loader, valid_loader) / .test() -- driving the sm_90a hot path (reference: training/sg_trainer/sg_trainer.py).

What is kept: the per-batch order of SURVEY.md Appendix B (H2D -> forward+loss -> backward -> optimizer -> EMA -> LR
step), named training_params of the reference recipes (max_epochs, initial_lr, lr_mode, cosine_final_lr_ratio,
lr_warmup_steps, optimizer, optimizer_params, zero_weight_decay_on_bias_and_bn, ema, ema_params, batch_accumulate,
loss, save_model, ...), the checkpoint dictionary keys, rank-0-only checkpointing.
What is different by design: one flat fp32 parameter / gradient buffer (training/flat_state.py), bf16 activations
without a GradScaler, two optimizer launches per step, ONE flat NCCL all-reduce of live gradients per step under
torchrun, and (optionally) the whole step captured in a CUDA graph.
Out of scope (SURVEY.md section 2): hydra recipes, dataset classes, loggers, metrics bookkeeping, QAT/PTQ, KD.
"""
import datetime
import inspect
import math
import os
import time
from typing import Any, Callable, Dict, Mapping, Optional

import torch
from torch import nn

from .. import functional as SF
from .. import kernels as K
from ..common.factories import LossesFactory, MetricsFactory, _fuzzy
from .flat_state import FlatState
from .utils.callbacks import CallbackHandler, PhaseContext

DEFAULT_TRAINING_PARAMS = {
    "max_epochs": 1,
    "initial_lr": 0.1,
    "lr_mode": "cosine",  # cosine | constant | step
    "cosine_final_lr_ratio": 0.01,
    "lr_updates": [],
    "lr_decay_factor": 0.1,
    "lr_warmup_steps": 0,  # LinearBatchLRWarmup
    "lr_warmup_epochs": 0,  # LinearEpochLRWarmup (and the epoch the schedulers start at)
    "lr_cooldown_epochs": 0,
    "warmup_mode": None,  # None: batch warm-up when lr_warmup_steps > 0, else epoch warm-up
    "warmup_initial_lr": None,
    "optimizer": "SGD",
    "optimizer_params": {},
    "zero_weight_decay_on_bias_and_bn": False,
    "loss": None,
    "criterion_params": {},
    "ema": False,
    "ema_params": {"decay": 0.9999, "decay_type": "constant"},
    "batch_accumulate": 1,
    "mixed_precision": True,  # informational: the compute path is always bf16 operands / fp32 accumulation
    "save_model": True,
    "save_ckpt_epoch_list": [],
    "run_validation_freq": 1,
    "max_train_batches": None,
    "max_valid_batches": None,
    "cuda_graph": False,
    "seed": 42,
    "silent_mode": True,
    "sync_bn": False,
    "phase_callbacks": [],
    "train_metrics_list": [],  # metrics updated with every train batch's outputs (sg_trainer.py:1729-1739); reported as train_<name>
    "valid_metrics_list": [],  # metric objects with update(...) / compute() / reset(), e.g. training.metrics.DetectionMetrics_050
    "metric_to_watch": None,  # None: the validation loss; else a key of the metrics' compute() dictionaries (fuzzy-matched like the reference)
    "greater_metric_to_watch_is_better": False,
    "resume": False,  # continue from <ckpt_root_dir>/<experiment_name>/<ckpt_name> (reference: sg_trainer.py:1877-1935)
    "resume_path": None,  # ... or from an explicit checkpoint file
    "ckpt_name": "ckpt_latest.pth",
    "resume_strict_load": True,
}

# defaults merged under user optimizer_params (reference: training/params.py:84-90)
OPTIMIZER_DEFAULTS = {"SGD": {"weight_decay": 1e-4, "momentum": 0.9}, "Adam": {"weight_decay": 1e-4}, "AdamW": {"weight_decay": 1e-2}}


def _match_metric_name(wanted: str, available: list) -> str:
    """metric_to_watch resolution (reference: sg_trainer.py:588-601, fuzzy_idx_in_list): exact name, else the unique name that
    is equal after dropping case, underscores and punctuation."""
    if wanted in available:
        return wanted
    hits = [a for a in available if _fuzzy(a) == _fuzzy(wanted)]
    if len(hits) != 1:
        raise ValueError(f"No match found for `metric_to_watch={wanted}`. Available metrics to monitor are: `{available}`.")
    return hits[0]


def cosine_lr(step: float, total_steps: float, initial_lr: float, final_lr_ratio: float) -> float:
    """CosineLRScheduler.compute_learning_rate (training/utils/callbacks/callbacks.py:506-511)."""
    lr = 0.5 * initial_lr * (1.0 + math.cos(step / (total_steps + 1) * math.pi))
    return lr * (1 - final_lr_ratio) + initial_lr * final_lr_ratio


def lr_schedule(tp: Mapping[str, Any], steps_per_epoch: int) -> list:
    """The learning rate the reference's callbacks leave in the optimizer at every optimisation step of a run, reproduced by
    replaying their order inside Trainer._train_epoch (training/utils/callbacks/callbacks.py; sg_trainer.py:499-600):
      epoch start  -> LinearEpochLRWarmup (:275-314), while lr_warmup_epochs >= epoch;
      batch start  -> LinearBatchLRWarmup (:317-380): linspace(warmup_initial_lr, initial_lr, min(lr_warmup_steps, len(loader)))[step];
      (the optimizer step uses the rate at this point)
      batch step   -> CosineLRScheduler (:489-512), i.e. its value takes effect from the NEXT step;
      epoch end    -> StepLRScheduler (:395-425), i.e. a milestone e takes effect from epoch e + 1."""
    lr0 = float(tp["initial_lr"])
    spe = max(int(steps_per_epoch), 1)
    max_epochs = int(tp["max_epochs"])
    warm_epochs = int(tp.get("lr_warmup_epochs") or 0)
    warm_steps = int(tp.get("lr_warmup_steps") or 0)
    cool = int(tp.get("lr_cooldown_epochs") or 0)
    mode_w = tp.get("warmup_mode")
    batch_warmup = warm_steps > 0 and (mode_w is None or "batch" in str(getattr(mode_w, "__name__", mode_w)).lower())
    epoch_warmup = not batch_warmup and warm_epochs > 0
    mode = tp.get("lr_mode")
    if mode not in (None, "constant", "none", "cosine", "CosineLRScheduler", "step", "StepLRScheduler"):
        raise NotImplementedError(f"lr_mode {mode}")
    n_batch = min(warm_steps, spe) if batch_warmup else 0
    w0 = tp.get("warmup_initial_lr")
    batch_start = float(w0) if w0 is not None else lr0 / (n_batch + 1)
    epoch_start = float(w0) if w0 is not None else lr0 / (warm_epochs + 1)
    ratio = float(tp.get("cosine_final_lr_ratio", 0.01))
    lr, out = lr0, []
    for epoch in range(max_epochs):
        if epoch_warmup and warm_epochs >= epoch:
            lr = epoch_start + epoch * (lr0 - epoch_start) / warm_epochs
        for b in range(spe):
            g = epoch * spe + b
            if g < n_batch:
                lr = batch_start + (lr0 - batch_start) * g / (n_batch - 1) if n_batch > 1 else batch_start
            out.append(float(lr))
            if mode in ("cosine", "CosineLRScheduler"):
                enabled = (g >= warm_steps) if warm_steps > 0 else (warm_epochs <= epoch < max_epochs - cool)
                if enabled:
                    cur = max(0, spe * (epoch - warm_epochs) + b - warm_steps)
                    total = spe * (max_epochs - warm_epochs - cool) - warm_steps
                    lr = cosine_lr(cur, total, lr0, ratio)
        if mode in ("step", "StepLRScheduler") and warm_epochs <= epoch:
            lr = lr0 * float(tp["lr_decay_factor"]) ** sum(1 for e in tp["lr_updates"] if e <= epoch)
    return out or [lr0]


def ema_decay(decay_type: str, decay: float, step: int, total_steps: int, beta: float = 15.0) -> float:
    """training/utils/ema_decay_schedules.py:22-51 (constant / threshold / exp)."""
    if decay_type == "constant":
        return decay
    if decay_type == "threshold":
        return min(decay, (1 + step) / (10 + step))
    if decay_type == "exp":
        return decay * (1 - math.exp(-beta * step / max(total_steps, 1)))
    raise ValueError(f"unknown ema decay_type {decay_type}")


def is_distributed() -> bool:
    return torch.distributed.is_available() and torch.distributed.is_initialized() and torch.distributed.get_world_size() > 1


def setup_device(device: Optional[str] = None):
    """torchrun-launched jobs (LOCAL_RANK set) are data parallel over NCCL, one process per GPU
    (reference: training/utils/distributed_training_utils.py:173-311, env:// rendezvous)."""
    if not torch.cuda.is_available():
        raise RuntimeError("super_gradients_b200 needs a CUDA device (sm_90a); there is no CPU execution path")
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local_rank)
    if int(os.environ.get("WORLD_SIZE", "1")) > 1 and not torch.distributed.is_initialized():
        # a finite timeout turns a lost rank / mismatched collective into an error instead of an endless wait
        torch.distributed.init_process_group("nccl", init_method="env://", device_id=torch.device("cuda", local_rank), timeout=datetime.timedelta(minutes=4))
    return torch.device("cuda", local_rank)


def _update_metrics(metrics, fields: Mapping[str, Any]):
    """Every metric's update() receives the batch fields it declares (MetricsUpdateCallback, callbacks.py:590-597)."""
    for m in metrics:
        accepted = inspect.signature(m.update).parameters
        m.update(**{k: v for k, v in fields.items() if k in accepted})


def _metric_values(metrics) -> Dict[str, float]:
    values = {}
    for m in metrics:
        res = m.compute()
        values.update({k: float(v) for k, v in res.items()} if isinstance(res, Mapping) else {type(m).__name__: float(res)})
    return values


class _SplitReplay:
    """replay() = graph A, an eagerly issued collective, graph B (TrainStep.capture under data parallelism)."""

    def __init__(self, first, between, second):
        self.first, self.between, self.second = first, between, second

    def replay(self):
        self.first.replay()
        self.between()
        self.second.replay()


class TrainStep:
    """One optimisation step over a FlatState: zero grads -> forward -> loss -> backward -> (all-reduce) -> optimizer
    (-> EMA).  The object owns every per-step device buffer, so the step can be captured in a CUDA graph."""

    STAGING_SLOTS = 8  # pinned host slots of the per-step hyper-parameters (how far the host may run ahead of the device)

    def __init__(self, model: nn.Module, criterion: Callable, optimizer: str, optimizer_params: Mapping[str, Any], zero_wd_on_bias_and_bn: bool, ema: bool = False, batch_accumulate: int = 1,
                 keep_outputs: bool = False):  # fmt: skip
        """keep_outputs: expose the detached model outputs of the last step as `last_outputs` (train metrics).  Under a captured graph
        that is the graph's static output buffer, so work enqueued after run() reads the step just replayed."""
        self.model, self.criterion = model, criterion
        self.keep_outputs = keep_outputs
        self.last_outputs = None
        self.flat = FlatState(model, zero_wd_on_bias_and_bn)
        self.device = self.flat.params.device
        self.opt_name = optimizer
        op = {**OPTIMIZER_DEFAULTS.get(optimizer, {}), **dict(optimizer_params)}
        self.op = op
        f = self.flat
        if optimizer == "SGD":
            self.state = [torch.zeros_like(f.params)]
            self.hp_host = torch.zeros((self.STAGING_SLOTS, 2, 5), dtype=torch.float32).pin_memory()
        elif optimizer in ("AdamW", "Adam"):
            if optimizer == "Adam":
                raise NotImplementedError("Adam (L2-coupled) is not implemented; use AdamW or SGD")
            self.state = [torch.zeros_like(f.params), torch.zeros_like(f.params)]
            self.hp_host = torch.zeros((self.STAGING_SLOTS, 2, 8), dtype=torch.float32).pin_memory()
        else:
            raise NotImplementedError(f"optimizer {optimizer} has no fused kernel (SGD, AdamW are implemented)")
        self.hp = torch.zeros_like(self.hp_host[0], device=self.device)
        self._slot, self._slot_events = 0, [None] * self.STAGING_SLOTS
        self.ema_on = ema
        if ema:
            self.ema_params = f.params.clone()
            self.ema_buffers = f.buffers.clone()
            self.ema_decay_host = torch.zeros((self.STAGING_SLOTS, 1), dtype=torch.float32).pin_memory()
            self.ema_decay = torch.zeros(1, dtype=torch.float32, device=self.device)
        self.world = torch.distributed.get_world_size() if is_distributed() else 1
        self.accumulate = batch_accumulate
        self.opt_steps = 0
        self.graph = None
        self.static_in = None
        self.static_out = None
        self._filters_stale = False
        self.batched_plumbing = True
        self.arena = K.StepArena()   # zero-initialised scratch of one step (owned here: a captured graph replays its addresses)
        self.ctx = SF.StepContext()  # filter caches + batched work tables of this model
        if self.device.type == "cuda" and os.environ.get("SGB_SIDE_WGRAD", "1") != "0":
            self.ctx.side_stream = torch.cuda.Stream(device=self.device)  # weight gradients overlap the dgrad / BN-backward chain
        self._nbt = [b for n, b in model.named_buffers() if n.endswith("num_batches_tracked")]

    # -------------------------------------------------------------------------------------------- host-side schedule
    def set_hyper_params(self, lr: float, ema_decay_value: Optional[float] = None):
        """Writes this step's LR (and Adam bias corrections) to the device; must precede run()."""
        t = self.opt_steps + 1
        # the reference's _backward_step (sg_trainer.py:611-644) calls loss.backward() on every micro-batch without dividing
        # by batch_accumulate: accumulated gradients are SUMMED; only the data-parallel average (DDP) divides
        gs = 1.0 / self.world
        wd = float(self.op.get("weight_decay", 0.0))
        # The host may run many steps ahead of the device (graph replays are enqueued without a sync): every call stages its
        # values in its own pinned slot, and a slot is only rewritten after the copy that read it has executed.
        k = self._slot
        self._slot = (k + 1) % self.STAGING_SLOTS
        if self._slot_events[k] is not None:
            self._slot_events[k].synchronize()
        hp_host = self.hp_host[k]
        if self.opt_name == "SGD":
            mu, nes = float(self.op.get("momentum", 0.0)), float(bool(self.op.get("nesterov", False)))
            hp_host[0] = torch.tensor([lr, mu, wd, gs, nes])
            hp_host[1] = torch.tensor([lr, mu, 0.0, gs, nes])
        else:
            b1, b2 = self.op.get("betas", (0.9, 0.999))
            eps = float(self.op.get("eps", 1e-8))
            row = [lr, b1, b2, eps, wd, 1 - b1**t, 1 - b2**t, gs]
            hp_host[0] = torch.tensor(row)
            row[4] = 0.0
            hp_host[1] = torch.tensor(row)
        self.hp.copy_(hp_host, non_blocking=True)
        if self.ema_on and ema_decay_value is not None:
            self.ema_decay_host[k, 0] = ema_decay_value
            self.ema_decay.copy_(self.ema_decay_host[k], non_blocking=True)
        if self.device.type == "cuda":
            ev = torch.cuda.Event()
            ev.record()
            self._slot_events[k] = ev

    # -------------------------------------------------------------------------------------------- device-side step
    def forward_backward(self, inputs, targets):
        # per-step plumbing that would otherwise cost one tiny launch per layer: one memset for every zero-initialised
        # scratch tensor (K.ARENA), one batched bf16 re-layout of all filters, one batched KRSC -> OIHW gradient pass and
        # one foreach add for the num_batches_tracked counters
        if not self.batched_plumbing:
            return self._forward_backward_plain(inputs, targets)
        self.arena.begin_step(self.device)
        K.ARENA = self.arena
        SF.set_step_context(self.ctx)
        SF._NBT_DEFERRED[0] = True
        try:
            if self._filters_stale:
                if SF.refresh_weight_caches(self.ctx, self.device):
                    self._filters_stale = False
            outputs = self.model(inputs)
            self._keep(outputs)
            out = self.criterion(outputs, targets)
            loss, items = out if isinstance(out, tuple) else (out, out.detach().reshape(1))
            loss.backward()
            SF.flush_wgrads(self.ctx, self.device)
            if self._nbt:
                torch._foreach_add_(self._nbt, 1)
        finally:
            SF._NBT_DEFERRED[0] = False
            SF.set_step_context(None)
            self.arena.end_step()
            K.ARENA = K.NO_ARENA
        # parameters whose gradient arrived through plain autograd (e.g. views created outside a fused Function)
        for _, p in self.flat.order:
            if p.grad is not None:
                p.main_grad.add_(p.grad)
                p.grad = None
        return loss.detach(), items

    def _forward_backward_plain(self, inputs, targets):
        """The same step with every per-layer launch in place (batched_plumbing = False): the reference behaviour the
        batched path is tested against."""
        outputs = self.model(inputs)
        self._keep(outputs)
        out = self.criterion(outputs, targets)
        loss, items = out if isinstance(out, tuple) else (out, out.detach().reshape(1))
        loss.backward()
        for _, p in self.flat.order:
            if p.grad is not None:
                p.main_grad.add_(p.grad)
                p.grad = None
        return loss.detach(), items

    def _keep(self, outputs):
        if self.keep_outputs:
            self.last_outputs = outputs.detach() if torch.is_tensor(outputs) else outputs

    def optimizer_step(self):
        if self.world > 1:
            self.flat.all_reduce_grads(self.world)
        self._apply_update()

    def _apply_update(self):
        """Optimizer + EMA over the (already reduced) flat gradients; no collective in here."""
        f = self.flat
        nd = f.n_decay
        ranges = [(0, nd, 0), (nd, f.n_live, 1)]
        for a, b, row in ranges:
            if b <= a:
                continue
            if self.opt_name == "SGD":
                K.sgd_step(f.params[a:b], f.grads[a:b], self.state[0][a:b], self.hp[row])
            else:
                K.adamw_step(f.params[a:b], f.grads[a:b], self.state[0][a:b], self.state[1][a:b], self.hp[row])
        if self.ema_on:
            K.ema_update(self.ema_params, f.params, self.ema_decay)
            if f.n_buf:
                K.ema_update(self.ema_buffers, f.buffers, self.ema_decay)
        f.zero_grad()
        SF.bump_weight_epoch()
        self._filters_stale = True

    def _step_eager(self, inputs, targets, do_optimizer_step=True):
        loss, items = self.forward_backward(inputs, targets)
        if do_optimizer_step:
            self.optimizer_step()
        return loss, items

    def run(self, inputs, targets, do_optimizer_step=True):
        """inputs / targets: device tensors (targets may be any structure the criterion accepts).  With a captured
        graph the tensors are copied into the static buffers first."""
        if self.graph is not None:
            if not do_optimizer_step:
                raise RuntimeError("gradient accumulation is not supported together with cuda_graph")
            self._copy_static(self.static_in, (inputs, targets))
            self.graph.replay()
            loss, items = self.static_out
        else:
            loss, items = self._step_eager(inputs, targets, do_optimizer_step)
        if do_optimizer_step:
            self.opt_steps += 1
        return loss, items

    @staticmethod
    def _copy_static(dst, src):
        if torch.is_tensor(dst):
            dst.copy_(src, non_blocking=True)
        else:
            for d, s in zip(dst, src):
                TrainStep._copy_static(d, s)

    def capture(self, inputs, targets, warmup: int = 3):
        """Captures the whole step in a CUDA graph (static shapes: pad the targets to a fixed n_max).  The LR is read
        from device memory, so set_hyper_params() keeps working between replays."""
        clone = lambda t: t.clone() if torch.is_tensor(t) else type(t)(clone(u) for u in t)  # noqa: E731
        warmup = max(warmup, 2)  # step 1 sizes the zero arena, step 2 builds the batched work tables the graph replays
        self.static_in = (clone(inputs), clone(targets))
        # The warm-up steps exist to size the arena / build the work tables, not to train: parameters, optimizer moments, EMA,
        # BatchNorm buffers and the step counter are restored afterwards, so a captured run follows the eager trajectory.
        live = [t for t in (self.flat.params, *self.state, getattr(self, "ema_params", None), getattr(self, "ema_buffers", None), self.flat.buffers, *self._nbt) if torch.is_tensor(t) and t.numel()]
        saved, steps0 = [t.clone() for t in live], self.opt_steps
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(warmup):
                self._step_eager(*self.static_in)
                self.opt_steps += 1
        torch.cuda.current_stream().wait_stream(s)
        with torch.no_grad():
            for t, v in zip(live, saved):
                t.copy_(v)
        self.opt_steps = steps0
        torch.cuda.synchronize()
        SF.bump_weight_epoch()
        split = (self.world > 1 and os.environ.get("SGB_NCCL_IN_GRAPH") != "1") or os.environ.get("SGB_SPLIT_GRAPH") == "1"
        if split:
            # Data parallel: TWO graphs around an eagerly issued all-reduce (forward + backward | NCCL | optimizer + EMA).  Capturing
            # the collective inside the graph saves one launch but depends on NCCL's capture support and on nothing else in the
            # process touching CUDA meanwhile; the split costs ~one extra graph launch per step and is as robust as the 1-GPU capture.
            g1, self.static_out = self._capture_region(lambda: self.forward_backward(*self.static_in))
            g2, _ = self._capture_region(self._apply_update, pool=g1.pool())
            self.graph = _SplitReplay(g1, (lambda: self.flat.all_reduce_grads(self.world)) if self.world > 1 else (lambda: None), g2)
        else:
            self.graph, self.static_out = self._capture_region(lambda: self._step_eager(*self.static_in))
        return self.graph

    def _capture_region(self, fn, pool=None):
        """Records fn() into a CUDA graph; returns (graph, fn's outputs = the graph's static output tensors)."""
        g = torch.cuda.CUDAGraph()
        # with NCCL in the process other threads (the process-group watchdog) touch CUDA during capture: thread-local capture mode
        # keeps those calls from invalidating it
        kw = {"capture_error_mode": "thread_local" if self.world > 1 else "global"}
        if pool is not None:
            kw["pool"] = pool
        with torch.cuda.graph(g, **kw):
            out = fn()
        return g, out

    # -------------------------------------------------------------------------------------------- EMA swap (validation)
    def swap_ema(self):
        if not self.ema_on:
            return
        for a, b in ((self.flat.params, self.ema_params), (self.flat.buffers, self.ema_buffers)):
            tmp = a.clone()
            a.copy_(b)
            b.copy_(tmp)
        SF.bump_weight_epoch()


class Trainer:
    def __init__(self, experiment_name: str, device: Optional[str] = None, multi_gpu=None, ckpt_root_dir: Optional[str] = None):
        self.experiment_name = experiment_name
        self.ckpt_root_dir = ckpt_root_dir or os.path.join(os.getcwd(), "checkpoints")
        self.checkpoints_dir_path = os.path.join(self.ckpt_root_dir, experiment_name)
        self.device = setup_device(device)
        self.net: Optional[nn.Module] = None
        self.step: Optional[TrainStep] = None
        self.history: Dict[str, list] = {"train_loss": [], "valid_loss": [], "lr": []}

    @property
    def ddp_silent_mode(self) -> bool:
        return is_distributed() and torch.distributed.get_rank() != 0

    # ------------------------------------------------------------------------------------------------ LR schedule
    def _lr_at(self, tp, global_step: int, steps_per_epoch: int) -> float:
        """Learning rate in the optimizer at one optimisation step (see lr_schedule)."""
        key = (id(tp), int(steps_per_epoch))
        if getattr(self, "_lr_table_key", None) != key:
            self._lr_table = lr_schedule(tp, steps_per_epoch)
            self._lr_table_key = key
        return self._lr_table[min(int(global_step), len(self._lr_table) - 1)]

    # ------------------------------------------------------------------------------------------------ train
    def train(self, model: nn.Module, training_params: Mapping[str, Any], train_loader, valid_loader=None, test_loaders=None, additional_configs_to_log=None):
        tp = {**DEFAULT_TRAINING_PARAMS, **dict(training_params or {})}
        ckpt = None
        if tp["resume"] or tp["resume_path"]:
            path = tp["resume_path"] or os.path.join(self.checkpoints_dir_path, tp["ckpt_name"])
            ckpt = torch.load(path, map_location="cpu", weights_only=False)
            model.load_state_dict(ckpt["net"], strict=bool(tp["resume_strict_load"]))
        self.net = model.to(self.device)
        if tp["sync_bn"] and is_distributed():
            # reference sg_trainer.py:449-456.  The conversion swaps module objects only: the Parameters and buffers (so the state-dict
            # keys, the flat-buffer layout and the adjacency requests) stay the same objects; the fused blocks see SyncBatchNorm modules
            # and reduce their statistics across ranks (functional.bn_sync).  On one rank SyncBatchNorm is plain BatchNorm, as in torch.
            self.net = torch.nn.SyncBatchNorm.convert_sync_batchnorm(self.net)
        torch.manual_seed(int(tp["seed"]) + (torch.distributed.get_rank() if is_distributed() else 0))
        criterion = tp["loss"]
        if isinstance(criterion, (str, Mapping)):
            criterion = LossesFactory().get({criterion: tp["criterion_params"]} if isinstance(criterion, str) else criterion)
        if criterion is None:
            raise ValueError("training_params['loss'] is required")
        if isinstance(criterion, nn.Module):
            criterion = criterion.to(self.device)
        self.criterion = criterion
        from . import metrics as _registered_metrics  # noqa: F401  (fills the METRICS registry)

        train_metrics = [MetricsFactory().get(m) for m in tp["train_metrics_list"] or []]
        self.step = TrainStep(self.net, criterion, tp["optimizer"], tp["optimizer_params"], bool(tp["zero_weight_decay_on_bias_and_bn"]), ema=bool(tp["ema"]), batch_accumulate=int(tp["batch_accumulate"]),
                              keep_outputs=bool(train_metrics))  # fmt: skip
        handler = CallbackHandler(tp["phase_callbacks"])
        context = PhaseContext(net=self.net, criterion=criterion, device=self.device, experiment_name=self.experiment_name, ckpt_dir=self.checkpoints_dir_path,
                               train_loader=train_loader, valid_loader=valid_loader, training_params=tp, optimizer=None, context_methods=self)  # fmt: skip
        steps_per_epoch = len(train_loader) if tp["max_train_batches"] is None else min(len(train_loader), int(tp["max_train_batches"]))
        total_steps = steps_per_epoch * int(tp["max_epochs"])
        ema_p = {**DEFAULT_TRAINING_PARAMS["ema_params"], **dict(tp["ema_params"] or {})}
        acc = int(tp["batch_accumulate"])
        best = None
        start_epoch = 0
        if ckpt is not None:
            start_epoch = int(ckpt.get("epoch", -1)) + 1
            best = ckpt.get("acc")
            self._restore_training_state(ckpt)
        t0 = time.time()
        handler.fire("on_training_start", context)
        for epoch in range(start_epoch, int(tp["max_epochs"])):
            if context.stop_training:
                break
            self.net.train()
            context.update_context(epoch=epoch, batch_idx=None)
            handler.fire("on_train_loader_start", context)
            if hasattr(getattr(train_loader, "sampler", None), "set_epoch"):
                train_loader.sampler.set_epoch(epoch)
            running, nb = None, 0
            for m in train_metrics:
                m.reset()
            for batch_idx, batch in enumerate(train_loader):
                if batch_idx >= steps_per_epoch:
                    break
                inputs, targets = batch[0], batch[1]
                inputs = inputs.to(self.device, non_blocking=True)
                if torch.is_tensor(targets) and not (hasattr(criterion, "forward") and type(criterion).__name__ == "PPYoloELoss"):
                    targets = targets.to(self.device, non_blocking=True)
                gstep = epoch * steps_per_epoch + batch_idx
                lr = self._lr_at(tp, gstep, steps_per_epoch)
                do_step = (batch_idx + 1 + steps_per_epoch * epoch) % acc == 0
                self.step.set_hyper_params(lr, ema_decay(ema_p["decay_type"], float(ema_p["decay"]), gstep + 1, total_steps, float(ema_p.get("beta", 15))) if tp["ema"] else None)
                if tp["cuda_graph"] and self.step.graph is None:
                    if torch.is_tensor(targets) and targets.is_cuda:
                        self.step.capture(inputs, targets)
                    elif not getattr(self, "_warned_no_graph", False):
                        # detection / pose targets stay on the host (ragged per-image lists padded by the loss): the step runs eagerly
                        import warnings

                        warnings.warn("training_params['cuda_graph'] is set but the targets are not a device tensor (detection / pose losses pad them on the "
                                      "host): the train step runs without a CUDA graph; TrainStep.capture() with device-resident padded targets (bench.py) captures it")
                        self._warned_no_graph = True
                if handler.callbacks:
                    context.update_context(batch_idx=batch_idx, inputs=inputs, target=targets, lr=lr)
                    handler.fire("on_train_batch_start", context)
                loss, _items = self.step.run(inputs, targets, do_step)
                running = loss.clone() if running is None else running + loss  # clone: with a captured graph `loss` is the static output buffer
                if train_metrics:  # MetricsUpdateCallback at TRAIN_BATCH_END (sg_trainer.py:1264), enqueued behind the step: no sync
                    _update_metrics(train_metrics, {"preds": self.step.last_outputs, "target": targets, "inputs": inputs, "device": self.device})
                nb += 1
                self.history["lr"].append(lr)
                if handler.callbacks:  # the fused step is over: the reference's per-batch events, in its order
                    context.update_context(loss_log_items=_items, preds=None)
                    handler.fire("on_train_batch_loss_end", context)
                    handler.fire("on_train_batch_backward_end", context)
                    if do_step:
                        handler.fire("on_train_batch_gradient_step_start", context)
                        handler.fire("on_train_batch_gradient_step_end", context)
                    handler.fire("on_train_batch_end", context)
            train_loss = float(running / max(nb, 1)) if running is not None else float("nan")
            self.history["train_loss"].append(train_loss)
            metrics = {"train_loss": train_loss}
            metrics.update({f"train_{k}": v for k, v in _metric_values(train_metrics).items()})  # never collides with the validation keys
            context.update_context(metrics_dict=metrics)
            handler.fire("on_train_loader_end", context)
            if valid_loader is not None and (epoch + 1) % int(tp["run_validation_freq"]) == 0:
                self.step.swap_ema()  # validate / checkpoint the EMA weights (sg_trainer.py:1566-1569)
                handler.fire("on_validation_loader_start", context)
                metrics["valid_loss"] = self._validate(valid_loader, tp, handler, context)
                metrics.update(self.valid_metric_values)
                self.history["valid_loss"].append(metrics["valid_loss"])
                context.update_context(metrics_dict=metrics)
                handler.fire("on_validation_loader_end", context)
                self.step.swap_ema()
            if tp["save_model"] and not self.ddp_silent_mode:
                # `best` always holds ONE metric: the watched validation metric when a validation loader exists (epochs that
                # skipped validation neither compare nor update it), else the training loss
                validated = "valid_loss" in metrics
                if validated and tp["metric_to_watch"]:
                    watch, greater = metrics[_match_metric_name(tp["metric_to_watch"], list(metrics))], bool(tp["greater_metric_to_watch_is_better"])
                elif validated:
                    watch, greater = metrics["valid_loss"], False
                elif valid_loader is None:
                    watch, greater = train_loss, False
                else:
                    watch, greater = None, False
                is_best = watch is not None and (best is None or (watch > best if greater else watch < best))
                best = watch if is_best else best
                self._save_checkpoint(epoch, metrics, tp, is_best, acc=best if best is not None else watch)
                if is_best and "valid_loss" in metrics:
                    handler.fire("on_validation_end_best_epoch", context)
            if not tp["silent_mode"] and not self.ddp_silent_mode:
                print(f"[{self.experiment_name}] epoch {epoch} " + " ".join(f"{k}={v:.5f}" for k, v in metrics.items()) + f" ({time.time() - t0:.1f}s)")
        handler.fire("on_training_end", context)
        return self.history

    @torch.no_grad()
    def _validate(self, loader, tp, handler=None, context=None) -> float:
        """One pass over `loader` in eval mode: mean loss (returned) and the `valid_metrics_list` objects' results
        (self.valid_metric_values).  As the reference's MetricsUpdateCallback does (callbacks.py:590-597), every metric's update()
        receives the batch context -- preds, target, inputs, device and the data set's additional batch items such as
        crowd_targets -- filtered to the arguments it declares."""
        loss, _items, self.valid_metric_values = self._evaluate(loader, tp.get("valid_metrics_list") or [], tp["max_valid_batches"], handler, context)
        return loss

    @torch.no_grad()
    def _evaluate(self, loader, metrics_list, max_batches=None, handler=None, context=None, phase="validation"):
        """-> (mean loss, mean loss-items tensor or None, {metric name: value}); fires on_<phase>_batch_start / _end."""
        from . import metrics as _registered_metrics  # noqa: F401  (fills the METRICS registry)

        self.net.eval()
        tot, items_tot, n = 0.0, None, 0
        valid_metrics = [MetricsFactory().get(m) for m in metrics_list]
        for m in valid_metrics:
            m.reset()
        for i, batch in enumerate(loader):
            if max_batches is not None and i >= int(max_batches):
                break
            inputs, targets = batch[0].to(self.device), batch[1]
            if torch.is_tensor(targets) and type(self.criterion).__name__ != "PPYoloELoss":
                targets = targets.to(self.device)
            if handler is not None and handler.callbacks:
                context.update_context(batch_idx=i, inputs=inputs, target=targets)
                handler.fire(f"on_{phase}_batch_start", context)
            preds = self.net(inputs)
            out = self.criterion(preds, targets) if self.criterion is not None else None
            if handler is not None and handler.callbacks:
                context.update_context(preds=preds, loss_log_items=out[1] if isinstance(out, tuple) else None)
                handler.fire(f"on_{phase}_batch_end", context)
            if out is not None:
                tot += float(out[0] if isinstance(out, tuple) else out)
                if isinstance(out, tuple):
                    items_tot = out[1].detach().double().cpu() if items_tot is None else items_tot + out[1].detach().double().cpu()
            n += 1
            if valid_metrics:
                extra = batch[2] if len(batch) > 2 and isinstance(batch[2], Mapping) else {}
                _update_metrics(valid_metrics, {"preds": preds, "target": targets, "inputs": inputs, "device": self.device, **extra})
        values = _metric_values(valid_metrics)
        self.net.train()
        return tot / max(n, 1), (items_tot / max(n, 1) if items_tot is not None else None), values

    def test(self, model: nn.Module = None, test_loader=None, loss=None, silent_mode: bool = False, test_metrics_list=None, loss_logging_items_names=None,
             metrics_progress_verbose=False, test_phase_callbacks=None, use_ema_net=True) -> Dict[str, float]:  # fmt: skip
        """Trainer.test (reference: sg_trainer.py:2096-2192): evaluates `model` (or the trained network -- its EMA weights when
        use_ema_net and EMA was on) on `test_loader` and returns {loss component name: mean, ..., metric name: value, ...}."""
        if test_loader is None:
            raise ValueError("test_loader is required")
        keep_net, keep_criterion = getattr(self, "net", None), getattr(self, "criterion", None)
        swapped = False
        try:
            if model is not None:
                self.net = model.to(self.device)
            elif keep_net is None:
                raise ValueError("Model is not defined. You should either train some model using trainer.train(...) or pass `model` to trainer.test(...)")
            elif use_ema_net and getattr(self, "step", None) is not None and self.step.ema_on:
                self.step.swap_ema()
                swapped = True
            if loss is not None:
                self.criterion = LossesFactory().get(loss) if isinstance(loss, (str, Mapping)) else loss
            handler = CallbackHandler(list(test_phase_callbacks or []))
            context = PhaseContext(net=self.net, criterion=self.criterion, device=self.device, experiment_name=self.experiment_name)
            handler.fire("on_test_loader_start", context)
            mean_loss, items, values = self._evaluate(test_loader, test_metrics_list or [], None, handler, context, phase="test")
            out = {}
            if self.criterion is not None:
                names = loss_logging_items_names or getattr(self.criterion, "component_names", None)
                if items is not None and names is not None and len(names) == len(items):
                    out.update({n_: float(v) for n_, v in zip(names, items)})
                else:
                    out[type(self.criterion).__name__] = mean_loss
            out.update(values)
            context.update_context(metrics_dict=out)
            handler.fire("on_test_loader_end", context)
            if not silent_mode and not self.ddp_silent_mode:
                print(f"[{self.experiment_name}] test " + " ".join(f"{k}={v:.5f}" for k, v in out.items()))
            return out
        finally:
            if swapped:
                self.step.swap_ema()
            self.net, self.criterion = keep_net, keep_criterion

    # ------------------------------------------------------------------------------------------------ checkpoints
    def _state_dict(self, use_ema=False):
        if use_ema and self.step.ema_on:
            self.step.swap_ema()
            sd = {k: v.detach().clone() for k, v in self.net.state_dict().items()}
            self.step.swap_ema()
            return sd
        return {k: v.detach().clone() for k, v in self.net.state_dict().items()}

    def _restore_training_state(self, ckpt: Mapping[str, Any]):
        """Optimizer moments, step counter and EMA weights of a checkpoint written by _save_checkpoint (the network weights were
        loaded into the model before the flat buffers were built)."""
        st = self.step
        osd = ckpt.get("optimizer_state_dict") or {}
        if osd:
            saved_order, mine_order = list(osd.get("flat_order", [])), [n for n, _ in st.flat.order]
            if osd.get("name") != st.opt_name or sorted(saved_order) != sorted(mine_order):
                raise ValueError("the checkpoint's optimizer state does not belong to this model / optimizer")
            if saved_order == mine_order:
                for mine, saved in zip(st.state, osd["state"]):
                    mine.copy_(saved.to(mine.device))
            else:
                # same parameters, another layout of the flat buffer (FlatState moves parameters that asked to be adjacent): by name
                off = 0
                for name in saved_order:
                    o, k = st.flat.offsets[name]
                    for mine, saved in zip(st.state, osd["state"]):
                        mine[o : o + k].copy_(saved[off : off + k].to(mine.device))
                    off += k
            st.opt_steps = int(osd.get("opt_steps", 0))
        if st.ema_on and ckpt.get("ema_net") is not None:
            ema = ckpt["ema_net"]
            with torch.no_grad():
                for name, (off, k) in st.flat.offsets.items():
                    st.ema_params[off : off + k].copy_(ema[name].reshape(-1).to(st.ema_params.device))
                off = 0
                for name in st.flat.buffer_names:
                    k = ema[name].numel()
                    st.ema_buffers[off : off + k].copy_(ema[name].reshape(-1).to(st.ema_buffers.device))
                    off += k

    def _save_checkpoint(self, epoch: int, metrics: dict, tp, is_best: bool, acc=None):
        """Same dictionary keys as the reference (sg_trainer.py:649-739): net, acc, epoch, metrics, optimizer_state_dict,
        ema_net, ..."""
        os.makedirs(self.checkpoints_dir_path, exist_ok=True)
        state = {
            "net": self._state_dict(False),
            "acc": acc if acc is not None else metrics.get("valid_loss", metrics.get("train_loss")),  # the watched metric, as the reference stores it
            "epoch": epoch,
            "metrics": metrics,
            "packages": {"torch": torch.__version__},
            "optimizer_state_dict": {"name": self.step.opt_name, "flat_order": [n for n, _ in self.step.flat.order], "state": [s.cpu() for s in self.step.state], "opt_steps": self.step.opt_steps},
            "scaler_state_dict": None,
            "processing_params": None,
        }
        if self.step.ema_on:
            state["ema_net"] = self._state_dict(True)
        torch.save(state, os.path.join(self.checkpoints_dir_path, "ckpt_latest.pth"))
        if is_best:
            torch.save(state, os.path.join(self.checkpoints_dir_path, "ckpt_best.pth"))
        if epoch in tp["save_ckpt_epoch_list"]:
            torch.save(state, os.path.join(self.checkpoints_dir_path, f"ckpt_epoch_{epoch}.pth"))
