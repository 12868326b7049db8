"""SGD, AdamW, Adam, RMSprop, RMSpropTF, Lion and Lamb on the flat parameter buffer: their constructor arguments, state tensors and
the per-step hyper-parameter rows of the csrc/optim.cu kernels (row layouts and most of the arithmetic: csrc/optim_math.cuh).

The reference builds these with build_optimizer (training/utils/optimizer_utils.py:88-141): the registry defaults of
training/params.py:88-94 are merged under the user's optimizer_params, and with zero_weight_decay_on_bias_and_bn the decay group
gets `optimizer_params.get("weight_decay", 0.0)` -- not the class default -- while the other group gets 0.  Every scalar the
kernels read is derived here in double (Python floats, as torch.optim computes them) and rounded to float32 once.  SGD and AdamW
take the merged optimizer_params as they are: unknown keys are ignored, and the decay group gets the merged weight_decay.
"""
import math
from typing import Any, List, Mapping

import torch

# registry defaults merged under the user's optimizer_params (training/params.py:84-94, optimizer_utils.py:24-29)
REGISTRY_DEFAULTS = {"SGD": {"weight_decay": 1e-4, "momentum": 0.9}, "AdamW": {"weight_decay": 1e-2}, "Adam": {"weight_decay": 1e-4},
                     "RMSprop": {"weight_decay": 1e-4, "momentum": 0.9}, "RMSpropTF": {"weight_decay": 1e-4, "momentum": 0.9}}

# constructor defaults: torch.optim.Adam / RMSprop, and training/utils/optimizers/{rmsprop_tf,lion,lamb}.py
CLASS_DEFAULTS = {
    "Adam": {"lr": 1e-3, "betas": (0.9, 0.999), "eps": 1e-8, "weight_decay": 0.0, "amsgrad": False, "foreach": None, "maximize": False, "capturable": False,
             "differentiable": False, "fused": None, "decoupled_weight_decay": False},
    "RMSprop": {"lr": 1e-2, "alpha": 0.99, "eps": 1e-8, "weight_decay": 0.0, "momentum": 0.0, "centered": False, "capturable": False, "foreach": None,
                "maximize": False, "differentiable": False},
    "RMSpropTF": {"lr": 1e-2, "alpha": 0.9, "eps": 1e-10, "weight_decay": 0.0, "momentum": 0.0, "centered": False, "decoupled_decay": False, "lr_in_momentum": True},
    "Lion": {"lr": 1e-4, "betas": (0.9, 0.99), "weight_decay": 0.0},
    "Lamb": {"lr": 1e-3, "bias_correction": True, "betas": (0.9, 0.999), "eps": 1e-6, "weight_decay": 0.01, "grad_averaging": True, "max_grad_norm": 1.0,
             "trust_clip": False, "always_adapt": False},
}  # fmt: skip

# the optimizers whose constructor arguments are checked against CLASS_DEFAULTS
NAMES = tuple(CLASS_DEFAULTS)
ALL_NAMES = ("SGD", "AdamW") + NAMES

# elements per Lamb reduction chunk (a chunk never spans two parameter tensors)
LAMB_CHUNK = 16384


def resolve(name: str, optimizer_params: Mapping[str, Any], zero_wd_on_bias_and_bn: bool):
    """-> (merged constructor arguments, weight decay of the decay group).  Refuses what the constructor would refuse, and the
    arguments that change torch's arithmetic beyond what the kernels implement (NAMES only)."""
    if name not in ALL_NAMES:
        raise NotImplementedError(f"optimizer {name} has no fused kernel ({', '.join(ALL_NAMES)} are implemented)")
    explicit = {**REGISTRY_DEFAULTS.get(name, {}), **dict(optimizer_params)}
    if name in ("SGD", "AdamW"):
        return explicit, float(explicit.get("weight_decay", 0.0))
    unknown = sorted(set(explicit) - set(CLASS_DEFAULTS[name]))
    if unknown:
        raise TypeError(f"{name}.__init__() got an unexpected keyword argument '{unknown[0]}'")
    op = {**CLASS_DEFAULTS[name], **explicit}
    for flag in ("amsgrad", "maximize", "decoupled_weight_decay"):
        if op.get(flag):
            raise NotImplementedError(f"{name}({flag}=True) has no fused kernel")
    wd = float(explicit.get("weight_decay", 0.0)) if zero_wd_on_bias_and_bn else float(op["weight_decay"])
    return op, wd


def state_tensors(name: str, op: Mapping[str, Any], like: torch.Tensor) -> List[torch.Tensor]:
    """The persistent per-element state, in checkpoint order: SGD [momentum_buffer] (also with momentum 0); AdamW / Adam / Lamb
    [exp_avg, exp_avg_sq]; RMSprop / RMSpropTF [square_avg, momentum_buffer if momentum > 0, grad_avg if centered] (RMSpropTF's
    square_avg starts at ones); Lion [exp_avg]."""
    z = lambda: torch.zeros_like(like)  # noqa: E731
    if name in ("AdamW", "Adam", "Lamb"):
        return [z(), z()]
    if name in ("SGD", "Lion"):
        return [z()]
    sq = torch.ones_like(like) if name == "RMSpropTF" else z()
    return [sq] + ([z()] if float(op["momentum"]) > 0 else []) + ([z()] if op["centered"] else [])


def hyper_param_rows(name: str, op: Mapping[str, Any], wd: float, lr: float, step: int, grad_scale: float) -> List[List[float]]:
    """[decay-group row, zero-decay-group row] of step `step` (1-based) in the layouts of csrc/optim_math.cuh."""
    lr, t, gs = float(lr), int(step), float(grad_scale)
    rows = []
    for w in (wd, 0.0):
        if name == "SGD":
            rows.append([lr, float(op.get("momentum", 0.0)), w, gs, float(bool(op.get("nesterov", False)))])
        elif name == "AdamW":
            b1, b2 = op.get("betas", (0.9, 0.999))
            rows.append([lr, b1, b2, float(op.get("eps", 1e-8)), w, 1 - b1**t, 1 - b2**t, gs])
        elif name == "Adam":
            b1, b2 = (float(b) for b in op["betas"])
            rows.append([w, 1 - b1, b2, 1 - b2, -(lr / (1 - b1**t)), (1 - b2**t) ** 0.5, float(op["eps"]), gs])
        elif name == "RMSprop":
            a = float(op["alpha"])
            rows.append([w, a, 1 - a, float(op["eps"]), float(op["momentum"]), -lr, float(bool(op["centered"])), gs])
        elif name == "RMSpropTF":
            flags = int(bool(op["centered"])) | 2 * int(bool(op["decoupled_decay"])) | 4 * int(bool(op["lr_in_momentum"]))
            rows.append([w, 1.0 - float(op["alpha"]), float(op["eps"]), float(op["momentum"]), lr, -lr, float(flags), gs])
        elif name == "Lion":
            b1, b2 = (float(b) for b in op["betas"])
            rows.append([1 - lr * w, b1, 1 - b1, -lr, b2, 1 - b2, gs])
        elif name == "Lamb":
            b1, b2 = (float(b) for b in op["betas"])
            bc1, bc2 = (1 - b1**t, 1 - b2**t) if op["bias_correction"] else (1.0, 1.0)
            beta3 = 1 - b1 if op["grad_averaging"] else 1.0
            adapt = w != 0 or bool(op["always_adapt"])
            rows.append([b1, beta3, b2, 1 - b2, math.sqrt(bc2), bc1, float(op["eps"]), w, -lr, gs, float(op["max_grad_norm"]), float(adapt), float(bool(op["trust_clip"]))])
        else:
            raise NotImplementedError(f"optimizer {name} has no fused kernel")
    return rows


def lamb_chunk_table(numels: List[int], chunk: int = LAMB_CHUNK) -> torch.Tensor:
    """int64 [nchunk, 4] rows {start, len, first chunk of its tensor, chunks of its tensor} over tensors laid out back to back
    with the given element counts (FlatState.order); every chunk lies inside one tensor and holds at most `chunk` elements."""
    rows, off = [], 0
    for k in numels:
        k = int(k)
        first, cnt = len(rows), max(1, -(-k // chunk)) if k else 0
        for j in range(cnt):
            rows.append([off + j * chunk, min(chunk, k - j * chunk), first, cnt])
        off += k
    return torch.tensor(rows, dtype=torch.int64).reshape(-1, 4)


HP_LEN = {"SGD": 5, "AdamW": 8, "Adam": 8, "RMSprop": 8, "RMSpropTF": 8, "Lion": 7, "Lamb": 13}

# the grad_scale column of every optimizer's hyper-parameter rows (SGD_GS, ADAMW_GS, ADAM_GS, ... of csrc/optim_math.cuh), where
# clip_grad_norm folds its coefficient
GRAD_SCALE_COLUMN = {"SGD": 3, "AdamW": 7, "Adam": 7, "RMSprop": 7, "RMSpropTF": 7, "Lion": 6, "Lamb": 9}


class FlatOptimizer:
    """The state and the per-step launches of one of ALL_NAMES over a FlatState: one kernel per weight-decay range for the elementwise
    optimizers; for Lamb three launches over both ranges at once (gradient sum of squares, m / v update with per-tensor sums,
    apply), reducing in a fixed order through a device-resident chunk table, with no host synchronisation."""

    def __init__(self, name: str, op: Mapping[str, Any], weight_decay: float, flat):
        self.name, self.op, self.weight_decay = name, op, weight_decay
        self.hp_len = HP_LEN[name]
        self.state = state_tensors(name, op, flat.params)
        if name == "Lamb":
            dev = flat.params.device
            self.chunks = flat.chunks
            self.partials = torch.zeros(3 * self.chunks.shape[0], dtype=torch.float64, device=dev)
            self.update = torch.zeros_like(flat.params)

    def rows(self, lr: float, step: int, grad_scale: float) -> List[List[float]]:
        return hyper_param_rows(self.name, self.op, self.weight_decay, lr, step, grad_scale)

    def step(self, flat, hp: torch.Tensor):
        """hp: device float32 [2, hp_len] (rows of this step); flat.grads already reduced across ranks."""
        from .. import kernels as K

        s = self.state
        if self.name == "Lamb":
            if self.chunks.shape[0]:
                K.lamb_grad_sqnorm(flat.grads, self.chunks, hp, self.partials)
                K.lamb_step(flat.params, flat.grads, s[0], s[1], self.update, flat.n_decay, self.chunks, hp, self.partials)
            return
        momentum = self.name in ("RMSprop", "RMSpropTF") and float(self.op["momentum"]) > 0
        centered = self.name in ("RMSprop", "RMSpropTF") and bool(self.op["centered"])
        for a, b, row in ((0, flat.n_decay, 0), (flat.n_decay, flat.n_live, 1)):
            if b <= a:
                continue
            p, g, st = flat.params[a:b], flat.grads[a:b], [t[a:b] for t in s]
            if self.name == "SGD":
                K.sgd_step(p, g, st[0], hp[row])
            elif self.name == "AdamW":
                K.adamw_step(p, g, st[0], st[1], hp[row])
            elif self.name == "Adam":
                K.adam_step(p, g, st[0], st[1], hp[row])
            elif self.name == "Lion":
                K.lion_step(p, g, st[0], hp[row])
            else:
                fn = K.rmsprop_step if self.name == "RMSprop" else K.rmsprop_tf_step
                fn(p, g, st[0], st[1] if momentum else None, st[-1] if centered else None, hp[row])
