"""Shared inputs of the optimizer goldens (tests/golden/make_optimizer_goldens.py) and the tests that replay them: the tiny YOLO-NAS
fixture's parameters, a gradient sequence from an integer hash (the same float32 values on every machine and torch version), the
per-step learning rates, and the cases.

Every case trains the whole model for STEPS steps; the golden keeps the parameters and optimizer state of RECORDED tensors after
every step.  The ZERO_GRAD tensors get exactly-zero gradients at every step, and ZERO_PARAM starts at zero with zero gradients (Lamb's
zero-norm branches, Lion's sign(0))."""
import copy
import os

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STEPS = 4
LRS = [1e-2, 3e-3, 1e-3, 2e-4]

# name: (optimizer, optimizer_params, zero_weight_decay_on_bias_and_bn, gradient scale)
CASES = {
    "adam_default": ("Adam", {}, True, 1.0),
    "adam_no_zero_wd": ("Adam", {"betas": (0.8, 0.95), "eps": 1e-6}, False, 1e-3),
    "rmsprop_default": ("RMSprop", {}, True, 1.0),
    "rmsprop_centered_momentum": ("RMSprop", {"centered": True, "momentum": 0.5, "alpha": 0.9}, True, 1.0),
    "rmsprop_plain": ("RMSprop", {"momentum": 0.0, "weight_decay": 1e-2}, False, 1e-2),
    "rmsprop_tf_default": ("RMSpropTF", {}, True, 1.0),
    "rmsprop_tf_centered_momentum": ("RMSpropTF", {"centered": True, "momentum": 0.5}, True, 1.0),
    "rmsprop_tf_decoupled": ("RMSpropTF", {"decoupled_decay": True, "weight_decay": 1e-2}, False, 1.0),
    "rmsprop_tf_lr_out_of_momentum": ("RMSpropTF", {"lr_in_momentum": False, "centered": True}, True, 3.0),
    "rmsprop_tf_no_momentum": ("RMSpropTF", {"momentum": 0.0}, False, 1.0),
    "lion_default": ("Lion", {}, True, 1.0),
    "lion_decay": ("Lion", {"weight_decay": 0.5, "betas": (0.95, 0.98)}, False, 1.0),
    "lamb_default": ("Lamb", {}, True, 1.0),
    "lamb_default_no_zero_wd": ("Lamb", {}, False, 1.0),
    "lamb_below_max_norm": ("Lamb", {"weight_decay": 0.01}, True, 1e-3),
    "lamb_above_max_norm": ("Lamb", {"weight_decay": 0.01, "max_grad_norm": 5.0}, True, 1.0),
    "lamb_trust_clip": ("Lamb", {"weight_decay": 0.01, "trust_clip": True}, False, 1e-3),
    "lamb_always_adapt": ("Lamb", {"weight_decay": 0.01, "always_adapt": True}, True, 1.0),
    "lamb_no_bias_correction": ("Lamb", {"weight_decay": 0.01, "bias_correction": False}, False, 1.0),
    "lamb_no_grad_averaging": ("Lamb", {"weight_decay": 0.01, "grad_averaging": False}, True, 1e-3),
}

ZERO_GRAD = ("backbone.stem.conv.post_bn.bias", "heads.head1.cls_pred.weight")
ZERO_PARAM = "heads.head1.reg_pred.bias"


def tiny_model():
    """The tiny YOLO-NAS of tests/golden/tiny_yolo_nas.pt (the product's module tree), in float32 on the host."""
    from super_gradients_b200.training.models.detection_models.yolo_nas import YoloNAS

    g = torch.load(os.path.join(ROOT, "tests", "golden", "tiny_yolo_nas.pt"), weights_only=False)
    torch.manual_seed(0)
    ap = copy.deepcopy(g["arch"])
    m = YoloNAS(backbone=ap["backbone"], neck=ap["neck"], heads=ap["heads"], num_classes=4, bn_eps=1e-3, bn_momentum=0.03, inplace_act=True, in_channels=3)
    m.load_state_dict({k: v.clone() for k, v in g["sd0"].items()}, strict=False)
    with torch.no_grad():
        dict(m.named_parameters())[ZERO_PARAM].zero_()
    return m


def is_live(name: str) -> bool:
    return "rbr_reparam" not in name  # the QARepVGG placeholders never receive a gradient (training/flat_state.py)


def recorded(model):
    """The tensors whose values the golden keeps: small ones of both weight-decay groups (16 to 48 elements: the vector body and the
    scalar tail of torch's CPU loops), two QARepVGG alphas, and the zero tensors."""
    live = [(n, p) for n, p in model.named_parameters() if is_live(n)]
    small = [n for n, p in live if p.numel() <= 48 and not n.endswith("alpha")][:6] + [n for n, p in live if n.endswith("alpha")][:2]
    return sorted(set(small + [*ZERO_GRAD, ZERO_PARAM]))


def unpack(want: dict, step: int) -> dict:
    """{recorded name: {"param" / state key: flat tensor}} after `step` (1-based) of a golden case, which stores each key as one
    [STEPS, n] tensor: per step the recorded tensors back to back in `recorded` order."""
    out = {}
    for key, rows in want["steps"].items():
        flat, off = rows[step - 1], 0
        for n, k in zip(want["recorded"], want["numel"]):
            out.setdefault(n, {})[key] = flat[off : off + k]
            off += k
    return out


def seeded_grad(numel: int, step: int, salt: int, scale: float) -> torch.Tensor:
    """float32 gradients in [-scale/2, scale/2) from a 32-bit integer hash of (element, step, tensor)."""
    i = torch.arange(numel, dtype=torch.int64)
    x = (i * 0x9E3779B1 + (step * 1000003 + salt) * 0x85EBCA77) & 0xFFFFFFFF
    x = x ^ (x >> 15)
    x = (x * 0x2C1B3C6D) & 0xFFFFFFFF
    x = x ^ (x >> 12)
    x = (x * 0x297A2D39) & 0xFFFFFFFF
    x = x ^ (x >> 15)
    return ((x.double() / 2.0**32 - 0.5) * scale).float()


def grads_of(model, step: int, scale: float):
    """{name: gradient} of every live parameter at `step` (1-based)."""
    out = {}
    for salt, (n, p) in enumerate(model.named_parameters()):
        if is_live(n):
            out[n] = torch.zeros_like(p) if n in (*ZERO_GRAD, ZERO_PARAM) else seeded_grad(p.numel(), step, salt, scale).reshape(p.shape)
    return out


def replay(case: str, want: dict, device="cpu"):
    """Runs the product's FlatOptimizer for `case` over the tiny model's flat buffer (on `device`, through whatever kernels.py
    functions are installed) and yields (step, {recorded name: {"param": .., state key: ..}} after the step, the golden's values after
    the step, the values before the step, flat).

    Every step starts from the golden's previous step on the recorded tensors, so each step is checked on its own (torch's
    vectorised CPU sqrt is not correctly rounded, and Lamb's norms add in another order: see assert_matches).  Lamb's global
    gradient norm depends on the gradients alone, and its trust ratio on the recorded tensor's own values."""
    from super_gradients_b200.training import fused_optimizers as FO
    from super_gradients_b200.training.flat_state import FlatState

    name, params, zero_wd, scale = CASES[case]
    model = tiny_model().to(device)
    flat = FlatState(model, zero_wd)
    op, wd = FO.resolve(name, params, zero_wd)
    opt = FO.FlatOptimizer(name, op, wd, flat)
    keys = STATE_KEYS[name](op)

    def values():
        out = {}
        for n in want["recorded"]:
            off, k = flat.offsets[n]
            out[n] = {"param": flat.params[off : off + k].cpu().clone(), **{key: s[off : off + k].cpu().clone() for key, s in zip(keys, opt.state)}}
        return out

    for t in range(1, STEPS + 1):
        grads = grads_of(model, t, scale)
        with torch.no_grad():
            if t > 1:
                for n, prev in unpack(want, t - 1).items():
                    off, k = flat.offsets[n]
                    flat.params[off : off + k].copy_(prev["param"].reshape(-1))
                    for key, s in zip(keys, opt.state):
                        s[off : off + k].copy_(prev[key].reshape(-1))
            for n, (off, k) in flat.offsets.items():
                flat.grads[off : off + k].copy_(grads[n].reshape(-1))
        hp = torch.tensor(opt.rows(LRS[t - 1], t, 1.0), dtype=torch.float32, device=device)
        before = values()
        opt.step(flat, hp)
        yield t, values(), unpack(want, t), before, flat


# the reference's state-dict keys of FlatOptimizer.state, in order
STATE_KEYS = {
    "Adam": lambda op: ["exp_avg", "exp_avg_sq"],
    "Lamb": lambda op: ["exp_avg", "exp_avg_sq"],
    "Lion": lambda op: ["exp_avg"],
    "RMSprop": lambda op: ["square_avg"] + (["momentum_buffer"] if float(op["momentum"]) > 0 else []) + (["grad_avg"] if op["centered"] else []),
    "RMSpropTF": lambda op: ["square_avg"] + (["momentum_buffer"] if float(op["momentum"]) > 0 else []) + (["grad_avg"] if op["centered"] else []),
}


def ulp_distance(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """|a - b| in float32 units in the last place (0 for equal bits; NaN never matches)."""
    ia, ib = a.float().view(torch.int32).long(), b.float().view(torch.int32).long()
    ia = torch.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = torch.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return (ia - ib).abs()


# the values downstream of a square root: torch's vectorised CPU sqrt (AVX2 / AVX-512 builds) is off by one ulp for about 0.6% of
# float32 inputs, where the kernels' sqrt is correctly rounded
SQRT_DOWNSTREAM = {"Adam": {"param"}, "RMSprop": {"param", "momentum_buffer"}, "RMSpropTF": {"param", "momentum_buffer"}, "Lion": set()}


def ulp(x: torch.Tensor) -> torch.Tensor:
    return (torch.nextafter(x.abs(), torch.tensor(float("inf"))) - x.abs()).float()


def assert_matches(case: str, got: dict, want: dict, before: dict, step: int):
    """Adam, RMSprop, RMSpropTF and Lion are bit-identical, except the SQRT_DOWNSTREAM values: there one ulp of the square root
    reaches the term it divides, so |got - want| <= 2^-22 (|want| + |before|) + ulp(want), the term being at most |want| + |before|.
    Lamb: the same bound with 1e-6 for 2^-22 -- its global and per-tensor norms add in another order than torch's CPU reductions,
    and the clip factor and trust ratio scale every term of the step."""
    name = CASES[case][0]
    for n, w in want.items():
        assert set(w) == set(got[n]), (n, sorted(w), sorted(got[n]))
        for key, ref in w.items():
            mine, prev = got[n][key], before[n][key]
            if name == "Lamb" or key in SQRT_DOWNSTREAM[name]:
                err = (mine.double() - ref.double()).abs()
                eps = 1e-6 if name == "Lamb" else 2.0**-22
                tol = eps * (ref.double().abs() + prev.double().abs()) + ulp(ref).double()
                assert bool((err <= tol).all()), f"{case} step {step} {n}.{key}: {int((err > tol).sum())} of {err.numel()} elements outside the bound, worst {float((err / tol).max()):.3g}x"
            else:
                d = ulp_distance(mine, ref)
                assert int(d.max()) == 0, f"{case} step {step} {n}.{key}: {int((d > 0).sum())} of {d.numel()} elements differ, max {int(d.max())} ulp"
