#!/usr/bin/env python
"""Prints the sequence of kernel-wrapper calls the autograd glue (functional.py and the model modules) makes, one line per call:
the wrapper's name, shape / dtype / stride / storage offset of every tensor argument and the scalar arguments (no pointers, no
values), plus the ATen ops other than views that the glue issues itself between wrapper calls.  Two runs of the same workloads must print the same
lines when only the glue's code changed: `diff` of two traces shows every launch, shape or stream that a refactor moved.

Default: the CPU stand-in of the wrappers (tests/cpu_backend.py); two train steps and one eval forward of tiny YOLO-NAS (batched
plumbing on and off, then with each experiment switch off), tiny YOLO-NAS-POSE and resnet18_cifar.
--device cuda: the real kernels, one model (tiny YOLO-NAS, batched plumbing), each line tagged with its stream (main / side).
Usage: python tests/diagnostics/glue_trace.py [--device cuda] > trace.txt"""
import argparse
import copy
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import torch  # noqa: E402
from _pytest.monkeypatch import MonkeyPatch  # noqa: E402
from torch.utils._python_dispatch import TorchDispatchMode  # noqa: E402

import cpu_backend  # noqa: E402
from super_gradients_b200 import functional as SF  # noqa: E402
from super_gradients_b200 import kernels as K  # noqa: E402

SWITCHES = ("QAREP_FOLD", "STEM_PATCHES", "KPAD", "DUAL_CONV", "DEFER_SHORTCUT", "FUSE_SHORTCUT")


class Trace:
    def __init__(self, device):
        self.depth = 0  # > 0 while a wrapper runs: its own ATen ops are the stand-in's business, not the glue's
        self.on = False
        self.cuda = device.type == "cuda"
        self.main = torch.cuda.current_stream().cuda_stream if self.cuda else None
        self.lines = []

    def fmt(self, a):
        if isinstance(a, torch.Tensor):
            return f"T{tuple(a.shape)}:{str(a.dtype)[6:]}:{tuple(a.stride())}+{a.storage_offset()}"
        if isinstance(a, (list, tuple)):
            inner = ",".join(self.fmt(v) for v in a)
            return f"[{inner}]" if isinstance(a, list) else f"({inner})"
        if isinstance(a, dict):
            return "{" + ",".join(f"{k}={self.fmt(v)}" for k, v in a.items()) + "}"
        if a is None or isinstance(a, (bool, int, float, str, torch.dtype, torch.device)):
            return repr(a)
        if hasattr(a, "__name__"):
            return a.__name__
        return type(a).__name__

    def emit(self, name, args, kwargs):
        if not self.on:
            return
        where = ""
        if self.cuda:
            where = "main " if torch.cuda.current_stream().cuda_stream == self.main else "side "
        kw = ",".join(f"{k}={self.fmt(v)}" for k, v in kwargs.items())
        self.lines.append(f"{where}{name}({','.join(self.fmt(a) for a in args)}{';' + kw if kw else ''})")

    def wrap(self, name, fn):
        def traced(*args, **kwargs):
            if self.depth == 0:
                self.emit("K." + name, args, kwargs)
            self.depth += 1
            try:
                return fn(*args, **kwargs)
            finally:
                self.depth -= 1

        return traced


class GlueOps(TorchDispatchMode):
    def __init__(self, trace):
        super().__init__()
        self.trace = trace

    def __torch_dispatch__(self, func, types, args=(), kwargs=None):
        # views (slice, select, reshape as a view, detach, ...) launch nothing: the tensor arguments of the calls that read them show
        # their shape, strides and offset
        if self.trace.depth == 0 and not func.is_view:
            self.trace.emit(str(func), args, kwargs or {})
        return func(*args, **(kwargs or {}))


def _yolo_nas(g, dev):
    from super_gradients_b200.training.models.detection_models.yolo_nas import YoloNAS

    ap = copy.deepcopy(g["arch"])
    m = YoloNAS(backbone=ap["backbone"], neck=ap["neck"], heads=ap["heads"], num_classes=4, bn_eps=1e-3, bn_momentum=0.03, inplace_act=True, in_channels=3)
    m.load_state_dict({k: v.clone() for k, v in g["sd0"].items()}, strict=False)
    return m.to(dev)


def _yolo_nas_pose(g, dev):
    from super_gradients_b200.training.models.pose_estimation_models import YoloNASPose

    ap = copy.deepcopy(g["arch"])
    m = YoloNASPose(backbone=ap["backbone"], neck=ap["neck"], heads=ap["heads"], num_classes=5, bn_eps=1e-3, bn_momentum=0.03, inplace_act=True, in_channels=3)
    m.load_state_dict({k: v.clone() for k, v in g["sd0"].items()}, strict=False)
    return m.to(dev)


def run(trace, title, model, crit, x, t, **attrs):
    from super_gradients_b200.training.sg_trainer import TrainStep

    model.train()
    st = TrainStep(model, crit, "SGD", {"weight_decay": 1e-5, "momentum": 0.9}, zero_wd_on_bias_and_bn=True, ema=True)
    for k, v in attrs.items():
        setattr(st, k, v)
    trace.lines.append(f"=== {title}")
    with GlueOps(trace):
        trace.on = True
        for i in range(2):
            trace.lines.append(f"--- train step {i}")
            st.set_hyper_params(1e-3, 0.99)
            st.forward_backward(x, t)
            st.optimizer_step()
            st.opt_steps += 1
        trace.lines.append("--- eval forward")
        model.eval()
        with torch.no_grad():
            model(x)
        trace.on = False


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--device", default="cpu", choices=["cpu", "cuda"])
    dev = torch.device(ap.parse_args().device)
    mp = MonkeyPatch()
    if dev.type == "cpu":
        cpu_backend.install_training(mp)
    trace = Trace(dev)
    for name in sorted({**cpu_backend._SUBSET, **cpu_backend._TRAINING}):
        mp.setattr(K, name, trace.wrap(name, getattr(K, name)))

    from super_gradients_b200.training.losses import CrossEntropyLoss, PPYoloELoss, YoloNASPoseLoss, pad_targets_host
    from super_gradients_b200.training import models

    load = lambda name: torch.load(os.path.join(ROOT, "tests", "golden", name + ".pt"), weights_only=False)  # noqa: E731
    g = load("tiny_yolo_nas")
    x, t = g["x"].to(dev), tuple(v.to(dev) for v in pad_targets_host(g["targets"], g["x"].shape[0], 16))
    det_loss = lambda: PPYoloELoss(num_classes=4, use_static_assigner=False)  # noqa: E731
    run(trace, "tiny YOLO-NAS, batched plumbing", _yolo_nas(g, dev), det_loss(), x, t)
    if dev.type == "cpu":
        run(trace, "tiny YOLO-NAS, per-layer plumbing", _yolo_nas(g, dev), det_loss(), x, t, batched_plumbing=False)
        g0, gp = load("tiny_yolo_nas_pose"), load("tiny_yolo_nas_pose_train")
        run(trace, "tiny YOLO-NAS-POSE", _yolo_nas_pose(g0, dev), YoloNASPoseLoss(oks_sigmas=gp["sigmas"], **gp["kw"]), gp["x"], gp["targets"])
        torch.manual_seed(0)
        gen = torch.Generator().manual_seed(6)
        xc, yc = torch.randn(8, 3, 32, 32, generator=gen), torch.randint(0, 10, (8,), generator=gen)
        run(trace, "resnet18_cifar", models.get("resnet18_cifar", num_classes=10), CrossEntropyLoss(), xc, yc)
        for sw in SWITCHES:
            flag = getattr(SF, sw)
            flag[0] = False
            run(trace, f"tiny YOLO-NAS, {sw} off", _yolo_nas(g, dev), det_loss(), x, t)
            flag[0] = True
    mp.undo()
    print("\n".join(trace.lines))
    print(f"# {len(trace.lines)} lines")


if __name__ == "__main__":
    main()
