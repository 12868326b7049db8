"""Generates tests/golden/optimizers.pt by running the UNMODIFIED reference build_optimizer (/root/reference, through
oracle/ref_shim.py) on the host in float32: for every case of tests/optimizer_cases.py, the tiny YOLO-NAS's parameters with and
without zero_weight_decay_on_bias_and_bn, STEPS steps of the seeded gradient sequence at the per-step learning rates LRS, and
after every step the recorded tensors' parameters and optimizer state (state key -> tensor).  The reference's names of the
zero-decay group (the same in every case) are stored once, so the replay can check that the flat buffer groups the same tensors.  Each key is stored as one
[STEPS, n] tensor (per step the recorded tensors back to back, tests/optimizer_cases.unpack) to keep the file small.

torch's CPU optimizers run their single-tensor path here (foreach is only the default for CUDA tensors).  RMSpropTF calls the
deprecated add_(Number, Tensor) overloads, which torch still accepts with a warning.  Run once in the build container:

    python tests/golden/make_optimizer_goldens.py
"""
import os
import sys
import types
import warnings

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import ref_shim  # noqa: E402
from optimizer_cases import CASES, LRS, STEPS, grads_of, recorded, tiny_model  # noqa: E402


def main():
    ref_shim.install()
    from super_gradients.training.utils import optimizer_utils
    from super_gradients.training.utils.optimizers import lamb, lion, rmsprop_tf  # noqa: F401  (register Lamb, Lion, RMSpropTF)

    warnings.simplefilter("ignore")
    out = {"torch": torch.__version__, "cases": {}}
    for case, (name, params, zero_wd, scale) in CASES.items():
        model = tiny_model()
        names = recorded(model)
        tp = types.SimpleNamespace(optimizer=name, optimizer_params=dict(params), zero_weight_decay_on_bias_and_bn=zero_wd, finetune=False)
        opt = optimizer_utils.build_optimizer(model, LRS[0], tp)
        by_id = {id(p): n for n, p in model.named_parameters()}
        no_decay = sorted(by_id[id(p)] for p in opt.param_groups[0]["params"]) if zero_wd else []  # the zero-decay group comes first
        params_by_name = dict(model.named_parameters())
        steps = []
        for t in range(1, STEPS + 1):
            for grp in opt.param_groups:
                grp["lr"] = LRS[t - 1]
            grads = grads_of(model, t, scale)
            for n, p in model.named_parameters():
                p.grad = grads.get(n)
            opt.step()
            state = {n: {"param": params_by_name[n].detach(), **{k: v for k, v in opt.state[params_by_name[n]].items() if torch.is_tensor(v) and v.shape == params_by_name[n].shape}}
                     for n in names}  # fmt: skip
            steps.append({k: torch.cat([state[n][k].reshape(-1) for n in names]) for k in state[names[0]]})
        steps = {k: torch.stack([s[k] for s in steps]) for k in steps[0]}
        if zero_wd:  # the grouping depends on the model alone: stored once
            assert out.setdefault("no_decay", no_decay) == no_decay
        out["cases"][case] = {"recorded": names, "numel": [params_by_name[n].numel() for n in names], "steps": steps, "optimizer_params": dict(tp.optimizer_params),
                              "group_weight_decay": sorted({float(g["weight_decay"]) for g in opt.param_groups})}  # fmt: skip
    torch.save(out, os.path.join(HERE, "optimizers.pt"))
    print({k: (len(v["recorded"]), v["group_weight_decay"]) for k, v in out["cases"].items()})


if __name__ == "__main__":
    main()
