"""Generates tests/golden/weight_averaging.pt by running the UNMODIFIED reference ModelWeightAveraging and EarlyStop (/root/reference,
through oracle/ref_shim.py) over the seeded sequences of tests/weight_averaging_cases.py:

  - averaging: for each case (loss and accuracy modes, NaN / Inf metrics, more validated epochs than slots, ties that must not
    replace, a run where no metric is ever finite), the BatchNorm model of `snapshot_states()` epoch by epoch through
    get_average_model(model, {metric: value}); per epoch the averaged state dict (or None) and snapshots_metric, and at the end the
    whole averaging_snapshots.pkl.  The states carry NaN, +-Inf, subnormals and values near the float32 maximum.
  - EarlyStop: for each case of EARLY_STOP_CASES (the pose recipe's arguments with patience exhaustion, a threshold, non-finite
    values with and without check_finite, min mode with min_delta at float32 resolution, a missing key with strict=False), per
    check the stop flag, wait_count and best score.

Under torch >= 2.6 the reference's own torch.load of the snapshot file fails (weights_only now defaults to True and the file holds a
numpy array), so that one call is run with weights_only=False; numpy 2 dropped the np.Inf alias EarlyStop's constructor reads,
so it is restored around that call.  Run once in the build container:

    python tests/golden/make_weight_averaging_goldens.py
"""
import functools
import os
import sys
import tempfile
from unittest import mock

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import ref_shim  # noqa: E402
from weight_averaging_cases import AVERAGING_CASES, EARLY_STOP_CASES, bn_model, snapshot_states  # noqa: E402


def main():
    ref_shim.install()
    from super_gradients.training.utils import weight_averaging_utils as W
    from super_gradients.training.utils.callbacks import Phase, PhaseContext
    from super_gradients.training.utils.early_stopping import EarlyStop

    states = snapshot_states()
    out = {"torch": torch.__version__, "averaging": {}, "early_stop": {}}
    load = functools.partial(torch.load, weights_only=False)
    for name, (greater, metrics) in AVERAGING_CASES.items():
        model = bn_model()
        steps = []
        with tempfile.TemporaryDirectory() as d, mock.patch.object(W.torch, "load", load):
            mwa = W.ModelWeightAveraging(d, greater_is_better=greater, metric_to_watch="m")
            for epoch, value in enumerate(metrics):
                model.load_state_dict(states[epoch])
                avg = mwa.get_average_model(model, validation_results_dict={"m": value})
                steps.append({"average": None if avg is None else {k: v.clone() for k, v in avg.items()},
                              "snapshots_metric": mwa._get_averaging_snapshots_dict()["snapshots_metric"].copy()})  # fmt: skip
            out["averaging"][name] = {"steps": steps, "pkl": load(mwa.averaging_snapshots_file, map_location="cpu")}
    for name, (kwargs, values) in EARLY_STOP_CASES.items():
        with mock.patch.object(np, "Inf", np.inf, create=True):  # numpy 2 removed the alias the reference's constructor uses
            cb = EarlyStop(**{**kwargs, "phase": Phase[kwargs["phase"]]})
        rows = []
        for v in values:
            ctx = PhaseContext(metrics_dict={} if v is None else {kwargs["monitor"]: v})
            cb(ctx)
            rows.append({"stop": bool(ctx.stop_training), "wait_count": cb.wait_count, "best_score": float(cb.best_score)})
        out["early_stop"][name] = rows
    torch.save(out, os.path.join(HERE, "weight_averaging.pt"))
    print({k: len(v["steps"]) for k, v in out["averaging"].items()}, {k: len(v) for k, v in out["early_stop"].items()})


if __name__ == "__main__":
    main()
