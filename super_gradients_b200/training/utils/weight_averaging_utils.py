"""ModelWeightAveraging (reference: training/utils/weight_averaging_utils.py:12-132): keeps the best `number_of_models_to_average`
validated snapshots of a model and returns their average, which Trainer.train(average_best_models=True) writes to average_model.pth.

What is kept: the constructor, update_snapshots_dict / get_average_model / cleanup, the slot choice (:105-129), the running mean in
slot order (:89-95) bit for bit, and averaging_snapshots.pkl in the reference's format (snapshot0 .. snapshotN-1 as CPU state dicts
or None, snapshots_metric as a float64 numpy array), read back with load_checkpoint=True.
What is different by design: the snapshots live on the device.  Each occupied slot is ONE float32 buffer holding the snapshot's
float32 entries concatenated in state-dict order, and get_average_model averages them in one kernel launch
(kernels.average_snapshots) and one device-to-host copy.  The few other entries (num_batches_tracked) are averaged on the host with
the reference's torch expression, so they come out float32 after two snapshots, as there.  The snapshot file is written at
construction and rewritten only when a slot changes (the reference rewrites it after every validated epoch with the same content).
update_snapshots_dict returns whether a slot changed instead of the snapshot dictionary."""
import os
from typing import Mapping, Optional, Union

import numpy as np
import torch
from torch import nn

from ... import kernels as K

MAX_SLOTS = 64  # SGB_AVG_MAX_SLOTS in include/sgb200.h


def _state_dict_of(model: Union[nn.Module, Mapping[str, torch.Tensor]]) -> Mapping[str, torch.Tensor]:
    if isinstance(model, nn.Module):
        return getattr(model, "module", model).state_dict()
    return model


class ModelWeightAveraging:
    def __init__(self, ckpt_dir: str, greater_is_better: bool, metric_to_watch: str, load_checkpoint: bool = False, number_of_models_to_average: int = 10):
        """
        :param ckpt_dir:                    directory of averaging_snapshots.pkl
        :param greater_is_better:           whether a greater value of the watched metric is better
        :param metric_to_watch:             the key of the watched metric in the validation results (the one ckpt_best.pth follows)
        :param load_checkpoint:             read the snapshots of an earlier run from averaging_snapshots.pkl, if it exists
        :param number_of_models_to_average: number of snapshot slots
        """
        if not 1 <= int(number_of_models_to_average) <= MAX_SLOTS:
            raise ValueError(f"number_of_models_to_average must be in [1, {MAX_SLOTS}], got {number_of_models_to_average}")
        self.averaging_snapshots_file = os.path.join(ckpt_dir, "averaging_snapshots.pkl")
        self.number_of_models_to_average = n = int(number_of_models_to_average)
        self.metric_to_watch = metric_to_watch
        self.greater_is_better = greater_is_better
        self._keys = None  # state-dict keys in order
        self._float = {}  # key -> (offset, numel, shape) of the float32 entries inside a slot
        self._numel = 0
        self._slots = [None] * n  # device float32 [numel] of each occupied slot
        self._other = [None] * n  # {key: CPU tensor} of each occupied slot's other entries
        self._pending = None  # CPU state dicts read from the snapshot file, moved to the device by the first call that sees the model
        if load_checkpoint and ckpt_dir is not None and os.path.isfile(self.averaging_snapshots_file):
            # the file holds a numpy array: torch >= 2.6 refuses it under the default weights_only=True
            saved = torch.load(self.averaging_snapshots_file, map_location="cpu", weights_only=False)
            self.snapshots_metric = np.asarray(saved["snapshots_metric"], dtype=np.float64).copy()
            self._pending = [saved.get(f"snapshot{i}") for i in range(n)]
            filled = [sd is not None for sd in self._pending]
            if len(self.snapshots_metric) != n or filled != sorted(filled, reverse=True):
                raise ValueError(f"{self.averaging_snapshots_file} does not hold {n} snapshot slots filled from slot 0 on")
        else:
            self.snapshots_metric = np.full(n, -np.inf if greater_is_better else np.inf)
            self._save()

    # ------------------------------------------------------------------------------------------------ public API
    def update_snapshots_dict(self, model: Union[nn.Module, Mapping[str, torch.Tensor]], validation_results_dict: Mapping[str, float]) -> bool:
        """Puts the model's state (a module or its state dict) into the slot it replaces, if its watched metric is better than that
        slot's (reference :54-72, :105-129).  Returns whether a slot changed; the snapshot file is rewritten only then."""
        sd = _state_dict_of(model)
        self._materialize(sd)
        val = float(validation_results_dict[self.metric_to_watch])
        if not np.isfinite(val):
            return False
        arr = self.snapshots_metric
        idx = int(np.argmin(arr) if self.greater_is_better else np.argmax(arr))
        if not ((self.greater_is_better and val > arr[idx]) or (not self.greater_is_better and val < arr[idx])):
            return False
        self._store(idx, sd)
        arr[idx] = val
        self._save()
        return True

    def get_average_model(self, model, validation_results_dict: Optional[Mapping[str, float]] = None) -> Optional[Mapping[str, torch.Tensor]]:
        """The average of the occupied slots as a CPU state dict with the model's keys, order and the reference's dtypes (float32
        entries in one pinned buffer), after updating the slots with `model` when validation_results_dict is given.  None while no
        slot is occupied (every validated metric so far was non-finite), as the reference returns."""
        sd = _state_dict_of(model)
        if validation_results_dict is not None:
            self.update_snapshots_dict(sd, validation_results_dict)
        else:
            self._materialize(sd)
        k = sum(s is not None for s in self._slots)
        if k == 0:
            return None
        dev = self._slots[0].device
        out = torch.empty(self._numel, dtype=torch.float32, device=dev)
        if self._numel:
            table = torch.tensor([s.data_ptr() for s in self._slots[:k]], dtype=torch.int64).to(dev)
            K.average_snapshots(table, k, out)
        host = torch.empty(self._numel, dtype=torch.float32, pin_memory=out.is_cuda)
        host.copy_(out)
        avg = {}
        for key in self._keys:
            if key in self._float:
                o, n, shape = self._float[key]
                avg[key] = host[o : o + n].view(shape)
            else:
                a = self._other[0][key].clone()
                for m in range(1, k):  # reference :93-95, verbatim
                    a = torch.true_divide(a * m + self._other[m][key], (m + 1))
                avg[key] = a
        return avg

    def cleanup(self):
        """Deletes the snapshot file (at the end of training)."""
        os.remove(self.averaging_snapshots_file)

    # ------------------------------------------------------------------------------------------------ slots
    def _layout(self, sd: Mapping[str, torch.Tensor]):
        if self._keys is None:
            self._keys = list(sd)
            off = 0
            for key, t in sd.items():
                if t.dtype == torch.float32:
                    self._float[key] = (off, t.numel(), tuple(t.shape))
                    off += t.numel()
            self._numel = off
        elif list(sd) != self._keys or any(tuple(sd[k].shape) != s for k, (_, _, s) in self._float.items()):
            raise ValueError("the state dict does not match the snapshots' keys and shapes")

    def _materialize(self, sd: Mapping[str, torch.Tensor]):
        """Fixes the slot layout from the first state dict seen and moves snapshots read from the file to that state's device."""
        self._layout(sd)
        if self._pending is not None:
            dev = next((t.device for t in sd.values() if t.dtype == torch.float32), torch.device("cpu"))
            pending, self._pending = self._pending, None
            for i, snap in enumerate(pending):
                if snap is not None:
                    self._store(i, snap, dev)

    def _store(self, i: int, sd: Mapping[str, torch.Tensor], device=None):
        self._layout(sd)
        dev = device if device is not None else next((t.device for t in sd.values() if t.dtype == torch.float32), torch.device("cpu"))
        if self._slots[i] is None:
            self._slots[i] = torch.empty(self._numel, dtype=torch.float32, device=dev)
        if self._numel:
            with torch.no_grad():
                torch.cat([sd[k].detach().reshape(-1).to(self._slots[i].device) for k in self._float], out=self._slots[i])
        self._other[i] = {k: sd[k].detach().cpu().clone() for k in self._keys if k not in self._float}

    def _snapshot(self, i: int) -> Optional[dict]:
        if self._slots[i] is None:
            return None
        flat = self._slots[i].cpu()
        return {k: flat[self._float[k][0] : self._float[k][0] + self._float[k][1]].view(self._float[k][2]) if k in self._float else self._other[i][k] for k in self._keys}

    def _save(self):
        d = {f"snapshot{i}": self._snapshot(i) for i in range(self.number_of_models_to_average)}
        d["snapshots_metric"] = self.snapshots_metric.copy()
        torch.save(d, self.averaging_snapshots_file)
