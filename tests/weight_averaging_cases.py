"""Inputs of the best-snapshot averaging and EarlyStop goldens (tests/golden/make_weight_averaging_goldens.py) and their replays
(tests/test_weight_averaging_cpu.py): a small BatchNorm model, its seeded per-epoch states, the validated metric sequences and the
EarlyStop argument / value sequences, the reference's averaging loop and a bitwise comparison."""
import torch
from torch import nn

NAN, INF = float("nan"), float("inf")
N_EPOCHS = 16


def bn_model() -> nn.Module:
    """Odd-sized float32 entries (216, 8, 40, 5 ...) and two num_batches_tracked counters."""
    torch.manual_seed(0)
    return nn.Sequential(nn.Conv2d(3, 8, 3), nn.BatchNorm2d(8), nn.ReLU(), nn.Conv2d(8, 5, 1), nn.BatchNorm2d(5))


def snapshot_states() -> list:
    """The model's state at every epoch: seeded values of varied magnitude, counters that grow by a different step each epoch, and
    float32 specials in the first convolution: NaN, +-Inf, subnormals, values near the float32 maximum (a * n overflows)."""
    keys = bn_model().state_dict()
    states = []
    for e in range(N_EPOCHS):
        g = torch.Generator().manual_seed(100 + e)
        sd = {}
        for k, v in keys.items():
            if v.dtype == torch.int64:
                sd[k] = torch.tensor(7 * e + e * e % 5, dtype=torch.int64)
            else:
                sd[k] = (torch.randn(v.shape, generator=g) * 10.0 ** (e % 7 - 3)).float()
        w = sd["0.weight"].view(-1)
        if e == 2:
            w[:4] = torch.tensor([NAN, INF, -INF, 1e38])
        if e in (3, 5):
            w[4:8] = torch.tensor([1e-40, -3e-42, 1.4e-45, 1.17e-38])
        if e in (4, 6, 9):
            w[8:11] = torch.tensor([3e38, -3.3e38, 2e38])
        states.append(sd)
    return states


# name -> (greater_is_better, the watched value of every validated epoch)
AVERAGING_CASES = {
    "loss": (False, [5.0, 4.0, NAN, 6.0, 3.0, INF, 2.5, 7.0, 1.0, 4.5, 3.5, 0.5, 8.0, 7.0, 2.0, 0.25]),
    "accuracy": (True, [0.1, -INF, 0.3, 0.2, NAN, 0.5, 0.05, 0.4, 0.6, 0.35, 0.7, 0.15, 0.05, 0.8, 0.1, 0.9]),
    "few_slots_first_nan": (False, [NAN, 3.0, 2.0, 2.0, 1.0, 5.0]),
    "never_finite": (True, [NAN, INF, -INF, NAN]),
}

POSE_EARLY_STOP = {"phase": "VALIDATION_EPOCH_END", "monitor": "AP", "mode": "max", "min_delta": 0.0001, "patience": 100, "verbose": True}

# name -> (EarlyStop arguments (phase by name), the monitored value at every check; None: the key is missing)
EARLY_STOP_CASES = {
    # the pose recipe's arguments: improvements, then gains below min_delta until patience runs out
    "pose_patience": (POSE_EARLY_STOP, [0.1, 0.2, 0.35, 0.3500999, 0.36] + [0.36 + 0.00005 * (i % 2) for i in range(100)]),
    "pose_threshold": ({**POSE_EARLY_STOP, "threshold": 0.5}, [0.1, 0.3, 0.5, 0.50000001, 0.6]),
    "pose_non_finite": (POSE_EARLY_STOP, [0.1, 0.2, NAN]),
    "pose_inf": (POSE_EARLY_STOP, [0.1, INF]),
    "max_unchecked_nan": ({**POSE_EARLY_STOP, "check_finite": False, "patience": 3}, [0.1, NAN, 0.2, NAN, NAN, NAN]),
    # min mode: min_delta 0.01 enters with the opposite sign; current - min_delta is rounded to float32
    "min_delta_float32": ({"phase": "TRAIN_EPOCH_END", "monitor": "loss", "mode": "min", "min_delta": 0.01, "patience": 2},
                          [0.5, 0.49, 0.48999998, 0.47, 0.4600001, 0.46, 0.455]),  # fmt: skip
    "min_threshold": ({"phase": "VALIDATION_EPOCH_END", "monitor": "loss", "mode": "min", "patience": 5, "threshold": 0.1}, [1.0, 0.5, 0.1, 0.0999999]),
    "missing_not_strict": ({"phase": "VALIDATION_EPOCH_END", "monitor": "AP", "mode": "max", "patience": 2, "strict": False}, [0.1, None, 0.05, None, 0.05]),
}


def reference_average(snaps):
    """weight_averaging_utils.py:89-95 of the reference, on CPU state dicts in slot order."""
    avg = {k: v.clone() for k, v in snaps[0].items()}
    for n in range(1, len(snaps)):
        for key in avg:
            avg[key] = torch.true_divide(avg[key] * n + snaps[n][key], (n + 1))
    return avg


def same_bits(a: torch.Tensor, b: torch.Tensor) -> bool:
    """Equal dtype, shape and bits; NaN matches NaN whatever its payload."""
    if a.dtype != b.dtype or a.shape != b.shape:
        return False
    if not a.is_floating_point():
        return torch.equal(a, b)
    a, b = a.contiguous().reshape(-1), b.contiguous().reshape(-1)
    nan = torch.isnan(a)
    return torch.equal(nan, torch.isnan(b)) and torch.equal(a[~nan].view(torch.int32), b[~nan].view(torch.int32))


def assert_same_state(a, b):
    assert (a is None) == (b is None)
    if a is None:
        return
    assert list(a) == list(b)
    for k in a:
        assert same_bits(a[k], b[k]), k
