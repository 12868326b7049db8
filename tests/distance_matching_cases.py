"""Shared helpers of the distance-matching tests: the fixture tests/golden/distance_matching.pt (made from the reference by
tests/golden/make_distance_matching_goldens.py) and the padded kernel inputs of one of its batches."""
import os

import torch

from super_gradients_b200.training.utils import detection_utils as DU

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = torch.load(os.path.join(HERE, "golden", "distance_matching.pt"), weights_only=False)
METRICS = {"euclidean": DU.EuclideanDistance, "manhattan": DU.ManhattanDistance}
CASES = [(name, metric) for name in sorted(GOLD) for metric in sorted(METRICS)]


def padded(batch, device="cpu"):
    """(rows, counts, t_pad, t_cnt, c_pad, c_cnt) of one fixture batch, the layout both matching kernels read."""
    rows, counts = DU.pad_predictions(batch["output"], device)
    B = len(batch["output"])
    t_pad, t_cnt = DU.pad_matching_targets_host(batch["targets"], B)
    c_pad = c_cnt = None
    if batch["crowd_targets"] is not None and len(batch["crowd_targets"]):
        c_pad, c_cnt = DU.pad_matching_targets_host(batch["crowd_targets"], B)
        c_pad, c_cnt = c_pad.to(device), c_cnt.to(device)
    return rows, counts, t_pad.to(device), t_cnt.to(device), c_pad, c_cnt


def assert_flags_equal(matched, ignore, counts, ref, where):
    """Kernel flags [B, P, T] against the reference's per-image (preds_matched, preds_to_ignore), bit for bit; padding rows zero."""
    matched, ignore, counts = matched.cpu(), ignore.cpu(), counts.cpu()
    for b, (ref_m, ref_g) in enumerate(ref):
        n = int(counts[b])
        assert n == len(ref_m), (where, b)
        assert torch.equal(matched[b, :n].bool(), ref_m), (where, b, matched[b, :n], ref_m)
        assert torch.equal(ignore[b, :n].bool(), ref_g), (where, b, ignore[b, :n], ref_g)
        assert not matched[b, n:].any() and not ignore[b, n:].any(), (where, b)


def assert_compute_equal(out, ref):
    """compute() against the reference's dictionary: the same keys in the same order, the same values (the summary is the same
    torch arithmetic; the score-threshold grid is a torch.linspace whose last bit depends on the SIMD width)."""
    assert list(out) == list(ref)
    for k, v in ref.items():
        tol = 1e-6 if k.startswith("Best_score_threshold") else 1e-7
        assert abs(out[k] - v) <= tol, (k, out[k], v)
