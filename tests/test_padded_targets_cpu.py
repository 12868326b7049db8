"""Host side of the captured detection / pose train step: padding into caller-owned (reused, dirty) buffers equals fresh padding bit
for bit, the per-batch need, and the n_max policy of TrainStep.run_padded, including the epoch-end agreement of two gloo ranks."""
import os
import socket
import subprocess
import sys

import pytest
import torch

from super_gradients_b200.training.losses import max_pose_targets_host, max_targets_host, pad_pose_targets_host, pad_targets_host
from super_gradients_b200.training.sg_trainer import padded_step_plan
from test_pose_loss_host import _random_case

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _det_targets(counts, seed=0):
    """flat [N, 6] targets with counts[b] rows for image b, rows of the images interleaved; a zero box (gt_valid 0) in every third row."""
    g = torch.Generator().manual_seed(seed)
    rows = []
    for b, n in enumerate(counts):
        for _ in range(n):
            rows.append(torch.cat([torch.tensor([float(b), float(torch.randint(0, 4, (1,), generator=g))]), torch.rand(4, generator=g) * 60 + 4]))
    if not rows:
        return torch.zeros(0, 6)
    t = torch.stack(rows)
    t[2::3, 2:] = 0.0
    return t[torch.randperm(t.shape[0], generator=g)]


def _det_cases(golden):
    return [(golden("tiny_yolo_nas")["targets"], 4), (_det_targets((3, 0, 5, 1)), 4), (_det_targets((0, 0, 0)), 3), (_det_targets((7,)), 1)]


def _equal(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert x.dtype == y.dtype and x.shape == y.shape and torch.equal(x, y)


def test_detection_padding_into_out_matches_fresh_padding(golden):
    B, n_max = 4, 9
    out = tuple(t.clone() for t in pad_targets_host(_det_targets((9, 9, 9, 9), seed=3), B, n_max))  # a dirty slot: every row written
    for t, b in _det_cases(golden):
        if b != B:
            continue
        got = pad_targets_host(t, B, n_max, out=out)
        assert all(g is o for g, o in zip(got, out))
        _equal(out, pad_targets_host(t, B, n_max))
    for t, b in _det_cases(golden):  # every fixture at its own batch size, into a fresh dirty buffer
        dirty = tuple(x.fill_(7) for x in (torch.empty(b, 8, 4), torch.empty(b, 8, dtype=torch.int32), torch.empty(b, 8, dtype=torch.uint8)))
        _equal(pad_targets_host(t, b, 8, out=dirty), pad_targets_host(t, b, 8))


def test_pose_padding_into_out_matches_fresh_padding(golden):
    cases = [_random_case(s, n_inst=n)[1] for s, n in ((0, (3, 0, 2)), (1, (1, 4, 1)), (2, (0, 0, 5)), (5, (0, 0, 0)))]
    big = _random_case(9, n_inst=(6, 6, 6), crowd_every=1)[1]
    out = tuple(t.clone() for t in pad_pose_targets_host(big, 3, 6))
    assert int(out[2].sum()) == 18  # the dirty slot has a crowd flag in every row
    for t in cases:
        _equal(pad_pose_targets_host(t, 3, 6, out=out), pad_pose_targets_host(t, 3, 6))
    g = golden("tiny_yolo_nas_pose_train")["targets"]
    J = g[1].shape[1]
    dirty = (torch.full((4, 5, 4), 3.0), torch.full((4, 5, J, 3), 3.0), torch.ones(4, 5, dtype=torch.uint8), torch.ones(4, 5, dtype=torch.uint8))
    _equal(pad_pose_targets_host(g, 4, 5, out=dirty), pad_pose_targets_host(g, 4, 5))


def test_padding_keeps_its_errors_and_checks_out():
    t = _det_targets((3, 1))
    out = pad_targets_host(t, 2, 3)
    with pytest.raises(ValueError, match="3 boxes but n_max=2"):
        pad_targets_host(t, 2, 2, out=tuple(x[:, :2].contiguous() for x in out))
    for bad in ((out[0], out[1]), (out[0], out[1].long(), out[2]), (out[0][:1].contiguous(), out[1], out[2]), (out[0].transpose(1, 2), out[1], out[2])):
        with pytest.raises(ValueError):
            pad_targets_host(t, 2, 3, out=bad)
    _, p, _ = _random_case(1, n_inst=(1, 4, 1))
    with pytest.raises(ValueError, match="4 instances but n_max=3"):
        pad_pose_targets_host(p, 3, 3, out=tuple(x[:, :3].contiguous() for x in pad_pose_targets_host(p, 3, 4)))
    swapped = (p[0], torch.cat([p[1][1:2], p[1][:1], p[1][2:]]), p[2])
    for fn in (lambda: pad_pose_targets_host(swapped, 3, 4), lambda: max_pose_targets_host(swapped)):
        with pytest.raises(ValueError, match="same instances"):
            fn()


def test_need_is_the_largest_per_image_count(golden):
    for t, b in _det_cases(golden):
        want = int(torch.bincount(t[:, 0].long(), minlength=b).max()) if t.numel() else 0
        assert max_targets_host(t) == want
    for s, n in ((0, (3, 0, 2)), (1, (1, 4, 1)), (5, (0, 0, 0))):
        assert max_pose_targets_host(_random_case(s, n_inst=n)[1]) == max(n)
    assert max_pose_targets_host(golden("tiny_yolo_nas_pose_train")["targets"]) == int(torch.bincount(golden("tiny_yolo_nas_pose_train")["targets"][0][:, 0].long()).max())


def test_n_max_policy():
    # first batch: the loss's floor, or the batch's need when larger (never 0: the loss pads to at least one slot)
    assert padded_step_plan(None, None, 16, 5, 32) == ("capture", 16)
    assert padded_step_plan(None, None, 0, 23, 32) == ("capture", 23)
    assert padded_step_plan(None, None, 0, 0, 32) == ("capture", 1)
    # a batch that fits replays; one that needs more, or has another batch size (a last partial batch), runs eagerly
    assert padded_step_plan(23, 32, 0, 23, 32) == ("replay", 23)
    assert padded_step_plan(23, 32, 0, 0, 32) == ("replay", 23)
    assert padded_step_plan(23, 32, 0, 24, 32) == ("eager", 23)
    assert padded_step_plan(23, 32, 0, 3, 17) == ("eager", 23)
    # after an epoch with an overflow the agreed n_max is the floor of the next capture
    assert padded_step_plan(None, None, 40, 30, 32) == ("capture", 40)


_DDP_SCRIPT = r"""
import sys, torch, torch.distributed as dist
sys.path.insert(0, sys.argv[1])
from super_gradients_b200.training.sg_trainer import TrainStep, padded_step_plan
dist.init_process_group("gloo", init_method="env://")
rank = dist.get_rank()

class Step:  # TrainStep's n_max state on the CPU; release_graph frees nothing here
    end_epoch = TrainStep.end_epoch
    def __init__(self):
        self.n_max, self.graph_batch, self._n_floor, self._overflow_need, self.device, self.captures = None, None, 0, 0, torch.device("cpu"), []
    def release_graph(self):
        self.n_max = None
    def step(self, epoch, need, batch, floor=4):
        action, n_max = padded_step_plan(self.n_max, self.graph_batch, max(floor, self._n_floor), need, batch)
        if action == "capture":
            self.n_max, self.graph_batch = n_max, batch
            self.captures.append((epoch, n_max))
        elif action == "eager" and need > n_max:
            self._overflow_need = max(self._overflow_need, need)
        return action

# per rank, per epoch: the needs of its batches.  Rank 0 captures n_max 6, rank 1 n_max 20.  Epoch 1: rank 0 overflows (need 12,
# below rank 1's n_max) and both ranks meet a short last batch.  Epoch 2: nothing overflows.
needs = {0: [[6, 3], [2, 12, 5], [6, 6]], 1: [[20, 1], [3, 4, 2], [9, 1]]}
actions = []
s = Step()
for epoch, ns in enumerate(needs[rank]):
    for i, n in enumerate(ns):
        actions.append(s.step(epoch, n, 4 if epoch == 1 and i == len(ns) - 1 else 8))
    s.end_epoch()
want_captures = {0: [(0, 6), (2, 12)], 1: [(0, 20), (2, 20)]}[rank]
assert s.captures == want_captures, (rank, s.captures)
want_actions = {0: ["capture", "replay", "replay", "eager", "eager", "capture", "replay"], 1: ["capture", "replay", "replay", "replay", "eager", "capture", "replay"]}[rank]
assert actions == want_actions, (rank, actions)
print("rank", rank, "ok")
"""


def test_regrow_is_agreed_by_every_rank_at_the_epoch_end(tmp_path):
    """Both ranks capture again at the same epoch although only one overflowed, and the short last batch alone regrows nothing."""
    script = tmp_path / "regrow.py"
    script.write_text(_DDP_SCRIPT)
    env = dict(os.environ, OMP_NUM_THREADS="1")
    with socket.socket() as sock:  # a port that is free now, not a fixed one another job may hold
        sock.bind(("127.0.0.1", 0))
        port = str(sock.getsockname()[1])
    out = subprocess.run(
        [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1", "--master-port", port, str(script), ROOT],
        capture_output=True, text=True, timeout=240, env=env,
    )  # fmt: skip
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.count("ok") == 2


def test_regrow_without_overflow_keeps_the_graph():
    from super_gradients_b200.training.sg_trainer import TrainStep

    class Step:
        end_epoch = TrainStep.end_epoch

        def __init__(self, overflow):
            self.n_max, self._n_floor, self._overflow_need, self.device, self.released = 8, 0, overflow, torch.device("cpu"), False

        def release_graph(self):
            self.released, self.n_max = True, None

    keep, grow = Step(0), Step(11)
    keep.end_epoch()
    grow.end_epoch()
    assert not keep.released and keep.n_max == 8
    assert grow.released and grow._n_floor == 11 and grow._overflow_need == 0
