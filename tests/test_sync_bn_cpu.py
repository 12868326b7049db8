"""sync_bn (torch.nn.SyncBatchNorm under data parallelism) on the CPU: the glue above kernels.py with the cross-rank stand-ins of
tests/cpu_backend_sync.py, on two gloo ranks (tests/sync_bn_cases.py states what every case compares), plus the C-ABI validation of
every synced call shape.  The CUDA kernels themselves are covered by tests/test_sync_bn_gpu.py."""
import collections
import ctypes
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)

import cpu_backend_sync  # noqa: E402
import sync_bn_cases  # noqa: E402
from super_gradients_b200 import functional as SF  # noqa: E402
from super_gradients_b200 import kernels as K  # noqa: E402
from super_gradients_b200 import lib as L  # noqa: E402

BLOCKS = [c for c in sync_bn_cases.CASES if c != "tiny_yolo_nas_step"]


def _run(rows, cases, port):
    codes, out = sync_bn_cases.launch(ROOT, "cpu", rows, cases, port)
    assert codes == [0] * len(rows), out[-4000:]
    for case in cases:
        assert out.count(f"{case} ok") == len(rows), out[-4000:]


def test_sync_bn_blocks_world2_gloo():
    """ConvBNReLU, a wide (stats-in-BatchNorm) layer, QARepVGG, a CSP layer (dual 1x1 pair + bottleneck shortcut fused into the apply
    pass) and a ResNet bottleneck with drop-path on two ranks of two images each, plus one tiny YOLO-NAS TrainStep (loss: the mean over
    images of a fixed linear functional of the raw head outputs, which decomposes over equal shards) against the full batch."""
    _run([2, 2], BLOCKS + ["tiny_yolo_nas_step"], 29561)


def test_sync_bn_blocks_unequal_shards_world2_gloo():
    """The same blocks with 3 images on rank 0 and 1 on rank 1: the global count, not world x local count, divides the sums."""
    _run([3, 1], BLOCKS, 29562)


def test_trainer_sync_bn_world2_gloo(tmp_path):
    """Trainer.train() with sync_bn: True on two ranks: converts the model, trains, the replicas stay identical, state-dict keys are
    unchanged and rank 0's checkpoint loads strictly into the unconverted model."""
    _run([1, 1], [f"trainer:{tmp_path}"], 29563)


@pytest.fixture
def one_rank_group(tmp_path):
    import torch.distributed as dist

    dist.init_process_group("gloo", init_method=f"file://{tmp_path / 'pg'}", rank=0, world_size=1)
    try:
        yield
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("name", ["tiny_yolo_nas", "yolo_nas_s"])
def test_synced_call_shapes_are_served(monkeypatch, one_rank_group, name):
    """Every synced BatchNorm / QARepVGG call of a train step (tiny YOLO-NAS fixture; YOLO-NAS-S at 64 x 64) goes to the product wrapper
    and the real libsgb200.so entry point with host addresses first (as tests/test_abi_validation_cpu.py does): the descriptors with
    the cross-rank count are accepted (the entry point gets as far as its first CUDA call), then the stand-in computes the result."""
    import copy

    from torch import nn

    from super_gradients_b200.training import models
    from super_gradients_b200.training.losses import PPYoloELoss
    from super_gradients_b200.training.sg_trainer import TrainStep

    real = {n: getattr(K, n) for n in cpu_backend_sync._SYNC}
    cpu_backend_sync.install(monkeypatch)
    seen, rejected = collections.Counter(), []
    lib = L.load()

    def call(fn, *args):
        rc = getattr(lib, fn)(*args)
        seen[fn] += 1
        d = args[0]._obj if args and hasattr(args[0], "_obj") else None
        if d is not None and hasattr(d, "count") and d.count:
            seen["with count"] += 1
        if rc in (-1, -2):
            msg = lib.sgb_last_error()
            rejected.append((fn, rc, msg.decode() if msg else ""))
        return rc

    monkeypatch.setattr(L, "call", call)
    monkeypatch.setattr(K, "_stream", lambda: None)
    for n, r in real.items():
        standin = getattr(K, n)

        def both(*a, _real=r, _standin=standin, **k):
            if "sync" in k:
                _real(*a, **k)
            return _standin(*a, **k)

        monkeypatch.setattr(K, n, both)
    if name == "tiny_yolo_nas":
        from super_gradients_b200.training.models.detection_models.yolo_nas import YoloNAS

        g = torch.load(os.path.join(HERE, "golden", "tiny_yolo_nas.pt"), weights_only=False)
        ap = copy.deepcopy(g["arch"])
        m = YoloNAS(backbone=ap["backbone"], neck=ap["neck"], heads=ap["heads"], num_classes=4, bn_eps=1e-3, bn_momentum=0.03, inplace_act=True, in_channels=3)
        m.load_state_dict({k: v.clone() for k, v in g["sd0"].items()}, strict=False)
        x, targets, ncls = g["x"], g["targets"], 4
    else:
        torch.manual_seed(0)
        m = models.get("yolo_nas_s", num_classes=80)
        x = torch.randn(2, 3, 64, 64)
        targets, ncls = torch.tensor([[0, 1, 30.0, 30.0, 20.0, 16.0], [1, 5, 20.0, 40.0, 12.0, 18.0]]), 80
    m = nn.SyncBatchNorm.convert_sync_batchnorm(m).train()
    st = TrainStep(m, PPYoloELoss(num_classes=ncls, use_static_assigner=False), "SGD", {"weight_decay": 1e-5, "momentum": 0.9}, zero_wd_on_bias_and_bn=True)
    calls0 = SF.SYNC_CALLS[0]
    st.set_hyper_params(1e-3)
    loss, _ = st.forward_backward(x, targets)
    assert torch.isfinite(loss)
    assert not rejected, rejected[:5]
    n_bn = sum(isinstance(mm, nn.SyncBatchNorm) for mm in m.modules())
    # one collective per synced launch and direction; a QARepVGG block or a dual pair is ONE launch for its two BatchNorms
    assert 0 < SF.SYNC_CALLS[0] - calls0 < 2 * n_bn and seen["with count"] == SF.SYNC_CALLS[0] - calls0
    assert seen["sgb_qarep_moments"] > 0 and seen["sgb_qarep_bwd_apply"] == seen["sgb_qarep_moments"]
    assert seen["sgb_bn_act_fwd"] > 0 and seen["sgb_bn_act_bwd_apply"] == seen["sgb_bn_act_fwd"]
    for fused in ("sgb_bn_act_fwd_fused", "sgb_bn_act_bwd_fused", "sgb_qarep_fwd_fused", "sgb_qarep_bwd_fused"):
        assert seen[fused] == 0, fused


def test_fused_entry_points_refuse_a_cross_rank_count():
    """The cooperative launches cannot host a collective between their passes: a descriptor with a count is refused, not mis-served."""
    L.load()
    x = torch.zeros(64, 16, dtype=torch.bfloat16)
    cnt = torch.zeros(1, dtype=torch.float64)
    d = L.BnDesc()
    d.M, d.C, d.x_pitch, d.y_pitch, d.stats_repl, d.eps = 64, 16, 16, 16, 1, 1e-5
    d.count, d.param_scale = cnt.data_ptr(), 0.5
    p = x.data_ptr()
    f = torch.zeros(16)
    with pytest.raises(L.SgbError, match="two-pass"):
        L.call("sgb_bn_act_fwd_fused", ctypes.byref(d), p, cnt.data_ptr(), f.data_ptr(), f.data_ptr(), None, None, None, p, f.data_ptr(), f.data_ptr(), None)
    d.param_scale = 0.0
    with pytest.raises(L.SgbError, match="param_scale"):
        L.call("sgb_bn_act_fwd", ctypes.byref(d), p, cnt.data_ptr(), f.data_ptr(), f.data_ptr(), None, None, None, p, f.data_ptr(), f.data_ptr(), None)
