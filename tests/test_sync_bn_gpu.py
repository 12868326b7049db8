"""sync_bn on the sm_90a kernels: the split BatchNorm / QARepVGG passes with the cross-rank count (SgbBnDesc / SgbQarepDesc .count,
.param_scale).  Two ranks share the one H100 over gloo (eager); one rank over NCCL checks the single-GPU split path, the CUDA graph
and the absence of host synchronisation."""
import copy
import os
import sys

import pytest
import torch
from torch import nn

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)

import sync_bn_cases  # noqa: E402

pytestmark = pytest.mark.gpu
BLOCKS = [c for c in sync_bn_cases.CASES if c != "tiny_yolo_nas_step"]


def _run(rows, cases, port):
    codes, out = sync_bn_cases.launch(ROOT, "cuda", rows, cases, port)
    assert codes == [0] * len(rows), out[-4000:]
    for case in cases:
        assert out.count(f"{case} ok") == len(rows), out[-4000:]


def test_sync_bn_blocks_two_ranks_one_gpu():
    """The block and tiny-YOLO-NAS equivalences of tests/sync_bn_cases.py on the real kernels, two ranks of two images each."""
    _run([2, 2], BLOCKS + ["tiny_yolo_nas_step"], 29571)


def test_sync_bn_blocks_unequal_shards_one_gpu():
    _run([3, 1], BLOCKS, 29572)


@pytest.fixture
def nccl_world1(tmp_path):
    import torch.distributed as dist

    dist.init_process_group("nccl", init_method=f"file://{tmp_path / 'pg'}", rank=0, world_size=1, device_id=torch.device("cuda", 0))
    try:
        yield
    finally:
        dist.destroy_process_group()


def _tiny(g, sync):
    from super_gradients_b200.training.models.detection_models.yolo_nas import YoloNAS

    ap = copy.deepcopy(g["arch"])
    m = YoloNAS(backbone=ap["backbone"], neck=ap["neck"], heads=ap["heads"], num_classes=4, bn_eps=1e-3, bn_momentum=0.03, inplace_act=True, in_channels=3)
    m.load_state_dict({k: v.clone() for k, v in g["sd0"].items()}, strict=False)
    if sync:
        m = nn.SyncBatchNorm.convert_sync_batchnorm(m)
    return m.cuda().train()


@pytest.mark.parametrize("name", BLOCKS)
def test_world1_split_path_equals_fused_path(nccl_world1, name):
    """At world size 1 the synced layer still takes the split path (statistics pass, identity reduce, apply pass with the count
    pointer): outputs within 1 bf16 ulp of the fused unsynced launches, gradients and running statistics to summation order."""
    from super_gradients_b200.training.flat_state import FlatState

    torch.manual_seed(0)
    ref, (c, h, w) = sync_bn_cases._blocks(name)
    sync_bn_cases._randomise_bn(ref, torch.Generator().manual_seed(1))
    syn = nn.SyncBatchNorm.convert_sync_batchnorm(copy.deepcopy(ref))
    x = torch.randn(4, c, h, w, generator=torch.Generator().manual_seed(3))
    res = []
    for m in (ref.cuda().train(), syn.cuda().train()):
        for blk in m.modules():
            if hasattr(blk, "drop_path") and hasattr(blk.drop_path, "sample_scale"):
                blk.drop_path.sample_scale = lambda t: torch.tensor([2.0, 0.0, 2.0, 2.0], device=t.device)
        f = FlatState(m)
        gen = torch.Generator().manual_seed(4)
        with torch.no_grad():
            shape = m(x.cuda().bfloat16().contiguous(memory_format=torch.channels_last)).shape
        f.buffers.zero_()
        g = torch.randn(tuple(shape), generator=gen)
        out, dx = sync_bn_cases._fwd_bwd(m, f, x, g, "cuda")
        res.append((out, dx, f.grads.cpu(), f.buffers.cpu()))
    sync_bn_cases._check(name, res[1], res[0], 1.0, 2e-2)


def test_synced_train_step_graph_world1_nccl(nccl_world1, golden):
    """The synced TrainStep of the tiny YOLO-NAS: eager under torch.cuda.set_sync_debug_mode("error") (no host synchronisation),
    captured into one CUDA graph whose replays follow the eager synced steps, and close to the unsynced step."""
    from super_gradients_b200 import functional as SF
    from super_gradients_b200.training.losses import PPYoloELoss, pad_targets_host
    from super_gradients_b200.training.sg_trainer import TrainStep

    g = golden("tiny_yolo_nas")
    x = g["x"].cuda()
    t = tuple(v.cuda() for v in pad_targets_host(g["targets"], g["x"].shape[0], 16))

    def step(sync):
        m = _tiny(g, sync)
        return TrainStep(m, PPYoloELoss(num_classes=4, use_static_assigner=False), "SGD", {"weight_decay": 1e-5, "momentum": 0.9}, zero_wd_on_bias_and_bn=True, ema=True)

    plain, eager, graphed = step(False), step(True), step(True)
    assert SF.bn_sync(next(mm for mm in eager.model.modules() if isinstance(mm, nn.SyncBatchNorm))) is not None
    # synced vs unsynced (the same statistics, taken in a different summation order); the first two steps size the step arena and
    # build the batched work tables (host-to-device copies), the third runs as every later step does
    for _ in range(3):
        plain.set_hyper_params(1e-3, 0.99)
        lp, _ = plain.run(x, t)
    for _ in range(2):
        eager.set_hyper_params(1e-3, 0.99)
        eager.run(x, t)
    eager.set_hyper_params(1e-3, 0.99)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        calls0 = SF.SYNC_CALLS[0]
        le, _ = eager.run(x, t)
        n_calls = SF.SYNC_CALLS[0] - calls0
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert n_calls > 0
    assert abs(float(lp) - float(le)) <= 2e-2 * abs(float(lp)), (float(lp), float(le))
    assert sync_bn_cases.l2rel(eager.flat.buffers, plain.flat.buffers) < 1e-3
    assert sync_bn_cases.l2rel(eager.flat.params, plain.flat.params) < 1e-3
    # graph: capture restores the state after its warm-up steps, so the replays follow the eager synced twin from step 2 on
    graphed.flat.params.copy_(eager.flat.params)
    graphed.flat.buffers.copy_(eager.flat.buffers)
    for q, r in zip(graphed.state, eager.state):
        q.copy_(r)
    graphed.ema_params.copy_(eager.ema_params)
    graphed.ema_buffers.copy_(eager.ema_buffers)
    graphed.opt_steps = eager.opt_steps
    SF.bump_weight_epoch()
    graphed.set_hyper_params(1e-3, 0.99)
    graphed.capture(x, t, warmup=2)
    assert isinstance(graphed.graph, torch.cuda.CUDAGraph)  # ONE graph (no split around a collective at world size 1)
    for i in range(2):
        eager.set_hyper_params(1e-3, 0.99)
        graphed.set_hyper_params(1e-3, 0.99)
        la, _ = eager.run(x, t)
        lb, _ = graphed.run(x, t)
        assert abs(float(la) - float(lb)) <= 2e-2 * abs(float(la)), (i, float(la), float(lb))
    assert sync_bn_cases.l2rel(graphed.flat.params, eager.flat.params) < 1e-3
    assert sync_bn_cases.l2rel(graphed.flat.buffers, eager.flat.buffers) < 1e-3


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_sync_bn_blocks_two_gpus_nccl():
    """One rank per GPU over NCCL: the same block and tiny-YOLO-NAS equivalences."""
    codes, out = sync_bn_cases.launch(ROOT, "cuda-nccl", [2, 2], BLOCKS + ["tiny_yolo_nas_step"], 29573)
    assert codes == [0, 0], out[-4000:]
