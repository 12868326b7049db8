"""Test infrastructure for SyncBatchNorm on the fused blocks: a worker that every rank of a torch.distributed group runs, and the
launcher that starts the ranks as direct child processes.

Every case compares the synced model on this rank's shard of a batch against ONE process running the unconverted model (plain
BatchNorm) on the whole batch, both on the same backend (the real kernels on a GPU, tests/cpu_backend_sync.py on the CPU):
  * outputs and input gradients: this rank's rows of the full-batch ones (outputs within one bf16 ulp);
  * running statistics: equal to the full-batch ones;
  * parameter gradients: the SUM over ranks of each rank's flat gradients equals the full-batch gradient, i.e. after the
    data-parallel 1 / world average each equals the full-batch gradient / world -- torch's DDP + SyncBatchNorm convention.
The upstream gradient of the whole batch is fixed (seeded); rank r's is its rows.

    python sync_bn_cases.py <repo root> <cpu|cuda|cuda-nccl> <rows of rank 0>,<rows of rank 1>,... <case> [<case> ...]
"""
import copy
import os
import subprocess
import sys
import time

import torch
import torch.distributed as dist
from torch import nn

COMPOSITE = ("csp_dual_shortcut", "resnet_bottleneck_droppath")  # blocks of several BatchNorm layers
CASES = ("conv_bn_relu", "wide_stats_in_bn", "qarepvgg", "csp_dual_shortcut", "resnet_bottleneck_droppath", "tiny_yolo_nas_step")


def _blocks(name):
    from super_gradients_b200.modules import ConvBNAct
    from super_gradients_b200.modules.qarepvgg_block import QARepVGGBlock
    from super_gradients_b200.training.models.classification_models.resnet import Bottleneck
    from super_gradients_b200.training.models.detection_models.yolo_nas.yolo_stages import YoloNASCSPLayer

    if name == "conv_bn_relu":
        return ConvBNAct(16, 32, 3, 1, nn.ReLU, bias=False), (16, 12, 12)
    if name == "wide_stats_in_bn":  # more than 96 output channels: statistics from sgb_channel_stats, not the GEMM epilogue
        return ConvBNAct(32, 128, 1, 0, nn.ReLU, bias=False), (32, 8, 8)
    if name == "qarepvgg":
        return QARepVGGBlock(32, 32, activation_type=nn.ReLU, use_alpha=True), (32, 10, 10)
    if name == "csp_dual_shortcut":  # the two 1x1 layers as one GEMM + one BatchNorm, the bottleneck's shortcut fused into its apply pass
        return YoloNASCSPLayer(32, 64, 1, QARepVGGBlock, nn.ReLU, shortcut=True, use_alpha=True), (32, 8, 8)
    if name == "resnet_bottleneck_droppath":
        return Bottleneck(64, 16, droppath_prob=0.5), (64, 8, 8)
    raise KeyError(name)


def _randomise_bn(model, gen):
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, nn.modules.batchnorm._BatchNorm):
                m.weight.copy_(1 + 0.3 * torch.randn(m.weight.shape, generator=gen))
                m.bias.copy_(0.2 * torch.randn(m.bias.shape, generator=gen))
                m.running_mean.copy_(0.1 * torch.randn(m.running_mean.shape, generator=gen))


def _fwd_bwd(model, flat, x, g, dev):
    xin = x.to(dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    out = model(xin)
    out.backward(g.to(dev).to(out.dtype).contiguous(memory_format=torch.channels_last))
    for _, p in flat.order:  # gradients that arrived through plain autograd (as TrainStep does)
        if p.grad is not None:
            p.main_grad.add_(p.grad)
            p.grad = None
    return out.detach().float().cpu(), xin.grad.float().cpu()


def l2rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _check(what, mine, full, tol_out, tol_grad):
    """tol_out: elementwise bound in units of the bf16 ulp of the full-batch value; tol_grad: relative L2 bound."""
    out, dx, grads, bufs = mine
    fo, fdx, fg, fb = full
    ulp = fo.abs().clamp_min(1e-3) * 2.0**-7
    err = (out - fo).abs() / ulp
    if what in COMPOSITE:
        # several layers: a last-bit difference of one stored activation (summation order of the statistics) propagates, so a
        # few outputs of the last layer move by more than one ulp
        assert float((err > tol_out).float().mean()) < 1e-2 and float(err.max()) <= 8 * tol_out, (what, "output", float((err > tol_out).float().mean()), float(err.max()))
    else:
        assert not bool((err > tol_out).any()), (what, "output", int((err > tol_out).sum()), float(err.max()))
    assert l2rel(dx, fdx) < tol_grad, (what, "input gradient", l2rel(dx, fdx))
    assert l2rel(grads, fg) < tol_grad, (what, "parameter gradients", l2rel(grads, fg))
    assert l2rel(bufs, fb) < 1e-5, (what, "running statistics", l2rel(bufs, fb))


def run_block(name, rows, dev, tol_out, tol_grad):
    from super_gradients_b200.training.flat_state import FlatState

    rank, world = dist.get_rank(), dist.get_world_size()
    lo, hi = sum(rows[:rank]), sum(rows[: rank + 1])
    torch.manual_seed(0)
    ref, (c, h, w) = _blocks(name)
    gen = torch.Generator().manual_seed(1)
    _randomise_bn(ref, gen)
    syn = nn.SyncBatchNorm.convert_sync_batchnorm(copy.deepcopy(ref))
    assert list(syn.state_dict()) == list(ref.state_dict())
    n = sum(rows)
    x = torch.randn(n, c, h, w, generator=gen)
    scale = torch.tensor([2.0 if i % 3 else 0.0 for i in range(n)])  # drop-path: a fixed keep pattern by global image index
    models = []
    for m, part in ((ref, slice(0, n)), (syn, slice(lo, hi))):
        m = m.to(dev).train()
        for blk in m.modules():
            if hasattr(blk, "drop_path") and hasattr(blk.drop_path, "sample_scale"):
                blk.drop_path.sample_scale = lambda t, _s=scale[part]: _s.to(t.device)
        models.append((m, FlatState(m), part))
    (mr, fr, _), (ms, fs, part) = models
    with torch.no_grad():
        probe = copy.deepcopy(ref).eval()(x[:1].to(dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last))
    g = torch.randn((n,) + tuple(probe.shape[1:]), generator=gen)
    fo, fdx = _fwd_bwd(mr, fr, x, g, dev)
    so, sdx = _fwd_bwd(ms, fs, x[part], g[part], dev)
    grads = fs.grads.clone()
    dist.all_reduce(grads)
    _check(name, (so, sdx, grads.cpu(), fs.buffers.cpu()), (fo[part], fdx[part], fr.grads.cpu(), fr.buffers.cpu()), tol_out, tol_grad)


class _LinearHeadLoss:
    """Mean over this rank's images of a fixed linear functional of the raw head outputs (cls logits, box distributions).  With equal
    shards the full-batch value is the mean of the ranks' values, so one data-parallel step (gradients averaged over ranks) equals one
    full-batch step on one process."""

    def __call__(self, outputs, weights):
        raw = outputs[1] if isinstance(outputs, tuple) and isinstance(outputs[1], (tuple, list)) else outputs
        loss = sum((t.float() * wt).sum() for t, wt in zip(raw[:2], weights)) / raw[0].shape[0]
        return loss, loss.detach().reshape(1)


def _update_check(root, rows, dev, tol):
    """One SGD step of the tiny YOLO-NAS: synced 2-rank step vs the one-process full-batch step, compared through the UPDATE (params after
    minus before), which is lr * gradient here (no momentum history)."""
    from super_gradients_b200.training.models.detection_models.yolo_nas import YoloNAS
    from super_gradients_b200.training.sg_trainer import TrainStep

    rank = dist.get_rank()
    assert len(set(rows)) == 1, "the loss decomposes over equal shards"
    lo, hi = sum(rows[:rank]), sum(rows[: rank + 1])
    fx = torch.load(os.path.join(root, "tests", "golden", "tiny_yolo_nas.pt"), weights_only=False)

    def build():
        ap = copy.deepcopy(fx["arch"])
        m = YoloNAS(backbone=ap["backbone"], neck=ap["neck"], heads=ap["heads"], num_classes=4, bn_eps=1e-3, bn_momentum=0.03, inplace_act=True, in_channels=3)
        m.load_state_dict({k: v.clone() for k, v in fx["sd0"].items()}, strict=False)
        return m.to(dev).train()

    n = sum(rows)
    gen = torch.Generator().manual_seed(2)
    reps = (n + fx["x"].shape[0] - 1) // fx["x"].shape[0]
    x = (torch.cat([fx["x"]] * reps)[:n] * (1 + 0.1 * torch.rand(n, 1, 1, 1, generator=gen))).contiguous()
    probe = build()
    raw = probe(x[:2].to(dev))
    raw = raw[1] if isinstance(raw, tuple) and isinstance(raw[1], (tuple, list)) else raw
    wts = [torch.randn((n,) + tuple(t.shape[1:]), generator=gen) for t in raw[:2]]
    del probe, raw
    # the whole model is sensitive to last-bit differences (one flipped bf16 activation grows layer by layer to percent-level changes
    # of the deep maps' statistics), so the full-batch step runs the SAME synced layers with a one-rank group: the two steps then
    # differ only in how the ranks' sums are combined
    own = [dist.new_group([r]) for r in range(dist.get_world_size())][rank]
    res = []
    for part, sync in ((slice(0, n), False), (slice(lo, hi), True)):
        m = nn.SyncBatchNorm.convert_sync_batchnorm(build(), process_group=None if sync else own)
        st = TrainStep(m, _LinearHeadLoss(), "SGD", {"weight_decay": 0.0, "momentum": 0.0}, zero_wd_on_bias_and_bn=True, ema=False)
        p0 = st.flat.params.clone()
        if not sync:
            st.world = 1  # the one-process full-batch step: no collective, no 1 / world average
        st.set_hyper_params(1.0)
        st.forward_backward(x[part].to(dev), [wt[part].to(dev) for wt in wts])
        st.optimizer_step() if sync else st._apply_update()
        res.append(((p0 - st.flat.params).cpu(), st.flat.buffers.cpu().clone(), [k for k in m.state_dict()]))
    (uf, bf, kf), (us, bs, ks) = res
    assert kf == ks, "state-dict keys changed by the conversion"
    assert l2rel(us, uf) < tol, ("update (lr 1: the gradient)", l2rel(us, uf))
    assert l2rel(bs, bf) < 1e-5, ("running statistics", l2rel(bs, bf))
    mine = [torch.zeros_like(us) for _ in range(dist.get_world_size())]
    dist.all_gather(mine, us)
    assert all(torch.equal(mine[0], t) for t in mine), "replicas diverged"


def _trainer_check(root, ckpt_dir):
    """Trainer.train() with the shipped YOLO-NAS recipe's sync_bn: True on every rank of the group (CPU stand-in backend)."""
    from super_gradients_b200.training import sg_trainer
    from super_gradients_b200.training.losses import PPYoloELoss
    from super_gradients_b200.training.models.detection_models.yolo_nas import YoloNAS

    fx = torch.load(os.path.join(root, "tests", "golden", "tiny_yolo_nas.pt"), weights_only=False)

    def build():
        ap = copy.deepcopy(fx["arch"])
        m = YoloNAS(backbone=ap["backbone"], neck=ap["neck"], heads=ap["heads"], num_classes=4, bn_eps=1e-3, bn_momentum=0.03, inplace_act=True, in_channels=3)
        m.load_state_dict({k: v.clone() for k, v in fx["sd0"].items()}, strict=False)
        return m

    rank = dist.get_rank()
    sg_trainer.setup_device = lambda device=None: torch.device("cpu")
    x = fx["x"] * (1.0 if rank == 0 else 0.9)  # each rank its own shard
    tp = dict(max_epochs=1, initial_lr=1e-3, lr_mode="cosine", cosine_final_lr_ratio=0.1, lr_warmup_steps=0, optimizer="SGD", optimizer_params={"momentum": 0.9, "weight_decay": 1e-5},
              zero_weight_decay_on_bias_and_bn=True, ema=True, ema_params={"decay": 0.99, "decay_type": "threshold"}, loss=PPYoloELoss(num_classes=4, use_static_assigner=False),
              save_model=True, sync_bn=True)  # fmt: skip
    model = build()
    keys = list(model.state_dict())
    tr = sg_trainer.Trainer("sync_bn", ckpt_root_dir=ckpt_dir)
    hist = tr.train(model, tp, [(x, fx["targets"])] * 2)
    assert all(torch.isfinite(torch.tensor(hist["train_loss"])))
    n_sync = sum(isinstance(m, nn.SyncBatchNorm) for m in tr.net.modules())
    assert n_sync > 20 and not any(type(m) is nn.BatchNorm2d for m in tr.net.modules()), n_sync
    assert list(tr.net.state_dict()) == keys, "state-dict keys changed by the conversion"
    for t in (tr.step.flat.params, tr.step.flat.buffers):
        both = [torch.zeros_like(t) for _ in range(dist.get_world_size())]
        dist.all_gather(both, t)
        assert all(torch.equal(both[0], b) for b in both), "replicas diverged"
    dist.barrier()
    if rank == 0:
        ck = torch.load(os.path.join(ckpt_dir, "sync_bn", "ckpt_latest.pth"), weights_only=False)
        build().load_state_dict(ck["net"])  # strict: a synced run's checkpoint loads into the unconverted model


def main(argv):
    root, dev, rows, cases = argv[0], argv[1], [int(r) for r in argv[2].split(",")], argv[3:]
    sys.path[:0] = [root, os.path.join(root, "tests")]
    backend = "nccl" if dev == "cuda-nccl" else "gloo"
    dev = "cuda" if dev.startswith("cuda") else dev
    if dev == "cuda":
        torch.cuda.set_device(int(os.environ["LOCAL_RANK"]) if backend == "nccl" else 0)
    dist.init_process_group(backend, init_method="env://")
    mp = None
    if dev == "cpu":
        from _pytest.monkeypatch import MonkeyPatch

        import cpu_backend_sync

        mp = MonkeyPatch()
        cpu_backend_sync.install(mp)
        tol_out, tol_grad = 1.0, 1e-2  # bf16 storage of every intermediate activation and gradient
    else:
        tol_out, tol_grad = 1.0, 2e-2
    try:
        for case in cases:
            if case == "tiny_yolo_nas_step":
                # percent-level bound: see the note in _update_check on the model's sensitivity to last-bit differences
                _update_check(root, rows, dev, 5e-2 if dev == "cpu" else 0.1)
            elif case.startswith("trainer:"):
                _trainer_check(root, case.split(":", 1)[1])
            else:
                run_block(case, rows, dev, tol_out, tol_grad)
            print("rank", dist.get_rank(), case, "ok", flush=True)
        dist.barrier()
    finally:
        dist.destroy_process_group()  # an orderly shutdown: a rank that exits while gloo's threads are alive can abort at exit


def launch(root, device, rows, cases, port, timeout=900):
    """Runs the worker on len(rows) ranks as direct child processes; returns (returncodes, combined output).  Every child is joined
    before returning, and killed and reaped on timeout."""
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), WORLD_SIZE=str(len(rows)), OMP_NUM_THREADS="2")
    procs = []
    try:
        for r in range(len(rows)):
            procs.append(subprocess.Popen([sys.executable, os.path.abspath(__file__), root, device, ",".join(map(str, rows)), *cases],
                                          env=dict(env, RANK=str(r), LOCAL_RANK=str(r)), stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))  # fmt: skip
        deadline = time.monotonic() + timeout
        outs = []
        for p in procs:
            outs.append(p.communicate(timeout=max(1.0, deadline - time.monotonic()))[0])
        return [p.returncode for p in procs], "\n".join(outs)
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
                p.wait()


if __name__ == "__main__":
    main(sys.argv[1:])
