"""Adam, RMSprop, RMSpropTF, Lion and Lamb on the sm_90a kernels (csrc/optim.cu): every case of the unmodified reference's goldens
(tests/golden/optimizers.pt, bounds in optimizer_cases.assert_matches), the kernels against the host build of their own header,
CUDA-graph replay against eager launches, Lamb's run-to-run reproducibility, a resume through the checkpoint's optimizer state,
and Trainer.train() of the tiny YOLO-NAS."""
import types

import pytest
import torch

import host_optim
from optimizer_cases import CASES, LRS, assert_matches, replay, seeded_grad, tiny_model

from super_gradients_b200.training import fused_optimizers as FO
from super_gradients_b200.training.flat_state import FlatState

pytestmark = pytest.mark.gpu
DEV = "cuda"
NAMES = {"Adam": {}, "RMSprop": {"centered": True}, "RMSpropTF": {"centered": True}, "Lion": {"weight_decay": 0.1}, "Lamb": {"weight_decay": 0.01, "always_adapt": True}}


@pytest.mark.parametrize("case", CASES)
def test_kernels_replay_the_reference(case, golden):
    want = golden("optimizers")["cases"][case]
    for step, got, ref, before, _flat in replay(case, want, DEV):
        assert_matches(case, got, ref, before, step)


def _flat_pair(case):
    """The tiny model's flat buffers twice: on the device and on the host, with one optimizer each."""
    name, params, zero_wd, scale = CASES[case]
    out = []
    for dev in (DEV, "cpu"):
        model = tiny_model().to(dev)
        flat = FlatState(model, zero_wd)
        op, wd = FO.resolve(name, params, zero_wd)
        out.append((flat, FO.FlatOptimizer(name, op, wd, flat)))
    return out


@pytest.mark.parametrize("case", CASES)
def test_kernels_match_their_host_build(case, monkeypatch):
    """The whole flat buffer for four steps: bit-identical to the g++ build of optim_math.cuh (both sqrt are correctly rounded).
    Lamb's sums are float64 in another order on the host; rounded to float32 they agree to 1e-6."""
    (fd, od), (fh, oh) = _flat_pair(case)
    name, scale = CASES[case][0], CASES[case][3]
    for t in range(1, 5):
        g = seeded_grad(fd.n_live, t, 7, scale)
        fd.grads.copy_(g)
        fh.grads.copy_(g)
        od.step(fd, torch.tensor(od.rows(LRS[t - 1], t, 1.0), device=DEV))
        with monkeypatch.context() as mp:
            host_optim.install(mp)
            oh.step(fh, torch.tensor(oh.rows(LRS[t - 1], t, 1.0)))
        for a, b in zip((fd.params, *od.state), (fh.params, *oh.state)):
            if name == "Lamb":
                torch.testing.assert_close(a.cpu(), b, rtol=1e-6, atol=1e-9)
            else:
                assert torch.equal(a.cpu(), b), (case, t, int((a.cpu() != b).sum()))


def _train_step(name, params):
    from super_gradients_b200.training.losses import PPYoloELoss
    from super_gradients_b200.training.sg_trainer import TrainStep

    return TrainStep(tiny_model().to(DEV).train(), PPYoloELoss(num_classes=4, use_static_assigner=False), name, params, zero_wd_on_bias_and_bn=True, ema=True)


@pytest.mark.parametrize("name", NAMES)
def test_graph_replay_is_bit_identical_to_eager(name):
    """TrainStep's optimizer + EMA region (the part after the all-reduce) captured in a CUDA graph and replayed with a new learning
    rate every step, against the same launches issued eagerly, on the same gradients."""
    sa, sb = _train_step(name, NAMES[name]), _train_step(name, NAMES[name])
    sb.set_hyper_params(LRS[0], 0.9)
    graph, _ = sb._capture_region(sb._apply_update)  # recorded, not run: both twins still hold the initial state
    assert torch.equal(sa.flat.params, sb.flat.params)
    for i in range(len(LRS)):
        g = seeded_grad(sa.flat.n_live, i + 1, 3, 1.0).to(DEV)
        for st in (sa, sb):
            st.set_hyper_params(LRS[i], 0.9)
            st.flat.grads.copy_(g)
        sa._apply_update()
        graph.replay()
        sa.opt_steps += 1
        sb.opt_steps += 1
        torch.cuda.synchronize()
        assert torch.equal(sa.flat.params, sb.flat.params), (name, i)
        assert all(torch.equal(a, b) for a, b in zip(sa.state, sb.state)) and torch.equal(sa.ema_params, sb.ema_params), (name, i)


@pytest.mark.parametrize("name", NAMES)
def test_captured_train_step_follows_eager(name, golden):
    """The whole train step (forward, loss, backward, optimizer, EMA) captured: it trains like the eager step (the forward and
    backward kernels add in a run-dependent order, so the comparison is close, not bitwise).  The learning rates keep each
    parameter's step near 1e-3: RMSprop's first steps are about 10 lr in every element, whatever the gradient's size, so a
    noise-level gradient turns into a full step of either sign."""
    lr = 1e-4 if name == "RMSprop" else 1e-3
    from super_gradients_b200.training.losses import pad_targets_host

    g = golden("tiny_yolo_nas")
    gb, gl, gv = pad_targets_host(g["targets"], g["x"].shape[0], 16)
    x, t = g["x"].to(DEV), (gb.to(DEV), gl.to(DEV), gv.to(DEV))
    sa, sb = _train_step(name, NAMES[name]), _train_step(name, NAMES[name])
    sb.set_hyper_params(lr, 0.9)
    sb.capture(x, t, warmup=2)
    assert torch.equal(sa.flat.params, sb.flat.params) and all(torch.equal(a, b) for a, b in zip(sa.state, sb.state))
    for _ in range(3):
        for st in (sa, sb):
            st.set_hyper_params(lr, 0.9)
            st.run(x, t)
    d = float((sa.flat.params - sb.flat.params).norm() / sa.flat.params.norm())
    assert d < 1e-3, d


def test_lamb_is_bit_identical_across_runs():
    """Two runs of three Lamb steps over 6.3 M parameters in 40 tensors (chunks of every size) give the same bits."""
    sizes = [1, 7, 16384, 16385, 3 * 16384 + 5] + [int(x) for x in torch.randint(1, 400000, (35,), generator=torch.Generator().manual_seed(1))]
    runs = []
    for _ in range(2):
        model = torch.nn.ParameterList([torch.nn.Parameter(seeded_grad(k, 0, i, 2.0)) for i, k in enumerate(sizes)]).to(DEV)
        flat = FlatState(model, False)
        flat.n_decay = sum(sizes[:20])  # two weight-decay ranges
        op, wd = FO.resolve("Lamb", {"weight_decay": 0.01}, True)
        opt = FO.FlatOptimizer("Lamb", op, wd, flat)
        for t in range(1, 4):
            flat.grads.copy_(seeded_grad(flat.n_live, t, 99, 1.0))
            opt.step(flat, torch.tensor(opt.rows(1e-2, t, 0.5), device=DEV))
        runs.append([flat.params.clone(), *[s.clone() for s in opt.state], opt.partials.clone()])
    assert all(torch.equal(a, b) for a, b in zip(*runs))


@pytest.mark.parametrize("name", NAMES)
def test_resume_continues_exactly(name):
    """Four steps straight against two steps, a checkpoint's optimizer_state_dict restored into a fresh TrainStep, two more steps."""
    from super_gradients_b200.training.sg_trainer import Trainer

    def run(st, steps):
        for t in steps:
            st.set_hyper_params(LRS[t - 1])
            st.flat.grads.copy_(seeded_grad(st.flat.n_live, t, 5, 1.0))
            st._apply_update()
            st.opt_steps += 1

    a = _train_step(name, NAMES[name])
    run(a, range(1, 5))
    b = _train_step(name, NAMES[name])
    run(b, range(1, 3))
    ckpt = {"optimizer_state_dict": {"name": b.opt_name, "flat_order": [n for n, _ in b.flat.order], "state": [s.cpu() for s in b.state], "opt_steps": b.opt_steps}}
    c = _train_step(name, NAMES[name])
    c.flat.params.copy_(b.flat.params)
    Trainer._restore_training_state(types.SimpleNamespace(step=c), ckpt)
    assert c.opt_steps == 2
    run(c, range(3, 5))
    assert torch.equal(a.flat.params, c.flat.params) and all(torch.equal(x, y) for x, y in zip(a.state, c.state))


@pytest.mark.parametrize("name", ["Adam", "Lamb"])
def test_trainer_tiny_yolo_nas(name, golden, tmp_path):
    from super_gradients_b200.training.losses import PPYoloELoss
    from super_gradients_b200.training.sg_trainer import Trainer

    g = golden("tiny_yolo_nas")
    params = {"Adam": {}, "Lamb": {"weight_decay": 0.01}}[name]
    tp = {"max_epochs": 6, "initial_lr": {"Adam": 2e-3, "Lamb": 2e-2}[name], "lr_mode": "constant", "optimizer": name, "optimizer_params": params, "zero_weight_decay_on_bias_and_bn": True, "ema": True,
          "loss": PPYoloELoss(num_classes=4, use_static_assigner=False)}  # fmt: skip
    hist = Trainer(f"tiny_{name}", ckpt_root_dir=str(tmp_path)).train(tiny_model(), tp, [(g["x"], g["targets"])] * 2)
    losses = hist["train_loss"]
    assert all(torch.isfinite(torch.tensor(losses))) and losses[-1] < losses[0], losses
