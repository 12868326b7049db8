"""SGD and AdamW through FlatOptimizer on the sm_90a kernels: TrainStep's update (clip_grad_norm, optimizer, EMA), eagerly and
replayed from a captured CUDA graph, bit-identical to the same launches issued by hand with the rows TrainStep.set_hyper_params
built before SGD and AdamW joined FlatOptimizer."""
import pytest
import torch

from optimizer_cases import LRS, seeded_grad, tiny_model
from test_sgd_adamw_cpu import old_op, old_rows

pytestmark = pytest.mark.gpu
DEV = "cuda"
CASES = {"sgd_momentum": ("SGD", {"momentum": 0.9, "weight_decay": 1e-4}), "sgd_no_momentum": ("SGD", {"momentum": 0.0}),
         "sgd_nesterov": ("SGD", {"nesterov": True}), "adamw": ("AdamW", {"weight_decay": 5e-2, "betas": (0.8, 0.95), "eps": 1e-6})}  # fmt: skip
MAX_NORM, DECAY, STEPS = 1.0, 0.9, 3


def _train_step(name, params):
    from super_gradients_b200.training.losses import PPYoloELoss
    from super_gradients_b200.training.sg_trainer import TrainStep

    return TrainStep(tiny_model().to(DEV).train(), PPYoloELoss(num_classes=4, use_static_assigner=False), name, params, zero_wd_on_bias_and_bn=True, ema=True,
                     clip_grad_norm=MAX_NORM)  # fmt: skip


def _by_hand(name, params, st):
    """STEPS updates of st's initial parameters through the kernel wrappers, rows from the old formula."""
    from super_gradients_b200 import kernels as K

    f = st.flat
    p, ema, ema_buf = f.params.clone(), f.params.clone(), f.buffers.clone()
    state = [torch.zeros_like(p) for _ in range(1 if name == "SGD" else 2)]
    partials = torch.zeros(f.chunks.shape[0], dtype=torch.float64, device=DEV)
    coef = torch.zeros(2, dtype=torch.float32, device=DEV)
    decay = torch.tensor([DECAY], dtype=torch.float32, device=DEV)
    for t in range(1, STEPS + 1):
        g = seeded_grad(f.n_live, t, 11, 1.0).to(DEV)
        hp = old_rows(name, old_op(name, params), LRS[t - 1], t, 1.0).to(DEV)
        K.clip_grad_norm(g, f.chunks, hp, 3 if name == "SGD" else 7, MAX_NORM, partials, coef)
        for a, b, row in ((0, f.n_decay, 0), (f.n_decay, f.n_live, 1)):
            if name == "SGD":
                K.sgd_step(p[a:b], g[a:b], state[0][a:b], hp[row])
            else:
                K.adamw_step(p[a:b], g[a:b], state[0][a:b], state[1][a:b], hp[row])
        K.ema_update(ema, p, decay)
        K.ema_update(ema_buf, f.buffers, decay)
    torch.cuda.synchronize()
    return [p, *state, ema, ema_buf, coef]


@pytest.mark.parametrize("case", CASES)
def test_update_matches_the_launches_by_hand(case):
    name, params = CASES[case]
    eager, graphed = _train_step(name, params), _train_step(name, params)
    graphed.set_hyper_params(LRS[0], DECAY)
    graph, _ = graphed._capture_region(graphed._apply_update)  # recorded, not run
    want = _by_hand(name, params, eager)
    for t in range(1, STEPS + 1):
        g = seeded_grad(eager.flat.n_live, t, 11, 1.0).to(DEV)
        for st in (eager, graphed):
            st.flat.grads.copy_(g)
            st.set_hyper_params(LRS[t - 1], DECAY)
        eager._apply_update()
        graph.replay()
        eager.opt_steps += 1
        graphed.opt_steps += 1
    torch.cuda.synchronize()
    assert 0 < float(want[-1][1]) < 1  # the clip acted
    for st, how in ((eager, "eager"), (graphed, "graph")):
        got = [st.flat.params, *st.state, st.ema_params, st.ema_buffers, st.clip_norm_coef]
        assert len(got) == len(want)
        for i, (x, y) in enumerate(zip(got, want)):
            assert torch.equal(x, y), (case, how, i, int((x != y).sum()))
