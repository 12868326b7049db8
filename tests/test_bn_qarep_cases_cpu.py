"""CPU checks of tests/bn_qarep_cases.py: the fp64 oracles against torch's BatchNorm modules, the fp32 transcription of the
BatchNorm / QARepVGG passes within every bound, and each deliberate defect of the transcription outside at least one bound."""
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import bn_qarep_cases as B

SMS = 132
SHAPES = {2: (2, 1, 1), 105: (3, 5, 7), 4096: (4, 32, 32)}


def _nchw(t, n, h, w):
    return t.view(n, h, w, -1).permute(0, 3, 1, 2)


@pytest.mark.parametrize("C", [8, 48])
@pytest.mark.parametrize("M", [2, 105, 4096])
@pytest.mark.parametrize("variant", ["plain", "residual", "droppath"])
def test_bn_oracle_matches_torch_batchnorm(C, M, variant):
    n, h, w = SHAPES[M]
    g = torch.Generator().manual_seed(M * 7 + C)
    x = B.channel_data(M, C, g, offsets=(0.0, 4.0), constant=False)
    gamma, beta = torch.randn(C, generator=g, dtype=torch.float64), torch.randn(C, generator=g, dtype=torch.float64)
    rm, rv = torch.randn(C, generator=g, dtype=torch.float64), torch.rand(C, generator=g, dtype=torch.float64) + 0.5
    res = B.round_bf16(torch.randn(M, C, generator=g, dtype=torch.float64)) if variant != "plain" else None
    ss_img = torch.tensor([0.0 if i % 3 == 0 else 1.25 for i in range(n)], dtype=torch.float64) if variant == "droppath" else None
    ss = ss_img.repeat_interleave(h * w).view(-1, 1) if ss_img is not None else None
    dy = B.round_bf16(torch.randn(M, C, generator=g, dtype=torch.float64))
    ref = B.bn_train_ref(x, gamma, beta, rm, rv, 1e-3, 0.03, "relu", res, ss, dy)
    bn = nn.BatchNorm2d(C, eps=1e-3, momentum=0.03).double().train()
    with torch.no_grad():
        bn.weight.copy_(gamma), bn.bias.copy_(beta), bn.running_mean.copy_(rm), bn.running_var.copy_(rv)
    xt = _nchw(x, n, h, w).clone().requires_grad_(True)
    rt = _nchw(res, n, h, w).clone().requires_grad_(True) if res is not None else None
    z = bn(xt)
    if ss_img is not None:
        z = z * ss_img.view(-1, 1, 1, 1)
    if rt is not None:
        z = z + rt
    y = F.relu(z)
    y.backward(_nchw(dy, n, h, w))
    tc = lambda a, b: torch.testing.assert_close(a, b, rtol=1e-10, atol=1e-10)  # noqa: E731
    tc(ref["y"], B.mc(y))
    tc(ref["rm"], bn.running_mean)
    tc(ref["rv"], bn.running_var)
    tc(ref["dx"], B.mc(xt.grad))
    tc(ref["dgamma"], bn.weight.grad)
    tc(ref["dbeta"], bn.bias.grad)
    if rt is not None:
        tc(ref["dres"], B.mc(rt.grad))


@pytest.mark.parametrize("C", [8, 48])
@pytest.mark.parametrize("M", [2, 105, 4096])
@pytest.mark.parametrize("post", [True, False])
def test_qarep_oracle_matches_two_batchnorms(C, M, post):
    n, h, w = SHAPES[M]
    g = torch.Generator().manual_seed(M + C)
    y3, u = B.channel_data(M, C, g, constant=False), B.round_bf16(torch.randn(M, C, generator=g, dtype=torch.float64))
    p = [torch.randn(C, generator=g, dtype=torch.float64) for _ in range(5)]
    rs = [torch.zeros(C, dtype=torch.float64), torch.ones(C, dtype=torch.float64)] * 2
    dout = B.round_bf16(torch.randn(M, C, generator=g, dtype=torch.float64))
    ref = B.qarep_train_ref(y3, u, *p, *rs, 1e-3, 1e-5, 0.1, "relu", post, dout=dout)
    bn3, bnp = nn.BatchNorm2d(C, eps=1e-3, momentum=0.1).double(), nn.BatchNorm2d(C, eps=1e-5, momentum=0.1).double()
    with torch.no_grad():
        bn3.weight.copy_(p[0]), bn3.bias.copy_(p[1]), bnp.weight.copy_(p[3]), bnp.bias.copy_(p[4])
    ab = p[2].clone().requires_grad_(True)
    a, b = _nchw(y3, n, h, w).clone().requires_grad_(True), _nchw(u, n, h, w).clone().requires_grad_(True)
    z = bn3(a) + b + ab.view(1, -1, 1, 1)
    o = F.relu(bnp(z) if post else z)
    o.backward(_nchw(dout, n, h, w))
    tc = lambda x, y: torch.testing.assert_close(x, y, rtol=1e-9, atol=1e-9)  # noqa: E731
    tc(ref["o"], B.mc(o))
    tc(ref["dy3"], B.mc(a.grad))
    tc(ref["du"], B.mc(b.grad))
    tc(ref["dgamma3"], bn3.weight.grad)
    tc(ref["rm3"], bn3.running_mean)
    tc(ref["rv3"], bn3.running_var)
    if post:
        tc(ref["dgamma_p"], bnp.weight.grad)
        tc(ref["dbeta_p"], bnp.bias.grad)
        tc(ref["rmp"], bnp.running_mean)
        tc(ref["rvp"], bnp.running_var)
        # post-BN removes every per-channel constant: the first BatchNorm's bias and the 1x1 bias get no gradient
        assert float(ref["autograd_dbeta3"].abs().max()) < 1e-9 * (1 + float(dout.abs().sum()))
        assert float(ref["autograd_dab"].abs().max()) < 1e-9 * (1 + float(dout.abs().sum()))
        assert not ref["dbeta3"].any() and not ref["dab"].any()
    else:
        tc(ref["dbeta3"], bn3.bias.grad)
        tc(ref["dab"], ab.grad)
    # the coefficient rows restate the same block
    c = ref["coef"]
    pre = c[4] * y3 + c[5] * u + c[6]
    tc(pre, ref["pre"])


# ------------------------------------------------------------------------------------------------ transcription against the bounds
def bn_case(M, C, seed, act="relu", residual=False, droppath=False, stats_repl=0, read_y=False, shards=1, no_beta=False, mut=None):
    """One BatchNorm forward + backward through the transcription, checked by verify_bn (raises on a bound violation)."""
    g = torch.Generator().manual_seed(seed)
    sizes = [M] if shards == 1 else [M, M // 2 + 8]
    xs = [B.channel_data(m, C, g, constant=not no_beta) for m in sizes]  # a constant channel with beta = 0: the ReLU mask is rounding noise
    gamma = (torch.randn(C, generator=g) * 0.8 + 0.4).float()
    gamma[0] = 0.0  # with beta[0] = 0: every pre-activation of channel 0 is exactly 0 (ties at the ReLU)
    beta = (torch.randn(C, generator=g) * 0.3).float()
    beta[0] = 0.0
    if no_beta:
        beta = None
    rm, rv = torch.randn(C, generator=g).float(), (torch.rand(C, generator=g) + 0.5).float()
    eps, mom = B.f32(1e-3), B.f32(0.07)
    res = [B.round_bf16(torch.randn(m, C, generator=g, dtype=torch.float64)) for m in sizes] if residual else None
    ss = None
    if droppath:
        hw = 3
        ss = []
        for m in sizes:
            img = torch.tensor([0.0 if i % 3 == 1 else B.f32(1 / 0.8) for i in range(m // hw)], dtype=torch.float64)
            ss.append(img.repeat_interleave(hw).view(-1, 1))
    dys = [B.round_bf16(torch.randn(m, C, generator=g, dtype=torch.float64)) for m in sizes]
    Mt = sum(sizes)
    ps = 0.5 if shards > 1 else 1.0
    if shards > 1:  # statistics: every shard's sums added (the all-reduce), then each shard's apply pass
        S = sum(B.chan_sums_t(torch.stack([x, x * x], -1), B.launch_grid(x.shape[0], SMS)) for x in xs).unsqueeze(0)
        fw = [B.bn_fwd_t(x, gamma, beta, rm, rv, eps, mom, act, r, s, stats=S, M_global=Mt, mut=mut) for x, r, s in zip(xs, res or [None] * 2, ss or [None] * 2)]
    else:
        stats = B.split_stats(xs[0], stats_repl, g) if stats_repl else None
        fw = [B.bn_fwd_t(xs[0], gamma, beta, rm, rv, eps, mom, act, res[0] if res else None, ss[0] if ss else None, stats=stats,
                         grid=B.launch_grid(M, SMS), mut=mut)]
    f0 = fw[0]
    dg0, db0 = torch.randn(C, generator=g).float(), torch.randn(C, generator=g).float()
    bw = B.bn_bwd_t([(x, dy, f["y"]) for x, dy, f in zip(xs, dys, fw)], gamma, beta, f0["mean"], f0["rstd"], act,
                    [B.launch_grid(m, SMS) for m in sizes], Mt, ss, read_y or residual or droppath or no_beta, dg0, db0, ps, mut=mut)
    inp = {"x": xs, "residual": res, "ss": ss, "dy": dys, "gamma": gamma, "beta": beta, "rm": rm, "rv": rv, "eps": eps, "mom": mom, "act": act,
           "ps": ps, "dgamma0": dg0, "dbeta0": db0, "stats_exact": bool(stats_repl), "read_y": read_y or residual or droppath or no_beta,
           "sum_extra": 1 if shards > 1 else 0}
    got = {"y": [f["y"] for f in fw], "mean": f0["mean"], "rstd": f0["rstd"], "rm": f0["rm"], "rv": f0["rv"], "dx": bw["dx"],
           "dres": bw["dres"] if residual else None, "dgamma": bw["dgamma"], "dbeta": bw["dbeta"]}
    return B.verify_bn(inp, got, SMS)


def qarep_case(M, C, seed, act="relu", post=True, residual=False, no_ab=False, shards=1, mut=None):
    g = torch.Generator().manual_seed(seed)
    sizes = [M] if shards == 1 else [M, M // 2 + 8]
    y3s = [B.channel_data(m, C, g) for m in sizes]
    us = [B.round_bf16(0.6 * y - 0.6 * y.mean(0) + torch.randn(m, C, generator=g, dtype=torch.float64) + 0.5) for y, m in zip(y3s, sizes)]
    gamma3 = (torch.randn(C, generator=g) * 0.8 + 0.2).float()
    beta3, ab = (torch.randn(C, generator=g) * 0.3).float(), None if no_ab else (torch.randn(C, generator=g) * 0.3).float()
    gp, bp = (torch.randn(C, generator=g) * 0.8 + 0.2).float(), (torch.randn(C, generator=g) * 0.3).float()
    gp[0], bp[0] = 0.0, 0.0  # channel 0: pre-activations exactly 0
    rs = [torch.randn(C, generator=g).float(), (torch.rand(C, generator=g) + 0.5).float(), torch.randn(C, generator=g).float(), (torch.rand(C, generator=g) + 0.5).float()]
    eps3, epsp, mom = B.f32(1e-3), B.f32(1e-5), B.f32(0.07)
    res = [B.round_bf16(torch.randn(m, C, generator=g, dtype=torch.float64)) for m in sizes] if residual else None
    alpha = B.f32(0.7) if residual else None
    # dout partly follows the output, so the backward sums are not all near zero
    douts = [B.round_bf16(0.5 * torch.tanh(y) + torch.randn(m, C, generator=g, dtype=torch.float64)) for y, m in zip(y3s, sizes)]
    acc0 = [torch.randn(C, generator=g).float() for _ in range(5)]
    ps = 0.5 if shards > 1 else 1.0
    Mt = sum(sizes)
    args = (gamma3, beta3, ab, gp if post else None, bp if post else None, *rs, eps3, epsp, mom, act, post)
    if shards > 1:
        y3c, uc = torch.cat(y3s), torch.cat(us)
        grid = B.launch_grid(Mt, SMS)  # sums of the concatenation stand in for the all-reduced shard sums
        fw = B.qarep_fwd_t(y3c, uc, *args, grid, torch.cat(res) if res else None, alpha, mut=mut)
        own = [B.qarep_bwd_t(y3s[i], us[i], douts[i], fw["coef"], gp, act, post, B.launch_grid(sizes[i], SMS), M_global=Mt)["sums"] for i in (0, 1)]
        bw_b = B.qarep_bwd_t(y3s[1], us[1], douts[1], fw["coef"], gp, act, post, B.launch_grid(sizes[1], SMS), param_scale=ps, M_global=Mt, extra_sums=own[0], mut=mut)
        bw = B.qarep_bwd_t(y3s[0], us[0], douts[0], fw["coef"], gp, act, post, B.launch_grid(sizes[0], SMS), acc0, ps, Mt, own[1], mut=mut)
        outs, dy3, du = [fw["out"]], [bw["dy3"], bw_b["dy3"]], [bw["du"], bw_b["du"]]
        shards_in = [torch.cat(y3s)], [torch.cat(us)]
    else:
        fw = B.qarep_fwd_t(y3s[0], us[0], *args, B.launch_grid(M, SMS), res[0] if res else None, alpha, mut=mut)
        bw = B.qarep_bwd_t(y3s[0], us[0], douts[0], fw["coef"], gp, act, post, B.launch_grid(M, SMS), acc0, mut=mut)
        outs, dy3, du = [fw["out"]], [bw["dy3"]], [bw["du"]]
        shards_in = y3s, us
    inp = {"y3": shards_in[0], "u": shards_in[1], "dout": douts if shards == 1 else [torch.cat(douts)], "residual": res if shards == 1 or not res else [torch.cat(res)],
           "gamma3": gamma3, "beta3": beta3, "ab": ab, "gamma_p": gp if post else None, "beta_p": bp if post else None, "rm3": rs[0], "rv3": rs[1],
           "rmp": rs[2], "rvp": rs[3], "eps3": eps3, "eps_post": epsp, "mom": mom, "act": act, "use_post_bn": post, "res_alpha": alpha, "acc0": acc0, "ps": ps}
    got = {"out": outs, "coef": fw["coef"], "rm3": fw["rm3"], "rv3": fw["rv3"], "rmp": fw["rmp"], "rvp": fw["rvp"], "dy3": [torch.cat(dy3)], "du": [torch.cat(du)], "acc": bw["acc"]}
    return B.verify_qarep(inp, got, SMS)


BN_CASES = {
    "fused_relu": dict(M=4096, C=48),
    "epilogue_stats": dict(M=105, C=24, stats_repl=8),
    "read_y": dict(M=105, C=64, read_y=True),
    "residual": dict(M=4096, C=24, residual=True),
    "droppath": dict(M=4095, C=8, droppath=True, residual=True),
    "no_beta_none": dict(M=105, C=64, act="none", no_beta=True),
    "no_beta_relu": dict(M=3200, C=8, no_beta=True),
    "two_pixels": dict(M=2, C=8),
    "sync": dict(M=600, C=24, shards=2),
    "wide": dict(M=40, C=2560),
    # recorded shapes (YOLO-NAS-S at 2 x 640^2, ResNet-50 at 2 x 224^2)
    "yolo_80x80x96": dict(M=12800, C=96),
    "resnet_7x7x2048": dict(M=98, C=2048, residual=True),
}
QAREP_CASES = {
    "post": dict(M=4096, C=24),
    "no_post": dict(M=105, C=64, post=False),
    "shortcut": dict(M=105, C=8, residual=True),
    "no_ab_none": dict(M=2, C=8, act="none", no_ab=True),
    "sync": dict(M=600, C=24, shards=2),
    "yolo_40x40x64": dict(M=3200, C=64),
}


@pytest.mark.parametrize("name", list(BN_CASES))
def test_bn_transcription_within_bounds(name):
    rep = bn_case(seed=sum(map(ord, name)), **BN_CASES[name])
    assert rep["dx"] <= 1.0


@pytest.mark.parametrize("name", list(QAREP_CASES))
def test_qarep_transcription_within_bounds(name):
    rep = qarep_case(seed=sum(map(ord, name)), **QAREP_CASES[name])
    assert rep["dy3"] <= 1.0


# each defect, and the case that must expose it
MUTATION_CASES = {
    "biased_rv": ("bn", dict(M=105, C=24)),
    "eps_post_first": ("qarep", dict(M=105, C=24)),
    "cov_half": ("qarep", dict(M=105, C=24)),
    "q_no_czy": ("qarep", dict(M=105, C=24)),
    "ps_one": ("bn", dict(M=600, C=24, shards=2)),
    "dres_scaled": ("bn", dict(M=4095, C=8, droppath=True, residual=True)),
    "repl0": ("bn", dict(M=105, C=24, stats_repl=8)),
    "ss_after_res": ("bn", dict(M=4095, C=8, droppath=True, residual=True)),
}


def test_mutation_list_is_complete():
    assert set(MUTATION_CASES) == set(B.MUTATIONS)


@pytest.mark.parametrize("mut", list(MUTATION_CASES))
def test_transcription_mutation_breaks_a_bound(mut):
    fam, kw = MUTATION_CASES[mut]
    run = bn_case if fam == "bn" else qarep_case
    run(seed=5, **kw)  # the correct transcription passes
    with pytest.raises(AssertionError):
        run(seed=5, mut=mut, **kw)


def test_qarep_sync_mutation_ps():
    qarep_case(M=600, C=24, seed=3, shards=2)
    with pytest.raises(AssertionError):
        qarep_case(M=600, C=24, seed=3, shards=2, mut="ps_one")


def test_chain_len_launch_formula():
    # one CTA of 256 pixels, C = 8: one channel vector, 256 lanes, one pixel each
    assert B.chain_len(256, 8, 132) == 1 + 256
    # C = 2048: 256 vectors, one lane; grid capped at the SM count
    assert B.chain_len(2 * 224 * 224, 2048, 132) == -(-2 * 224 * 224 // 132) + 1
    assert B.chain_len(2 * 224 * 224, 2048, 114) > B.chain_len(2 * 224 * 224, 2048, 132)
