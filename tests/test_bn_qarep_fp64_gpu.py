"""The BatchNorm and QARepVGG train / inference kernels (csrc/bn_kernels.cu) on every launch path against the fp64 oracles of
tests/bn_qarep_cases.py, with the error bounds derived there from the kernels' arithmetic, plus the checks that need no tolerance:
the mask recomputed from x equals the mask read from y, the fused shortcut equals the shortcut pass it replaced, accumulators
receive exactly their increment, and the post-BN block leaves the first BatchNorm's bias gradients untouched."""
import pytest
import torch

import bn_qarep_cases as B

pytestmark = pytest.mark.gpu

DEV = "cuda"


def K():
    from super_gradients_b200 import kernels

    return kernels


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def dev_nhwc(m, n, h, w, pitch=None, off=0):
    """fp64 [M, C] holding bf16 values -> CUDA bf16 NHWC [n, C, h, w] view, a channel slice [off, off + C) of a `pitch`-wide buffer."""
    C = m.shape[1]
    pitch = pitch or C
    buf = torch.full((n, h, w, pitch), -7.0, dtype=torch.bfloat16, device=DEV)
    buf[..., off : off + C] = m.view(n, h, w, C).to(DEV).bfloat16()
    return buf.permute(0, 3, 1, 2)[:, off : off + C]


class TwoRankSync:
    """Duck-typed functional.BnSync of rank A of two ranks on one GPU: every sync(buffer) call records the buffer as this rank made it
    and adds the other rank's buffer of the same call (captured by an earlier run of that rank)."""

    def __init__(self, other=None):
        self.param_scale, self.count, self.other, self.seen = 0.5, None, other, []

    def __call__(self, buf):
        self.seen.append(buf.clone())
        if self.other is not None:
            buf += self.other[len(self.seen) - 1]


def _shape(M):
    return {2: (2, 1, 1), 105: (3, 5, 7), 40: (2, 4, 5), 98: (2, 7, 7)}.get(M) or (M // 1600, 40, 40)


# ------------------------------------------------------------------------------------------------ BatchNorm
def run_bn(M, C, seed, act="relu", residual=False, droppath=False, stats_repl=0, x_slice=False, dy_slice=False, dy2=False, no_beta=False,
           want_res=None, mom=0.07):
    k = K()
    n, h, w = _shape(M)
    g = torch.Generator().manual_seed(seed)
    x = B.channel_data(M, C, g, constant=not no_beta)  # a constant channel with beta = 0 leaves the ReLU mask to rounding noise
    gamma = (torch.randn(C, generator=g) * 0.8 + 0.4).float()
    gamma[0] = 0.0  # with beta[0] = 0 every pre-activation of channel 0 is exactly 0: ReLU ties
    beta = (torch.randn(C, generator=g) * 0.3).float()
    beta[0] = 0.0
    if no_beta:
        beta = None
    rm, rv = torch.randn(C, generator=g).float(), (torch.rand(C, generator=g) + 0.5).float()
    eps, momf = B.f32(1e-3), B.f32(mom)
    res = B.round_bf16(torch.randn(M, C, generator=g, dtype=torch.float64)) if residual else None
    ss_img = torch.tensor([0.0 if i % 3 == 1 else 1 / 0.8 for i in range(n)], dtype=torch.float32) if droppath else None
    dy = B.round_bf16(torch.randn(M, C, generator=g, dtype=torch.float64))
    dg0, db0 = torch.randn(C, generator=g).float(), torch.randn(C, generator=g).float()
    xg = dev_nhwc(x, n, h, w, C + 16 if x_slice else None, 8 if x_slice else 0)
    resg = dev_nhwc(res, n, h, w) if residual else None
    ssg = ss_img.to(DEV) if droppath else None
    stats = B.split_stats(x, stats_repl, g).to(DEV) if stats_repl else None
    cu = lambda t: None if t is None else t.to(DEV)  # noqa: E731
    rmg, rvg = rm.clone().to(DEV), rv.clone().to(DEV)
    y, mean, rstd = k.bn_act_fwd(xg, stats, cu(gamma), cu(beta), rmg, rvg, eps, momf, act, resg, sample_scale=ssg)
    want_res = residual if want_res is None else want_res
    kw = {}
    if dy2:
        sp = (C // 2) // 8 * 8
        kw["dy2"] = dev_nhwc(dy[:, sp:].contiguous(), n, h, w, C - sp + 8, 8)
        dyg = dev_nhwc(dy[:, :sp].contiguous(), n, h, w)
    else:
        dyg = dev_nhwc(dy, n, h, w, C + 24 if dy_slice else None, 16 if dy_slice else 0)
    dgg, dbg = dg0.clone().to(DEV), db0.clone().to(DEV)
    dx, dres, dgo, dbo = k.bn_act_bwd(dyg, xg, y, cu(gamma), mean, rstd, eps, act, want_residual_grad=want_res, dgamma=dgg, dbeta=dbg, beta=cu(beta), sample_scale=ssg, **kw)
    ss = ss_img.double().repeat_interleave(h * w).view(-1, 1).to(DEV) if droppath else None
    inp = {"x": [x.to(DEV)], "residual": [res.to(DEV)] if residual else None, "ss": [ss] if droppath else None, "dy": [dy.to(DEV)], "gamma": gamma, "beta": beta,
           "rm": rm, "rv": rv, "eps": eps, "mom": momf, "act": act, "dgamma0": dg0, "dbeta0": db0, "stats_exact": bool(stats_repl),
           "read_y": want_res or no_beta or droppath}
    got = {"y": [B.mc(y)], "mean": mean, "rstd": rstd, "rm": rmg, "rv": rvg, "dx": [B.mc(dx)], "dres": [B.mc(dres)] if want_res else None, "dgamma": dgo, "dbeta": dbo}
    rep = B.verify_bn(inp, got, sms())
    return rep, locals()


BN_MATRIX = {
    # name: kwargs
    "epilogue_stats_repl8": dict(M=105, C=24, stats_repl=8),
    "fused_stats_C8_M2": dict(M=2, C=8),
    "fused_stats_C64_big": dict(M=51200, C=64),
    "fused_C2048": dict(M=98, C=2048, residual=True),
    "fused_C2560": dict(M=40, C=2560, stats_repl=8),
    "x_slice_split_bwd": dict(M=105, C=24, x_slice=True),
    "dy_concat_slice": dict(M=3200, C=64, dy_slice=True),
    "dy2_two_sources": dict(M=105, C=48, dy2=True),
    "droppath_residual": dict(M=3200, C=24, droppath=True, residual=True),
    "residual_grad": dict(M=105, C=64, residual=True),
    "act_none_no_beta": dict(M=105, C=24, act="none", no_beta=True),
    "relu_no_beta": dict(M=3200, C=8, no_beta=True),
}


@pytest.mark.parametrize("name", list(BN_MATRIX))
def test_bn_train_against_fp64(name):
    rep, _ = run_bn(seed=sum(map(ord, name)), **BN_MATRIX[name])
    print(name, {k: round(v, 3) for k, v in rep.items()})


@pytest.mark.parametrize("C,M", [(8, 105), (24, 3200), (2560, 40)])
@pytest.mark.parametrize("residual", [False, True])
def test_bn_infer_against_fp64(C, M, residual):
    k = K()
    n, h, w = _shape(M)
    g = torch.Generator().manual_seed(C + M)
    x = B.channel_data(M, C, g)
    gamma, beta = (torch.randn(C, generator=g) * 0.8).float(), (torch.randn(C, generator=g) * 0.3).float()
    rm, rv = (x.mean(0) + torch.randn(C, generator=g, dtype=torch.float64) * 0.1).float(), (x.var(0) + 0.5).float()
    res = B.round_bf16(torch.randn(M, C, generator=g, dtype=torch.float64)) if residual else None
    eps = B.f32(1e-3)
    y = k.bn_act_infer(dev_nhwc(x, n, h, w), gamma.to(DEV), beta.to(DEV), rm.to(DEV), rv.to(DEV), eps, "relu", dev_nhwc(res, n, h, w) if residual else None)
    xd = x.to(DEV)
    rd = res.to(DEV) if residual else None
    ref = B.bn_infer_ref(xd, gamma.to(DEV), beta.to(DEV), rm.to(DEV), rv.to(DEV), eps, "relu", rd)
    iv = B.bn_infer_bounds(xd, gamma, beta, rm, rv, eps, "relu", rd)
    B.check("y", B.mc(y), ref["y"], iv["y"], bf16=True)


def test_bn_mask_from_x_equals_mask_from_y():
    """With beta given and no residual the backward recomputes the ReLU mask with the forward's own FMA: bit-identical to reading y."""
    k = K()
    for M, C in ((105, 24), (51200, 64)):
        _, v = run_bn(M=M, C=C, seed=M + C)
        a = k.bn_act_bwd(v["dyg"], v["xg"], v["y"], v["gamma"].to(DEV), v["mean"], v["rstd"], v["eps"], "relu", beta=v["beta"].to(DEV))
        b = k.bn_act_bwd(v["dyg"], v["xg"], v["y"], v["gamma"].to(DEV), v["mean"], v["rstd"], v["eps"], "relu", want_residual_grad=True, beta=v["beta"].to(DEV))
        assert torch.equal(a[0], b[0])
        assert torch.equal(b[1], torch.where(v["y"] > 0, v["dyg"], torch.zeros_like(v["dyg"])))


def test_bn_accumulate_and_repeat():
    """Parameter gradients are added into the given accumulators: acc in plus the increment, bit for bit.  At M <= 256 the fused launch
    has one CTA, so every channel sum is one fp64 atomic and repeated launches are bit-identical."""
    k = K()
    _, v = run_bn(M=105, C=64, seed=3)
    args = (v["dyg"], v["xg"], v["y"], v["gamma"].to(DEV), v["mean"], v["rstd"], v["eps"], "relu")
    r0 = k.bn_act_bwd(*args, beta=v["beta"].to(DEV))
    for _ in range(3):
        acc_g, acc_b = v["dg0"].to(DEV), v["db0"].to(DEV)
        r1 = k.bn_act_bwd(*args, dgamma=acc_g.clone(), dbeta=acc_b.clone(), beta=v["beta"].to(DEV))
        assert torch.equal(r1[0], r0[0])
        assert torch.equal(r1[2], acc_g + r0[2]) and torch.equal(r1[3], acc_b + r0[3])


def test_bn_fused_repeat_many_ctas():
    """Repeated fused launches over a grid of many CTAs (the grid barrier is reused) stay within the bounds every time."""
    for _ in range(3):
        run_bn(M=51200, C=64, seed=3)


def _bn_sync_inputs(Ms, C, seed):
    g = torch.Generator().manual_seed(seed)
    xs = [B.channel_data(m, C, g) for m in Ms]
    dys = [B.round_bf16(torch.randn(m, C, generator=g, dtype=torch.float64)) for m in Ms]
    gamma = (torch.randn(C, generator=g) * 0.8 + 0.4).float()
    beta = (torch.randn(C, generator=g) * 0.3).float()
    rm, rv = torch.randn(C, generator=g).float(), (torch.rand(C, generator=g) + 0.5).float()
    dg0, db0 = torch.randn(C, generator=g).float(), torch.randn(C, generator=g).float()
    return xs, dys, gamma, beta, rm, rv, dg0, db0


@pytest.mark.parametrize("C", [24, 2048])
def test_bn_sync_two_ranks(C):
    """Cross-rank statistics (split passes, count and param_scale from the sync object) emulated with two ranks on one GPU: rank A's
    outputs against the oracle over [A; B], parameter gradients x 1/2."""
    k = K()
    Ms = [3200, 1600] if C == 24 else [98, 49]
    shapes = [(m // 1600, 40, 40) if C == 24 else (m // 49, 7, 7) for m in Ms]
    xs, dys, gamma, beta, rm, rv, dg0, db0 = _bn_sync_inputs(Ms, C, C)
    eps, mom = B.f32(1e-3), B.f32(0.05)
    xg = [dev_nhwc(x, *s) for x, s in zip(xs, shapes)]
    dyg = [dev_nhwc(d, *s) for d, s in zip(dys, shapes)]
    G, Bt = gamma.to(DEV), beta.to(DEV)

    def rank(i, sync):
        rmg, rvg = rm.clone().to(DEV), rv.clone().to(DEV)
        y, mean, rstd = k.bn_act_fwd(xg[i], None, G, Bt, rmg, rvg, eps, mom, "relu", sync=sync)
        out = k.bn_act_bwd(dyg[i], xg[i], y, G, mean, rstd, eps, "relu", dgamma=dg0.clone().to(DEV), dbeta=db0.clone().to(DEV), beta=Bt, sync=sync)
        return y, mean, rstd, rmg, rvg, out

    a_alone = TwoRankSync()
    rank(0, a_alone)  # A's forward buffer, as A makes it
    b = TwoRankSync([a_alone.seen[0], torch.zeros_like(a_alone.seen[1])])
    rank(1, b)  # B with the global statistics: its backward sums are B's share of the global reduction
    a = TwoRankSync([b.seen[0], b.seen[1]])
    y, mean, rstd, rmg, rvg, (dx, _, dgo, dbo) = rank(0, a)
    inp = {"x": [x.to(DEV) for x in xs], "dy": [d.to(DEV) for d in dys], "residual": None, "ss": None, "gamma": gamma, "beta": beta, "rm": rm, "rv": rv,
           "eps": eps, "mom": mom, "act": "relu", "ps": 0.5, "dgamma0": dg0, "dbeta0": db0, "read_y": False, "sum_extra": 1, "check_rows": (0, Ms[0])}
    got = {"y": [B.mc(y)], "mean": mean, "rstd": rstd, "rm": rmg, "rv": rvg, "dx": [B.mc(dx)], "dgamma": dgo, "dbeta": dbo}
    B.verify_bn(inp, got, sms())


# ------------------------------------------------------------------------------------------------ QARepVGG
def _qarep_inputs(M, C, seed, post, no_ab, residual):
    g = torch.Generator().manual_seed(seed)
    y3 = B.channel_data(M, C, g)
    u = B.round_bf16(0.6 * y3 - 0.6 * y3.mean(0) + torch.randn(M, C, generator=g, dtype=torch.float64) + 0.5)
    gamma3 = (torch.randn(C, generator=g) * 0.8 + 0.2).float()
    gamma3[2] = -abs(float(gamma3[2])) - 0.3
    beta3, ab = (torch.randn(C, generator=g) * 0.3).float(), None if no_ab else (torch.randn(C, generator=g) * 0.3).float()
    gp, bp = (torch.randn(C, generator=g) * 0.8 + 0.2).float(), (torch.randn(C, generator=g) * 0.3).float()
    gp[0], bp[0] = 0.0, 0.0  # channel 0: pre-activations exactly 0
    rs = [torch.randn(C, generator=g).float(), (torch.rand(C, generator=g) + 0.5).float(), torch.randn(C, generator=g).float(), (torch.rand(C, generator=g) + 0.5).float()]
    res = B.round_bf16(torch.randn(M, C, generator=g, dtype=torch.float64)) if residual else None
    dout = B.round_bf16(0.5 * torch.tanh(y3) + torch.randn(M, C, generator=g, dtype=torch.float64))
    acc0 = [torch.randn(C, generator=g).float() for _ in range(5)]
    return y3, u, gamma3, beta3, ab, gp if post else None, bp if post else None, rs, res, dout, acc0


def run_qarep(M, C, seed, act="relu", post=True, residual=False, no_ab=False, sliced=False, dout_slice=False, mom=0.07):
    k = K()
    n, h, w = _shape(M)
    y3, u, gamma3, beta3, ab, gp, bp, rs, res, dout, acc0 = _qarep_inputs(M, C, seed, post, no_ab, residual)
    eps3, epsp, momf = B.f32(1e-3), B.f32(1e-5), B.f32(mom)
    cu = lambda t: None if t is None else t.to(DEV)  # noqa: E731
    if sliced:  # y3 / u as the two halves of one [N, 2K, H, W] GEMM output, gradients into the halves of one buffer
        cat = dev_nhwc(torch.cat([y3, u], 1), n, h, w)
        y3g, ug = cat[:, :C], cat[:, C:]
        dcat = torch.zeros_like(cat)
        out_grads = (dcat[:, :C], dcat[:, C:])
    else:
        y3g, ug, out_grads = dev_nhwc(y3, n, h, w), dev_nhwc(u, n, h, w), None
    rsg = [r.clone().to(DEV) for r in rs]
    alpha = torch.tensor([0.7], device=DEV) if residual else None
    out, coef = k.qarep_fwd(y3g, ug, cu(gamma3), cu(beta3), cu(ab), cu(gp), cu(bp), *rsg, eps3, epsp, momf, act, post,
                            **({"residual": dev_nhwc(res, n, h, w), "res_alpha": alpha} if residual else {}))
    dg = dev_nhwc(dout, n, h, w, C + 16 if dout_slice else None, 8 if dout_slice else 0)
    accg = [a.clone().to(DEV) for a in acc0]
    dy3, du, *accs = k.qarep_bwd(dg, out, y3g, ug, coef, cu(gamma3), cu(gp), eps3, epsp, act, post, acc=accg, out_grads=out_grads)
    inp = {"y3": [y3.to(DEV)], "u": [u.to(DEV)], "dout": [dout.to(DEV)], "residual": [res.to(DEV)] if residual else None, "gamma3": gamma3, "beta3": beta3, "ab": ab,
           "gamma_p": gp, "beta_p": bp, "rm3": rs[0], "rv3": rs[1], "rmp": rs[2], "rvp": rs[3], "eps3": eps3, "eps_post": epsp, "mom": momf, "act": act,
           "use_post_bn": post, "res_alpha": B.f32(0.7) if residual else None, "acc0": acc0}
    got = {"out": [B.mc(out)], "coef": coef, "rm3": rsg[0], "rv3": rsg[1], "rmp": rsg[2], "rvp": rsg[3], "dy3": [B.mc(dy3)], "du": [B.mc(du)], "acc": accs}
    rep = B.verify_qarep(inp, got, sms())
    return rep, locals()


QAREP_MATRIX = {
    "post_C8_M2": dict(M=2, C=8),
    "post_C24": dict(M=105, C=24),
    "post_C64_big": dict(M=51200, C=64),
    "post_C2048": dict(M=98, C=2048),
    "shortcut_res_alpha": dict(M=3200, C=24, residual=True),
    "no_post_bn": dict(M=105, C=64, post=False),
    "no_ab_act_none": dict(M=105, C=24, act="none", no_ab=True),
    "sliced_y3_u_out_grads": dict(M=3200, C=64, sliced=True),
    "dout_concat_slice": dict(M=105, C=24, dout_slice=True),
}


@pytest.mark.parametrize("name", list(QAREP_MATRIX))
def test_qarep_train_against_fp64(name):
    rep, _ = run_qarep(seed=sum(map(ord, name)), **QAREP_MATRIX[name])
    print(name, {k: round(v, 3) for k, v in rep.items()})


def test_qarep_shortcut_equals_separate_pass():
    """The fused res_alpha shortcut is bit-identical to the block output followed by the scale_add pass it replaced."""
    k = K()
    _, v = run_qarep(M=3200, C=24, seed=9, residual=True)
    n, h, w = _shape(3200)
    cu = lambda t: None if t is None else t.to(DEV)  # noqa: E731
    rsg = [r.clone().to(DEV) for r in v["rs"]]
    plain, _ = k.qarep_fwd(v["y3g"], v["ug"], cu(v["gamma3"]), cu(v["beta3"]), cu(v["ab"]), cu(v["gp"]), cu(v["bp"]), *rsg, v["eps3"], v["epsp"], v["momf"], "relu", True)
    two_pass = k.scale_add(dev_nhwc(v["res"], n, h, w), v["alpha"], plain)
    assert torch.equal(two_pass, v["out"])


def test_qarep_mask_is_forward_output_sign():
    """Without post-BN du is the masked dout: the backward's mask equals out > 0 of its own forward, element for element."""
    _, v = run_qarep(M=51200, C=64, seed=4, post=False)
    assert torch.equal(v["du"], torch.where(v["out"] > 0, v["dg"], torch.zeros_like(v["dg"])))


@pytest.mark.parametrize("C", [24, 64])
def test_qarep_post_bn_mask_is_forward_output_sign(C):
    """With post-BN: dout pre-masked with out > 0 gives bit-identical gradients, and dout kept only where out <= 0 gives the gradients of
    dout = 0.  Both hold only if the backward's mask is out > 0 of its own forward.  M <= 256: one CTA, one fp64 atomic per sum, so
    the runs are deterministic."""
    k = K()
    _, v = run_qarep(M=105, C=C, seed=C)
    cu = lambda t: None if t is None else t.to(DEV)  # noqa: E731
    pos = v["out"] > 0

    def bwd(dout):
        return k.qarep_bwd(dout, v["out"], v["y3g"], v["ug"], v["coef"], cu(v["gamma3"]), cu(v["gp"]), v["eps3"], v["epsp"], "relu", True)

    full, kept = bwd(v["dg"]), bwd(torch.where(pos, v["dg"], torch.zeros_like(v["dg"])))
    neg, zero = bwd(torch.where(pos, torch.zeros_like(v["dg"]), v["dg"])), bwd(torch.zeros_like(v["dg"]))
    assert 0.2 < float(pos.double().mean()) < 0.8
    for a, b in zip(full, kept):
        assert torch.equal(a, b)
    for a, b in zip(neg, zero):
        assert torch.equal(a, b)


def test_qarep_post_bn_leaves_bias_accumulators():
    _, v = run_qarep(M=3200, C=24, seed=6)
    assert torch.equal(v["accs"][1].cpu(), v["acc0"][1]) and torch.equal(v["accs"][2].cpu(), v["acc0"][2])


def test_qarep_sync_two_ranks():
    k = K()
    C, Ms = 24, [3200, 1600]
    shapes = [(2, 40, 40), (1, 40, 40)]
    ins = [_qarep_inputs(m, C, 20 + i, True, False, False) for i, m in enumerate(Ms)]
    y3s, us, douts = [t[0] for t in ins], [t[1] for t in ins], [t[9] for t in ins]
    _, _, gamma3, beta3, ab, gp, bp, rs, _, _, acc0 = ins[0]
    eps3, epsp, mom = B.f32(1e-3), B.f32(1e-5), B.f32(0.05)
    y3g = [dev_nhwc(t, *s) for t, s in zip(y3s, shapes)]
    ug = [dev_nhwc(t, *s) for t, s in zip(us, shapes)]
    dg = [dev_nhwc(t, *s) for t, s in zip(douts, shapes)]
    P = [t.to(DEV) for t in (gamma3, beta3, ab, gp, bp)]

    def rank(i, sync):
        rsg = [r.clone().to(DEV) for r in rs]
        out, coef = k.qarep_fwd(y3g[i], ug[i], *P, *rsg, eps3, epsp, mom, "relu", True, sync=sync)
        accg = [a.clone().to(DEV) for a in acc0]
        dy3, du, *accs = k.qarep_bwd(dg[i], out, y3g[i], ug[i], coef, P[0], P[3], eps3, epsp, "relu", True, acc=accg, sync=sync)
        return out, coef, rsg, dy3, du, accs

    a_alone = TwoRankSync()
    rank(0, a_alone)
    b = TwoRankSync([a_alone.seen[0], torch.zeros_like(a_alone.seen[1])])
    rank(1, b)
    a = TwoRankSync([b.seen[0], b.seen[1]])
    out, coef, rsg, dy3, du, accs = rank(0, a)
    inp = {"y3": [t.to(DEV) for t in y3s], "u": [t.to(DEV) for t in us], "dout": [t.to(DEV) for t in douts], "residual": None, "gamma3": gamma3, "beta3": beta3,
           "ab": ab, "gamma_p": gp, "beta_p": bp, "rm3": rs[0], "rv3": rs[1], "rmp": rs[2], "rvp": rs[3], "eps3": eps3, "eps_post": epsp, "mom": mom, "act": "relu",
           "use_post_bn": True, "acc0": acc0, "ps": 0.5, "check_rows": (0, Ms[0])}
    got = {"out": [B.mc(out)], "coef": coef, "rm3": rsg[0], "rv3": rsg[1], "rmp": rsg[2], "rvp": rsg[3], "dy3": [B.mc(dy3)], "du": [B.mc(du)], "acc": accs}
    B.verify_qarep(inp, got, sms())


# ------------------------------------------------------------------------------------------------ the one-pass variance
def test_one_pass_variance_report():
    """Worst save_rstd / coef[1] (rstd3) relative error per |mean| / std: the one-pass S2 / M - mean^2 loses (mean / std)^2 digits.
    At |mean| <= 4 std it stays below half a bf16 ulp (2^-9 relative) of the outputs."""
    report = {}
    for off in (0.0, 4.0, 64.0):
        k = K()
        M, C = 51200, 64
        n, h, w = _shape(M)
        g = torch.Generator().manual_seed(int(off) + 1)
        x = B.channel_data(M, C, g, offsets=(off,), constant=False)
        xg = dev_nhwc(x, n, h, w)
        ones = torch.ones(C, device=DEV)
        _, _, rstd = k.bn_act_fwd(xg, None, ones, torch.zeros(C, device=DEV), None, None, B.f32(1e-5), 0.1, "none")
        xd = x.to(DEV)
        ref = 1 / torch.sqrt(xd.var(0, unbiased=False) + B.f32(1e-5))
        e_bn = float(((rstd.double() - ref).abs() / ref).max())
        _, coef = k.qarep_fwd(xg, xg, ones, torch.zeros(C, device=DEV), None, ones, torch.zeros(C, device=DEV), None, None, None, None, B.f32(1e-5), B.f32(1e-5), 0.1, "none", True)
        e_q = float(((coef[1].double() - ref).abs() / ref).max())
        report[off] = (e_bn, e_q)
        if off <= 4.0:
            assert e_bn < 2.0**-9 and e_q < 2.0**-9
    print("one-pass variance: |mean|/std -> (save_rstd, coef[1]) worst relative error", report)


# ------------------------------------------------------------------------------------------------ recorded train steps
# launch paths each model must reach; every recorded call is checked against the oracle and bounds by replay_bn_qarep
REQUIRED = {
    "yolo_nas_s": {"bn_fwd:epilogue_stats", "bn_fwd:fused_stats", "bn_bwd:fused", "bn_bwd:dy2", "bn_bwd:dy_slice", "qarep_fwd:post_bn", "qarep_fwd:res_alpha",
                   "qarep_fwd:y3_u_slices", "qarep_bwd:post_bn", "qarep_bwd:out_grads_slices", "qarep_bwd:dout_slice", "channel_stats"},
    "resnet50": {"bn_fwd:epilogue_stats", "bn_fwd:fused_stats", "bn_fwd:residual", "bn_bwd:fused", "bn_bwd:residual_grad"},
    "resnet18_droppath": {"bn_fwd:sample_scale", "bn_bwd:sample_scale", "bn_fwd:residual", "bn_bwd:residual_grad"},
    "qarep_alpha": {"qarep_fwd:post_bn", "qarep_bwd:post_bn", "qarep_fwd:ab_none", "qarep_fwd:y3_u_slices", "qarep_bwd:out_grads_slices", "qarep_bwd:dout_slice"},
}
DRIVERS = {
    "yolo_nas_s": lambda: B.yolo_nas_s_step_record(batch=2, img=640),
    "resnet50": lambda: B.resnet_step_record("resnet50", batch=2, img=224),
    "resnet18_droppath": lambda: B.resnet_step_record("resnet18", batch=4, img=64, droppath_prob=0.5),
    "qarep_alpha": lambda: B.qarep_alpha_step_record(),
}


@pytest.mark.parametrize("model", list(DRIVERS))
def test_recorded_step_against_fp64(model):
    """Every BatchNorm / QARepVGG call of one train step at the model's real layer shapes, against the oracle and bounds."""
    calls = DRIVERS[model]()
    assert calls, "nothing was recorded"
    seen = B.replay_bn_qarep(calls, sms())
    print(model, len(calls), "calls, paths:", sorted(seen))
    assert REQUIRED[model] <= seen, f"paths not reached: {sorted(REQUIRED[model] - seen)}"
