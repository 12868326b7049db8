"""fp64 oracles, arithmetic-derived error bounds, an fp32 transcription and a launch recorder for the BatchNorm and QARepVGG passes of
csrc/bn_kernels.cu (bn_act_fwd / bn_act_infer / bn_act_bwd, qarep_fwd / qarep_bwd).

Layout.  Everything here works on [M, C] fp64 matrices in the kernels' pixel order (NHWC: pixel = (n * H + h) * W + w); `mc()` makes one
from an [N, C, H, W] tensor of any layout.  The drop-path scale is a per-pixel column [M, 1].  Cross-rank (sync) statistics are the
statistics of the concatenated shards; the oracles take the concatenation.

Oracles.  The exact bf16 inputs in float64, the operation written out (two-pass statistics) and torch autograd for the gradients.

Bounds.  Every kernel output is bounded by an interval (`Iv`) that contains the value the kernel can produce, evaluated from the
exact inputs through the kernel's own arithmetic:
  - a channel sum is a sum of fp32 partial sums: |error| <= gamma_L * sum|term| with gamma_L = L u / (1 - L u), u = 2^-24, and L the
    longest fp32 chain of the launch (`chain_len`): ceil(pixels per CTA / lanes) per-thread additions, then `lanes` in the cross-lane
    sum, with the grid at least min(ceil(M / 256), SM count);
  - every fp32 rounding the kernel makes widens the interval by u times the magnitude of the rounded quantity (`rnd`); formulas are
    evaluated in their centred form (x - mean) * scale, so the cancellation in x * scale + shift is not counted twice, while the
    one-pass variance S2 / M - mean^2 keeps its (mean / std)^2 growth;
  - a bf16 store adds half a bf16 ulp of the result;
  - statistics a convolution epilogue computed are bounded with the longest chain any grid can give (`epilogue_chain_len`).
The exact result lies in the same interval, so |kernel - oracle| <= width + rounding (`check`).  A ReLU whose pre-activation interval
contains 0 may take either mask value: the gradient intervals of that element and of the sums it enters take both (`ambiguous`).

Transcription.  `bn_fwd_t` / `bn_bwd_t` / `qarep_fwd_t` / `qarep_bwd_t` restate BnStatsOp, BnFwdOp, BnBwdRedOp / BnBwdApplyOp,
QarepMomOp, QarepFwdOpT, QarepBwdRedOp / QarepBwdApplyOp in fp32 torch on the CPU, with the launch's summation order and fmaf
emulated in fp64.  `mut` selects one deliberate defect; the CPU suite shows the bounds hold for the transcription and break for each
defect.

Recorder.  `record_bn_qarep()` patches the kernel front ends (functional.py and the models call them as `K.<name>`) the way
plumbing_cases.record_plumbing does and keeps, for every call, clones of the inputs, of the in-place state before the call (running
statistics, gradient accumulators) and of the outputs and that state after it.  `replay_bn_qarep()` checks every recorded call with
verify_bn / verify_qarep and returns the launch paths it saw.
"""
import contextlib
import math

import torch

U32 = 2.0**-24
U64 = 2.0**-53
TPB = 256
F64 = torch.float64


# ------------------------------------------------------------------------------------------------ layout, rounding
def mc(t):
    """[N, C, H, W] (any layout / device) -> fp64 [M, C] in NHWC pixel order."""
    return t.detach().permute(0, 2, 3, 1).reshape(-1, t.shape[1]).double()


def bf16_ulp(x):
    _, e = torch.frexp(x.abs())
    return torch.ldexp(torch.ones_like(x), (e.clamp_min(-125) - 8).to(torch.int32))


def round_bf16(x):
    u = bf16_ulp(x)
    return torch.round(x / u) * u


def f32(x):
    return x.float().double() if torch.is_tensor(x) else float(torch.tensor(x, dtype=torch.float32))


def fma32(a, b, c):
    """fmaf emulated in fp64: a * b is exact for fp32 operands, one rounding of the sum (then to fp32)."""
    return (a.double() * b.double() + c.double()).float()


# ------------------------------------------------------------------------------------------------ intervals
class Iv:
    """Closed interval [lo, hi] of fp64 tensors (broadcasting)."""

    __slots__ = ("lo", "hi")

    def __init__(self, lo, hi=None):
        self.lo = lo
        self.hi = lo if hi is None else hi

    @staticmethod
    def of(v):
        return v if isinstance(v, Iv) else Iv(v, v)

    def __add__(a, b):
        b = Iv.of(b)
        return Iv(a.lo + b.lo, a.hi + b.hi)

    __radd__ = __add__

    def __neg__(a):
        return Iv(-a.hi, -a.lo)

    def __sub__(a, b):
        return a + (-Iv.of(b))

    def __rsub__(a, b):
        return Iv.of(b) + (-a)

    def __mul__(a, b):
        b = Iv.of(b)
        p = [a.lo * b.lo, a.lo * b.hi, a.hi * b.lo, a.hi * b.hi]
        return Iv(torch.minimum(torch.minimum(p[0], p[1]), torch.minimum(p[2], p[3])) if torch.is_tensor(p[0]) or torch.is_tensor(p[1]) else min(p),
                  torch.maximum(torch.maximum(p[0], p[1]), torch.maximum(p[2], p[3])) if torch.is_tensor(p[0]) or torch.is_tensor(p[1]) else max(p))

    __rmul__ = __mul__

    def __truediv__(a, m):  # by a positive scalar
        return Iv(a.lo / m, a.hi / m)

    def inv(a):  # 1 / a, a > 0
        return Iv(1.0 / a.hi, 1.0 / a.lo)

    def sq(a):
        lo2, hi2 = a.lo * a.lo, a.hi * a.hi
        return Iv(torch.where(a.lo > 0, lo2, torch.where(a.hi < 0, hi2, torch.zeros_like(lo2))), torch.maximum(lo2, hi2))

    def sqrt(a):
        return Iv(a.lo.clamp_min(0).sqrt(), a.hi.clamp_min(0).sqrt())

    def clamp0(a):
        return Iv(a.lo.clamp_min(0), a.hi.clamp_min(0))

    def mag(a):
        return torch.maximum(a.lo.abs(), a.hi.abs())

    def width(a):
        return a.hi - a.lo

    def widen(a, e):
        return Iv(a.lo - e, a.hi + e)

    def sum0(a):
        return Iv(a.lo.sum(0), a.hi.sum(0))


def rnd(a, n=1, u=U32):
    """n roundings (fp32 by default) of a quantity in interval a."""
    a = Iv.of(a)
    m = a.mag()
    return a.widen(1.0001 * n * u * m + n * 2.0**-149 * (m > 0))  # rounding 0 is exact


def _abs_err(e):
    """An fp32 rounding bound e (fp64 tensor) plus the subnormal spacing wherever e is not 0 (rounding 0 is exact)."""
    return e + 4 * 2.0**-149 * (e > 0)


def act_iv(a, act):
    return a.clamp0() if act == "relu" else a


def mask_iv(pre, act):
    """The kernel's `pre > 0` for pre in the interval: [1, 1] certain, [0, 0] certain, [0, 1] ambiguous.  A bf16-stored
    pre-activation below 2^-133 rounds to 0, so the certain-1 side starts there."""
    if act != "relu":
        one = torch.ones_like(pre.lo)
        return Iv(one, one)
    lo = (pre.lo > 2.0**-133).double()
    hi = (pre.hi > 0).double()
    return Iv(lo, hi)


def ambiguous(m):
    return m.lo != m.hi


def gamma_n(L):
    return L * U32 / (1 - L * U32)


def chain_len(M, C, sms):
    """Longest fp32 rounding chain of one channel sum of chan_body over M pixels (per-thread run, then the lanes), for any grid the
    launch can pick (grid >= min(ceil(M / 256), SM count): at least one CTA per SM is resident)."""
    grid = max(1, min(math.ceil(M / 256), sms))
    per = math.ceil(M / grid)
    cvb = min(C // 8, TPB)
    lanes = TPB // cvb
    return math.ceil(per / lanes) + lanes


def epilogue_chain_len(M):
    """Longest fp32 rounding chain of one channel sum a convolution epilogue hands to bn_act_fwd (stats != None).  conv_mma.cu's
    epilogue adds a thread's rows of the 128-row tile, then 3 shuffle steps, then the WARPS_M warp rows, per CTA; conv_sm100.cu's
    wgmma epilogues add a thread's rows, 3 shuffle steps and the 8 (4) warps of a tile, then add every tile of the persistent CTA into
    one fp32 slot of s_stats (the halo kernel then adds its two warpgroups' slots) before one fp64 atomic.  The number of tiles a
    persistent CTA takes depends on its grid, so the bound takes the worst case over grids: every fp32 rounding on a value's path is
    one of those additions, and a CTA's slot covers at most all M rows of the layer, so no chain is longer than M."""
    return M


def sum_iv(terms, Ls, sizes):
    """Interval of the kernel's channel sums of `terms` (Iv [M, ...]) over shards of `sizes` rows, shard i summed with an fp32 chain of
    length Ls[i] (fp64 across CTAs and shards)."""
    out, r = None, 0
    for L, n in zip(Ls, sizes):
        part = Iv(terms.lo[r : r + n], terms.hi[r : r + n])
        s = part.sum0()
        mag = part.mag().sum(0)
        s = s.widen(gamma_n(L) * mag + (n + 8) * U64 * mag)
        out = s if out is None else out + s
        r += n
    return out


def check(name, k, ref, iv, bf16=False, extra=0.0):
    """|k - ref| <= width(iv) (+ half a bf16 ulp of the interval's magnitude for bf16 stores) + extra; returns the worst error /
    allowed ratio (for reports)."""
    k, ref = k.double().to(ref.device), ref.double()
    allow = iv.width() + extra
    if bf16:
        allow = allow + 0.5 * bf16_ulp(iv.mag() + iv.width())
    allow = torch.broadcast_to(allow, ref.shape)
    err = (k - ref).abs()
    bad = ~(err <= allow)
    if bool(bad.any()):
        i = int(bad.flatten().nonzero()[0])
        raise AssertionError(f"{name}: {int(bad.sum())} of {bad.numel()} outside the bound; first at flat {i}: kernel {float(k.flatten()[i])!r} "
                             f"oracle {float(ref.flatten()[i])!r} allowed {float(allow.flatten()[i]):.3e}")
    return float((err / allow.clamp_min(1e-300)).max()) if err.numel() else 0.0


# ------------------------------------------------------------------------------------------------ fp64 oracles
def _act(t, act):
    return torch.relu(t) if act == "relu" else t


def _req(t):
    return t.detach().double().clone().requires_grad_(True)


def bn_train_ref(x, gamma, beta, rm, rv, eps, mom, act, residual=None, sample_scale=None, dy=None, param_scale=1.0):
    """Train-mode BatchNorm (+ drop-path scale, + residual) + activation of x [M, C] (all shards).  eps / mom as the kernel sees them
    (fp32 values).  Returns y, pre (before the activation), mean, rstd, rm, rv and, with dy: dx, dres (the unscaled masked gradient),
    dgamma, dbeta (x param_scale)."""
    M, C = x.shape
    xr = _req(x)
    g = _req(gamma if gamma is not None else torch.ones(C, dtype=F64, device=x.device))
    b = _req(beta if beta is not None else torch.zeros(C, dtype=F64, device=x.device))
    res = _req(residual) if residual is not None else None
    mean = xr.mean(0)
    var = ((xr - mean) ** 2).mean(0)
    rstd = 1.0 / torch.sqrt(var + eps)
    pre = (xr - mean) * rstd * g + b
    if sample_scale is not None:  # drop-path scales the normalised branch before the residual joins
        pre = pre * sample_scale.double()
    if res is not None:
        pre = pre + res
    y = _act(pre, act)
    unb = var * (M / (M - 1)) if M > 1 else var
    out = {"y": y.detach(), "pre": pre.detach(), "mean": mean.detach(), "rstd": rstd.detach(),
           "rm": (1 - mom) * rm.double() + mom * mean.detach(), "rv": (1 - mom) * rv.double() + mom * unb.detach()}
    if dy is not None:
        ins = [xr, g, b] + ([res] if res is not None else [])
        gr = torch.autograd.grad(y, ins, dy.double())
        out.update(dx=gr[0], dgamma=gr[1] * param_scale, dbeta=gr[2] * param_scale, dres=gr[3] if res is not None else None)
    return out


def bn_infer_ref(x, gamma, beta, rm, rv, eps, act, residual=None):
    C = x.shape[1]
    g = gamma.double() if gamma is not None else torch.ones(C, dtype=F64, device=x.device)
    b = beta.double() if beta is not None else torch.zeros(C, dtype=F64, device=x.device)
    pre = (x.double() - rm.double()) / torch.sqrt(rv.double() + eps) * g + b
    if residual is not None:
        pre = pre + residual.double()
    return {"y": _act(pre, act), "pre": pre}


def qarep_train_ref(y3, u, gamma3, beta3, ab, gamma_p, beta_p, rm3, rv3, rmp, rvp, eps3, eps_post, mom, act, use_post_bn=True, residual=None,
                    res_alpha=None, dout=None, param_scale=1.0):
    """QARepVGG branch algebra on [M, C]: z = gamma3 (y3 - mu3) / sqrt(var3 + eps3) + beta3 + u + ab, out = act(post_bn(z)) (+ res_alpha
    * res after rounding the block output to bf16).  Returns out, pre, coef [9, C] (include/sgb200.h rows), the running statistics and,
    with dout: dy3, du, dgamma3, dbeta3, dab, dgamma_p, dbeta_p (x param_scale; dbeta3 / dab exactly 0 with post-BN)."""
    M, C = y3.shape
    dev = y3.device
    a, bu = _req(y3), _req(u)
    g3, b3 = _req(gamma3), _req(beta3)
    abr = _req(ab if ab is not None else torch.zeros(C, dtype=F64, device=dev))
    gp = _req(gamma_p if gamma_p is not None else torch.ones(C, dtype=F64, device=dev))
    bp = _req(beta_p if beta_p is not None else torch.zeros(C, dtype=F64, device=dev))
    mu3 = a.mean(0)
    var3 = ((a - mu3) ** 2).mean(0)
    rstd3 = 1.0 / torch.sqrt(var3 + eps3)
    s3 = g3 * rstd3
    z = s3 * (a - mu3) + b3 + bu + abr
    muz = z.mean(0)
    varz = ((z - muz) ** 2).mean(0)
    if use_post_bn:
        rstdz = 1.0 / torch.sqrt(varz + eps_post)
        pre = gp * (z - muz) * rstdz + bp
    else:
        rstdz = torch.ones_like(muz)
        pre = z
    o = _act(pre, act)
    d = lambda t: t.detach()  # noqa: E731
    muu = bu.mean(0)
    if use_post_bn:
        a3, au = gp * rstdz * s3, gp * rstdz
        c0 = gp * rstdz * (-s3 * mu3 - muu) + bp
        czy = ((z - muz) * (a - mu3)).mean(0) * rstdz * rstd3
    else:
        a3, au = s3, torch.ones_like(s3)
        c0 = b3 + abr - s3 * mu3
        czy = torch.zeros_like(s3)
    coef = torch.stack([d(mu3), d(rstd3), d(muu), d(rstdz), d(a3), d(au), d(c0), d(czy), d(s3)])
    unb = M / (M - 1) if M > 1 else 1.0
    out = {"pre": d(pre), "o": d(o), "coef": coef,
           "rm3": (1 - mom) * rm3.double() + mom * d(mu3), "rv3": (1 - mom) * rv3.double() + mom * d(var3) * unb,
           "rmp": (1 - mom) * rmp.double() + mom * d(muz) if use_post_bn else rmp.double(),
           "rvp": (1 - mom) * rvp.double() + mom * d(varz) * unb if use_post_bn else rvp.double()}
    out["out"] = round_bf16(d(o)) + res_alpha * residual.double() if residual is not None else d(o)
    if dout is not None:
        gr = torch.autograd.grad(o, [a, bu, g3, b3, abr, gp, bp], dout.double(), allow_unused=True)
        zero = torch.zeros(C, dtype=F64, device=dev)
        out.update(dy3=gr[0], du=gr[1], dgamma3=gr[2] * param_scale, dbeta3=zero if use_post_bn else gr[3] * param_scale,
                   dab=zero if use_post_bn else gr[4] * param_scale, dgamma_p=gr[5] * param_scale if use_post_bn else zero,
                   dbeta_p=gr[6] * param_scale if use_post_bn else zero, autograd_dbeta3=gr[3], autograd_dab=gr[4])
    return out


# ------------------------------------------------------------------------------------------------ bounds
def _cv(v, C, dev, default):
    return v.double().to(dev) if v is not None else torch.full((C,), float(default), dtype=F64, device=dev)


def bn_fwd_bounds(x, sums, M, gamma, beta, rm, rv, eps, mom, act, residual=None, sample_scale=None):
    """Intervals of the forward outputs given the channel-sum intervals `sums` = (S1, S2) over the global count M.  Returns a dict
    of Iv: mean (save_mean), rstd (save_rstd), rm, rv, scale, pre_bn (the kernel's fma, what the backward recomputes), pre (before the
    activation), y."""
    C, dev = x.shape[1], x.device
    g, b = _cv(gamma, C, dev, 1.0), _cv(beta, C, dev, 0.0)
    S1, S2 = sums
    mean = rnd(S1 / M, 2, U64)
    var = rnd(rnd(S2 / M, 1, U64) - rnd(mean.sq(), 1, U64), 1, U64).clamp0()
    rstd = rnd(rnd((var + eps).sqrt(), 2, U64).inv(), 1)  # the fp64 chain, then (float)
    meanf = rnd(mean)
    gr = g * rstd
    scale = rnd(gr)
    mgr = (meanf.mag() * g.abs() * rstd.mag())
    xs = (x - meanf) * gr
    pre_bn = (xs + b)
    pre_bn = pre_bn.widen(_abs_err(1.01 * U32 * (3 * mgr + b.abs() + x.abs() * scale.mag() + pre_bn.mag())))
    pre = pre_bn
    if sample_scale is not None:
        pre = rnd(pre * sample_scale.double())
    if residual is not None:
        pre = rnd(pre + residual.double())
    out = {"mean": meanf, "rstd": rstd, "scale": scale, "pre_bn": pre_bn, "pre": pre, "y": act_iv(pre, act)}
    if rm is not None:
        m = f32(mom)
        a = rnd((1 - m) * rm.double().to(dev), 2) + rnd(m * meanf)
        out["rm"] = rnd(a)
        unb = rnd(var * (M / (M - 1.0)), 2, U64) if M > 1 else var
        a = rnd((1 - m) * rv.double().to(dev), 2) + rnd(m * rnd(unb))
        out["rv"] = rnd(a)
    return out


def bn_fwd_sums(x, Ls, sizes):
    xi = Iv(x)
    return sum_iv(xi, Ls, sizes), sum_iv(Iv(x * x), Ls, sizes)


def bn_bwd_bounds(fw, x, dy, M, gamma, act, Ls, sizes, mask_from, sample_scale=None, dgamma0=None, dbeta0=None, param_scale=1.0):
    """Intervals of dx, dres, dgamma, dbeta given the forward intervals `fw` (the kernel's save_mean / save_rstd lie in fw['mean'] /
    fw['rstd']); `mask_from`: the pre-activation interval the kernel's mask is taken from.  Also returns the ambiguous-mask map."""
    C, dev = x.shape[1], x.device
    g = _cv(gamma, C, dev, 1.0)
    mk = mask_iv(mask_from, act)
    dyv = dy.double()
    dres = dyv * mk
    dz = dres if sample_scale is None else rnd(dres * sample_scale.double())
    rs = fw["rstd"]
    xh = (x - fw["mean"]) * rs
    xh = xh.widen(2.01 * U32 * xh.mag())
    S0 = sum_iv(dz, Ls, sizes)
    S1 = sum_iv(dz * xh, Ls, sizes)
    m0, m1 = rnd(S0 / M), rnd(S1 / M)
    xm = rnd(xh * m1)
    inner = rnd(rnd(dz - m0) - xm)
    scale = rnd(g * rs)
    dx = rnd(scale * inner)
    z = torch.zeros(C, dtype=F64, device=dev)
    dg0 = dgamma0.double().to(dev) if dgamma0 is not None else z
    db0 = dbeta0.double().to(dev) if dbeta0 is not None else z
    return {"dx": dx, "dres": dres, "dgamma": rnd(dg0 + rnd(S1 * param_scale)), "dbeta": rnd(db0 + rnd(S0 * param_scale)),
            "amb": ambiguous(mk), "m0": m0, "m1": m1}


def bn_infer_bounds(x, gamma, beta, rm, rv, eps, act, residual=None):
    C, dev = x.shape[1], x.device
    g, b = _cv(gamma, C, dev, 1.0), _cv(beta, C, dev, 0.0)
    rmv = rm.double().to(dev)
    r = 1.0 / torch.sqrt(rv.double().to(dev) + eps)
    rstd = Iv(r).widen(6.01 * U32 * r)  # fp32 add, rsqrtf (2 ulp)
    gr = g * rstd
    pre = (x - rmv) * gr + b
    pre = pre.widen(_abs_err(1.01 * U32 * (3 * rmv.abs() * gr.mag() + b.abs() + x.abs() * gr.mag() * 1.01 + pre.mag())))
    if residual is not None:
        pre = rnd(pre + residual.double())
    return {"pre": pre, "y": act_iv(pre, act)}


def qarep_moment_sums(y3, u, Ls, sizes):
    return [sum_iv(Iv(t), Ls, sizes) for t in (y3, y3 * y3, u, u * u, y3 * u)]


def qarep_fwd_bounds(y3, u, mom_iv, M, gamma3, beta3, ab, gamma_p, beta_p, rm3, rv3, rmp, rvp, eps3, eps_post, mom, act, use_post_bn,
                     residual=None, res_alpha=None):
    """Intervals of coef (list of 9 Iv, the fp32 rows), the running statistics, pre (the kernel's fp32 pre-activation) and out."""
    C, dev = y3.shape[1], y3.device
    S3, S33, Su, Suu, S3u = mom_iv
    d = lambda a, n=1: rnd(a, n, U64)  # noqa: E731
    mu3, muu = d(S3 / M), d(Su / M)
    var3 = d(d(S33 / M) - d(mu3.sq())).clamp0()
    varu = d(d(Suu / M) - d(muu.sq())).clamp0()
    cov = d(d(S3u / M) - d(mu3 * muu))
    rstd3 = d(d((var3 + eps3).sqrt(), 2).inv())
    g3, b3 = gamma3.double().to(dev), beta3.double().to(dev)
    abv = _cv(ab, C, dev, 0.0)
    s3 = d(g3 * rstd3)
    muz = d(b3 + muu + abv, 2)
    varz = d(d(s3.sq() * var3, 2) + varu + d(2.0 * s3 * cov, 2), 2).clamp0()
    if use_post_bn:
        gp, bp = gamma_p.double().to(dev), beta_p.double().to(dev)
        rstdz = d(d((varz + eps_post).sqrt(), 2).inv())
        au = d(gp * rstdz)
        a3 = d(au * s3)
        c0 = d(au * d(-s3 * mu3 - muu, 2) + bp, 2)
        czy = d((d(s3 * var3) + cov) * rstdz * rstd3, 4)
        centred = au * (s3 * (y3 - mu3) + (u - muu)) + bp
    else:
        one = torch.ones(C, dtype=F64, device=dev)
        rstdz, a3, au = Iv(one), s3, Iv(one)
        c0 = d(b3 + abv - s3 * mu3, 3)
        czy = Iv(torch.zeros(C, dtype=F64, device=dev))
        centred = s3 * (y3 - mu3) + u + b3 + abv
    coef = [rnd(v) for v in (mu3, rstd3, muu, rstdz, a3, au, c0, czy, s3)]
    a3f, auf, c0f = coef[4], coef[5], coef[6]
    inner = auf.mag() * u.abs() + c0f.mag()
    pre = centred.widen(_abs_err(1.01 * U32 * (a3f.mag() * y3.abs() + auf.mag() * u.abs() + c0f.mag() + inner + centred.mag())))
    o = act_iv(pre, act)
    out = {"coef": coef, "pre": pre, "o": o}
    m = f32(mom)
    unb = M / (M - 1.0) if M > 1 else 1.0
    run = lambda r0, v: rnd(rnd((1 - m) * r0.double().to(dev), 2) + rnd(m * rnd(v)))  # noqa: E731
    if rm3 is not None:
        out["rm3"], out["rv3"] = run(rm3, mu3), run(rv3, d(var3 * unb))
    if use_post_bn and rmp is not None:
        out["rmp"], out["rvp"] = run(rmp, muz), run(rvp, d(varz * unb))
    if residual is not None:
        # |bf16(o_k) - bf16(o_ref)| <= width + one bf16 ulp; then one fma rounding and the bf16 store (added by check)
        a = float(res_alpha)
        tot = o + a * residual.double()
        out["out"] = tot.widen(bf16_ulp(o.mag() + o.width()) + 1.01 * U32 * (tot.mag() + bf16_ulp(o.mag() + o.width())))
    else:
        out["out"] = o
    return out


def qarep_bwd_bounds(fw, y3, u, dout, M, gamma_p, act, use_post_bn, Ls, sizes, acc0=None, param_scale=1.0):
    """Intervals of dy3, du and the five accumulators, from the forward intervals `fw` (coef rows and pre)."""
    C, dev = y3.shape[1], y3.device
    mu3, rstd3, muu, rstdz, _, _, _, czy, s3 = fw["coef"]
    mk = mask_iv(fw["pre"], act)
    dzp = dout.double() * mk
    y3c = y3 - mu3
    y3c = y3c.widen(1.01 * U32 * y3c.mag())
    y3h = y3c * rstd3
    y3h = y3h.widen(1.01 * U32 * y3h.mag())
    T0 = sum_iv(dzp, Ls, sizes)
    T2 = sum_iv(dzp * y3h, Ls, sizes)
    m0, m2 = rnd(T0 / M), rnd(T2 / M)
    z = torch.zeros(C, dtype=F64, device=dev)
    acc0 = [a.double().to(dev) if a is not None else z for a in (acc0 or (None,) * 5)]
    if use_post_bn:
        s3y = s3 * y3c
        um = u - muu
        zh = (s3y + um) * rstdz
        zh = zh.widen(1.01 * U32 * (rstdz.mag() * (um.mag() + 2 * s3y.mag() + (s3y + um).mag()) + zh.mag()))
        T1 = sum_iv(dzp * zh, Ls, sizes)
        m1 = rnd(T1 / M)
        g = rnd(gamma_p.double().to(dev) * rstdz)
        q = rnd(g * rnd(m2 - rnd(m1 * czy)))
        dz = rnd(g * rnd(rnd(dzp - m0) - rnd(zh * m1)))
        dy3 = rnd(s3 * rnd(dz - rnd(y3h * q)))
        acc = [rnd(acc0[0] + rnd(M * q * param_scale, 2)), Iv(acc0[1]), Iv(acc0[2]), rnd(acc0[3] + rnd(T1 * param_scale)), rnd(acc0[4] + rnd(T0 * param_scale))]
    else:
        dz = dzp
        dy3 = rnd(s3 * rnd(rnd(dzp - m0) - rnd(y3h * m2)))
        acc = [rnd(acc0[0] + rnd(T2 * param_scale)), rnd(acc0[1] + rnd(T0 * param_scale)), rnd(acc0[2] + rnd(T0 * param_scale)), Iv(acc0[3]), Iv(acc0[4])]
    return {"dy3": dy3, "du": dz, "acc": acc, "amb": ambiguous(mk)}


# ------------------------------------------------------------------------------------------------ fp32 transcription
CHAN_GRID_CAP = 132 * 6  # sgb_chan_grid_cap() of common.cuh


def launch_grid(M, sms, per_sm=1):
    """launch_chan's grid: one CTA per 256 pixels, at most `per_sm` resident CTAs per SM and the common grid cap."""
    return int(max(1, min(math.ceil(M / 256), sms * per_sm, CHAN_GRID_CAP)))


def chan_sums_t(terms, grid):
    """chan_body's reduction of fp64 per-element increments terms [M, C, A] (each exact: a bf16 value, or an fp32 product an fmaf adds
    with one rounding): per thread in pixel order in fp32, then the lanes in order, fp64 across CTAs.  Returns fp64 [A, C]."""
    M, C, A = terms.shape
    cvb = min(C // 8, TPB)
    lanes = TPB // cvb
    per = math.ceil(M / grid)
    steps = math.ceil(per / lanes)
    T = torch.zeros(grid * per, C, A, dtype=F64)
    T[:M] = terms
    T2 = torch.zeros(grid, steps * lanes, C, A, dtype=F64)
    T2[:, :per] = T.view(grid, per, C, A)
    T2 = T2.view(grid, steps, lanes, C, A)
    acc = torch.zeros(grid, lanes, C, A, dtype=torch.float32)
    for s in range(steps):
        acc = (acc.double() + T2[:, s]).float()
    tot = torch.zeros(grid, C, A, dtype=torch.float32)
    for q in range(lanes):
        tot = tot + acc[:, q]
    return tot.double().sum(0).T.contiguous()


def _bn_coef_t(S1, S2, M, eps, g, b):
    mean = S1 / M
    var = (S2 / M - mean * mean).clamp_min(0)
    rstd = (1.0 / torch.sqrt(var + eps)).float()
    meanf = mean.float()
    scale = g * rstd
    shift = fma32(-(meanf * g), rstd, b)
    return mean, var, meanf, rstd, scale, shift


def bn_fwd_t(x, gamma, beta, rm, rv, eps, mom, act, residual=None, sample_scale=None, stats=None, grid=None, M_global=None, mut=None):
    """BnStatsOp + BnFwdOp in fp32.  x [M, C] fp64 holding bf16 values; stats: fp64 [repl, 2, C] given sums (else BnStatsOp's, on
    `grid` CTAs).  Returns y (bf16 values as fp64), mean, rstd, rm, rv (fp32)."""
    M, C = x.shape
    if stats is None:
        stats = chan_sums_t(torch.stack([x, x * x], -1), grid).unsqueeze(0)
    repl = stats[:1] if mut == "repl0" else stats
    S1, S2 = repl[:, 0].sum(0), repl[:, 1].sum(0)
    Mt = float(M_global or M)
    g = gamma.float() if gamma is not None else torch.ones(C)
    b = beta.float() if beta is not None else torch.zeros(C)
    mean, var, meanf, rstd, scale, shift = _bn_coef_t(S1, S2, Mt, eps, g, b)
    pre = fma32(x.float(), scale, shift)
    if sample_scale is not None:
        ss = sample_scale.float()
        r = residual.float() if residual is not None else torch.zeros_like(pre)
        pre = ((pre + r) * ss) if mut == "ss_after_res" else fma32(pre, ss, r)
    elif residual is not None:
        pre = pre + residual.float()
    y = torch.relu(pre) if act == "relu" else pre
    m = torch.tensor(mom, dtype=torch.float32)
    unb = var if (mut == "biased_rv" or Mt <= 1) else var * Mt / (Mt - 1.0)
    rmn = fma32((1 - m) * rm.float(), torch.ones(()), m * meanf)
    rvn = fma32((1 - m) * rv.float(), torch.ones(()), m * unb.float())
    return {"y": round_bf16(y.double()), "mean": meanf, "rstd": rstd, "rm": rmn, "rv": rvn}


def bn_bwd_t(shards, gamma, beta, mean, rstd, act, grids, M_global, sample_scale=None, read_y=False, dgamma0=None, dbeta0=None, param_scale=1.0, mut=None):
    """BnBwdRedOp + BnBwdApplyOp in fp32.  shards: list of (x, dy, y) [M_i, C] (y: the forward output, read for the mask when read_y);
    sample_scale: list of per-pixel columns or None.  Returns dx / dres per shard and the accumulated dgamma, dbeta."""
    C = shards[0][0].shape[1]
    g = gamma.float() if gamma is not None else torch.ones(C)
    b = beta.float() if beta is not None else torch.zeros(C)
    scale = g * rstd
    shift = fma32(-(mean * g), rstd, b)
    ps = 1.0 if mut == "ps_one" else param_scale
    per = []
    S = torch.zeros(2, C, dtype=F64)
    for i, (x, dy, y) in enumerate(shards):
        xf = x.float()
        pre = y.float() if read_y else fma32(xf, scale, shift)
        dzr = torch.where(pre > 0, dy.float(), torch.zeros_like(pre)) if act == "relu" else dy.float()
        ss = sample_scale[i].float() if sample_scale is not None else None
        dz = dzr * ss if ss is not None else dzr
        xh = (xf - mean) * rstd
        S += chan_sums_t(torch.stack([dz.double(), dz.double() * xh.double()], -1), grids[i])
        per.append((xf, dz, dzr, xh))
    Mt = float(M_global)
    m0, m1 = (S[0] / Mt).float(), (S[1] / Mt).float()
    out = {"dx": [], "dres": []}
    for xf, dz, dzr, xh in per:
        o = scale * fma32(-xh, m1, dz - m0)
        out["dx"].append(round_bf16(o.double()))
        out["dres"].append(round_bf16((dz if mut == "dres_scaled" else dzr).double()))
    z = torch.zeros(C)
    out["dgamma"] = (dgamma0.float() if dgamma0 is not None else z) + (S[1] * ps).float()
    out["dbeta"] = (dbeta0.float() if dbeta0 is not None else z) + (S[0] * ps).float()
    return out


def qarep_fwd_t(y3, u, gamma3, beta3, ab, gamma_p, beta_p, rm3, rv3, rmp, rvp, eps3, eps_post, mom, act, use_post_bn, grid, residual=None,
                res_alpha=None, mut=None):
    """QarepMomOp + QarepFwdOpT in fp32 on `grid` CTAs.  Returns out (bf16 values), coef [9, C] fp32 and the running statistics."""
    M, C = y3.shape
    S3, S33, Su, Suu, S3u = chan_sums_t(torch.stack([y3, y3 * y3, u, u * u, y3 * u], -1), grid)
    Mt = float(M)
    mu3 = S3 / Mt
    var3 = (S33 / Mt - mu3 * mu3).clamp_min(0)
    muu = Su / Mt
    varu = (Suu / Mt - muu * muu).clamp_min(0)
    cov = S3u / Mt - mu3 * muu
    rstd3 = 1.0 / torch.sqrt(var3 + (eps_post if mut == "eps_post_first" else eps3))
    g3, b3 = gamma3.double(), beta3.double()
    abc = ab.double() if ab is not None else torch.zeros(C, dtype=F64)
    s3 = g3 * rstd3
    muz = b3 + muu + abc
    varz = (s3 * s3 * var3 + varu + (1.0 if mut == "cov_half" else 2.0) * s3 * cov).clamp_min(0)
    if use_post_bn:
        rstdz = 1.0 / torch.sqrt(varz + eps_post)
        gp, bp = gamma_p.double(), beta_p.double()
        a3, au = gp * rstdz * s3, gp * rstdz
        c0 = gp * rstdz * (-s3 * mu3 - muu) + bp
        czy = (s3 * var3 + cov) * rstdz * rstd3
    else:
        rstdz = torch.ones(C, dtype=F64)
        a3, au, c0, czy = s3, torch.ones(C, dtype=F64), b3 + abc - s3 * mu3, torch.zeros(C, dtype=F64)
    coef = torch.stack([mu3, rstd3, muu, rstdz, a3, au, c0, czy, s3]).float()
    pre = fma32(coef[4], y3.float(), fma32(coef[5], u.float(), coef[6]))
    o = torch.relu(pre) if act == "relu" else pre
    if residual is not None:
        o = fma32(torch.tensor(float(res_alpha), dtype=torch.float32), residual.float(), round_bf16(o.double()).float())
    m = torch.tensor(mom, dtype=torch.float32)
    unb = Mt / (Mt - 1.0) if Mt > 1 else 1.0
    run = lambda r0, v: fma32((1 - m) * r0.float(), torch.ones(()), m * v.float())  # noqa: E731
    out = {"out": round_bf16(o.double()), "coef": coef, "rm3": run(rm3, mu3), "rv3": run(rv3, var3 * unb)}
    out["rmp"] = run(rmp, muz) if use_post_bn else rmp.float()
    out["rvp"] = run(rvp, varz * unb) if use_post_bn else rvp.float()
    return out


def qarep_bwd_t(y3, u, dout, coef, gamma_p, act, use_post_bn, grid, acc0=None, param_scale=1.0, M_global=None, extra_sums=None, mut=None):
    """QarepBwdRedOp + QarepBwdApplyOp in fp32.  extra_sums: fp64 [3, C] added to the reduction (another rank's).  Returns dy3, du
    (bf16 values) and the five accumulators."""
    C = y3.shape[1]
    r = coef.float()
    a, b, gv = y3.float(), u.float(), dout.float()
    pre = fma32(r[4], a, fma32(r[5], b, r[6]))
    dzp = torch.where(pre > 0, gv, torch.zeros_like(gv)) if act == "relu" else gv
    y3c = a - r[0]
    zh = fma32(r[8], y3c, b - r[2]) * r[3]
    y3h = y3c * r[1]
    T = chan_sums_t(torch.stack([dzp.double(), dzp.double() * zh.double() if use_post_bn else torch.zeros_like(y3), dzp.double() * y3h.double()], -1), grid)
    if extra_sums is not None:
        T = T + extra_sums
    Mt = float(M_global or y3.shape[0])
    ps = 1.0 if mut == "ps_one" else param_scale
    m0, m1, m2 = (T[0] / Mt).float(), (T[1] / Mt).float(), (T[2] / Mt).float()
    z = torch.zeros(C)
    acc = [t.float() if t is not None else z.clone() for t in (acc0 or (None,) * 5)]
    if use_post_bn:
        g = gamma_p.float() * r[3]
        q = g * m2 if mut == "q_no_czy" else g * (m2 - m1 * r[7])
        dz = g * fma32(-zh, m1, dzp - m0)
        o3 = r[8] * fma32(-y3h, q, dz)
        acc[0] = acc[0] + (Mt * q.double() * ps).float()
        acc[3] = acc[3] + (T[1] * ps).float()
        acc[4] = acc[4] + (T[0] * ps).float()
    else:
        dz = dzp
        o3 = r[8] * fma32(-y3h, m2, dzp - m0)
        acc[0] = acc[0] + (T[2] * ps).float()
        acc[1] = acc[1] + (T[0] * ps).float()
        acc[2] = acc[2] + (T[0] * ps).float()
    return {"dy3": round_bf16(o3.double()), "du": round_bf16(dz.double()), "acc": acc, "sums": T}


MUTATIONS = ("biased_rv", "eps_post_first", "cov_half", "q_no_czy", "ps_one", "dres_scaled", "repl0", "ss_after_res")


# ------------------------------------------------------------------------------------------------ synthetic data
def channel_data(M, C, gen, offsets=(0.0, 4.0, 64.0), constant=True):
    """bf16 values [M, C] fp64: channel c has |mean| / std = offsets[c % len]; channel 1 constant (var = 0) when `constant`."""
    std = torch.rand(C, generator=gen, dtype=F64) * 1.5 + 0.5
    off = torch.tensor([offsets[c % len(offsets)] for c in range(C)], dtype=F64) * std * torch.where(torch.arange(C) % 2 == 0, 1.0, -1.0)
    x = torch.randn(M, C, generator=gen, dtype=F64) * std + off
    if constant and C > 1:
        x[:, 1] = 2.75
    return round_bf16(x)


def split_stats(x, repl, gen):
    """Exact channel sums of x spread unevenly over `repl` replicas (as GEMM epilogues leave them): fp64 [repl, 2, C]."""
    C = x.shape[1]
    w = torch.rand(repl, C, generator=gen, dtype=F64)
    w[0] *= 3
    w = w / w.sum(0)
    s = torch.stack([x.sum(0), (x * x).sum(0)])
    out = (w.unsqueeze(1) * s.unsqueeze(0))
    out[-1] = s - out[:-1].sum(0)
    return out


# ------------------------------------------------------------------------------------------------ one case, checked
AMBIGUOUS_MAX = 0.05  # share of elements whose ReLU mask the bounds leave open


def _cat(v):
    return None if v is None else torch.cat(v, 0)


def _rows(inp, t):
    r = inp.get("check_rows")
    if r is None or t is None:
        return t
    if isinstance(t, Iv):
        return Iv(t.lo[r[0] : r[1]], t.hi[r[0] : r[1]])
    return t[r[0] : r[1]]


def verify_bn(inp, got, sms):
    """Checks one BatchNorm forward (+ backward) against bn_train_ref with the bounds above.  inp: x / residual / ss / dy (lists of
    shards [M_i, C] fp64, residual / ss / dy may be None), gamma, beta, rm, rv, dgamma0, dbeta0 (fp32 tensors or None), eps, mom (fp32
    values), act, ps, stats_exact (the sums were given exactly), stats_epilogue (the sums came from a convolution epilogue),
    read_y (the backward reads the forward output for its mask),
    sum_extra (extra rounding steps of the statistics pass).  got: y / dx / dres (lists), mean, rstd, rm, rv, dgamma, dbeta.
    Returns {output: worst error / allowed}."""
    xs = inp["x"]
    x, C = _cat(xs), xs[0].shape[1]
    sizes = [t.shape[0] for t in xs]
    M = x.shape[0]
    inp = {k: (v.to(x.device) if torch.is_tensor(v) else v) for k, v in inp.items()}
    res, ss, dy = _cat(inp.get("residual")), _cat(inp.get("ss")), _cat(inp.get("dy"))
    if inp.get("stats_exact"):
        Lf = [0] * len(sizes)
    elif inp.get("stats_epilogue"):
        Lf = [epilogue_chain_len(n) for n in sizes]
    else:
        Lf = [chain_len(n, C, sms) + inp.get("sum_extra", 0) for n in sizes]
    ref = bn_train_ref(x, inp["gamma"], inp["beta"], inp["rm"], inp["rv"], inp["eps"], inp["mom"], inp["act"], res, ss, dy, inp.get("ps", 1.0))
    fw = bn_fwd_bounds(x, bn_fwd_sums(x, Lf, sizes), M, inp["gamma"], inp["beta"], inp["rm"], inp["rv"], inp["eps"], inp["mom"], inp["act"], res, ss)
    rep = {}
    if got.get("y") is not None:
        rep["y"] = check("y", _cat(got["y"]), _rows(inp, ref["y"]), _rows(inp, fw["y"]), bf16=True)
    if got.get("mean") is not None:
        rep["save_mean"] = check("save_mean", got["mean"], ref["mean"], fw["mean"])
        rep["save_rstd"] = check("save_rstd", got["rstd"], ref["rstd"], fw["rstd"])
    if got.get("rm") is not None:
        rep["running_mean"] = check("running_mean", got["rm"], ref["rm"], fw["rm"])
        rep["running_var"] = check("running_var", got["rv"], ref["rv"], fw["rv"])
    if dy is None:
        return rep
    Lb = [chain_len(n, C, sms) for n in sizes]
    bw = bn_bwd_bounds(fw, x, dy, M, inp["gamma"], inp["act"], Lb, sizes, fw["pre"] if inp.get("read_y") else fw["pre_bn"], ss,
                       inp.get("dgamma0"), inp.get("dbeta0"), inp.get("ps", 1.0))
    amb = float(bw["amb"].double().mean())
    assert int(bw["amb"].sum()) <= AMBIGUOUS_MAX * bw["amb"].numel() + 2, f"{amb:.3f} of the ReLU masks are ambiguous under the bounds"
    rep["ambiguous"] = amb
    rep["dx"] = check("dx", _cat(got["dx"]), _rows(inp, ref["dx"]), _rows(inp, bw["dx"]), bf16=True)
    if got.get("dres") is not None:
        rep["dres"] = check("dres", _cat(got["dres"]), _rows(inp, ref["dres"]), _rows(inp, bw["dres"]), bf16=True)
    z = torch.zeros(C, dtype=F64, device=x.device)
    dg0 = inp["dgamma0"].double().to(x.device) if inp.get("dgamma0") is not None else z
    db0 = inp["dbeta0"].double().to(x.device) if inp.get("dbeta0") is not None else z
    rep["dgamma"] = check("dgamma", got["dgamma"], dg0 + ref["dgamma"], bw["dgamma"])
    if inp["beta"] is not None or got.get("dbeta") is not None:
        rep["dbeta"] = check("dbeta", got["dbeta"], db0 + ref["dbeta"], bw["dbeta"])
    return rep


def verify_qarep(inp, got, sms):
    """QARepVGG counterpart of verify_bn.  inp: y3 / u / dout / residual (lists of shards), gamma3, beta3, ab, gamma_p, beta_p, rm3, rv3,
    rmp, rvp, acc0 (5-tuple or None), eps3, eps_post, mom (fp32 values), act, use_post_bn, res_alpha (float or None), ps.  got: out
    (list), coef [9, C], rm3 ... rvp, dy3 / du (lists), acc (5 tensors)."""
    y3s = inp["y3"]
    y3, u, C = _cat(y3s), _cat(inp["u"]), y3s[0].shape[1]
    sizes = [t.shape[0] for t in y3s]
    M = y3.shape[0]
    inp = {k: (v.to(y3.device) if torch.is_tensor(v) else v) for k, v in inp.items()}
    if inp.get("acc0") is not None:
        inp["acc0"] = [t.to(y3.device) for t in inp["acc0"]]
    dout, res = _cat(inp.get("dout")), _cat(inp.get("residual"))
    Ls = [chain_len(n, C, sms) for n in sizes]
    a = (inp["gamma3"], inp["beta3"], inp["ab"], inp["gamma_p"], inp["beta_p"], inp["rm3"], inp["rv3"], inp["rmp"], inp["rvp"], inp["eps3"], inp["eps_post"], inp["mom"], inp["act"], inp["use_post_bn"])
    ref = qarep_train_ref(y3, u, *a, residual=res, res_alpha=inp.get("res_alpha"), dout=dout, param_scale=inp.get("ps", 1.0))
    fw = qarep_fwd_bounds(y3, u, qarep_moment_sums(y3, u, Ls, sizes), M, *a, residual=res, res_alpha=inp.get("res_alpha"))
    rep = {}
    if got.get("out") is not None:
        rep["out"] = check("out", _cat(got["out"]), _rows(inp, ref["out"]), _rows(inp, fw["out"]), bf16=True)
    if got.get("coef") is not None:
        for i, nm in enumerate(("mu3", "rstd3", "mu_u", "rstd_z", "a3", "au", "c0", "czy", "s3")):
            rep["coef_" + nm] = check("coef[%d] %s" % (i, nm), got["coef"][i], ref["coef"][i], fw["coef"][i])
    for k in ("rm3", "rv3", "rmp", "rvp"):
        if got.get(k) is not None and k in fw:
            rep[k] = check(k, got[k], ref[k], fw[k])
    if dout is None:
        return rep
    bw = qarep_bwd_bounds(fw, y3, u, dout, M, inp["gamma_p"], inp["act"], inp["use_post_bn"], Ls, sizes, inp.get("acc0"), inp.get("ps", 1.0))
    amb = float(bw["amb"].double().mean())
    assert int(bw["amb"].sum()) <= AMBIGUOUS_MAX * bw["amb"].numel() + 2, f"{amb:.3f} of the ReLU masks are ambiguous under the bounds"
    rep["ambiguous"] = amb
    rep["dy3"] = check("dy3", _cat(got["dy3"]), _rows(inp, ref["dy3"]), _rows(inp, bw["dy3"]), bf16=True)
    rep["du"] = check("du", _cat(got["du"]), _rows(inp, ref["du"]), _rows(inp, bw["du"]), bf16=True)
    z = torch.zeros(C, dtype=F64, device=y3.device)
    acc0 = [t.double().to(y3.device) if t is not None else z for t in (inp.get("acc0") or (None,) * 5)]
    for i, nm in enumerate(("dgamma3", "dbeta3", "dab", "dgamma_p", "dbeta_p")):
        rep[nm] = check(nm, got["acc"][i], acc0[i] + ref[nm], bw["acc"][i])
    return rep


# ------------------------------------------------------------------------------------------------ recorder
REC_OPS = ("bn_act_fwd", "bn_act_bwd", "bn_act_infer", "qarep_fwd", "qarep_bwd", "channel_stats")
_RUNNING = {"bn_act_fwd": ("running_mean", "running_var"), "qarep_fwd": ("rm3", "rv3", "rmp", "rvp")}


def _clone(v):
    if torch.is_tensor(v):
        return v.detach().clone()
    if isinstance(v, (tuple, list)):
        return type(v)(_clone(t) for t in v)
    return v


def _pitch(t):
    """Channel pitch of an NHWC operand (the pixel stride), or None."""
    return t.stride(3) if torch.is_tensor(t) and t.dim() == 4 else None


# per-channel vectors the kernels read C entries of: _DualConvBnAct passes the first layer's parameters, running statistics and gradient
# slots for both layers, the second layer's following the first's in memory
_PER_CHANNEL = {"bn_act_fwd": ("gamma", "beta", "running_mean", "running_var"), "bn_act_bwd": ("gamma", "beta", "mean", "rstd", "dgamma", "dbeta"),
                "bn_act_infer": ("gamma", "beta", "running_mean", "running_var"),
                "qarep_fwd": ("gamma3", "beta3", "bias1a", "gamma_p", "beta_p", "rm3", "rv3", "rmp", "rvp"), "qarep_bwd": ("gamma3", "gamma_p")}


def _layer_channels(name, a):
    t = a.get("x") if name.startswith("bn_") or name == "channel_stats" else a.get("y3")
    return t.shape[1]


def _full(t, C):
    """The C-entry vector a kernel reads through t's pointer (t itself when it has C entries)."""
    if t is None or not torch.is_tensor(t) or t.dim() != 1 or t.numel() >= C:
        return t
    return t.as_strided((C,), (1,))


@contextlib.contextmanager
def record_bn_qarep():
    """Patches K.bn_act_fwd / bn_act_bwd / bn_act_infer / qarep_fwd / qarep_bwd / channel_stats for the block and yields the list of
    calls made in it: {"op", "a" (the bound arguments, cloned before the call), "pitch" (pixel stride of every 4-d argument), "ptr"
    (data_ptr of every tensor argument), "out" / "out_ptr" (the results), "after" (running statistics after the call)}."""
    import inspect

    from super_gradients_b200 import kernels as K

    orig = {n: getattr(K, n) for n in REC_OPS}
    calls = []

    def wrap(name):
        sig = inspect.signature(orig[name])

        def f(*args, **kw):
            torch.cuda.synchronize()
            b = sig.bind(*args, **kw)
            b.apply_defaults()
            C = _layer_channels(name, b.arguments)
            for k in _PER_CHANNEL.get(name, ()):
                b.arguments[k] = _full(b.arguments[k], C)
            if name == "qarep_bwd" and b.arguments.get("acc") is not None:
                b.arguments["acc"] = tuple(_full(t, C) for t in b.arguments["acc"])
            a = {k: (v if k == "sync" else _clone(v)) for k, v in b.arguments.items()}
            entry = {"op": name, "a": a, "pitch": {k: _pitch(v) for k, v in b.arguments.items() if torch.is_tensor(v) and v.dim() == 4},
                     "ptr": {k: v.data_ptr() for k, v in b.arguments.items() if torch.is_tensor(v)}}
            if name == "qarep_bwd" and b.arguments.get("out_grads") is not None:
                entry["pitch"]["out_grads"] = _pitch(b.arguments["out_grads"][0])
            out = orig[name](*args, **kw)
            torch.cuda.synchronize()
            outs = out if isinstance(out, tuple) else (out,)
            entry["out"] = _clone(tuple(_full(t, C) if torch.is_tensor(t) and t.dim() == 1 else t for t in outs))
            entry["out_ptr"] = [t.data_ptr() if torch.is_tensor(t) else None for t in outs]
            entry["after"] = {k: _clone(b.arguments[k]) for k in _RUNNING.get(name, ()) if b.arguments.get(k) is not None}
            calls.append(entry)
            return out

        return f

    for n in REC_OPS:
        setattr(K, n, wrap(n))
    try:
        yield calls
    finally:
        for n, fn in orig.items():
            setattr(K, n, fn)


def _run_steps(m, loss, opt_kw, x, t, lr, steps=1, recorder=record_bn_qarep):
    """`steps` eager TrainSteps (SGD) of m, with the calls `recorder()` (a context manager yielding its list of calls) keeps."""
    from super_gradients_b200.training.sg_trainer import TrainStep

    st = TrainStep(m, loss, "SGD", opt_kw, zero_wd_on_bias_and_bn=True)
    with recorder() as calls:
        for _ in range(steps):
            st.set_hyper_params(lr)
            st.run(x, t)
        torch.cuda.synchronize()
    return calls


def yolo_nas_s_step_record(batch=2, img=640, seed=0, recorder=record_bn_qarep):
    """One eager TrainStep of YOLO-NAS-S (80 classes) on random images with detection targets (plumbing_cases' driver), recorded."""
    from super_gradients_b200.training import models
    from super_gradients_b200.training.losses import PPYoloELoss, pad_targets_host

    torch.manual_seed(seed)
    m = models.get("yolo_nas_s", num_classes=80).cuda().train()
    g = torch.Generator().manual_seed(seed + 1)
    x = torch.randn(batch, 3, img, img, generator=g).cuda()
    rows = []
    for b in range(batch):
        for _ in range(6):
            cx, cy = (torch.rand(2, generator=g) * (img - 200) + 100).tolist()
            w, h = (torch.rand(2, generator=g) * 150 + 30).tolist()
            rows.append([b, int(torch.randint(0, 80, (1,), generator=g)), cx, cy, w, h])
    t = tuple(a.cuda() for a in pad_targets_host(torch.tensor(rows), batch, 16))
    return _run_steps(m, PPYoloELoss(num_classes=80, use_static_assigner=False), {"weight_decay": 1e-5, "momentum": 0.9}, x, t, 1e-3, recorder=recorder)


def resnet_step_record(name="resnet50", batch=2, img=224, seed=0, droppath_prob=0.0, recorder=record_bn_qarep):
    """One eager TrainStep of a ResNet (1000 classes), optionally with drop-path in every block, recorded."""
    from super_gradients_b200.training import models
    from super_gradients_b200.training.losses import CrossEntropyLoss

    torch.manual_seed(seed)
    m = models.get(name, num_classes=1000, arch_params={"droppath_prob": droppath_prob} if droppath_prob else None).cuda().train()
    g = torch.Generator().manual_seed(seed + 1)
    x, y = torch.randn(batch, 3, img, img, generator=g).cuda(), torch.randint(0, 1000, (batch,), generator=g).cuda()
    return _run_steps(m, CrossEntropyLoss(), {"weight_decay": 1e-4, "momentum": 0.9}, x, y, 0.1, recorder=recorder)


def qarep_alpha_step_record(batch=2, seed=0):
    """One TrainStep of a stack of QARepVGG blocks with use_alpha=True (plumbing_cases' driver), recorded."""
    import torch.nn as nn

    from super_gradients_b200.modules.qarepvgg_block import QARepVGGBlock

    torch.manual_seed(seed)
    m = nn.Sequential(
        QARepVGGBlock(32, 32, use_alpha=True),
        QARepVGGBlock(32, 64, stride=2, use_alpha=True, use_residual_connection=False),
        QARepVGGBlock(64, 64, use_alpha=True, use_1x1_bias=False),
        QARepVGGBlock(64, 48, use_alpha=True, use_residual_connection=False),
    ).cuda().train()
    g = torch.Generator().manual_seed(seed + 1)
    x, wt = torch.randn(batch, 32, 24, 24, generator=g).cuda(), torch.randn(batch, 48, 12, 12, generator=g).cuda()

    def loss(out, w):
        v = (out.float() * w).sum() / out.shape[0]
        return v, v.detach().reshape(1)

    return _run_steps(m, loss, {"momentum": 0.9}, x, wt, 1e-3)


# ------------------------------------------------------------------------------------------------ replay
def _act_name(act):
    return "none" if act in (None, "none") else act


def _pix_ss(ss, t):
    """Per-image drop-path scale [N] -> per-pixel column [M, 1] of the [N, C, H, W] tensor t."""
    return None if ss is None else ss.double().repeat_interleave(t.shape[2] * t.shape[3]).view(-1, 1)


def _zeros_if_none(v, C, dev):
    return v if v is not None else torch.zeros(C, dtype=torch.float32, device=dev)


def _find(calls, i, op, out_index, ptr):
    for j in range(i - 1, -1, -1):
        if calls[j]["op"] == op and calls[j]["out_ptr"][out_index] == ptr:
            return calls[j]
    raise AssertionError(f"call {i}: no earlier {op} produced its statistics")


def _bn_fwd_inp(r):
    a = r["a"]
    x = a["x"]
    C, dev = x.shape[1], x.device
    return {"x": [mc(x)], "residual": [mc(a["residual"])] if a["residual"] is not None else None, "ss": [_pix_ss(a["sample_scale"], x)] if a["sample_scale"] is not None else None,
            "gamma": a["gamma"], "beta": a["beta"], "rm": _zeros_if_none(a["running_mean"], C, dev), "rv": _zeros_if_none(a["running_var"], C, dev),
            "eps": f32(a["eps"]), "mom": f32(a["momentum"]), "act": _act_name(a["act"]), "stats_epilogue": a["stats"] is not None}


def _qarep_fwd_inp(r):
    a = r["a"]
    y3 = a["y3"]
    C, dev = y3.shape[1], y3.device
    z = lambda k: _zeros_if_none(a[k], C, dev)  # noqa: E731
    return {"y3": [mc(y3)], "u": [mc(a["u"])], "residual": [mc(a["residual"])] if a["residual"] is not None else None, "gamma3": a["gamma3"], "beta3": a["beta3"],
            "ab": a["bias1a"], "gamma_p": a["gamma_p"], "beta_p": a["beta_p"], "rm3": z("rm3"), "rv3": z("rv3"), "rmp": z("rmp"), "rvp": z("rvp"),
            "eps3": f32(a["eps3"]), "eps_post": f32(a["eps_post"]), "mom": f32(a["momentum"]), "act": _act_name(a["act"]), "use_post_bn": bool(a["use_post_bn"]),
            "res_alpha": float(a["res_alpha"]) if a["res_alpha"] is not None else None}


def replay_bn_qarep(calls, sms):
    """Checks every recorded call against the oracles and bounds; returns the set of launch paths seen."""
    seen = set()
    for i, r in enumerate(calls):
        a, op = r["a"], r["op"]
        if op in ("bn_act_fwd", "bn_act_bwd", "qarep_fwd", "qarep_bwd") and _act_name(a["act"]) not in ("none", "relu"):
            seen.add(op + ":act_" + str(a["act"]))
            continue
        if op == "bn_act_fwd":
            inp = _bn_fwd_inp(r)
            y, mean, rstd = r["out"]
            after = r["after"]
            got = {"y": [mc(y)], "mean": mean, "rstd": rstd, "rm": after.get("running_mean"), "rv": after.get("running_var")}
            verify_bn(inp, got, sms)
            seen.add("bn_fwd:" + ("epilogue_stats" if a["stats"] is not None else "fused_stats"))
            seen.update("bn_fwd:" + k for k in ("residual", "sample_scale") if a[k] is not None)
            seen.add("bn_fwd:act_" + inp["act"])
        elif op == "bn_act_bwd":
            f = _find(calls, i, "bn_act_fwd", 1, r["ptr"]["mean"])
            inp = _bn_fwd_inp(f)
            dy = a["dy"] if a["dy2"] is None else torch.cat([a["dy"], a["dy2"]], 1)
            C, dev = dy.shape[1], dy.device
            inp.update(dy=[mc(dy)], dgamma0=_zeros_if_none(a["dgamma"], C, dev), dbeta0=_zeros_if_none(a["dbeta"], C, dev),
                       read_y=bool(a["want_residual_grad"]) or a["beta"] is None or a["sample_scale"] is not None, act=_act_name(a["act"]))
            dx, dres, dg, db = r["out"]
            verify_bn(inp, {"dx": [mc(dx)], "dres": [mc(dres)] if dres is not None else None, "dgamma": dg, "dbeta": db}, sms)
            x_dense = r["pitch"]["x"] == C
            seen.add("bn_bwd:" + ("fused" if x_dense else "split_x_slice"))
            if a["dy2"] is not None:
                seen.add("bn_bwd:dy2")
            elif r["pitch"]["dy"] != C:
                seen.add("bn_bwd:dy_slice")
            seen.update("bn_bwd:" + k for k in ("sample_scale",) if a[k] is not None)
            if a["want_residual_grad"]:
                seen.add("bn_bwd:residual_grad")
            if a["beta"] is None:
                seen.add("bn_bwd:beta_none")
        elif op == "qarep_fwd":
            inp = _qarep_fwd_inp(r)
            out, coef = r["out"]
            aft = r["after"]
            verify_qarep(inp, {"out": [mc(out)], "coef": coef, **{k: aft.get(k) for k in ("rm3", "rv3", "rmp", "rvp")}}, sms)
            seen.add("qarep_fwd:" + ("post_bn" if inp["use_post_bn"] else "no_post_bn"))
            if a["residual"] is not None:
                seen.add("qarep_fwd:res_alpha")
            if a["bias1a"] is None:
                seen.add("qarep_fwd:ab_none")
            if r["pitch"]["y3"] != a["y3"].shape[1]:
                seen.add("qarep_fwd:y3_u_slices")
        elif op == "qarep_bwd":
            f = _find(calls, i, "qarep_fwd", 1, r["ptr"]["coef"])
            inp = _qarep_fwd_inp(f)
            C = a["y3"].shape[1]
            acc0 = a["acc"]
            inp.update(dout=[mc(a["dout"])], acc0=None if acc0 is None else [_zeros_if_none(t, C, a["y3"].device) for t in acc0])
            dy3, du, *acc = r["out"]
            verify_qarep(inp, {"dy3": [mc(dy3)], "du": [mc(du)], "acc": acc}, sms)
            seen.add("qarep_bwd:" + ("post_bn" if inp["use_post_bn"] else "no_post_bn"))
            if a["out_grads"] is not None and r["pitch"]["out_grads"] != C:
                seen.add("qarep_bwd:out_grads_slices")
            if r["pitch"]["dout"] != r["pitch"]["out"]:
                seen.add("qarep_bwd:dout_slice")
        elif op == "channel_stats":
            x = mc(a["x"])
            n, C = x.shape
            st = r["out"][0].double()[0]
            L = chain_len(n, C, sms) + 1
            for j, t in enumerate((x, x * x)):
                err = (st[j] - t.sum(0)).abs()
                assert bool((err <= gamma_n(L) * t.abs().sum(0) + (n + 8) * U64 * t.abs().sum(0)).all()), "channel_stats outside its bound"
            seen.add("channel_stats")
        elif op == "bn_act_infer":
            seen.add("bn_infer")
    return seen
