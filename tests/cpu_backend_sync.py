"""Test infrastructure: CPU stand-ins for the cross-rank (SyncBatchNorm) form of the BatchNorm / QARepVGG kernel wrappers, installed on
top of cpu_backend.install_training.  Calls without `sync` go to cpu_backend unchanged.

Written from the textbook SyncBatchNorm formulation, not from the kernels' algebra: the per-channel sums and the element count are
summed over the group by torch.distributed.nn's differentiable all_reduce, the statistics follow from them, and the backward pass is
torch autograd through that graph (its all_reduce backward sums the gradients of the statistics over the ranks, which is what
torch.nn.SyncBatchNorm's backward does).  The parameter gradients are therefore torch's per-rank ones, computed from local terms;
the kernels' scheme (global sums scaled by 1 / ranks) differs per rank and agrees after the data-parallel average.

Only tests may import this module.
"""
import torch
import torch.distributed.nn.functional as DF

import cpu_backend as CB
from super_gradients_b200 import kernels as K


def _reduce(sums, count, sync):
    """[k, C] fp64 local sums and the local element count -> the group's sums and count (differentiable)."""
    buf = torch.cat([sums.reshape(-1), torch.tensor([float(count)], dtype=torch.float64)])
    if sync.size > 1:
        buf = DF.all_reduce(buf, group=sync.group)
    return buf[:-1].view(sums.shape), buf[-1]


def _bn_sync(t, gamma, beta, eps, sync):
    """Train-mode BatchNorm of t (fp32 NCHW) over every rank's pixels; returns (out, mean, biased var, global count)."""
    td = t.double()
    s, m = _reduce(torch.stack([td.sum((0, 2, 3)), (td * td).sum((0, 2, 3))]), t.shape[0] * t.shape[2] * t.shape[3], sync)
    mean = s[0] / m
    var = (s[1] / m - mean * mean).clamp_min(0)
    out = (t - CB._cv(mean)) * CB._cv(torch.rsqrt(var + eps))
    if gamma is not None:
        out = out * CB._cv(gamma)
    if beta is not None:
        out = out + CB._cv(beta)
    return out, mean, var, m


def _running(rm, rv, mean, var, m, momentum):
    if rm is not None:
        m = float(m)
        rm.mul_(1 - momentum).add_(momentum * mean.detach().float())
        rv.mul_(1 - momentum).add_(momentum * (var.detach() * (m / max(m - 1, 1))).float())


def bn_act_fwd(x, stats, gamma, beta, running_mean, running_var, eps, momentum, act, residual=None, sample_scale=None, sync=None):
    if sync is None:
        return CB.bn_act_fwd(x, stats, gamma, beta, running_mean, running_var, eps, momentum, act, residual, sample_scale)
    n, c, h, w = x.shape
    gamma, beta, running_mean, running_var = CB._span(gamma, c), CB._span(beta, c), CB._span(running_mean, c), CB._span(running_var, c)
    with torch.no_grad():
        z, mean, var, m = _bn_sync(x.float(), gamma.float(), beta.float(), eps, sync)
    y = z if sample_scale is None else z * sample_scale.float().view(-1, 1, 1, 1)
    if residual is not None:
        y = y + residual.float()
    out = K.empty_nhwc(n, c, h, w, x.device)
    out.copy_(CB._bf16(CB._act(y, act)))
    _running(running_mean, running_var, mean, var, m, momentum)
    return out, mean.float(), torch.rsqrt(var + eps).float()


def bn_act_bwd(dy, x, y, gamma, mean, rstd, eps, act, want_residual_grad=False, dgamma=None, dbeta=None, beta=None, sample_scale=None, dy2=None, sync=None):
    if sync is None:
        return CB.bn_act_bwd(dy, x, y, gamma, mean, rstd, eps, act, want_residual_grad, dgamma, dbeta, beta, sample_scale, dy2)
    n, c, h, w = x.shape
    gamma, beta, dgamma, dbeta = CB._span(gamma, c), CB._span(beta, c), CB._span(dgamma, c), CB._span(dbeta, c)
    if dy2 is not None:
        dy = torch.cat([dy.float(), dy2.float()], 1)
    if y is None:  # the mask is recomputed from x, as the kernels do
        scale = gamma.float() * rstd
        y = x.float() * CB._cv(scale) + CB._cv(beta.float() - mean * scale)
    dz_res = CB._mask(dy, y, act)
    dz = dz_res if sample_scale is None else dz_res * sample_scale.float().view(-1, 1, 1, 1)
    xl, gl, bl = x.float().requires_grad_(True), gamma.detach().float().requires_grad_(True), beta.detach().float().requires_grad_(True)
    with torch.enable_grad():
        z, _, _, _ = _bn_sync(xl, gl, bl, eps, sync)
        gx, gg, gb = torch.autograd.grad(z, [xl, gl, bl], dz)
    dx = K.empty_nhwc(n, c, h, w, x.device)
    dx.copy_(CB._bf16(gx))
    dres = None
    if want_residual_grad:
        dres = K.empty_nhwc(n, c, h, w, x.device)
        dres.copy_(CB._bf16(dz_res))
    dgamma = K.zeros((c,), torch.float32, x.device) if dgamma is None else dgamma
    dbeta = K.zeros((c,), torch.float32, x.device) if dbeta is None else dbeta
    dgamma += gg
    dbeta += gb
    return dx, dres, dgamma, dbeta


def _qarep_pre_sync(y3, u, gamma3, beta3, bias1a, gamma_p, beta_p, eps3, eps_post, use_post_bn, sync):
    """bn3(y3) + u + alpha*b1 [-> post_bn], both BatchNorms over every rank's pixels (qarepvgg_block.py:184-204)."""
    b3, m3, v3, m = _bn_sync(y3, gamma3, beta3, eps3, sync)
    z = b3 + u
    if bias1a is not None:
        z = z + bias1a.view(1, -1, 1, 1)
    if not use_post_bn:
        return z, (m3, v3, None, None, m)
    zp, mz, vz, _ = _bn_sync(z, gamma_p, beta_p, eps_post, sync)
    return zp, (m3, v3, mz, vz, m)


def qarep_fwd(y3, u, gamma3, beta3, bias1a, gamma_p, beta_p, rm3, rv3, rmp, rvp, eps3, eps_post, momentum, act, use_post_bn=True, residual=None, res_alpha=None, sync=None):
    if sync is None:
        return CB.qarep_fwd(y3, u, gamma3, beta3, bias1a, gamma_p, beta_p, rm3, rv3, rmp, rvp, eps3, eps_post, momentum, act, use_post_bn, residual, res_alpha)
    n, c, h, w = y3.shape
    f = lambda t: None if t is None else t.detach().float()  # noqa: E731
    with torch.no_grad():
        pre, (m3, v3, mz, vz, m) = _qarep_pre_sync(y3.float(), u.float(), f(gamma3), f(beta3), f(bias1a), f(gamma_p), f(beta_p), eps3, eps_post, use_post_bn, sync)
    out = K.empty_nhwc(n, c, h, w, y3.device)
    res = CB._act(pre, act)
    if residual is not None:
        res = res_alpha.detach().float() * residual.float() + CB._bf16(res).float()
    out.copy_(CB._bf16(res))
    _running(rm3, rv3, m3, v3, m, momentum)
    if use_post_bn:
        _running(rmp, rvp, mz, vz, m, momentum)
    coef = torch.zeros((9, c), dtype=torch.float32)
    CB._QAREP_MASK[coef.data_ptr()] = (coef, pre > 0)  # the stand-in keeps its own activation mask (see cpu_backend.qarep_fwd)
    return out, coef


def qarep_bwd(dout, out, y3, u, coef, gamma3, gamma_p, eps3, eps_post, act, use_post_bn=True, acc=None, out_grads=None, sync=None):
    if sync is None:
        return CB.qarep_bwd(dout, out, y3, u, coef, gamma3, gamma_p, eps3, eps_post, act, use_post_bn, acc, out_grads)
    n, c, h, w = y3.shape
    kept = CB._QAREP_MASK.pop(coef.data_ptr())
    dpre = dout.float() * kept[1] if K.act_code(act) == K.ACT_RELU else dout.float()
    leaf = lambda t: t.detach().float().clone().requires_grad_(True)  # noqa: E731
    y3l, ul, g3l = leaf(y3), leaf(u), leaf(gamma3)
    b3l, abl = torch.zeros(c, requires_grad=True), torch.zeros(c, requires_grad=True)
    gpl = leaf(gamma_p) if use_post_bn else None
    bpl = torch.zeros(c, requires_grad=True) if use_post_bn else None
    with torch.enable_grad():
        pre, _ = _qarep_pre_sync(y3l, ul, g3l, b3l, abl, gpl, bpl, eps3, eps_post, use_post_bn, sync)
        wrt = [y3l, ul, g3l, b3l, abl] + ([gpl, bpl] if use_post_bn else [])
        grads = torch.autograd.grad(pre, wrt, dpre, allow_unused=True)
    gy3, gu, gg3, gb3, gab = grads[:5]
    ggp, gbp = (grads[5], grads[6]) if use_post_bn else (None, None)
    dy3, du = out_grads if out_grads is not None else (K.empty_nhwc(n, c, h, w, y3.device), K.empty_nhwc(n, c, h, w, y3.device))
    dy3.copy_(CB._bf16(gy3))
    du.copy_(CB._bf16(gu))
    acc = acc or (None,) * 5
    outs = []
    for slot, g in zip(acc, (gg3, gb3, gab, ggp, gbp)):
        t = slot if slot is not None else K.zeros((c,), torch.float32, y3.device)
        if g is not None:
            t += g
        outs.append(t)
    return (dy3, du, *outs)


_SYNC = dict(bn_act_fwd=bn_act_fwd, bn_act_bwd=bn_act_bwd, qarep_fwd=qarep_fwd, qarep_bwd=qarep_bwd)


def install(monkeypatch):
    """cpu_backend.install_training plus the cross-rank forms of the BatchNorm / QARepVGG wrappers."""
    CB.install_training(monkeypatch)
    for name, fn in _SYNC.items():
        monkeypatch.setattr(K, name, fn)
