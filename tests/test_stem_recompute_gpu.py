"""The train-mode QARepVGG stem without stored pre-activations (functional.STEM_RECOMPUTE, sgb_stem_qarep_*): every pass recomputes
[y3 | u] from the 32-channel patch tensor instead of reading the stored GEMM output.

Kernel level, at the stem widths of the recipes (32, 48, 64) and a pixel count that is not a multiple of the 128-pixel tile:
  - the recomputed [y3 | u] (sgb_stem_gemm) is bit-equal to what sgb_conv_fprop stores;
  - the moments and the backward sums are those of the fused stored-operand launches up to the order of fp64 atomics (the recompute
    passes sum in the same order), and coef, out, [dy3 | du] and the parameter gradients are bit-equal to theirs.
Block level, YOLO-NAS-S stem at the benchmark's size (32 x 3 x 640²) and a ragged size: output, parameter gradients and running
statistics of the two paths, and the launch counter of the recompute path.
"""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _bits(t):
    return t.contiguous().view(torch.int16) if t.dtype == torch.bfloat16 else t.contiguous().view(torch.int32)


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


@pytest.mark.parametrize("kout,act", [(48, "relu"), (32, "relu"), (64, "none")])
def test_stem_passes_match_the_stored_operand_passes(kout, act):
    from super_gradients_b200 import kernels as K
    from super_gradients_b200 import lib as L

    torch.manual_seed(kout)
    n, h, w = 3, 35, 27  # 2835 pixels: the last 128-pixel tile is ragged
    x = torch.randn(n, 3, 2 * h, 2 * w, device=DEV)
    xp = K.stem_patches(x, 3, 2, 1, 32)
    kf = torch.zeros(2 * kout, 1, 1, 32, device=DEV)
    kf[..., :27] = 0.3 * torch.randn(2 * kout, 1, 1, 27, device=DEV)
    kf = kf.bfloat16().contiguous()
    ycat = K.conv_fprop(xp, kf, 2 * kout, 1, 1, 1, 0)
    launches = L.load().sgb_stem_recompute_launches()
    assert torch.equal(_bits(K.stem_gemm(xp, kf, kout)), _bits(ycat))
    y3, u = ycat[:, :kout], ycat[:, kout:]

    f = lambda s=1.0, o=0.0: (o + s * torch.randn(kout, device=DEV)).float()  # noqa: E731
    g3, b3, bias1, gp, bp = f(0.2, 1.0), f(0.1), f(0.1), f(0.2, 1.0), f(0.1)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = K._ptr
    ds = K._stem_desc(xp, kf, kout, 1e-3, 0.03, act)
    ds.pitcho = kout
    dq = K.qarep_desc(y3, u, K.empty_nhwc(n, kout, h, w, DEV), 1e-3, 1e-3, 0.03, act, True)

    # forward: against the fused stored-operand launch (moments, grid barrier, apply); the sums agree up to the order of the fp64
    # atomics (the fp32 partial sums are the same), the coefficients and the output bit for bit
    mom = torch.zeros(5, kout, dtype=torch.float64, device=DEV)
    mom_ref = torch.zeros(5, kout, dtype=torch.float64, device=DEV)
    out, out_ref = K.empty_nhwc(n, kout, h, w, DEV), K.empty_nhwc(n, kout, h, w, DEV)
    coef, coef_ref = torch.empty(9, kout, device=DEV), torch.empty(9, kout, device=DEV)
    prm = [p(t) for t in (g3, b3, bias1, gp, bp)] + [None] * 4
    L.call("sgb_qarep_fwd_fused", ctypes.byref(dq), p(y3), p(u), p(mom_ref), *prm, p(out_ref), p(coef_ref), st)
    L.call("sgb_stem_qarep_moments", ctypes.byref(ds), p(xp), p(kf), p(mom), st)
    L.call("sgb_stem_qarep_fwd", ctypes.byref(ds), p(xp), p(kf), p(mom), *prm, p(out), p(coef), st)
    for r in range(5):
        assert _rel(mom[r], mom_ref[r]) <= 1e-12, (r, _rel(mom[r], mom_ref[r]))
    assert torch.equal(_bits(coef), _bits(coef_ref)) and torch.equal(_bits(out), _bits(out_ref))

    # backward: against the fused stored-operand launch, the same way
    dout = (0.1 * torch.randn(n, kout, h, w, device=DEV)).bfloat16().contiguous(memory_format=torch.channels_last)
    ds.pitcho = dq.pitcho = kout
    ds.pitch3 = ds.pitchu = 2 * kout
    res = []
    for stem in (True, False):
        sums = torch.zeros(3, kout, dtype=torch.float64, device=DEV)
        dcat = K.empty_nhwc(n, 2 * kout, h, w, DEV)
        grads = [torch.zeros(kout, device=DEV) for _ in range(5)]
        if stem:
            L.call("sgb_stem_qarep_bwd_reduce", ctypes.byref(ds), p(dout), p(xp), p(kf), p(coef), p(sums), st)
            L.call("sgb_stem_qarep_bwd_apply", ctypes.byref(ds), p(dout), p(xp), p(kf), p(coef), p(sums), p(g3), p(gp), p(dcat), p(dcat[:, kout:]), *[p(t) for t in grads], st)
        else:
            L.call("sgb_qarep_bwd_fused", ctypes.byref(dq), p(dout), p(y3), p(u), p(coef), p(sums), p(g3), p(gp), p(dcat), p(dcat[:, kout:]), *[p(t) for t in grads], st)
        res.append((sums, dcat, grads))
    for r in range(3):
        assert _rel(res[0][0][r], res[1][0][r]) <= 1e-12, (r, _rel(res[0][0][r], res[1][0][r]))
    assert torch.equal(_bits(res[0][1]), _bits(res[1][1]))
    for a, b in zip(res[0][2], res[1][2]):
        assert torch.equal(_bits(a), _bits(b))
    torch.cuda.synchronize()
    assert L.load().sgb_stem_recompute_launches() == launches + 5


@pytest.mark.parametrize("shape", [(32, 3, 640, 640), (3, 3, 70, 54)], ids=["config2", "ragged"])
def test_stem_block_recompute_matches_the_stored_path(monkeypatch, shape):
    from super_gradients_b200 import functional as SF
    from super_gradients_b200 import lib as L
    from super_gradients_b200.modules import QARepVGGBlock

    torch.manual_seed(0)
    x = torch.randn(*shape, device=DEV)
    blk0 = QARepVGGBlock(3, 48, stride=2, use_residual_connection=False)
    with torch.no_grad():
        for q in blk0.parameters():
            q.add_(0.05 * torch.randn_like(q))

    def run(recompute):
        monkeypatch.setattr(SF, "STEM_RECOMPUTE", [recompute])
        blk = QARepVGGBlock(3, 48, stride=2, use_residual_connection=False)
        blk.load_state_dict(blk0.state_dict())
        blk = blk.to(DEV).train()
        assert SF.stem_patches_supported(blk, x)
        n0 = L.load().sgb_stem_recompute_launches()
        y = blk(x)
        gy = torch.linspace(-1, 1, y.numel(), device=DEV).reshape(y.shape).bfloat16()
        y.backward(gy)
        torch.cuda.synchronize()
        assert L.load().sgb_stem_recompute_launches() - n0 == (4 if recompute else 0)
        return y.detach(), {k: q.grad.clone() for k, q in blk.named_parameters() if q.grad is not None}, {k: v.clone() for k, v in blk.state_dict().items() if "running" in k}

    y0, g0, r0 = run(False)
    y1, g1, r1 = run(True)
    # the recompute passes sum the statistics in the stored path's order: the same output bit for bit, the same statistics and
    # BatchNorm gradients up to the order of fp64 atomics.  The filter gradients come from the stem's weight-gradient kernel, whose
    # CTAs add their partial sums with fp32 reductions in arrival order, which changes from run to run (3.9e-5 between the two paths
    # at 32 x 640², with [dy3 | du] bit-equal).
    nd = int((_bits(y1) != _bits(y0)).sum())
    print(f"{shape}: out differs in {nd} of {y0.numel()} elements")
    assert nd == 0
    assert set(g0) == set(g1)
    for k in g0:
        print(f"  {k}: rel {_rel(g1[k], g0[k]):.2e}")
        assert _rel(g1[k], g0[k]) <= (2e-4 if k.endswith("weight") and "bn" not in k else 1e-6), (k, _rel(g1[k], g0[k]))
    for k in r0:
        print(f"  {k}: rel {_rel(r1[k], r0[k]):.2e}")
        assert _rel(r1[k], r0[k]) <= 1e-6, (k, _rel(r1[k], r0[k]))
