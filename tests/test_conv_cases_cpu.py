"""The convolution oracles, integer cases, route mirror and bounds of tests/conv_cases.py on the CPU: the oracles agree with torch's own
double-precision convolution gradients, every integer case stays under its cap and sums exactly in fp32 in any order, the route mirror
reaches every row of the route table, the fp32 transcription of the kernels passes the checks the GPU suite applies, and each planted
defect fails at least one of them."""
import random

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import conv_cases as CC

F64 = torch.float64


def _g(seed):
    return torch.Generator().manual_seed(seed)


@pytest.mark.parametrize("shape", [(2, 16, 9, 11, 24, 3, 1, 1), (2, 8, 13, 12, 16, 3, 2, 1), (1, 16, 10, 10, 32, 1, 2, 0), (2, 8, 15, 14, 8, 7, 2, 3),
                                   (1, 8, 8, 10, 16, 2, 2, 0), (1, 16, 7, 9, 16, 3, 1, 0)])
def test_oracles_match_torch(shape):
    n, c, h, w, k, r, s, p = shape
    g = _g(sum(shape))
    x = torch.randn(n, c, h, w, generator=g, dtype=F64)
    wt = torch.randn(k, c, r, r, generator=g, dtype=F64)
    y = F.conv2d(x, wt, stride=s, padding=p)
    dy = torch.randn(y.shape, generator=g, dtype=F64)
    torch.testing.assert_close(CC.fprop_ref(x, wt, s, p), y)
    sc, sh, res = torch.rand(k, generator=g, dtype=F64), torch.randn(k, generator=g, dtype=F64), torch.randn(y.shape, generator=g, dtype=F64)
    z = y * sc.view(1, -1, 1, 1) + sh.view(1, -1, 1, 1) + res
    torch.testing.assert_close(CC.fprop_ref(x, wt, s, p, sc, sh, res, "relu"), z.clamp_min(0))
    torch.testing.assert_close(CC.fprop_ref(x, wt, s, p, sc, sh, res, "silu"), F.silu(z))
    dx = torch.nn.grad.conv2d_input(x.shape, wt, dy, stride=s, padding=p)
    old = torch.randn(x.shape, generator=g, dtype=F64)
    torch.testing.assert_close(CC.dgrad_ref(dy, wt, x.shape, s, p), dx)
    torch.testing.assert_close(CC.dgrad_ref(dy, wt, x.shape, s, p, old, accumulate=True), dx + old)
    dw = torch.nn.grad.conv2d_weight(x, wt.shape, dy, stride=s, padding=p).permute(0, 2, 3, 1)
    dw_old = torch.randn(dw.shape, generator=g, dtype=F64)
    torch.testing.assert_close(CC.wgrad_ref(x, dy, r, r, s, p), dw)
    torch.testing.assert_close(CC.wgrad_ref(x, dy, r, r, s, p, dw_old), dw_old + dw)
    if r == 3 and s == 1 and p == 1 and k > 16:
        got = CC.wgrad_ref(x, dy, 3, 3, 1, 1, dw_old, centre_from=16)
        torch.testing.assert_close(got[:16], dw_old[:16] + dw[:16])
        torch.testing.assert_close(got[16:, 1, 1], dw_old[16:, 1, 1] + dw[16:, 1, 1])
        off = torch.ones(3, 3, dtype=torch.bool)
        off[1, 1] = False
        torch.testing.assert_close(got[16:][:, off], dw_old[16:][:, off])


def test_convt2x2_oracle_is_the_scatter():
    g = _g(3)
    x = torch.randn(2, 16, 4, 5, generator=g, dtype=F64)
    w = torch.randn(16, 24, 2, 2, generator=g, dtype=F64)
    b = torch.randn(24, generator=g, dtype=F64)
    want = torch.zeros(2, 24, 8, 10, dtype=F64)
    for dh in range(2):
        for dw in range(2):
            want[:, :, dh::2, dw::2] = torch.einsum("nchw,co->nohw", x, w[:, :, dh, dw]) + b.view(1, -1, 1, 1)
    torch.testing.assert_close(CC.convt2x2_ref(x, w, b), want)


def _small(c):
    d = CC.desc_of(c)
    return c["N"] * max(c["C"], c["K"]) * max(c["H"] * c["W"], d["P"] * d["Q"]) <= 400_000


INT_CASES = [c for c in CC.all_cases() if _small(c)][::3]


@pytest.mark.parametrize("case", INT_CASES, ids=[c["id"] for c in INT_CASES])
def test_integer_case_meets_cap_and_sums_exactly_in_any_order(case):
    g = _g(7)
    o = CC.case_operands(case, False, g, "cpu")
    assert o["cap_seen"] <= case["cap"]
    # the products of a few outputs, summed in fp32 in shuffled orders, rounding to nearest and truncating: always the exact sum
    op = case["op"]
    if op == "fprop" or op == "wgrad":
        A = CC._im2col(o["x"], case["R"], case["R"], case["stride"], case["pad"]).double().reshape(-1, case["R"] ** 2 * case["C"])
        B = (o["w"].permute(0, 2, 3, 1).reshape(case["K"], -1) if op == "fprop" else o["dy"].permute(0, 2, 3, 1).reshape(-1, case["K"]))
        terms = (lambda i, j: A[i] * B[j]) if op == "fprop" else (lambda i, j: A[:, i] * B[:, j])
        ni, nj = (A.shape[0], B.shape[0]) if op == "fprop" else (A.shape[1], B.shape[1])
    else:
        return  # dgrad / convt2x2 reduce over the same kind of integer products; their caps are asserted above
    rng = random.Random(case["id"])
    for _ in range(8):
        i, j = rng.randrange(ni), rng.randrange(nj)
        t = terms(i, j).numpy()
        exact = float(t.sum())
        for _ in range(3):
            order = np.random.default_rng(rng.randrange(2**32)).permutation(len(t))
            s_rn, s_tr = np.float32(0), np.float32(0)
            for v in t[order]:
                s_rn = np.float32(s_rn + np.float32(v))
                q = float(s_tr) + float(v)
                s_tr = np.float32(np.trunc(q)) if abs(q) < 2**24 else np.float32(q)
                assert float(s_tr) == q, "a partial sum needed more than fp32's 24 bits"
            assert float(s_rn) == exact and float(s_tr) == exact


def test_route_mirror_covers_the_table():
    missing, seen = CC.missing_routes(CC.all_cases())
    assert not missing, f"no case reaches {missing}"


def test_route_mirror_rules():
    m = lambda **kw: CC.route(kw.pop("op"), CC.desc_of(CC.make_case(kw.pop("op2", "fprop"), **kw)), {})  # noqa: E731
    assert CC.halo_tiles_fit(40, 40) and CC.halo_tiles_fit(60, 62) and not CC.halo_tiles_fit(28, 28) and not CC.halo_tiles_fit(7, 7)
    assert [CC.pick_bn(n) for n in (8, 40, 100, 192, 256, 320, 384)] == [16, 48, 128, 96, 128, 64, 128]
    assert m(op="fprop", n=2, c=64, h=40, w=40, k=64).kernel == "conv3x3_halo_kernel"
    assert m(op="fprop", n=2, c=64, h=28, w=28, k=64).kernel == "conv_wgmma_kernel"
    assert m(op="fprop", n=2, c=24, h=28, w=28, k=64).engine == "mma"
    r = m(op="dgrad", op2="dgrad", n=2, c=64, h=40, w=40, k=64, stride=2)
    assert r.launches == 4 and r.variant.startswith("parity4_")
    assert m(op="dgrad", op2="dgrad", n=2, c=64, h=41, w=40, k=64, stride=2).engine == "mma"
    assert m(op="wgrad", op2="wgrad", n=2, c=24, h=16, w=16, k=160).variant == "bmw128"
    assert m(op="wgrad", op2="wgrad", n=2, c=24, h=16, w=16, k=96).variant == "bmw32"


# ------------------------------------------------------------------------------------------------ transcription and defects
DEFECT_CASES = [
    CC.make_case("fprop", 1, 32, 12, 12, 32, stats=8, scale=True, shift=True, residual=True, act="relu"),
    CC.make_case("fprop", 1, 64, 10, 10, 32, stride=2, shift=True, act="silu"),
    CC.make_case("dgrad", 1, 16, 12, 12, 32, stride=2, accumulate=True),
    CC.make_case("dgrad", 1, 16, 12, 10, 32, accumulate=True),
    CC.make_case("wgrad", 1, 16, 10, 10, 32, centre_from=16),
]


def _run_t(c, real, mut, seed=11):
    o = CC.case_operands(c, real, _g(seed), "cpu")
    got = CC.TRANSCRIPTION[c["op"]](c, o, mut)
    d = CC.desc_of(c)
    chain = c["N"] * d["P"] * d["Q"] + 1 if c["op"] == "wgrad" else None
    CC.VERIFY[c["op"]](c, o, got, exact=not real, chain=chain)


@pytest.mark.parametrize("real", [False, True], ids=["integer", "real"])
@pytest.mark.parametrize("case", DEFECT_CASES, ids=[c["id"] for c in DEFECT_CASES])
def test_transcription_passes_the_checks(case, real):
    _run_t(case, real, None)


@pytest.mark.parametrize("mut", CC.MUTATIONS)
def test_planted_defect_fails_a_check(mut):
    caught = []
    for c in DEFECT_CASES:
        for real in (False, True):
            try:
                _run_t(c, real, mut)
            except AssertionError as e:
                caught.append((c["id"], real, str(e)[:80]))
    assert caught, f"defect {mut} passed every check"


LAYER_CASES = [
    CC.make_case("fprop", 1, 64, 40, 40, 64, scale=True, shift=True, act="relu", stats=8),  # YOLO-NAS stage 2 block
    CC.make_case("fprop", 1, 96, 40, 40, 192, stride=2, shift=True, act="relu"),  # YOLO-NAS downsample
    CC.make_case("fprop", 1, 256, 14, 14, 256, stats=8),  # ResNet-50 layer3 3x3
    CC.make_case("fprop", 1, 1024, 14, 14, 256, r=1, stats=8),  # ResNet-50 layer3 1x1 reduce
    CC.make_case("fprop", 1, 64, 20, 20, 128, shift=True, residual=True, act="silu"),
    CC.make_case("dgrad", 1, 96, 40, 40, 192, stride=2, accumulate=True),
    CC.make_case("dgrad", 1, 128, 28, 28, 128, accumulate=True),
    CC.make_case("wgrad", 1, 64, 40, 40, 64),
    CC.make_case("wgrad", 1, 128, 28, 28, 128, centre_from=64),
]


@pytest.mark.parametrize("case", LAYER_CASES, ids=[c["id"] for c in LAYER_CASES])
def test_bounds_hold_for_the_transcription_at_layer_shapes(case):
    _run_t(case, True, None, seed=5)
