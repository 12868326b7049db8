"""Skipping the zero taps of folded QARepVGG filters (SgbConvDesc.centre_from) changes no result.

A folded filter [K3 ; centre(alpha * K1 + I)] has 2K output channels whose rows [K, 2K) are zero except at the centre tap.  Each
call below runs twice on the same inputs, with centre_from = K and with centre_from = 0 (every tap):
  - fprop and dgrad: the bf16 outputs equal bit for bit (-0 and +0 count as equal: a dropped product by an exact zero can turn one
    into the other), the BatchNorm statistics equal up to the order of the fp64 atomics that combine CTAs;
  - wgrad: rows [0, K) on all taps and the centre tap of rows [K, 2K) equal within fp32 reordering -- the kernel adds per-CTA
    partial sums with fp32 atomics in no fixed order, so two runs with the same setting differ the same way -- bounded by
    1e-5 x the same gradient computed over |x| and |dy|;
  - the same engine (halo-tile or im2col kernel) serves both calls.
Shapes: the folded blocks (C -> 2K, map) of YOLO-NAS-S / -M training at batch 2, plus ragged maps (60 x 62 gives edge tiles in
the halo kernel; 20 x 28 stays on the im2col kernel), each also with the im2col kernel forced."""
import pytest
import torch

from super_gradients_b200 import kernels as K
from super_gradients_b200 import lib

pytestmark = pytest.mark.gpu

# (C, 2K, H, W): the folded blocks of YOLO-NAS-S (bench config 2) and YOLO-NAS-M (config 3), then ragged maps
MODEL_SHAPES = [(32, 64, 160, 160), (48, 96, 80, 80), (64, 128, 80, 80), (64, 128, 40, 40), (96, 192, 40, 40),
                (64, 128, 160, 160), (96, 96, 80, 80), (128, 128, 80, 80), (192, 192, 40, 40)]  # fmt: skip
RAGGED_SHAPES = [(32, 64, 60, 62), (48, 96, 60, 62), (96, 192, 60, 62), (48, 96, 20, 28), (64, 128, 20, 28), (96, 192, 20, 28)]
SHAPES = MODEL_SHAPES + RAGGED_SHAPES
IDS = ["c%d_k%d_%dx%d" % s for s in SHAPES]


def _lib():
    return lib.load()


def _nhwc(n, c, h, w, g):
    return torch.randn(n, h, w, c, generator=g, device="cuda").to(torch.bfloat16).permute(0, 3, 1, 2)


def _folded_filter(c, k2, g):
    """fp32 OIHW [2K, C, 3, 3]: rows [0, K) a 3x3 filter, rows [K, 2K) a 1x1 filter at the centre tap."""
    kk = k2 // 2
    w = torch.zeros(k2, c, 3, 3, device="cuda")
    w[:kk] = torch.randn(kk, c, 3, 3, generator=g, device="cuda") * 0.05
    w[kk:, :, 1, 1] = torch.randn(k2 - kk, c, generator=g, device="cuda") * 0.2
    return w


def _arms(fn, kk, force_im2col):
    """(fn(0), fn(kk)), after checking that the same engine served both calls."""
    L = _lib()
    L.sgb_conv_force_im2col(1 if force_im2col else 0)
    out = []
    try:
        for cf in (0, kk):
            s0, h0 = L.sgb_sm100_launches(), L.sgb_conv_halo_launches()
            r = fn(cf)
            torch.cuda.synchronize()
            out.append((r, L.sgb_sm100_launches() - s0, L.sgb_conv_halo_launches() - h0))
    finally:
        L.sgb_conv_force_im2col(0)
    (_, s_full, h_full), (_, s_skip, h_skip) = out
    assert s_full == s_skip >= 1 and h_full == h_skip, "a different engine served the call with centre_from"
    return out[0][0], out[1][0]


def _equal(a, b):
    return bool((a.float() == b.float()).all())  # -0 == +0


def _stats_close(a, b, y):
    a, b = a.sum(0), b.sum(0)
    yf = y.double()
    bound = torch.stack([yf.abs().sum((0, 2, 3)), (yf * yf).sum((0, 2, 3))]) * 1e-9
    return bool(((a - b).abs() <= bound + 1e-12).all())


@pytest.mark.parametrize("force_im2col", [False, True], ids=["auto", "im2col"])
@pytest.mark.parametrize("shape", SHAPES, ids=IDS)
def test_fprop_skips_zero_taps(shape, force_im2col):
    c, k2, h, w = shape
    g = torch.Generator(device="cuda").manual_seed(11)
    x = _nhwc(2, c, h, w, g)
    krsc, _ = K.weight_prepare(_folded_filter(c, k2, g))

    def run(cf):
        st = K.new_stats(k2, "cuda")
        return K.conv_fprop(x, krsc, k2, 3, 3, 1, 1, stats=st, centre_from=cf), st

    (y0, s0), (y1, s1) = _arms(run, k2 // 2, force_im2col)
    assert _equal(y0, y1)
    assert _stats_close(s0, s1, y0)


@pytest.mark.parametrize("force_im2col", [False, True], ids=["auto", "im2col"])
@pytest.mark.parametrize("shape", SHAPES, ids=IDS)
def test_dgrad_skips_zero_taps(shape, force_im2col):
    c, k2, h, w = shape
    g = torch.Generator(device="cuda").manual_seed(12)
    dy = _nhwc(2, k2, h, w, g)
    _, crsk = K.weight_prepare(_folded_filter(c, k2, g))

    def run(cf):
        return K.conv_dgrad(dy, crsk, (2, c, h, w), 3, 3, 1, 1, centre_from=cf)

    dx0, dx1 = _arms(run, k2 // 2, force_im2col)
    assert _equal(dx0, dx1)


@pytest.mark.parametrize("shape", SHAPES, ids=IDS)
def test_wgrad_skips_unwanted_taps(shape):
    c, k2, h, w = shape
    kk = k2 // 2
    g = torch.Generator(device="cuda").manual_seed(13)
    x = _nhwc(2, c, h, w, g)
    dy = _nhwc(2, k2, h, w, g)

    def run(cf):
        return K.conv_wgrad(x, dy, 3, 3, 1, 1, centre_from=cf)

    full, skip = _arms(run, kk, False)
    scale = K.conv_wgrad(x.abs(), dy.abs(), 3, 3, 1, 1)  # sum over pixels of |dy| |x|: bounds the fp32 reordering error
    tol = 1e-5 * scale + 1e-6
    assert bool(((full[:kk] - skip[:kk]).abs() <= tol[:kk]).all())
    centre = (slice(kk, None), 1, 1)
    assert bool(((full[centre] - skip[centre]).abs() <= tol[centre]).all())
    # the off-centre entries of rows [K, 2K) past the 64-row block that holds row K are never written
    first_unwritten = (kk + 63) // 64 * 64
    if first_unwritten < k2:
        rest = skip[first_unwritten:].clone()
        rest[:, 1, 1] = 0
        assert bool((rest == 0).all())


def test_centre_from_is_refused_where_it_does_not_apply():
    g = torch.Generator(device="cuda").manual_seed(14)
    x = _nhwc(1, 32, 16, 16, g)
    krsc, _ = K.weight_prepare(_folded_filter(32, 64, g))
    for cf in (8, 64, 80, -16):
        with pytest.raises(lib.SgbError):
            K.conv_fprop(x, krsc, 64, 3, 3, 1, 1, centre_from=cf)
    k1, _ = K.weight_prepare(torch.randn(64, 32, 1, 1, generator=g, device="cuda"))
    with pytest.raises(lib.SgbError):
        K.conv_fprop(x, k1, 64, 1, 1, 1, 0, centre_from=32)
