"""The halo-tile weight-gradient kernel of 3x3 / stride-1 convolutions (wgrad3x3_halo_kernel) against the per-tap wgmma kernel
it replaces on those shapes (wgrad_wgmma_kernel, selected through the library's test-only sgb_conv_wgrad_force_im2col switch).
Both add fp32 partial sums into dW with atomics in no fixed order, so results agree within fp32 reordering, bounded by 1e-5 x the
same gradient computed over |x| and |dy| (the tolerance of test_conv_zero_taps_gpu.py).  dW starts non-zero, so entries a kernel
does not write keep their value, and both engines must leave the same entries untouched."""
import pytest
import torch

from super_gradients_b200 import kernels as K
from super_gradients_b200 import lib

pytestmark = pytest.mark.gpu

# (C, K, H, W) of the 3x3 / stride-1 weight gradients the shape rule takes in bench configurations 2 (YOLO-NAS-S), 3 (YOLO-NAS-M)
# and 4 (ResNet-50), run at batch 2 (the batch only changes the number of tiles), then maps that are not multiples of 8
MODEL_SHAPES = [(32, 64, 160, 160), (64, 128, 80, 80), (96, 192, 40, 40), (48, 96, 80, 80), (64, 128, 40, 40), (64, 64, 40, 40),
                (128, 256, 40, 40), (64, 128, 160, 160), (128, 128, 80, 80), (192, 192, 40, 40), (256, 256, 40, 40),
                (96, 192, 80, 80), (192, 384, 40, 40), (64, 64, 56, 56)]  # fmt: skip
RAGGED_SHAPES = [(32, 64, 60, 62), (48, 96, 62, 60), (16, 32, 46, 39)]
SHAPES = MODEL_SHAPES + RAGGED_SHAPES
IDS = ["c%d_k%d_%dx%d" % s for s in SHAPES]
# weight gradients the per-tap kernel keeps: 20² / 28² / 14² maps (8 x 8 tiles waste MMA rows), 1x1, stride 2
OTHER = [(64, 64, 20, 20, 3, 1), (128, 128, 28, 28, 3, 1), (256, 256, 14, 14, 3, 1), (64, 128, 40, 40, 1, 1), (64, 128, 40, 40, 3, 2)]


def _lib():
    return lib.load()


def _nhwc(n, c, h, w, g, extra=0):
    """bf16 NCHW view of channels-last storage; extra > 0: channels [extra, extra + c) of a (c + 2 extra)-channel buffer."""
    t = torch.randn(n, h, w, c + 2 * extra, generator=g, device="cuda").to(torch.bfloat16)
    return t[..., extra : extra + c].permute(0, 3, 1, 2)


def _run(x, dy, dw0, R, stride, centre_from, force):
    L = _lib()
    dw = dw0.clone()
    L.sgb_conv_wgrad_force_im2col(1 if force else 0)
    try:
        s0, h0 = L.sgb_sm100_launches(), L.sgb_conv_wgrad_halo_launches()
        K.conv_wgrad(x, dy, R, R, stride, R // 2, dw_krsc=dw, centre_from=centre_from)
        torch.cuda.synchronize()
        s1, h1 = L.sgb_sm100_launches(), L.sgb_conv_wgrad_halo_launches()
    finally:
        L.sgb_conv_wgrad_force_im2col(0)
    return dw, s1 - s0, h1 - h0


def _check(c, k, h, w, n=2, centre_from=0, extra=0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = _nhwc(n, c, h, w, g, extra)
    dy = _nhwc(n, k, h, w, g, extra)
    dw0 = torch.randn(k, 3, 3, c, generator=g, device="cuda")
    ref, s_ref, h_ref = _run(x, dy, dw0, 3, 1, centre_from, True)
    out, s_out, h_out = _run(x, dy, dw0, 3, 1, centre_from, False)
    assert (s_ref, h_ref) == (1, 0), "the forced call did not run on wgrad_wgmma_kernel"
    assert (s_out, h_out) == (1, 1), "the halo-tile wgrad kernel did not serve the call"
    cl = torch.channels_last
    scale = K.conv_wgrad(x.abs().contiguous(memory_format=cl), dy.abs().contiguous(memory_format=cl), 3, 3, 1, 1)
    tol = 1e-5 * scale + 1e-6
    assert bool(((out - ref).abs() <= tol).all()), float((out - ref).abs().max())
    if centre_from:
        # the off-centre entries of rows past the 64-row block that holds row centre_from - 1 keep their value
        first_unwritten = (centre_from + 63) // 64 * 64
        if first_unwritten < k:
            keep = torch.ones(k - first_unwritten, 3, 3, c, dtype=torch.bool, device="cuda")
            keep[:, 1, 1] = False
            assert bool((out[first_unwritten:][keep] == dw0[first_unwritten:][keep]).all())


@pytest.mark.parametrize("shape", SHAPES, ids=IDS)
def test_wgrad_halo_matches_per_tap_kernel(shape):
    _check(*shape)


@pytest.mark.parametrize("shape", SHAPES, ids=IDS)
def test_wgrad_halo_centre_from(shape):
    c, k, h, w = shape
    _check(c, k, h, w, centre_from=k // 2, seed=1)


@pytest.mark.parametrize("shape", [(32, 64, 160, 160), (64, 128, 40, 40), (48, 96, 62, 60)], ids=["c32_k64", "c64_k128", "c48_k96_ragged"])
def test_wgrad_halo_channel_slices(shape):
    c, k, h, w = shape
    _check(c, k, h, w, centre_from=k // 2, extra=16, seed=2)


def test_wgrad_halo_many_images():
    # 5 images of 7 x 6 tiles over ~132 tile ranges: ranges start and end inside images
    _check(32, 64, 56, 48, n=5, seed=3)
    _check(64, 128, 40, 40, n=7, centre_from=64, seed=4)


@pytest.mark.parametrize("shape", OTHER, ids=["20x20", "28x28", "14x14", "1x1", "stride2"])
def test_other_weight_gradients_stay_on_per_tap_kernel(shape):
    c, k, h, w, r, stride = shape
    g = torch.Generator(device="cuda").manual_seed(5)
    x = _nhwc(2, c, h, w, g)
    p = (h + 2 * (r // 2) - r) // stride + 1
    dy = _nhwc(2, k, p, p, g)
    dw0 = torch.zeros(k, r, r, c, device="cuda")
    _, s, hl = _run(x, dy, dw0, r, stride, 0, False)
    assert (s, hl) == (1, 0)
