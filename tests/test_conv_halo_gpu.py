"""The halo-tile kernel of 3x3 / stride-1 convolutions (conv3x3_halo_kernel) against the im2col wgmma kernel it replaces on
those shapes: the bf16 outputs must be equal bit for bit (-0 and +0 count as equal: the im2col kernel's zero-filled k16 steps
past C = 48 / 96 can turn one into the other), the BatchNorm statistics equal up to fp32 summation order.  The im2col engine is
selected through the library's test-only sgb_conv_force_im2col switch."""
import pytest
import torch

from super_gradients_b200 import kernels as K
from super_gradients_b200 import lib

pytestmark = pytest.mark.gpu

# (C_in, C_out, H, W) of the 3x3 / stride-1 convolutions of the bench configurations (YOLO-NAS-S / M, ResNet-50, YOLO-NAS-POSE-L
# blocks), run at batch 2: the batch only changes the number of tiles
MODEL_SHAPES = [
    (32, 64, 160, 160), (48, 96, 80, 80), (64, 128, 80, 80), (64, 64, 40, 40), (64, 128, 40, 40), (96, 192, 40, 40),
    (128, 256, 40, 40), (192, 192, 20, 20), (64, 64, 20, 20), (256, 512, 20, 20),
    (48, 48, 160, 160), (96, 96, 80, 80), (192, 192, 40, 40),
    (64, 64, 56, 56), (128, 128, 28, 28), (256, 256, 14, 14), (512, 512, 7, 7),
]
# edge tiles (W not a multiple of 8, H not a multiple of 16) on both engines: 28 x 28 and 44 x 20 stay on the im2col kernel
EDGE_SHAPES = [(32, 64, 60, 62), (64, 32, 62, 60), (32, 64, 28, 28), (64, 32, 44, 20)]
# shapes the shape rule must send to the halo kernel (fprop: C_in -> C_out; dgrad gathers C_out channels)
HALO_FPROP = {(32, 64, 160, 160), (48, 96, 80, 80), (64, 128, 80, 80), (64, 64, 56, 56), (64, 64, 40, 40), (96, 192, 40, 40),
              (32, 64, 60, 62), (64, 32, 62, 60)}
HALO_DGRAD = {(32, 64, 160, 160), (48, 96, 80, 80), (64, 128, 80, 80), (64, 64, 56, 56), (64, 64, 40, 40), (32, 64, 60, 62),
              (64, 32, 62, 60)}


def _lib():
    return lib.load()


def _both(fn):
    """(im2col result, halo-or-auto result, whether the halo kernel served the second call)."""
    L = _lib()
    L.sgb_conv_force_im2col(1)
    try:
        ref = fn()
    finally:
        L.sgb_conv_force_im2col(0)
    h0 = L.sgb_conv_halo_launches()
    out = fn()
    torch.cuda.synchronize()
    return ref, out, L.sgb_conv_halo_launches() > h0


def _equal(a, b):
    return bool((a.float() == b.float()).all())  # -0 == +0


def _nhwc(n, c, h, w, g, pitch=None, off=0):
    buf = torch.randn(n, h, w, pitch or c, generator=g, device="cuda").to(torch.bfloat16)
    return buf[..., off:off + c].permute(0, 3, 1, 2)


def _stats_close(a, b, y):
    a, b = a.sum(0), b.sum(0)
    yf = y.double()
    bound = torch.stack([yf.abs().sum((0, 2, 3)), (yf * yf).sum((0, 2, 3))]) * 1e-6
    return bool(((a - b).abs() <= bound + 1e-12).all())


@pytest.mark.parametrize("shape", MODEL_SHAPES + EDGE_SHAPES, ids=lambda s: "c%d_k%d_%dx%d" % s)
def test_fprop_with_statistics_matches_im2col(shape):
    c, k, h, w = shape
    g = torch.Generator(device="cuda").manual_seed(1)
    x = _nhwc(2, c, h, w, g)
    krsc, _ = K.weight_prepare(torch.randn(k, c, 3, 3, generator=g, device="cuda") * 0.1)

    def run():
        st = K.new_stats(k, "cuda")
        y = K.conv_fprop(x, krsc, k, 3, 3, 1, 1, stats=st)
        return y, st

    (y0, s0), (y1, s1), halo = _both(run)
    assert _equal(y0, y1)
    assert _stats_close(s0, s1, y1)
    if shape in HALO_FPROP:
        assert halo, "the shape rule should send this shape to the halo kernel"


@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("shape", MODEL_SHAPES + EDGE_SHAPES, ids=lambda s: "c%d_k%d_%dx%d" % s)
def test_dgrad_matches_im2col(shape, accumulate):
    c, k, h, w = shape
    g = torch.Generator(device="cuda").manual_seed(2)
    dy = _nhwc(2, k, h, w, g)
    _, crsk = K.weight_prepare(torch.randn(k, c, 3, 3, generator=g, device="cuda") * 0.1)
    dx0 = _nhwc(2, c, h, w, g)

    def run():
        dx = K.empty_nhwc(2, c, h, w, "cuda")
        dx.copy_(dx0)
        return K.conv_dgrad(dy, crsk, (2, c, h, w), 3, 3, 1, 1, out=dx, accumulate=accumulate)

    ref, out, halo = _both(run)
    assert _equal(ref, out)
    if shape in HALO_DGRAD:
        assert halo, "the shape rule should send this shape to the halo kernel"


@pytest.mark.parametrize("act", [lib.ACT_NONE, lib.ACT_RELU])
def test_fprop_scale_shift_residual_act(act):
    c, k, h, w = 48, 96, 80, 80
    g = torch.Generator(device="cuda").manual_seed(3)
    x = _nhwc(2, c, h, w, g)
    krsc, _ = K.weight_prepare(torch.randn(k, c, 3, 3, generator=g, device="cuda") * 0.1)
    scale = torch.rand(k, generator=g, device="cuda") + 0.5
    shift = torch.randn(k, generator=g, device="cuda")
    res = _nhwc(2, k, h, w, g)
    (y0, y1, halo) = _both(lambda: K.conv_fprop(x, krsc, k, 3, 3, 1, 1, scale=scale, shift=shift, residual=res, act=act))
    assert halo
    assert _equal(y0, y1)


def test_channel_slices_in_and_out():
    # input: channels [32, 96) of a 128-channel tensor; output: channels [64, 128) of a 192-channel tensor
    c, k, h, w = 64, 64, 56, 56
    g = torch.Generator(device="cuda").manual_seed(4)
    x = _nhwc(2, c, h, w, g, pitch=128, off=32)
    krsc, _ = K.weight_prepare(torch.randn(k, c, 3, 3, generator=g, device="cuda") * 0.1)
    base = _nhwc(2, 192, h, w, g)

    def run():
        buf = base.clone(memory_format=torch.channels_last)
        K.conv_fprop(x, krsc, k, 3, 3, 1, 1, out=buf[:, 64:128])
        return buf

    ref, out, halo = _both(run)
    assert halo
    assert _equal(ref, out)
    assert _equal(out[:, :64], base[:, :64]) and _equal(out[:, 128:], base[:, 128:]), "channels outside the output slice changed"
