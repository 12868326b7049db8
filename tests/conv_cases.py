"""fp64 oracles, exact integer-operand cases, arithmetic-derived error bounds, a mirror of the routing rules, an fp32 transcription and a
launch recorder for the convolution entry points (csrc/conv.cu -> conv_sm100.cu / conv_mma.cu): conv_fprop, conv_dgrad, conv_wgrad and
convt2x2_fprop.

Layout.  Oracles and checks work on fp64 NCHW tensors on whatever device the operands live on; weight gradients are KRSC [K, R, S, C]
as the kernels write them.

Oracles.  The bf16 operands in float64 through torch.nn.functional: conv2d (fprop, plus the scale / shift / residual / activation
epilogue), conv_transpose2d (dgrad, convt2x2), and conv2d over the batch axis with the stride as dilation (wgrad, added to the fp32
gradient already in dw; with centre_from the off-centre entries of rows >= centre_from keep it).

Exact integer cases.  x, w and dy hold sparse integers in {-2..2}, the residual small integers, scale is in +-{1/2, 1, 2} and shift a
multiple of 1/4.  The density is chosen per shape so that every output has sum |x w| <= cap (2^11 by default; `int_operands` asserts it
with an fp64 convolution of |x| and |w|).  Every partial sum any kernel can form is then an integer of at most 12 bits, which an fp32
accumulator holds exactly in any order, split or atomic, and the epilogue's products and sums stay below 2^16 in steps of 1/4.  So
the result is known to the bit: round_bf16(oracle) for bf16 stores, the oracle itself for fp32 ones, dw_old + oracle for weight
gradients.  A dropped, duplicated or misplaced product, a wrong tap, parity class or pitch changes it.  SiLU (__expf) is the one
inexact epilogue step: it is checked with its bound on top of the exact pre-activation.

Bounds for real-valued operands (bf16-rounded normals).  |acc - exact| <= gamma_L sum|x w| with u = 2^-23 (covers a truncating
tensor-core adder as well as round-to-nearest), L the longest fp32 addition chain of the launch: the reduction length (C rounded up to
the 64-channel box, times the taps) for fprop / dgrad / convt2x2, the pixels per CTA plus the number of pixel splits plus the add into
dw for wgrad (`wgrad_chain`, from the route mirror).  Each fp32 rounding of scale, shift and residual adds u |value|; SiLU adds the
__expf error of the CUDA C Programming Guide (2 + floor(|1.173 x|) ulp) and two roundings; a bf16 store adds half an ulp.  Epilogue
statistics of the stored y are bounded with bn_qarep_cases.epilogue_chain_len.

Route mirror.  `route(op, d, flags, sms)` restates conv.cu / conv_sm100.cu / conv_mma.cu's choices (supported, row_pairs, pick_bn,
halo_tiles_fit, halo_bn, the KC choice, wgrad_supported, wgrad_halo_nb, nb / CB, rb_all / rb_off and the even-ring rule, the dgrad
branches, dispatch_igemm's waste rule, wgrad_kernel's BMW rule) and returns the engine, kernel, tile variant and the launch-counter
deltas it implies (sgb_sm100_launches / sgb_conv_halo_launches / sgb_conv_wgrad_halo_launches).

Transcription.  `t_fprop` / `t_dgrad` / `t_wgrad` restate the kernels' arithmetic in fp32 torch on the CPU (implicit GEMM in 16-channel
k-steps, the stride-2 dgrad parity classes with their tap tables, 64-pixel wgrad steps, per-warp statistics partials); `mut` plants one
defect (MUTATIONS).  The CPU suite runs them through the same verify_* functions the GPU suite uses.

Recorder.  `record_conv()` patches K.conv_fprop / conv_dgrad / conv_wgrad / convt2x2_fprop and keeps, for every call, the inputs, the
in-place state before the call (accumulate targets, dw, statistics), the state after it and the launch-counter deltas.
"""
import contextlib
import functools
import inspect
import math
from collections import namedtuple

import torch
import torch.nn.functional as F

from bn_qarep_cases import U32, U64, _clone, _pitch, bf16_ulp, epilogue_chain_len, gamma_n, round_bf16

F64 = torch.float64
CAP = 2**11
BF16_NAN = 0x7FC0  # what channels outside an input slice hold: any read of them turns the result into NaN
SENTINEL = 0x5A5A  # bit pattern of the channels outside an output slice: a write to them shows
ACTS = ("none", "relu", "silu")


# ------------------------------------------------------------------------------------------------ fp64 oracles
def conv64(x, w, stride, pad):
    return F.conv2d(x.double(), w.double(), stride=stride, padding=pad)


def _out_padding(H, P, R, stride, pad):
    return H - ((P - 1) * stride - 2 * pad + R)


def dgrad64(dy, w, x_shape, stride, pad):
    N, C, H, W = x_shape
    R, S = w.shape[2], w.shape[3]
    P, Q = dy.shape[2], dy.shape[3]
    op = (_out_padding(H, P, R, stride, pad), _out_padding(W, Q, S, stride, pad))
    return F.conv_transpose2d(dy.double(), w.double(), stride=stride, padding=pad, output_padding=op)


def wgrad64(x, dy, R, S, stride, pad):
    """sum over pixels of dy[k] x[c] at tap (r, s): fp64 KRSC [K, R, S, C]."""
    g = F.conv2d(x.double().transpose(0, 1), dy.double().transpose(0, 1), padding=pad, dilation=stride)
    return g[:, :, :R, :S].permute(1, 2, 3, 0).contiguous()


def epilogue64(acc, scale=None, shift=None, residual=None, act="none"):
    """(pre-activation, y) of act(acc * scale + shift + residual) in fp64; scale / shift per output channel."""
    v = acc
    if scale is not None:
        v = v * scale.double().view(1, -1, 1, 1)
    if shift is not None:
        v = v + shift.double().view(1, -1, 1, 1)
    if residual is not None:
        v = v + residual.double()
    return v, act64(v, act)


def act64(v, act):
    if act == "relu":
        return v.clamp_min(0)
    if act == "silu":
        return v * torch.sigmoid(v)
    return v


def fprop_ref(x, w, stride, pad, scale=None, shift=None, residual=None, act="none"):
    return epilogue64(conv64(x, w, stride, pad), scale, shift, residual, act)[1]


def dgrad_ref(dy, w, x_shape, stride, pad, dx_old=None, accumulate=False):
    g = dgrad64(dy, w, x_shape, stride, pad)
    return g + dx_old.double() if accumulate else g


def centre_mask(K, R, S, C, centre_from, device):
    """True at the KRSC entries a centre_from weight gradient writes: every entry of rows < centre_from, the centre tap of the rest."""
    m = torch.ones(K, R, S, C, dtype=torch.bool, device=device)
    if centre_from:
        m[centre_from:] = False
        m[centre_from:, R // 2, S // 2] = True
    return m


def wgrad_ref(x, dy, R, S, stride, pad, dw_old=None, centre_from=0):
    g = wgrad64(x, dy, R, S, stride, pad)
    g = torch.where(centre_mask(*g.shape, centre_from, g.device), g, torch.zeros_like(g))
    return g if dw_old is None else dw_old.double() + g


def convt2x2_ref(x, w_t, bias=None):
    """ConvTranspose2d(k=2, s=2): x [N, Cin, P, Q], w_t [Cin, Cout, 2, 2]."""
    return F.conv_transpose2d(x.double(), w_t.double(), None if bias is None else bias.double(), stride=2)


def stats_ref(y):
    """[2, K]: per-channel sum of y and of y^2 over the stored (bf16) tensor."""
    y = y.double()
    return torch.stack([y.sum((0, 2, 3)), (y * y).sum((0, 2, 3))])


# ------------------------------------------------------------------------------------------------ bounds
def gamma23(L):
    """gamma_L with u = 2^-23 (gamma_n counts in u = 2^-24)."""
    return gamma_n(2 * L)


def rnd_err(v, e):
    """One fp32 rounding of a value near v (fp64 tensor) known to within e."""
    return e + 1.0001 * U32 * (v.abs() + e)


def expf_rel(v):
    """Relative error bound of __expf(-v): 2 + floor(|1.173 v|) ulp (CUDA C Programming Guide, intrinsic functions)."""
    return (2 + torch.floor((1.173 * v).abs())) * 2.0**-23


def epilogue_err(acc, e, scale=None, shift=None, residual=None, act="none"):
    """(y_ref, |y_kernel - y_ref| bound before the store) of the fp32 epilogue on an accumulator known to within e."""
    v = acc
    if scale is not None:
        sc = scale.double().view(1, -1, 1, 1)
        v, e = v * sc, e * sc.abs()
        e = rnd_err(v, e)
    if shift is not None:
        v = v + shift.double().view(1, -1, 1, 1)
        e = rnd_err(v, e)
    if residual is not None:
        v = v + residual.double()
        e = rnd_err(v, e)
    y = act64(v, act)
    if act == "silu":
        t = torch.exp(-v.clamp(-80, 80))
        e = 1.1 * e + y.abs() * (expf_rel(v) * t / (1 + t) + 3 * U32) + torch.where(v < -80, y.abs(), torch.zeros_like(v))
    return y, e


def fprop_chain(C, R, S):
    """Additions into one fprop / dgrad accumulator: the taps times C rounded up to a whole 64-channel box (boxes past C add zeros)."""
    return R * S * (-(-C // 64) * 64)


# ------------------------------------------------------------------------------------------------ comparisons
def _fail(name, bad, got, want, allow=None):
    i = int(bad.flatten().nonzero()[0])
    extra = "" if allow is None else f" allowed {float(allow.flatten()[i]):.3e}"
    raise AssertionError(f"{name}: {int(bad.sum())} of {bad.numel()} wrong; first at flat {i}: kernel {float(got.flatten()[i])!r} "
                         f"expected {float(want.flatten()[i])!r}{extra}")


def expect_exact(name, got, want):
    """Bit equality of the values (-0 == +0; NaN equals nothing)."""
    got, want = got.double().to(want.device), want.double()
    bad = ~(got == want)
    if bool(bad.any()):
        _fail(name, bad, got, want)


def expect_within(name, got, ref, err, bf16=False):
    """|got - ref| <= err (+ half a bf16 ulp of |ref| + err for a bf16 store)."""
    got, ref = got.double().to(ref.device), ref.double()
    allow = err + 0.5 * bf16_ulp(ref.abs() + err) if bf16 else err
    allow = torch.broadcast_to(allow, ref.shape)
    bad = ~((got - ref).abs() <= allow)
    if bool(bad.any()):
        _fail(name, bad, got, ref, allow)


def expect_stats(name, got, y_stored):
    """Epilogue statistics [2, K] (summed over replicas) of the stored y, within the epilogue chain bound."""
    M = y_stored.numel() // y_stored.shape[1]
    y = y_stored.double()
    L = epilogue_chain_len(M) + 1  # + the rounding of y * y
    for j, t in enumerate((y, y * y)):
        mag = t.abs().sum((0, 2, 3))
        expect_within(f"{name}[{j}]", got[j], t.sum((0, 2, 3)), gamma_n(L) * mag + (M + 8) * U64 * mag)


def expect_bits(name, after, before):
    """The bits of a buffer region the call must not write are unchanged."""
    if not torch.equal(after.view(torch.int16), before.view(torch.int16)):
        bad = after.view(torch.int16) != before.view(torch.int16)
        raise AssertionError(f"{name}: {int(bad.sum())} of {bad.numel()} elements outside the output slice were written")


# ------------------------------------------------------------------------------------------------ operands
def sparse_int(shape, density, gen, device="cpu"):
    """Integers in {-2, -1, 1, 2} at `density` of the entries, 0 elsewhere (fp64)."""
    v = torch.randint(1, 3, shape, generator=gen).double() * (torch.randint(0, 2, shape, generator=gen).double() * 2 - 1)
    keep = torch.rand(shape, generator=gen, dtype=F64) < density
    return (v * keep).to(device)


def real_bf16(shape, gen, scale=1.0, device="cpu"):
    return round_bf16(torch.randn(shape, generator=gen, dtype=F64) * scale).to(device)


def int_operands(shape_a, shape_b, absfn, L, cap, gen, device):
    """Two sparse integer operands whose reduction absfn(|a|, |b|) stays <= cap everywhere; the density is lowered until it does."""
    d = min(1.0, math.sqrt(cap / (2.25 * max(L, 1) * 1.5)))
    for _ in range(40):
        a, b = sparse_int(shape_a, d, gen, device), sparse_int(shape_b, d, gen, device)
        worst = float(absfn(a.abs(), b.abs()).max())
        if worst <= cap:
            assert worst <= cap, worst
            return a, b, worst
        d *= 0.75
    raise AssertionError(f"no density keeps sum |a b| <= {cap}")


def zero_off_centre(w, centre_from):
    """A folded filter: rows >= centre_from keep only their centre tap."""
    if centre_from:
        w = w.clone()
        c = w[centre_from:, :, 1, 1].clone()
        w[centre_from:] = 0
        w[centre_from:, :, 1, 1] = c
    return w


# ------------------------------------------------------------------------------------------------ cases
def make_case(op, n, c, h, w, k, r=3, stride=1, pad=None, **kw):
    """One call of the matrix.  op: fprop / dgrad / wgrad / convt2x2 (convt2x2: c = C_up, k = input channels, h, w = input size).
    Options: x_pitch / x_off (the gathered input as a channel slice), y_pitch / y_off (the written output as one), scale, shift,
    residual, act, stats (replicas, 0 = none), out_f32, centre_from, accumulate, force (force_im2col), cap, real (also run with
    real-valued operands against the bounds), bias (convt2x2)."""
    pad = r // 2 if pad is None else pad
    d = dict(op=op, N=n, C=c, H=h, W=w, K=k, R=r, S=r, stride=stride, pad=pad, x_pitch=None, x_off=0, y_pitch=None, y_off=0, scale=False,
             shift=False, residual=False, act="none", stats=0, out_f32=False, centre_from=0, accumulate=False, force=False, cap=CAP,
             real=False, bias=True)
    for key in kw:
        if key not in d and key != "id":
            raise KeyError(key)
    d.update(kw)
    if op == "convt2x2":
        d.update(R=2, S=2, stride=2, pad=0)
    d["id"] = kw.get("id") or case_id(d)
    return d


def case_id(d):
    s = f"{d['op']}_n{d['N']}c{d['C']}h{d['H']}w{d['W']}k{d['K']}r{d['R']}s{d['stride']}p{d['pad']}"
    for key, tag in (("x_pitch", "xp"), ("y_pitch", "yp"), ("stats", "st"), ("centre_from", "cf")):
        if d[key]:
            s += f"_{tag}{d[key]}"
    for key in ("scale", "shift", "residual", "out_f32", "accumulate", "force"):
        if d[key]:
            s += "_" + key
    if d["act"] != "none":
        s += "_" + d["act"]
    if d["cap"] != CAP:
        s += f"_cap{d['cap']}"
    return s


def desc_of(c):
    """The SgbConvDesc fields the front ends (kernels.py) set for case c: the pitches of the slices, offsets folded into the pointers."""
    N, C, H, W, K, R, S, st, pad = (c[k] for k in ("N", "C", "H", "W", "K", "R", "S", "stride", "pad"))
    if c["op"] == "convt2x2":  # the equivalent convolution: upsampled (H, W, C) -> small (P, Q, K)
        H, W, P, Q = 2 * c["H"], 2 * c["W"], c["H"], c["W"]
        return dict(N=N, H=H, W=W, C=C, K=K, R=2, S=2, stride=2, pad=0, P=P, Q=Q, x_pitch=-(-C // 8) * 8, x_off=0,
                    y_pitch=c["x_pitch"] or -(-K // 8) * 8, y_off=0, centre_from=0)
    P = (H + 2 * pad - R) // st + 1
    Q = (W + 2 * pad - S) // st + 1
    xp = c["x_pitch"] or -(-C // 8) * 8
    yp = c["y_pitch"] or -(-K // 8) * 8
    return dict(N=N, H=H, W=W, C=C, K=K, R=R, S=S, stride=st, pad=pad, P=P, Q=Q, x_pitch=xp, x_off=0, y_pitch=yp, y_off=0,
                centre_from=c["centre_from"])


# For dgrad the "x" slice options describe dx (written) and the "y" ones dy (gathered); for wgrad both are read.
def _legacy_cases():
    """The shapes the fp32-tolerance test of test_kernels_gpu.py covered, each as fprop (statistics over 8 replicas), fp32-out fprop,
    dgrad, accumulating dgrad and wgrad."""
    shapes = [
        (2, 16, 12, 12, 24, 3, 1, 1), (2, 16, 13, 11, 24, 3, 2, 1), (3, 32, 20, 20, 32, 3, 1, 1), (2, 48, 10, 10, 96, 3, 2, 1),
        (2, 64, 9, 9, 64, 1, 1, 0), (2, 96, 8, 8, 192, 1, 2, 0), (1, 8, 33, 33, 48, 3, 2, 1), (2, 8, 30, 30, 64, 7, 2, 3),
        (2, 128, 7, 7, 256, 3, 1, 1), (4, 64, 10, 10, 68, 1, 1, 0), (2, 192, 5, 5, 80, 1, 1, 0), (2, 16, 6, 6, 16, 2, 2, 0),
        (16, 32, 48, 48, 32, 3, 1, 1), (8, 64, 40, 40, 64, 3, 1, 1), (6, 96, 40, 40, 96, 3, 1, 1), (8, 48, 40, 40, 96, 3, 2, 1),
        (4, 192, 20, 20, 384, 3, 2, 1), (2, 384, 20, 20, 768, 1, 1, 0), (6, 64, 31, 29, 128, 1, 1, 0), (4, 16, 16, 16, 16, 3, 1, 1),
        (4, 32, 16, 16, 32, 3, 1, 1), (4, 16, 16, 16, 16, 1, 1, 0), (2, 64, 24, 24, 64, 3, 1, 1), (2, 16, 32, 32, 48, 3, 2, 1),
        (3, 32, 24, 24, 64, 3, 2, 1), (2, 48, 20, 20, 48, 3, 1, 1), (2, 192, 20, 20, 192, 3, 1, 1), (3, 32, 13, 37, 32, 3, 1, 1),
        (2, 128, 19, 16, 128, 3, 1, 1), (40, 32, 64, 64, 32, 3, 1, 1), (4, 96, 20, 20, 192, 3, 2, 1), (4, 96, 20, 20, 96, 3, 2, 1),
        (4, 96, 20, 20, 64, 1, 1, 0), (4, 192, 20, 20, 64, 1, 1, 0), (2, 288, 20, 20, 96, 1, 1, 0), (2, 48, 40, 40, 96, 1, 2, 0),
        (2, 80, 12, 12, 80, 1, 1, 0), (9, 48, 192, 192, 96, 3, 2, 1), (8, 96, 200, 200, 64, 1, 2, 0), (9, 64, 96, 96, 80, 1, 1, 0),
        (4, 96, 40, 40, 96, 2, 2, 0), (2, 192, 20, 20, 192, 2, 2, 0), (3, 32, 18, 22, 48, 2, 2, 0),
    ]
    return [c for shape in shapes for c in shape_modes(*shape)]


def shape_modes(n, c, h, w, k, r, stride, pad):
    """One convolution shape as fprop with statistics over 8 replicas, fp32-out fprop, dgrad, accumulating dgrad and wgrad."""
    g = dict(n=n, c=c, h=h, w=w, k=k, r=r, stride=stride, pad=pad)
    return [make_case("fprop", **g, stats=8), make_case("fprop", **g, out_f32=True), make_case("dgrad", **g), make_case("dgrad", **g, accumulate=True),
            make_case("wgrad", **g)]


def _matrix_cases():
    m = make_case
    cs = []
    # fprop, conv3x3_halo_kernel: every N tile, the narrowed 96 / 64 tiles, statistics, epilogues, edge maps, slices
    for k in (16, 32, 48, 64, 96, 128):
        cs.append(m("fprop", 2, 32, 40, 40, k, stats=8, real=k in (48, 128)))
    cs += [m("fprop", 1, 96, 40, 40, 384, id="fprop_halo_narrowed96", real=True), m("fprop", 1, 96, 40, 40, 256, id="fprop_halo_narrowed64"),
           m("fprop", 2, 64, 40, 40, 64, stats=1), m("fprop", 2, 64, 40, 40, 64, stats=8, scale=True, shift=True, residual=True, act="relu", real=True),
           m("fprop", 2, 64, 40, 40, 64, scale=True, shift=True, act="silu", real=True), m("fprop", 2, 64, 40, 40, 64, shift=True, residual=True),
           m("fprop", 2, 32, 60, 62, 48, stats=1, scale=True, shift=True, act="relu"), m("fprop", 2, 32, 62, 60, 32, act="silu", shift=True),
           m("fprop", 3, 16, 47, 45, 64, stats=8, real=True), m("fprop", 1, 48, 45, 47, 96, shift=True, act="relu"),
           m("fprop", 2, 32, 40, 40, 48, x_pitch=64, x_off=16, y_pitch=96, y_off=24, scale=True, shift=True, residual=True, act="relu", stats=8),
           m("fprop", 2, 64, 56, 56, 32, x_pitch=96, x_off=8, y_pitch=48, y_off=8, real=True)]
    # fprop, conv_wgmma_kernel: 1x1 s1 / s2, 3x3 s2, 3x3 s1 on maps the halo kernel leaves alone or under force_im2col, every KC and N tile
    cs += [m("fprop", 2, 64, 20, 20, 64, r=1, stats=8), m("fprop", 2, 64, 21, 19, 128, r=1, stride=2, scale=True, shift=True, act="relu"),
           m("fprop", 2, 32, 21, 23, 64, stride=2, stats=1, real=True), m("fprop", 2, 64, 28, 28, 64, act="silu", shift=True),
           m("fprop", 3, 32, 20, 20, 96), m("fprop", 4, 64, 14, 14, 128, residual=True, shift=True, act="relu"), m("fprop", 8, 128, 7, 7, 128, real=True),
           m("fprop", 2, 64, 40, 40, 64, force=True, stats=8, scale=True, shift=True, residual=True, act="relu", real=True)]
    for c in (16, 32, 48, 96, 288):  # KC 16 / 32 / 64, and the 64-channel boxes with zero-filled tails
        cs.append(m("fprop", 2, c, 14, 14, 48, stats=8))
    for k in (16, 32, 48, 64, 96, 128):
        cs.append(m("fprop", 2, 64, 20, 20, k, r=1))
    cs += [m("fprop", 2, 64, 20, 20, 128, centre_from=64, real=True), m("fprop", 2, 32, 28, 28, 64, centre_from=32, stats=8),
           m("fprop", 2, 64, 40, 40, 128, centre_from=64, force=True), m("fprop", 3, 32, 13, 37, 32),  # M = 1443, not a multiple of 128
           m("fprop", 16, 64, 64, 64, 64, r=1, stats=8)]  # 512 row tiles: more tiles than CTAs
    # fprop, the 2 x 2 / stride-2 row-pair re-description (dense x) and its decline (x as a slice: mma.sync)
    cs += [m("fprop", 2, 48, 20, 20, 64, r=2, stride=2, pad=0, real=True), m("fprop", 2, 48, 20, 20, 64, r=2, stride=2, pad=0, x_pitch=64, x_off=8)]
    # fprop, mma.sync: fp32 out, ragged channel counts, 7x7 s2, 3x3 without padding, K = 68, each dispatch_igemm BN
    cs += [m("fprop", 2, 32, 12, 12, 48, out_f32=True, real=True), m("fprop", 2, 8, 15, 13, 40, stats=8), m("fprop", 2, 24, 12, 12, 128, scale=True, shift=True, act="silu"),
           m("fprop", 2, 40, 10, 10, 68, residual=True, shift=True, act="relu", real=True), m("fprop", 2, 8, 30, 30, 64, r=7, stride=2, pad=3),
           m("fprop", 2, 32, 12, 12, 32, pad=0, stats=1), m("fprop", 2, 24, 9, 9, 40, x_pitch=48, x_off=16, y_pitch=64, y_off=8, scale=True, shift=True)]
    # convt2x2: the four parity launches on the wgmma kernel, and the mma.sync fallback (24 output channels)
    cs += [m("convt2x2", 2, 32, 10, 12, 64, real=True), m("convt2x2", 2, 64, 20, 20, 128), m("convt2x2", 2, 48, 7, 9, 32, x_pitch=48),
           m("convt2x2", 2, 24, 5, 6, 32, real=True)]
    # dgrad, stride-1 flip (halo and im2col), SKIP via centre_c, accumulate in place
    cs += [m("dgrad", 2, 64, 40, 40, 64, real=True), m("dgrad", 2, 64, 40, 40, 64, accumulate=True), m("dgrad", 2, 64, 40, 40, 128, centre_from=64, real=True),
           m("dgrad", 2, 32, 40, 40, 64, centre_from=32, accumulate=True), m("dgrad", 2, 64, 20, 20, 64), m("dgrad", 2, 64, 20, 20, 128, centre_from=64, accumulate=True),
           m("dgrad", 2, 64, 40, 40, 128, centre_from=64, force=True), m("dgrad", 2, 48, 20, 20, 64, r=1, accumulate=True),
           m("dgrad", 2, 32, 40, 40, 48, x_pitch=64, x_off=8, y_pitch=64, y_off=16, accumulate=True)]
    # dgrad, stride-2 3x3: the four parity classes (even maps), odd maps on mma.sync
    cs += [m("dgrad", 2, 32, 40, 40, 64, stride=2, real=True), m("dgrad", 2, 64, 20, 28, 64, stride=2, accumulate=True),
           m("dgrad", 2, 32, 21, 19, 64, stride=2, accumulate=True)]
    # dgrad, 1x1 stride 2: dense without accumulate (memset), accumulate (odd-parity pixels untouched), a slice without accumulate
    cs += [m("dgrad", 2, 64, 40, 40, 128, r=1, stride=2, real=True), m("dgrad", 2, 64, 40, 40, 128, r=1, stride=2, accumulate=True),
           m("dgrad", 2, 64, 40, 40, 128, r=1, stride=2, x_pitch=96, x_off=16)]
    # dgrad, mma.sync: K = 8 / 24 / 68 with padded dy, 7x7, 2x2 s2
    cs += [m("dgrad", 2, 32, 16, 16, 8), m("dgrad", 2, 32, 16, 16, 24, accumulate=True, real=True), m("dgrad", 2, 32, 12, 12, 68, y_pitch=80),
           m("dgrad", 2, 8, 30, 30, 64, r=7, stride=2, pad=3), m("dgrad", 2, 48, 20, 20, 64, r=2, stride=2, pad=0, accumulate=True)]
    # wgrad, wgrad3x3_halo_kernel: nb 16 / 32 / 48, edge maps, centre_from, accumulation into a non-zero dw
    cs += [m("wgrad", 2, 32, 40, 40, 64, real=True), m("wgrad", 2, 48, 40, 40, 64), m("wgrad", 2, 80, 40, 40, 32), m("wgrad", 2, 16, 47, 45, 48, real=True),
           m("wgrad", 2, 32, 60, 62, 128, centre_from=64), m("wgrad", 2, 64, 62, 60, 192, centre_from=128, real=True),
           m("wgrad", 2, 32, 40, 40, 64, x_pitch=64, x_off=16, y_pitch=96, y_off=8),
           m("wgrad", 2, 48, 40, 40, 96, centre_from=48, real=True)]  # centre_from inside a 64-row block (YOLO-NAS-S's 96-channel stage)
    # wgrad, wgrad_wgmma_kernel: every nb / CB, odd and even row-block counts with and without centre_from, pixel splits, 1x1, 3x3 s2
    for c in (16, 32, 48, 64, 96, 128):
        cs.append(m("wgrad", 2, c, 20, 20, 64))
    for k, cf in ((64, 0), (128, 0), (192, 0), (128, 64), (192, 128), (192, 64)):
        cs.append(m("wgrad", 2, 96, 14, 14, k, centre_from=cf, real=k == 192 and cf == 64))
    cs += [m("wgrad", 2, 96, 14, 14, 96, centre_from=48), m("wgrad", 2, 64, 20, 20, 128, centre_from=32, real=True),
           m("wgrad", 16, 64, 28, 28, 64, real=True), m("wgrad", 2, 64, 40, 40, 64, force=True), m("wgrad", 2, 64, 40, 40, 128, centre_from=64, force=True),
           m("wgrad", 2, 64, 20, 20, 128, r=1), m("wgrad", 2, 64, 21, 19, 128, r=1, stride=2), m("wgrad", 2, 32, 21, 23, 64, stride=2, real=True)]
    # wgrad, row pairs and mma.sync: C % 16 != 0, K % 8 != 0, 7x7, every BMW, centre_from with C = 24
    cs += [m("wgrad", 2, 48, 20, 20, 64, r=2, stride=2, pad=0, real=True), m("wgrad", 2, 24, 16, 16, 32), m("wgrad", 2, 32, 16, 16, 68, y_pitch=72, real=True),
           m("wgrad", 2, 8, 30, 30, 64, r=7, stride=2, pad=3), m("wgrad", 2, 24, 12, 12, 96), m("wgrad", 2, 24, 12, 12, 160),
           m("wgrad", 2, 24, 16, 16, 32, centre_from=16), m("wgrad", 2, 24, 16, 16, 64, centre_from=32, real=True)]
    # the epilogue / slice test of test_kernels_gpu.py, and its convt2x2 shape (mma.sync)
    cs += [m("fprop", 2, 32, 9, 9, 40, x_pitch=64, x_off=16, y_pitch=96, y_off=48, scale=True, shift=True, residual=True, act="relu", real=True, id="fprop_slices_epilogue")]
    return cs


def all_cases():
    out, ids = [], set()
    for c in _matrix_cases() + _legacy_cases():
        while c["id"] in ids:
            c["id"] += "+"
        ids.add(c["id"])
        out.append(c)
    return out


# ------------------------------------------------------------------------------------------------ route mirror
Route = namedtuple("Route", "engine kernel variant launches halo whalo chain")


def _ceil(a, b):
    return -(-a // b)


def pick_bn(n):
    for bn in (16, 32, 48, 64, 96, 128):
        if n <= bn:
            return bn
    best, bw = 128, _ceil(n, 128) * 128 - n
    for bn in (96, 64):
        w = _ceil(n, bn) * bn - n
        if w < bw:
            best, bw = bn, w
    return best


def halo_tiles_fit(P, Q):
    return 20 * P * Q >= 17 * (_ceil(P, 8) * 8) * (_ceil(Q, 8) * 8)


def halo_smem(C, bn, n, stats, stages):
    b = (9 * C * bn * 2 + 1023) & ~1023
    a = ((C // 8) * 1664 + 1023) & ~1023
    return 1024 + b + stages * a + (16 * 8 + 16) + ((8 * 2 * bn + 4 * n) * 4 if stats else 0)


def _supported(q):
    return (q["C"] % 16 == 0 and q["b_rows"] % 8 == 0 and q["R"] == q["S"] and q["R"] in (1, 3) and q["stride"] in (1, 2) and q["a_pitch"] % 8 == 0
            and q["y_pitch"] % 8 == 0 and q["N"] * q["P"] * q["Q"] < 2**31 and q["b_rows"] <= 4096)


def _halo_bn(q):
    if q["R"] != 3 or q["stride"] != 1 or q["pad"] != 1 or q["ntaps"] or q["out_mode"] or q["P"] != q["H"] or q["Q"] != q["W"]:
        return 0
    if not halo_tiles_fit(q["P"], q["Q"]):
        return 0
    n = q["b_rows"]
    full = pick_bn(n)
    waste = lambda bn: _ceil(n, bn) * bn - n  # noqa: E731
    for bn in (full, 96, 64):
        if bn <= full and (bn == full or (q["C"] <= 96 and bn >= 64 and waste(bn) <= waste(full))) and halo_smem(q["C"], bn, n, q["stats"], 2) <= 227 * 1024:
            return bn
    return 0


def _launch(q, force, nlaunch=1):
    """The wgmma engine's choice for one GEMM: conv3x3_halo_kernel or conv_wgmma_kernel, its N tile and KC."""
    C = q["C"]
    kc = 64 if C % 64 == 0 else (32 if C % 32 == 0 else 16)
    if kc < 64 and C > 32:
        kc = 64
    chain = q["taps"] * _ceil(C, kc) * kc
    skip = q["centre_from"] > 0
    hbn = 0 if force else _halo_bn(q)
    if hbn:
        tag = f"bn{hbn}" + ("_narrowed" if hbn != pick_bn(q["b_rows"]) else "") + ("_skip" if skip and q["flip"] else "")
        return Route("wgmma", "conv3x3_halo_kernel", tag, nlaunch, nlaunch, 0, chain)
    tag = f"bn{pick_bn(q['b_rows'])}_kc{kc}" + ("_skip" if skip else "")
    return Route("wgmma", "conv_wgmma_kernel", tag, nlaunch, 0, 0, chain)


def _gemm(C, a_pitch, b_rows, R, stride, pad, N, H, W, P, Q, y_pitch, taps=None, **kw):
    q = dict(C=C, a_pitch=a_pitch, b_rows=b_rows, R=R, S=R, stride=stride, pad=pad, N=N, H=H, W=W, P=P, Q=Q, y_pitch=y_pitch, ntaps=0, out_mode=0,
             flip=0, centre_from=0, stats=False, taps=taps or R * R)
    q.update(kw)
    return q


def _igemm_bn(n):
    waste = lambda bn: _ceil(n, bn) * bn - n  # noqa: E731
    best, bw = 128, waste(128)
    for bn in (64, 32):
        if waste(bn) < bw:
            best, bw = bn, waste(bn)
    return best


def _mma(op, d):
    if op == "wgrad":
        K = d["K"]
        bmw = 32 if K <= 32 else (64 if K <= 64 else 128)
        if 64 < K <= 96:
            bmw = 32
        mt, nt = _ceil(K, bmw), _ceil(d["R"] * d["S"] * d["C"], 64)
        total = _ceil(d["N"] * d["P"] * d["Q"], 32)
        splits = max(1, 132 * 4 // (mt * nt))
        splits = min(splits, total)
        if total // splits < 8:
            splits = total // 8 if total // 8 > 0 else 1
        per = _ceil(total, splits)
        splits = _ceil(total, per)
        return Route("mma", "wgrad_kernel", f"bmw{bmw}", 0, 0, 0, per * 32 + splits + 1)
    n = 4 * d["C"] if op == "convt2x2" else (d["C"] if op == "dgrad" else d["K"])
    red = d["K"] if op == "convt2x2" else (_ceil(d["K"], 8) * 8 * d["R"] * d["S"] if op == "dgrad" else d["C"] * d["R"] * d["S"])
    return Route("mma", "igemm_conv_kernel", f"bn{_igemm_bn(n)}", 0, 0, 0, _ceil(red, 32) * 32)


def _row_pairs(d):
    return (d["R"] == 2 and d["S"] == 2 and d["stride"] == 2 and d["pad"] == 0 and d["x_pitch"] == d["C"] and d["x_off"] == 0 and d["H"] % 2 == 0
            and d["W"] % 2 == 0 and d["P"] == d["H"] // 2 and d["Q"] == d["W"] // 2 and (2 * d["C"]) % 16 == 0 and d["K"] % 8 == 0 and d["y_pitch"] % 8 == 0)


def _wgrad_route(d, R, S, C, x_pitch, N, H, W, P, Q, stride, pad, flags, sms):
    K, cf = d["K"], d["centre_from"]
    if not (C % 16 == 0 and K % 8 == 0 and ((R == 1 and S == 1) or (R == 3 and S == 3) or (R == 2 and S == 1)) and x_pitch % 8 == 0 and d["y_pitch"] % 8 == 0):
        return None
    nb = next((c for c in (128, 96, 64, 48, 32) if C % c == 0), 16)
    cb = 64 if nb % 64 == 0 else (32 if nb % 32 == 0 else 16)
    rb_all = _ceil(K, 64)
    rb_off = _ceil(cf, 64) if cf else rb_all
    taps = R * S
    items = sum((_ceil(rb_off if (taps == 9 and t != 4) else rb_all, 1) + 1) // 2 for t in range(taps))
    npix = N * P * Q
    if not flags.get("wgrad_force") and R == 3 and stride == 1 and pad == 1 and P == H and Q == W and halo_tiles_fit(P, Q):
        hnb = 32 if C % 32 == 0 else (48 if C % 48 == 0 else 16)
        tiles = N * _ceil(P, 8) * _ceil(Q, 8)
        hitems = rb_all * (C // hnb)
        chain = 0
        for ctas in (1, 2):  # the launch's CTAs per SM come from the kernel's register count: take the longer chain of either
            splits = max(1, sms * ctas // hitems)
            per = _ceil(tiles, splits)
            chain = max(chain, per * 64 + _ceil(tiles, per) + 1)
        return Route("wgmma", "wgrad3x3_halo_kernel", f"nb{hnb}" + ("_cf" if cf else ""), 1, 0, 1, chain)
    stage_bytes = 2 * 64 * 128 + (nb // cb) * 64 * cb * 2
    stages = min(8, (200 * 1024 - 128 - 1024) // stage_bytes)
    odd = rb_all % 2 or rb_off % 2
    even_forced = bool(odd and stages % 2)
    base = items * (C // nb)
    total = _ceil(npix, 64)
    splits = min(_ceil(2 * sms, base), total // 8)
    splits = max(splits, 1)
    per = _ceil(total, splits) * 64
    splits = _ceil(npix, per)
    tag = f"nb{nb}_cb{cb}_rb{rb_all}.{rb_off}" + ("_even_ring" if even_forced else "") + ("_split" if splits > 1 else "")
    return Route("wgmma", "wgrad_wgmma_kernel", tag, 1, 0, 0, per + splits + 1)


def route(op, d, flags=None, sms=132):
    """The engine, kernel, tile variant and launch-counter deltas the library picks for one call.  d: SgbConvDesc fields (desc_of);
    flags: accumulate, out_f32, stats, force (sgb_conv_force_im2col), wgrad_force (sgb_conv_wgrad_force_im2col).  Operand pointers are
    taken to be 16-byte aligned (every front end and case here passes such)."""
    f = flags or {}
    N, H, W, C, K, R, S, st, pad, P, Q = (d[k] for k in ("N", "H", "W", "C", "K", "R", "S", "stride", "pad", "P", "Q"))
    if op == "fprop":
        if f.get("out_f32"):
            return _mma(op, d)
        if pad == R // 2:
            q = _gemm(C, d["x_pitch"], K, R, st, pad, N, H, W, P, Q, d["y_pitch"], centre_from=d["centre_from"], stats=bool(f.get("stats")))
            if _supported(q):
                return _launch(q, f.get("force"))
        if _row_pairs(d):
            q = _gemm(2 * C, 2 * C, K, 1, 1, 0, N * (H // 2), 2, W // 2, 1, W // 2, d["y_pitch"], taps=2, ntaps=2, stats=bool(f.get("stats")))
            r = _launch(q, f.get("force"))
            return r._replace(variant="row_pairs_" + r.variant)
        return _mma(op, d)
    if op == "convt2x2":
        if K % 16 or C % 16:
            return _mma(op, d)
        q = _gemm(K, d["y_pitch"], C, 1, 1, 0, N, P, Q, P, Q, d["x_pitch"], out_mode=1)
        if not _supported(q):
            return _mma(op, d)
        r = _launch(q, f.get("force"), nlaunch=4)
        return r._replace(variant="parity4_" + r.variant)
    if op == "dgrad":
        acc = bool(f.get("accumulate"))
        if st == 1 and pad == R // 2 and K % 16 == 0:
            q = _gemm(K, d["y_pitch"], C, R, 1, R - 1 - pad, N, P, Q, H, W, d["x_pitch"], flip=1, centre_from=d["centre_from"])
            if _supported(q):
                r = _launch(q, f.get("force"))
                return r._replace(variant=r.variant + ("_acc" if acc else ""))
        if st == 2 and K % 16 == 0 and R == 3 and S == 3 and pad == 1 and H == 2 * P and W == 2 * Q:
            q = _gemm(K, d["y_pitch"], C, 3, 1, 0, N, P, Q, P, Q, d["x_pitch"], taps=4, ntaps=4, out_mode=1)
            if not _supported(q):
                return _mma(op, d)
            r = _launch(q, f.get("force"), nlaunch=4)
            return r._replace(variant="parity4_" + r.variant + ("_acc" if acc else ""))
        if st == 2 and K % 16 == 0 and R == 1 and S == 1 and pad == 0 and H == 2 * P and W == 2 * Q:
            q = _gemm(K, d["y_pitch"], C, 1, 1, 0, N, P, Q, P, Q, d["x_pitch"], out_mode=1)
            dense = d["x_pitch"] == C and d["x_off"] == 0
            if _supported(q) and (acc or dense):
                r = _launch(q, f.get("force"))
                return r._replace(variant="s2_1x1_" + ("acc" if acc else "memset") + "_" + r.variant)
        return _mma(op, d)
    if op == "wgrad":
        r = None
        if pad == R // 2 and st in (1, 2) and R == S and R in (1, 3):
            r = _wgrad_route(d, R, S, C, d["x_pitch"], N, H, W, P, Q, st, pad, f, sms)
        elif _row_pairs(d):
            r = _wgrad_route(dict(d, centre_from=0), 2, 1, 2 * C, 2 * C, N * (H // 2), 2, W // 2, 1, W // 2, 1, 0, f, sms)
            r = r._replace(variant="row_pairs_" + r.variant) if r else None
        return r or _mma(op, d)
    raise ValueError(op)


def case_flags(c):
    return dict(accumulate=c["accumulate"], out_f32=c["out_f32"], stats=c["stats"] > 0, force=c["force"] and c["op"] != "wgrad",
                wgrad_force=c["force"] and c["op"] == "wgrad")


def case_route(c, sms=132):
    return route(c["op"], desc_of(c), case_flags(c), sms)


def route_tags(c, r):
    """What one case reaches: '<op>:<kernel>:<variant>' plus one tag per epilogue / layout / mode option."""
    op, k = c["op"], r.kernel
    tags = {f"{op}:{k}", f"{op}:{k}:{r.variant}"}
    opts = []
    if c["stats"]:
        opts.append(f"stats_repl{c['stats']}")
    for key in ("scale", "shift", "residual", "out_f32", "accumulate", "force"):
        if c[key]:
            opts.append(key)
    if c["act"] != "none":
        opts.append("act_" + c["act"])
    if c["centre_from"]:
        opts.append("centre_from")
        if c["centre_from"] % 64:
            opts.append("centre_from_inside_row_block")
    if c["x_pitch"] and c["x_pitch"] != c["C"]:
        opts.append("x_slice")
    if c["y_pitch"] and c["y_pitch"] != c["K"]:
        opts.append("y_slice")
    if c["op"] != "convt2x2" and (c["H"] % 2 or c["W"] % 2):
        opts.append("odd_map")
    tags.update(f"{op}:{k}:{o}" for o in opts)
    return tags


# Every (op, kernel, variant / option) the matrix must reach, row by row of the route table.
REQUIRED = {
    # conv3x3_halo_kernel
    *(f"fprop:conv3x3_halo_kernel:bn{b}" for b in (16, 32, 48, 64, 96, 128)), "fprop:conv3x3_halo_kernel:bn96_narrowed",
    "fprop:conv3x3_halo_kernel:bn64_narrowed", "fprop:conv3x3_halo_kernel:stats_repl1", "fprop:conv3x3_halo_kernel:stats_repl8",
    "fprop:conv3x3_halo_kernel:scale", "fprop:conv3x3_halo_kernel:shift", "fprop:conv3x3_halo_kernel:residual", "fprop:conv3x3_halo_kernel:act_relu",
    "fprop:conv3x3_halo_kernel:act_silu", "fprop:conv3x3_halo_kernel:odd_map", "fprop:conv3x3_halo_kernel:x_slice", "fprop:conv3x3_halo_kernel:y_slice",
    # conv_wgmma_kernel
    *(f"fprop:conv_wgmma_kernel:bn{b}_kc64" for b in (16, 32, 48, 64, 96, 128)), "fprop:conv_wgmma_kernel:bn48_kc16", "fprop:conv_wgmma_kernel:bn48_kc32",
    "fprop:conv_wgmma_kernel:bn128_kc64_skip", "fprop:conv_wgmma_kernel:force", "fprop:conv_wgmma_kernel:act_silu", "fprop:conv_wgmma_kernel:stats_repl1",
    "fprop:conv_wgmma_kernel:row_pairs_bn64_kc64",
    # mma.sync fprop
    "fprop:igemm_conv_kernel:out_f32", "fprop:igemm_conv_kernel:bn32", "fprop:igemm_conv_kernel:bn64", "fprop:igemm_conv_kernel:bn128",
    "fprop:igemm_conv_kernel:x_slice", "fprop:igemm_conv_kernel:act_silu", "fprop:igemm_conv_kernel:stats_repl8",
    # convt2x2
    "convt2x2:conv_wgmma_kernel:parity4_bn32_kc64", "convt2x2:conv_wgmma_kernel:parity4_bn48_kc32", "convt2x2:igemm_conv_kernel",
    # dgrad
    "dgrad:conv3x3_halo_kernel:bn64", "dgrad:conv3x3_halo_kernel:bn64_skip", "dgrad:conv3x3_halo_kernel:accumulate", "dgrad:conv_wgmma_kernel:bn64_kc64",
    "dgrad:conv_wgmma_kernel:bn64_kc64_skip_acc", "dgrad:conv_wgmma_kernel:force", "dgrad:conv_wgmma_kernel:parity4_bn32_kc64",
    "dgrad:conv_wgmma_kernel:parity4_bn64_kc64_acc", "dgrad:igemm_conv_kernel:odd_map", "dgrad:conv_wgmma_kernel:s2_1x1_memset_bn64_kc64",
    "dgrad:conv_wgmma_kernel:s2_1x1_acc_bn64_kc64", "dgrad:igemm_conv_kernel:x_slice", "dgrad:igemm_conv_kernel:y_slice",
    "dgrad:igemm_conv_kernel:accumulate", "dgrad:conv3x3_halo_kernel:x_slice",
    # wgrad
    "wgrad:wgrad3x3_halo_kernel:nb16", "wgrad:wgrad3x3_halo_kernel:nb32", "wgrad:wgrad3x3_halo_kernel:nb48", "wgrad:wgrad3x3_halo_kernel:nb32_cf",
    "wgrad:wgrad3x3_halo_kernel:odd_map", "wgrad:wgrad3x3_halo_kernel:centre_from_inside_row_block",
    "wgrad:wgrad_wgmma_kernel:centre_from_inside_row_block", "wgrad:wgrad3x3_halo_kernel:x_slice",
    "wgrad:wgrad_wgmma_kernel:nb16_cb16_rb1.1", "wgrad:wgrad_wgmma_kernel:nb32_cb32_rb1.1", "wgrad:wgrad_wgmma_kernel:nb64_cb64_rb1.1",
    "wgrad:wgrad_wgmma_kernel:nb128_cb64_rb1.1",
    "wgrad:wgrad_wgmma_kernel:nb48_cb16_rb1.1", "wgrad:wgrad_wgmma_kernel:nb96_cb32_rb1.1_even_ring", "wgrad:wgrad_wgmma_kernel:nb96_cb32_rb2.2",
    "wgrad:wgrad_wgmma_kernel:nb96_cb32_rb3.3_even_ring", "wgrad:wgrad_wgmma_kernel:nb96_cb32_rb2.1_even_ring", "wgrad:wgrad_wgmma_kernel:nb96_cb32_rb3.2_even_ring",
    "wgrad:wgrad_wgmma_kernel:force", "wgrad:wgrad_wgmma_kernel:nb64_cb64_rb1.1_split", "wgrad:wgrad_wgmma_kernel:row_pairs_nb96_cb32_rb1.1_even_ring",
    "wgrad:wgrad_kernel:bmw32", "wgrad:wgrad_kernel:bmw64", "wgrad:wgrad_kernel:bmw128", "wgrad:wgrad_kernel:centre_from",
}


def missing_routes(cases, sms=132):
    seen = set()
    for c in cases:
        seen |= route_tags(c, case_route(c, sms))
    return sorted(REQUIRED - seen), seen


# ------------------------------------------------------------------------------------------------ operands of a case
def case_operands(c, real, gen, device):
    """fp64 NCHW operands (bf16-exact values) of case c: integer (exact checks, cap asserted) or real-valued (bounds)."""
    op, N, C, H, W, K, R, st, pad = (c[k] for k in ("op", "N", "C", "H", "W", "K", "R", "stride", "pad"))
    d = desc_of(c)
    P, Q = d["P"], d["Q"]
    o = {}
    if op == "convt2x2":
        xs, ws = (N, K, H, W), (K, C, 2, 2)
        absfn = lambda a, b: convt2x2_ref(a, b)  # noqa: E731
        L = K
    elif op == "fprop":
        xs, ws = (N, C, H, W), (K, C, R, R)
        absfn = lambda a, b: conv64(a, zero_off_centre(b, c["centre_from"]), st, pad)  # noqa: E731
        L = C * R * R
    elif op == "dgrad":
        xs, ws = (N, K, P, Q), (K, C, R, R)
        absfn = lambda a, b: dgrad64(a, zero_off_centre(b, c["centre_from"]), (N, C, H, W), st, pad)  # noqa: E731
        L = K * R * R
    else:
        xs, ws = (N, C, H, W), (N, K, P, Q)
        absfn = lambda a, b: wgrad64(a, b, R, R, st, pad)  # noqa: E731
        L = N * P * Q
    if real:
        a = real_bf16(xs, gen, device=device)
        b = real_bf16(ws, gen, 1.0 if op == "wgrad" else 0.2, device=device)
        o["cap_seen"] = None
    else:
        a, b, o["cap_seen"] = int_operands(xs, ws, absfn, L, c["cap"], gen, device)
    if op == "wgrad":
        o["x"], o["dy"] = a, b
        K_, R_ = K, R
        o["dw_old"] = (torch.randint(-32, 33, (K_, R_, R_, C), generator=gen).double() / 4).to(device)
    elif op == "dgrad":
        o["dy"], o["w"] = a, zero_off_centre(b, c["centre_from"])
        o["dx_old"] = torch.randint(-8, 9, (N, C, H, W), generator=gen).double().to(device) if c["accumulate"] else None
        if real and c["accumulate"]:
            o["dx_old"] = real_bf16((N, C, H, W), gen, device=device)
    elif op == "fprop":
        o["x"], o["w"] = a, zero_off_centre(b, c["centre_from"])
    else:
        o["x"], o["w"] = a, b
        o["bias"] = (torch.randint(-8, 9, (C,), generator=gen).double() / 4).to(device) if c["bias"] else None
    if op == "fprop":
        if c["scale"]:
            s = torch.tensor([0.5, 1.0, 2.0], dtype=F64)[torch.randint(0, 3, (K,), generator=gen)] * (torch.randint(0, 2, (K,), generator=gen) * 2 - 1)
            o["scale"] = (s if not real else (torch.rand(K, generator=gen, dtype=F64) + 0.5).float().double()).to(device)
        if c["shift"]:
            s = torch.randint(-16, 17, (K,), generator=gen).double() / 4
            o["shift"] = (s if not real else torch.randn(K, generator=gen, dtype=F64).float().double()).to(device)
        if c["residual"]:
            o["residual"] = (torch.randint(-8, 9, (N, K, P, Q), generator=gen).double().to(device) if not real else real_bf16((N, K, P, Q), gen, device=device))
    return o


# ------------------------------------------------------------------------------------------------ verification
def verify_fprop(c, o, got, exact, chain=None):
    """got: {"y": fp64 NCHW (the stored output), "stats": [2, K] summed over replicas or absent}."""
    acc = conv64(o["x"], o["w"], c["stride"], c["pad"])
    ep = dict(scale=o.get("scale"), shift=o.get("shift"), residual=o.get("residual"), act=c["act"])
    pre, y = epilogue64(acc, **ep)
    bf16 = not c["out_f32"]
    if exact and c["act"] != "silu":
        expect_exact("fprop y", got["y"], round_bf16(y) if bf16 else y)
    else:
        e = torch.zeros_like(acc)
        if not exact:
            e = gamma23(chain or fprop_chain(c["C"], c["R"], c["R"])) * conv64(o["x"].abs(), o["w"].abs(), c["stride"], c["pad"])
        y, e = epilogue_err(acc, e, **ep)
        expect_within("fprop y", got["y"], y, e, bf16=bf16)
    if got.get("stats") is not None:
        expect_stats("fprop stats", got["stats"], got["y"])


def verify_dgrad(c, o, got, exact, chain=None):
    """got: {"dx": fp64 NCHW}."""
    N, C, H, W = c["N"], c["C"], c["H"], c["W"]
    g = dgrad64(o["dy"], o["w"], (N, C, H, W), c["stride"], c["pad"])
    old = o.get("dx_old") if c["accumulate"] else None
    if exact:
        expect_exact("dgrad dx", got["dx"], round_bf16(g if old is None else g + old))
    else:
        e = gamma23(chain or fprop_chain(_ceil(c["K"], 8) * 8, c["R"], c["R"])) * dgrad64(o["dy"].abs(), o["w"].abs(), (N, C, H, W), c["stride"], c["pad"])
        y, e = epilogue_err(g, e, residual=old)
        expect_within("dgrad dx", got["dx"], y, e, bf16=True)


def verify_wgrad(c, o, got, exact, chain):
    """got: {"dw": fp32 KRSC after the call}; o["dw_old"]: before it."""
    R, st, pad = c["R"], c["stride"], c["pad"]
    g = wgrad64(o["x"], o["dy"], R, R, st, pad)
    keep = centre_mask(*g.shape, c["centre_from"], g.device)
    g = torch.where(keep, g, torch.zeros_like(g))
    want = o["dw_old"] + g
    if exact:
        expect_exact("wgrad dw", got["dw"], want)
    else:
        e = gamma23(chain) * wgrad64(o["x"].abs(), o["dy"].abs(), R, R, st, pad)
        e = torch.where(keep, e + 1.0001 * U32 * (want.abs() + e), torch.zeros_like(e))
        expect_within("wgrad dw", got["dw"], want, e)
    if c["centre_from"]:
        expect_exact("wgrad dw (entries centre_from leaves alone)", got["dw"][~keep], o["dw_old"][~keep])


def verify_convt2x2(c, o, got, exact, chain=None):
    y = convt2x2_ref(o["x"], o["w"], o.get("bias"))
    if exact:
        expect_exact("convt2x2 y", got["y"], round_bf16(y))
    else:
        acc = convt2x2_ref(o["x"], o["w"])
        e = gamma23(chain or _ceil(c["K"], 64) * 64) * convt2x2_ref(o["x"].abs(), o["w"].abs())
        y, e = epilogue_err(acc, e, shift=o.get("bias"))
        expect_within("convt2x2 y", got["y"], y, e, bf16=True)


VERIFY = {"fprop": verify_fprop, "dgrad": verify_dgrad, "wgrad": verify_wgrad, "convt2x2": verify_convt2x2}


# ------------------------------------------------------------------------------------------------ fp32 transcription (CPU)
MUTATIONS = ("drop_kstep", "halo_shift", "parity_taps", "oh_add", "acc_bf16", "truncate_store", "shift_first", "residual_twice", "stats_drop_warp",
             "wgrad_offcentre")


def _bf16(t, mut=None):
    t = t.float()
    if mut == "truncate_store":
        return (t.view(torch.int32) & ~0xFFFF).view(torch.float32).double()
    return t.bfloat16().double()


def t_gemm(A, B, mut=None, kstep=16):
    """fp32 implicit GEMM: A [M, T, Kc], B [N, T, Kc] -> [M, N], accumulated tap by tap in k-steps of `kstep` channels."""
    A, B = A.float(), B.float()
    M, T, Kc = A.shape
    acc = torch.zeros(M, B.shape[0], dtype=torch.float32)
    steps = list(range(0, Kc, kstep))
    for t in range(T):
        for k0 in steps:
            if mut == "drop_kstep" and t == T // 2 and k0 == steps[-1]:
                continue
            acc = acc + A[:, t, k0 : k0 + kstep] @ B[:, t, k0 : k0 + kstep].T
            if mut == "acc_bf16":
                acc = acc.bfloat16().float()
    return acc


def _im2col(x, R, S, stride, pad, mut=None):
    """[N, C, H, W] -> [N * P * Q, R * S, C] (NHWC pixel order)."""
    N, C = x.shape[:2]
    xp = F.pad(x.float(), (pad, pad, pad, pad))
    if mut == "halo_shift":  # every tap reads one column to the right
        xp = F.pad(xp[..., 1:], (0, 1))
    cols = F.unfold(xp, (R, S), stride=stride)  # [N, C * R * S, L]
    L = cols.shape[-1]
    return cols.view(N, C, R * S, L).permute(0, 3, 2, 1).reshape(N * L, R * S, C)


def _nchw(rows, N, P, Q):
    return rows.view(N, P, Q, -1).permute(0, 3, 1, 2)


def t_epilogue(acc, scale=None, shift=None, residual=None, act="none", mut=None):
    v = acc.float()
    if mut == "shift_first" and shift is not None:
        v = v + shift.float().view(1, -1, 1, 1)
    if scale is not None:
        v = v * scale.float().view(1, -1, 1, 1)
    if shift is not None and mut != "shift_first":
        v = v + shift.float().view(1, -1, 1, 1)
    if residual is not None:
        v = v + residual.float()
        if mut == "residual_twice":
            v = v + residual.float()
    if act == "relu":
        v = v.clamp_min(0)
    elif act == "silu":
        v = v / (1 + torch.exp(-v))
    return v


def t_stats(y, mut=None, rows=128, warp_rows=16):
    """Per-channel sum of y and y^2 as the epilogues form them: fp32 per 16-row warp slice, fp32 per 128-row tile, fp64 across tiles."""
    m = y.permute(0, 2, 3, 1).reshape(-1, y.shape[1]).float()
    out = torch.zeros(2, y.shape[1], dtype=F64)
    for t0 in range(0, m.shape[0], rows):
        tile = m[t0 : t0 + rows]
        s1 = torch.zeros(y.shape[1])
        s2 = torch.zeros(y.shape[1])
        for w0 in range(0, tile.shape[0], warp_rows):
            if mut == "stats_drop_warp" and t0 == 0 and w0 == warp_rows:
                continue
            part = tile[w0 : w0 + warp_rows]
            s1, s2 = s1 + part.sum(0), s2 + (part * part).sum(0)
        out[0] += s1.double()
        out[1] += s2.double()
    return out


def t_fprop(c, o, mut=None):
    x, w = o["x"], o["w"]
    N, K, R, st, pad = c["N"], c["K"], c["R"], c["stride"], c["pad"]
    A = _im2col(x, R, R, st, pad, mut)
    B = w.float().reshape(K, w.shape[1], R * R).permute(0, 2, 1)
    d = desc_of(c)
    acc = _nchw(t_gemm(A, B, mut), N, d["P"], d["Q"])
    y = t_epilogue(acc, o.get("scale"), o.get("shift"), o.get("residual"), c["act"], mut)
    y = y.double() if c["out_f32"] else _bf16(y, mut)
    return {"y": y, "stats": t_stats(y, mut) if c["stats"] else None}


def stride2_taps(ph, pw, pad, R=3, S=3):
    """(dh, dw, r, s) of the taps that reach input-gradient parity class (ph, pw) of a stride-2 convolution."""
    return [((ph + pad - r) // 2, (pw + pad - s) // 2, r, s) for r in range(R) if (ph + pad - r) % 2 == 0 for s in range(S) if (pw + pad - s) % 2 == 0]


def t_dgrad(c, o, mut=None):
    dy, w = o["dy"], o["w"]
    N, C, H, W, K, R, st, pad = (c[k] for k in ("N", "C", "H", "W", "K", "R", "stride", "pad"))
    old = o.get("dx_old") if c["accumulate"] else None
    if st == 1:
        wf = w.transpose(0, 1).flip(2, 3)  # [C, K, R, S]
        A = _im2col(dy, R, R, 1, R - 1 - pad, mut)
        acc = _nchw(t_gemm(A, wf.float().reshape(C, K, R * R).permute(0, 2, 1), mut), N, H, W)
        return {"dx": _bf16(t_epilogue(acc, residual=old, mut=mut), mut)}
    assert st == 2 and R == 3 and pad == 1 and H % 2 == 0 and W % 2 == 0
    P, Q = H // 2, W // 2
    dx = torch.zeros(N, C, H, W, dtype=F64)
    dyp = F.pad(dy.float(), (1, 1, 1, 1))  # dy rows / columns -1 .. P
    for cls in range(4):
        ph, pw = cls >> 1, cls & 1
        taps = stride2_taps(*((1, 0) if mut == "parity_taps" and cls == 3 else (ph, pw)), pad)
        A = torch.stack([dyp[:, :, 1 + dh : 1 + dh + P, 1 + dw_ : 1 + dw_ + Q].permute(0, 2, 3, 1).reshape(-1, K) for dh, dw_, _, _ in taps], 1)
        B = torch.stack([w[:, :, r, s].T for _, _, r, s in taps], 1)  # [C, T, K]
        acc = _nchw(t_gemm(A, B, mut), N, P, Q)
        oh = 0 if mut == "oh_add" and ph == 1 else ph
        res = None if old is None else old[:, :, ph::2, pw::2]
        dx[:, :, oh::2, pw::2] = _bf16(t_epilogue(acc, residual=res, mut=mut), mut)
    return {"dx": dx}


def t_wgrad(c, o, mut=None, wpix=64):
    x, dy = o["x"], o["dy"]
    N, C, K, R, st, pad, cf = (c[k] for k in ("N", "C", "K", "R", "stride", "pad", "centre_from"))
    A = _im2col(x, R, R, st, pad).reshape(-1, R * R * C)  # [pix, (r, s, c)]
    D = dy.float().permute(0, 2, 3, 1).reshape(-1, K)
    acc = torch.zeros(K, R * R * C)
    for p0 in range(0, A.shape[0], wpix):
        acc = acc + D[p0 : p0 + wpix].T @ A[p0 : p0 + wpix]
    acc = acc.view(K, R, R, C)
    dw = (o["dw_old"].float() + acc).double()
    if cf and mut != "wgrad_offcentre":
        dw = torch.where(centre_mask(K, R, R, C, cf, dw.device), dw, o["dw_old"])
    return {"dw": dw}


TRANSCRIPTION = {"fprop": t_fprop, "dgrad": t_dgrad, "wgrad": t_wgrad}


# ------------------------------------------------------------------------------------------------ recorder
REC_OPS = ("conv_fprop", "conv_dgrad", "conv_wgrad", "convt2x2_fprop")
_INPLACE = {"conv_fprop": ("stats",)}  # the in-place outputs (dgrad's out, wgrad's dw_krsc) are the results


def _counters():
    from super_gradients_b200 import lib

    L = lib.load()
    return (L.sgb_sm100_launches(), L.sgb_conv_halo_launches(), L.sgb_conv_wgrad_halo_launches())


@contextlib.contextmanager
def record_conv():
    """Patches K.conv_fprop / conv_dgrad / conv_wgrad / convt2x2_fprop for the block and yields the list of calls made in it:
    {"op", "a" (the bound arguments, cloned before the call), "pitch" (pixel stride of every 4-d argument), "align" (every tensor
    argument's data_ptr is 16-byte aligned), "out" (the result, cloned after the call), "after" (the in-place state after it),
    "launches" (deltas of the three launch counters)}.  The device is synchronised around each call: the weight gradients run on
    the step's side stream.  functools.wraps keeps each front end's signature visible: functional._centre_kw reads it to decide whether
    to pass centre_from."""
    from super_gradients_b200 import kernels as K

    orig = {n: getattr(K, n) for n in REC_OPS}
    calls = []

    def wrap(name):
        fn = orig[name]
        sig = inspect.signature(fn)

        @functools.wraps(fn)
        def f(*args, **kw):
            torch.cuda.synchronize()
            b = sig.bind(*args, **kw)
            b.apply_defaults()
            a = {k: _clone(v) for k, v in b.arguments.items()}
            tens = {k: v for k, v in b.arguments.items() if torch.is_tensor(v)}
            entry = {"op": name, "a": a, "pitch": {k: _pitch(v) for k, v in tens.items() if v.dim() == 4},
                     "align": all(v.data_ptr() % 16 == 0 for v in tens.values())}
            n0 = _counters()
            out = fn(*args, **kw)
            torch.cuda.synchronize()
            entry["launches"] = tuple(b_ - a_ for a_, b_ in zip(n0, _counters()))
            entry["out"] = _clone(out)
            entry["pitch"]["result"] = _pitch(out)
            entry["after"] = {k: _clone(b.arguments[k]) for k in _INPLACE.get(name, ()) if torch.is_tensor(b.arguments.get(k))}
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


def pose_infer_record(name="yolo_nas_pose_s", batch=2, img=640, seed=0):
    """One inference forward of a YOLO-NAS-POSE model (folded BatchNorm: the scale / shift / activation epilogues), recorded."""
    from super_gradients_b200.training import models

    torch.manual_seed(seed)
    m = models.get(name, num_classes=17).cuda().eval()
    g = torch.Generator().manual_seed(seed + 1)
    x = torch.randn(batch, 3, img, img, generator=g).cuda()
    with record_conv() as calls, torch.no_grad():
        m(x)
        torch.cuda.synchronize()
    return calls


# ------------------------------------------------------------------------------------------------ replay
def _act_name(act):
    from super_gradients_b200 import lib

    return {lib.ACT_NONE: "none", lib.ACT_RELU: "relu", lib.ACT_SILU: "silu"}[act] if isinstance(act, int) else ("none" if act is None else act)


def _recorded_desc(r):
    """(op, SgbConvDesc fields, flags, case-like dict, operands) of one recorded call."""
    a, op = r["a"], r["op"]
    if op == "conv_fprop":
        x, krsc = a["x"], a["w_krsc"]
        N, C, H, W = x.shape
        K, R, S = a["K"], a["R"], a["S"]
        st, pad = a["stride"], a["pad"]
        out = r["out"]
        c = make_case("fprop", N, C, H, W, K, r=R, stride=st, pad=pad, x_pitch=r["pitch"]["x"], y_pitch=r["pitch"]["result"], act=_act_name(a["act"]),
                      out_f32=bool(a["out_f32"]), centre_from=a["centre_from"], stats=a["stats"].shape[0] if a["stats"] is not None else 0,
                      scale=a["scale"] is not None, shift=a["shift"] is not None, residual=a["residual"] is not None)
        w = krsc.double()[:K].permute(0, 3, 1, 2)
        o = {"x": x.double(), "w": w, "scale": None if a["scale"] is None else a["scale"][:K], "shift": None if a["shift"] is None else a["shift"][:K], "residual": None if a["residual"] is None else a["residual"].double()}
        got = {"y": out.double()}
        if a["stats"] is not None:
            got["stats"] = (r["after"]["stats"] - a["stats"]).sum(0)
        return "fprop", c, o, got
    if op == "conv_dgrad":
        dy, crsk = a["dy"], a["w_crsk"]
        N, C, H, W = a["x_shape"]
        K = dy.shape[1]
        R = a["R"]
        out = r["out"]
        c = make_case("dgrad", N, C, H, W, K, r=R, stride=a["stride"], pad=a["pad"], x_pitch=r["pitch"]["result"], y_pitch=r["pitch"]["dy"],
                      accumulate=bool(a["accumulate"]), centre_from=a["centre_from"])
        w = crsk.double()[..., :K].permute(3, 0, 1, 2)  # [C, R, S, Kp] -> [K, C, R, S]
        o = {"dy": dy.double(), "w": w, "dx_old": a["out"].double() if a["accumulate"] else None}
        return "dgrad", c, o, {"dx": out.double()}
    if op == "conv_wgrad":
        x, dy = a["x"], a["dy"]
        N, C, H, W = x.shape
        K, R = dy.shape[1], a["R"]
        c = make_case("wgrad", N, C, H, W, K, r=R, stride=a["stride"], pad=a["pad"], x_pitch=r["pitch"]["x"], y_pitch=r["pitch"]["dy"],
                      centre_from=a["centre_from"])
        dw_old = a["dw_krsc"].double() if a["dw_krsc"] is not None else torch.zeros(K, R, a["S"], C, dtype=F64, device=x.device)
        return "wgrad", c, {"x": x.double(), "dy": dy.double(), "dw_old": dw_old}, {"dw": r["out"].double()}
    x, w_up = a["x_small"], a["w_up"]
    N, Kin, P, Q = x.shape
    Cu = a["C_up"]
    c = make_case("convt2x2", N, Cu, P, Q, Kin, x_pitch=r["pitch"]["x_small"])
    w_t = w_up.double().view(2, 2, Cu, Kin).permute(3, 2, 0, 1)
    return "convt2x2", c, {"x": x.double(), "w": w_t, "bias": a["bias"]}, {"y": r["out"].double()}


def replay_conv(calls, sms):
    """Checks every recorded call against the fp64 oracle with the real-valued bounds and its launch-counter deltas against the route
    mirror; frees each call once checked.  Returns {op:kernel:variant tags seen}."""
    seen = set()
    for i in range(len(calls)):
        r = calls[i]
        calls[i] = None
        op, c, o, got = _recorded_desc(r)
        rt = route(op, desc_of(c), case_flags(c), sms)
        assert r["align"], f"call {i} ({c['id']}): an unaligned operand (the route mirror assumes 16-byte alignment)"
        assert r["launches"] == (rt.launches, rt.halo, rt.whalo), f"call {i} ({c['id']}): launches {r['launches']}, the route mirror says {rt}"
        try:
            VERIFY[op](c, o, got, exact=False, chain=rt.chain)
        except AssertionError as e:
            raise AssertionError(f"call {i} ({c['id']}, {rt.kernel} {rt.variant}): {e}") from None
        seen |= route_tags(c, rt)
        del r, o, got
    return seen
