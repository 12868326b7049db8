"""Thin torch-tensor front end of the C ABI (lib.py).  Every function here launches CUDA kernels from libsgb200.so on
the current torch stream; torch is used only for device memory and streams.  No function has a non-CUDA fallback.

Activation tensors are NCHW-shaped torch tensors in channels_last memory format (physically NHWC bf16).  A channel
slice ``buf[:, a:b]`` of such a tensor is a valid operand: its channel pitch is ``buf.shape[1]``.
"""
import ctypes
import os
from typing import Optional

import torch

from . import lib as L
from .lib import ACT_NONE, ACT_RELU, ACT_SILU  # noqa: F401

STATS_REPL = 8  # replicas of the per-channel sum buffers (spreads fp64 atomics)

# Optional per-launch timing (bench.py roofline pass): (name, start_event, end_event) on the launching stream.
PROFILE_ON = [False]
PROFILE = []


def _timed(name, *args):
    if not PROFILE_ON[0]:
        return L.call(name, *args)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    L.call(name, *args)
    b.record()
    d = args[0]._obj if args and hasattr(args[0], "_obj") else None  # ctypes.byref(desc)
    tag = tuple(getattr(d, f) for f in ("N", "H", "W", "C", "K", "R", "stride") if hasattr(d, f)) if d is not None else ()
    PROFILE.append((name, a, b, tag))

class StepArena:
    """Zero-initialised scratch of ONE training step (BatchNorm / moment accumulators, fp32 weight-gradient buffers).

    Outside a step (`active` False) `zeros()` is plain torch.zeros.  training/sg_trainer.TrainStep brackets every step with
    begin_step() / end_step(): the first bracketed step only measures the demand, later steps sub-allocate from one buffer
    that a single memset clears, instead of one fill kernel per tensor (~360 launches per YOLO-NAS-S step).  Tensors
    handed out never outlive the step that requested them."""

    ALIGN = 256

    def __init__(self):
        self.buf = None
        self.off = 0
        self.need = 0
        self.active = False

    def begin_step(self, device):
        if self.buf is None and self.need > 0:
            self.buf = torch.empty(int(self.need * 1.25) + (1 << 20), dtype=torch.uint8, device=device)
            self.high = self.buf.numel()
        if self.buf is not None:
            self.buf[: min(self.high, self.buf.numel())].zero_()
            self.high = 0
        self.off = 0
        self.need = 0
        self.active = True

    def end_step(self):
        self.active = False
        if self.buf is not None:
            self.high = self.off

    def zeros(self, shape, dtype, device):
        if not self.active:
            return torch.zeros(shape, dtype=dtype, device=device)
        n = 1
        for d in shape:
            n *= d
        nbytes = n * torch.empty((), dtype=dtype).element_size()
        span = (nbytes + self.ALIGN - 1) // self.ALIGN * self.ALIGN
        self.need += span
        if self.buf is None or self.off + span > self.buf.numel() or self.buf.device != torch.device(device):
            return torch.zeros(shape, dtype=dtype, device=device)
        out = self.buf[self.off : self.off + nbytes].view(dtype).view(shape)
        self.off += span
        return out


NO_ARENA = StepArena()  # never activated: zeros() is torch.zeros
ARENA = NO_ARENA        # the arena of the TrainStep that is executing (training/sg_trainer.py swaps it in and out)


def zeros(shape, dtype, device):
    return ARENA.zeros(tuple(shape) if not isinstance(shape, int) else (shape,), dtype, device)


# BatchNorm / QARepVGG backward as one cooperative launch per layer instead of a reduction launch + an apply launch (SGB_FUSED_BWD=0: two passes)
FUSED_BWD = [os.environ.get("SGB_FUSED_BWD", "1") != "0"]
FUSED_FWD = [os.environ.get("SGB_FUSED_FWD", "1") != "0"]  # QARepVGG forward: moments + apply as one cooperative launch

_ACT = {None: ACT_NONE, "none": ACT_NONE, "relu": ACT_RELU, "silu": ACT_SILU}


def act_code(act) -> int:
    if isinstance(act, int):
        return act
    return _ACT[act]


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def require_cuda(t: torch.Tensor, name="tensor"):
    if not t.is_cuda:
        raise L.SgbError(f"{name} must live on a CUDA device: super_gradients_b200 has no CPU execution path")


def nhwc_pitch(t: torch.Tensor) -> int:
    """Channel pitch (elements) of an NHWC operand; raises if `t` is not laid out as (a channel slice of) NHWC."""
    if t.dim() != 4:
        raise L.SgbError(f"expected a 4-d activation tensor, got shape {tuple(t.shape)}")
    n, c, h, w = t.shape
    sn, sc, sh, sw = t.stride()
    if c > 1 and sc != 1:
        raise L.SgbError(f"tensor with shape {tuple(t.shape)} strides {t.stride()} is not NHWC (channel stride != 1)")
    if w > 1:
        pitch = sw
    elif h > 1:
        pitch = sh
    elif n > 1:
        pitch = sn
    else:
        return ((c + 7) // 8) * 8  # a single pixel: any pitch describes it
    ok = pitch >= c and (w == 1 or sw == pitch) and (h == 1 or sh == w * pitch) and (n == 1 or sn == h * w * pitch)
    if not ok:
        raise L.SgbError(f"tensor with shape {tuple(t.shape)} strides {t.stride()} is not NHWC")
    return pitch


def as_nhwc(t: torch.Tensor) -> torch.Tensor:
    """Returns `t` itself if it is a valid NHWC bf16 operand, else a channels_last bf16 copy."""
    require_cuda(t)
    if t.dtype == torch.bfloat16:
        try:
            p = nhwc_pitch(t)
            if p % 8 == 0 and t.data_ptr() % 16 == 0:
                return t
        except L.SgbError:
            pass
    n, c, h, w = t.shape
    out = empty_nhwc(n, c, h, w, t.device)
    out.copy_(t)
    return out


def empty_nhwc(n, c, h, w, device, c_alloc=None) -> torch.Tensor:
    """bf16 NHWC tensor with logical channels c; storage pitch is c rounded up to 8 (padding channels are zero)."""
    ca = c_alloc or ((c + 7) // 8) * 8
    if ca == c:
        return torch.empty((n, c, h, w), dtype=torch.bfloat16, device=device, memory_format=torch.channels_last)
    buf = zeros((n, h, w, ca), torch.bfloat16, device).permute(0, 3, 1, 2)  # NHWC storage; inside a train step: the step arena (no fill launch)
    return buf[:, :c].detach()  # a plain alias of the storage (not an autograd view: outputs of custom Functions are written in place)


def conv_desc(x: torch.Tensor, K: int, R: int, S: int, stride: int, pad: int, y: Optional[torch.Tensor] = None, P=None, Q=None) -> L.ConvDesc:
    n, c, h, w = x.shape
    P = (h + 2 * pad - R) // stride + 1 if P is None else P
    Q = (w + 2 * pad - S) // stride + 1 if Q is None else Q
    d = L.ConvDesc()
    d.N, d.H, d.W, d.C = n, h, w, c
    d.K, d.R, d.S, d.P, d.Q = K, R, S, P, Q
    d.stride, d.pad = stride, pad
    d.x_pitch, d.x_off = nhwc_pitch(x), 0
    d.y_pitch, d.y_off = (nhwc_pitch(y), 0) if y is not None else (((K + 7) // 8) * 8, 0)
    d.up2 = 0
    return d


def new_stats(C: int, device, nacc=2, count=None) -> torch.Tensor:
    """[STATS_REPL, nacc, C] fp64 accumulators of a GEMM epilogue.  count (cross-rank statistics, bn_act_fwd(sync=...)): the local
    element count is stored right after the sums, so that ONE all-reduce of the buffer yields the global sums and count."""
    if count is None:
        return zeros((STATS_REPL, nacc, C), torch.float64, device)
    return new_sync_sums(STATS_REPL * nacc * C, count, device)[:-1].view(STATS_REPL, nacc, C)


def new_sync_sums(n: int, count, device) -> torch.Tensor:
    """fp64 [n + 1]: n zeroed sums followed by the element count (one fill launch; zeros() is a memset inside a step)."""
    buf = zeros((n + 1,), torch.float64, device)
    buf[n:].fill_(float(count))
    return buf


def _with_count(sums: torch.Tensor) -> torch.Tensor:
    """The flat buffer of sums allocated with their element count behind them (new_stats(count=...), new_sync_sums)."""
    return torch.as_strided(sums, (sums.numel() + 1,), (1,), sums.storage_offset())


# ------------------------------------------------------------------------------------------------ conv family
def conv_fprop(x, w_krsc, K, R, S, stride, pad, *, scale=None, shift=None, residual=None, stats=None, act=ACT_NONE, out=None, out_f32=False):
    """y = act(conv(x, w) * scale + shift + residual); optionally accumulates per-channel sum / sum-of-squares."""
    require_cuda(x, "x")
    n, c, h, w = x.shape
    P = (h + 2 * pad - R) // stride + 1
    Q = (w + 2 * pad - S) // stride + 1
    if out is None:
        if out_f32:
            out = torch.empty((n, K, P, Q), dtype=torch.float32, device=x.device, memory_format=torch.channels_last)
        else:
            out = empty_nhwc(n, K, P, Q, x.device)
    d = conv_desc(x, K, R, S, stride, pad, out, P, Q)
    ep = L.Epilogue()
    ep.scale = scale.data_ptr() if scale is not None else None
    ep.shift = shift.data_ptr() if shift is not None else None
    ep.residual = residual.data_ptr() if residual is not None else None
    ep.stats = stats.data_ptr() if stats is not None else None
    ep.stats_repl = stats.shape[0] if stats is not None else 1
    ep.act = act_code(act)
    ep.out_f32 = 1 if out_f32 else 0
    if residual is not None and nhwc_pitch(residual) != d.y_pitch:
        raise L.SgbError("residual must share the output's channel pitch")
    _timed("sgb_conv_fprop", ctypes.byref(d), _ptr(x), _ptr(w_krsc), _ptr(out), ctypes.byref(ep), _stream())
    return out


def conv_dgrad(dy, w_crsk, x_shape, R, S, stride, pad, out=None, accumulate=False):
    n, c, h, w = x_shape
    K = dy.shape[1]
    if out is None:
        out = empty_nhwc(n, c, h, w, dy.device)
    d = L.ConvDesc()
    d.N, d.H, d.W, d.C = n, h, w, c
    d.K, d.R, d.S, d.P, d.Q = K, R, S, dy.shape[2], dy.shape[3]
    d.stride, d.pad = stride, pad
    d.x_pitch, d.x_off = nhwc_pitch(out), 0
    d.y_pitch, d.y_off = nhwc_pitch(dy), 0
    _timed("sgb_conv_dgrad", ctypes.byref(d), _ptr(dy), _ptr(w_crsk), _ptr(out), 1 if accumulate else 0, _stream())
    return out


def conv_wgrad(x, dy, R, S, stride, pad, dw_krsc=None):
    """Returns fp32 [K, R, S, C] (C = x.shape[1], i.e. including any channel padding of x)."""
    n, c, h, w = x.shape
    K = dy.shape[1]
    if dw_krsc is None:
        dw_krsc = zeros((K, R, S, c), torch.float32, x.device)
    d = conv_desc(x, K, R, S, stride, pad, dy, dy.shape[2], dy.shape[3])
    _timed("sgb_conv_wgrad", ctypes.byref(d), _ptr(x), _ptr(dy), _ptr(dw_krsc), _stream())
    return dw_krsc


def weight_prepare(w_oihw: torch.Tensor, c_pad=None, want_crsk=True, scale=None, add_identity=False, out=None):
    """fp32 OIHW -> (bf16 KRSC [K,R,S,c_pad], bf16 CRSK [C,R,S,Kp] or None); `out` reuses a previous result's storage."""
    require_cuda(w_oihw, "weight")
    K, C, R, S = w_oihw.shape
    c_pad = c_pad or ((C + 7) // 8) * 8
    w = w_oihw.detach().contiguous().float()
    if out is not None and out[0] is not None and tuple(out[0].shape) == (K, R, S, c_pad):
        krsc, crsk = out
    else:
        krsc = torch.empty((K, R, S, c_pad), dtype=torch.bfloat16, device=w.device)
        crsk = None
        if want_crsk and c_pad == C:
            crsk = torch.empty((C, R, S, ((K + 7) // 8) * 8), dtype=torch.bfloat16, device=w.device)
    _timed("sgb_weight_prepare", _ptr(w), K, C, R, S, c_pad, _ptr(krsc), _ptr(crsk), _ptr(scale), 1 if add_identity else 0, _stream())
    return krsc, crsk


def wgrad_to_oihw(dw_krsc: torch.Tensor, C: int, out: Optional[torch.Tensor] = None, accumulate=False) -> torch.Tensor:
    K, R, S, cp = dw_krsc.shape
    g = out if out is not None else torch.empty((K, C, R, S), dtype=torch.float32, device=dw_krsc.device)
    _timed("sgb_wgrad_to_oihw", _ptr(dw_krsc), K, C, R, S, cp, _ptr(g), 1 if accumulate else 0, _stream())
    return g


def _item_table(items) -> torch.Tensor:
    """ctypes item structs -> device byte tensor (the batched kernels read their work list from device memory)."""
    arr = (type(items[0]) * len(items))(*items)
    host = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8)
    return host


def weight_prepare_batch(entries, device) -> torch.Tensor:
    """entries: (w fp32 OIHW, scale or None, krsc, crsk or None, c_pad, add_identity).  Returns the device item table
    to pass to run_weight_prepare_batch (build once, replay every step)."""
    items, start = [], 0
    for w, scale, krsc, crsk, c_pad, add_identity, *extra in entries:
        Kk, C, R, S = w.shape
        it = L.WeightItem()
        it.w, it.scale, it.krsc, it.crsk = w.data_ptr(), (scale.data_ptr() if scale is not None else None), krsc.data_ptr(), (crsk.data_ptr() if crsk is not None else None)
        it.K, it.C, it.R, it.S, it.c_pad, it.add_identity, it.start = Kk, C, R, S, c_pad, 1 if add_identity else 0, start
        # optional 7th element: placement inside a wider destination filter (SgbWeightItem: kp, koff, etaps, etap)
        it.kp, it.koff, it.etaps, it.etap = extra[0] if extra else (0, 0, 0, 0)
        start += Kk * R * S * c_pad + (C * R * S * (((Kk + 7) // 8) * 8) if crsk is not None else 0)  # the kernel walks the SOURCE-shaped index space
        items.append(it)
    return _item_table(items).to(device), len(items), start


def run_weight_prepare_batch(table, n, total):
    _timed("sgb_weight_prepare_batch", _ptr(table), n, total, _stream())


def wgrad_to_oihw_batch_table(entries, device):
    """entries: (dw fp32 KRSC, C, slot fp32 OIHW, accumulate)."""
    items, start = [], 0
    for dw, C, g, accumulate in entries:
        Kk, R, S, cp = dw.shape
        if R == 1 and S == 1:
            cp = dw.stride(0)  # a [K, 1, 1, c] view of one tap of a wider gradient buffer (the folded QARepVGG filter): rows are further apart
        elif not dw.is_contiguous():
            raise L.SgbError("wgrad_to_oihw_batch: a multi-tap gradient must be contiguous KRSC")
        it = L.WgradItem()
        it.dw, it.g = dw.data_ptr(), g.data_ptr()
        it.K, it.C, it.R, it.S, it.c_pad, it.accumulate, it.start = Kk, C, R, S, cp, 1 if accumulate else 0, start
        start += Kk * C * R * S
        items.append(it)
    return _item_table(items).to(device), len(items), start


def run_wgrad_to_oihw_batch(table, n, total):
    _timed("sgb_wgrad_to_oihw_batch", _ptr(table), n, total, _stream())


def qarep_alpha_finish_table(entries, device):
    """entries: (dw1 fp32 KRSC [K,1,1,c_pad], C, w1, alpha, dab or None, bias1 or None, g_w1, g_bias or None, g_alpha)."""
    items = []
    for dw1, C, w1, alpha, dab, bias1, g_w1, g_bias, g_alpha in entries:
        it = L.AlphaItem()
        p = lambda t: None if t is None else t.data_ptr()  # noqa: E731
        it.dw1, it.w1, it.alpha, it.dab, it.bias1, it.g_w1, it.g_bias, it.g_alpha = p(dw1), p(w1), p(alpha), p(dab), p(bias1), p(g_w1), p(g_bias), p(g_alpha)
        it.K, it.C, it.c_pad, it.pad_ = dw1.shape[0], C, dw1.stride(0), 0  # stride(0): the row pitch (a one-tap view of a wider buffer has a larger one)
        items.append(it)
    return _item_table(items).to(device), len(items)


def run_qarep_alpha_finish(table, n):
    _timed("sgb_qarep_alpha_finish_batch", _ptr(table), n, _stream())


def convt2x2_fprop(x_small, w_up, bias, C_up):
    """ConvTranspose2d(k=2, s=2): x_small [N,K,P,Q] -> [N,C_up,2P,2Q]; w_up bf16 [(dh,dw,c_up)][K]."""
    n, K, P, Q = x_small.shape
    out = empty_nhwc(n, C_up, 2 * P, 2 * Q, x_small.device)
    d = L.ConvDesc()
    d.N, d.H, d.W, d.C = n, 2 * P, 2 * Q, C_up
    d.K, d.R, d.S, d.P, d.Q = K, 2, 2, P, Q
    d.stride, d.pad = 2, 0
    d.x_pitch, d.x_off = nhwc_pitch(out), 0
    d.y_pitch, d.y_off = nhwc_pitch(x_small), 0
    _timed("sgb_convt2x2_fprop", ctypes.byref(d), _ptr(x_small), _ptr(w_up), _ptr(bias), _ptr(out), _stream())
    return out


# ------------------------------------------------------------------------------------------------ layout
def nchw_f32_to_nhwc_bf16(x: torch.Tensor, c_align: int = 8) -> torch.Tensor:
    """c_align: channel count of the result is C rounded up to a multiple of it (16 lets a 3-channel image use the
    wgmma path, whose K-chunk is 16 channels)."""
    require_cuda(x, "x")
    n, c, h, w = x.shape
    x = x.contiguous().float()
    out = torch.empty((n, ((c + c_align - 1) // c_align) * c_align, h, w), dtype=torch.bfloat16, device=x.device, memory_format=torch.channels_last)
    _timed("sgb_nchw_f32_to_nhwc_bf16", _ptr(x), n, c, h, w, _ptr(out), out.shape[1], 0, out.shape[1], _stream())
    return out


def stem_patches(x: torch.Tensor, R: int, stride: int, pad: int, c_out: int) -> torch.Tensor:
    """fp32 NCHW image -> bf16 NHWC [N, c_out, P, Q] patch tensor (channel (r * R + s) * C + c; see include/sgb200.h)."""
    require_cuda(x, "x")
    n, c, h, w = x.shape
    x = x.contiguous().float()
    P, Q = (h + 2 * pad - R) // stride + 1, (w + 2 * pad - R) // stride + 1
    out = torch.empty((n, c_out, P, Q), dtype=torch.bfloat16, device=x.device, memory_format=torch.channels_last)
    _timed("sgb_stem_patches_f32", _ptr(x), n, c, h, w, R, stride, pad, _ptr(out), P, Q, c_out, _stream())
    return out


def nhwc_bf16_to_nchw_f32(x: torch.Tensor) -> torch.Tensor:
    n, c, h, w = x.shape
    out = torch.empty((n, c, h, w), dtype=torch.float32, device=x.device)
    L.call("sgb_nhwc_bf16_to_nchw_f32", _ptr(x), n, c, h, w, nhwc_pitch(x), 0, _ptr(out), _stream())
    return out


def preprocess_u8(src, out_slot, dst_hw, pad_tl, pad_value=114.0, max_value=255.0, reverse_channels=False, mean=None, std=None):
    """Fused predict() pre-processing of ONE image.  src: uint8 [H, W, C] (C <= 4) on the device; out_slot: bf16 NHWC view
    [1 or -, c_pad, out_h, out_w] of the batch tensor (one image), channels >= C are zeroed.  dst_hw: size after the rescale
    step; pad_tl: (top, left) position of the resized image on the canvas."""
    require_cuda(src, "image")
    if src.dtype != torch.uint8 or src.dim() != 3 or not src.is_contiguous():
        raise L.SgbError("image must be a contiguous uint8 [H, W, C] tensor")
    slot = out_slot if out_slot.dim() == 4 else out_slot.unsqueeze(0)
    d = L.PreprocDesc()
    d.src_h, d.src_w, d.src_c = src.shape
    d.src_pitch = src.shape[1] * src.shape[2]
    d.dst_h, d.dst_w = int(dst_hw[0]), int(dst_hw[1])
    d.out_h, d.out_w = slot.shape[2], slot.shape[3]
    d.pad_top, d.pad_left = int(pad_tl[0]), int(pad_tl[1])
    d.out_pitch = nhwc_pitch(slot)
    d.reverse_channels = 1 if reverse_channels else 0
    d.pad_value = float(pad_value)
    d.max_value = float(max_value) if max_value else 0.0
    d.normalize = 1 if mean is not None else 0
    for i in range(4):
        d.mean[i] = float(mean[i]) if mean is not None and i < len(mean) else 0.0
        d.std[i] = float(std[i]) if std is not None and i < len(std) else 1.0
    if slot.shape[0] != 1 or slot.shape[1] != d.out_pitch:
        raise L.SgbError("out_slot must be one image of a dense NHWC batch (all its channels)")
    _timed("sgb_preprocess_u8", ctypes.byref(d), _ptr(src), _ptr(slot), _stream())
    return out_slot


RS_FIELDS = 8  # SGB_RS_FIELDS: (offset, h, w, pitch, resized_h, resized_w, crop_top, crop_left) per image


def resample_crop_u8(table_host, table, src, out, max_value=255.0, reverse_channels=False, mean=None, std=None):
    """Resize + center-crop pre-processing of a whole batch in one launch.  table_host: int64 [B, 8] CPU tensor (offset into `src`,
    h, w, row pitch, resized h, w, crop top, left), table: the same on the device; src: device uint8 buffer holding the HWC RGB images;
    out: bf16 NHWC [B, c_pad, out_h, out_w] (channels >= 3 are zeroed)."""
    require_cuda(src, "src")
    if table_host.dtype != torch.int64 or table_host.dim() != 2 or table_host.shape[1] != RS_FIELDS or not table_host.is_contiguous() or table_host.is_cuda:
        raise L.SgbError(f"table_host must be a contiguous int64 [B, {RS_FIELDS}] host tensor")
    if table.dtype != torch.int64 or tuple(table.shape) != tuple(table_host.shape) or not table.is_contiguous() or src.dtype != torch.uint8:
        raise L.SgbError("table must be the device copy of table_host and src a uint8 buffer")
    B, pitch = table_host.shape[0], nhwc_pitch(out)
    if out.dtype != torch.bfloat16 or out.shape[0] != B or out.shape[1] != pitch:
        raise L.SgbError("out must be a dense bf16 NHWC batch [B, c_pad, out_h, out_w]")
    m = s = None
    if mean is not None:
        m, s = (ctypes.c_float * 4)(*[float(v) for v in mean][:4]), (ctypes.c_float * 4)(*[float(v) for v in std][:4])
    _timed("sgb_resample_crop_u8", ctypes.c_void_p(table_host.data_ptr()), _ptr(table), _ptr(src), src.numel(), B, 3, out.shape[2], out.shape[3], pitch,
           1 if reverse_channels else 0, float(max_value) if max_value else 0.0, m, s, _ptr(out), _stream())  # fmt: skip
    return out


def classify_rows(logits, target=None, k=1, counters=None, label=None, confidence=None):
    """Row-wise classification decode of fp32 / bf16 logits [N, C] (unit column stride).  target: int64 [N] class indices or a
    float [N, C] soft-label tensor (argmax per row); counters: int64 [4] device accumulators (top-1 correct, top-k correct, rows,
    invalid targets); label int32 [N] / confidence f32 [N]: the top-1 index and the softmax maximum."""
    require_cuda(logits, "logits")
    if logits.dim() != 2 or logits.dtype not in (torch.float32, torch.bfloat16) or (logits.shape[1] > 1 and logits.stride(1) != 1):
        raise L.SgbError(f"logits must be a float32 / bfloat16 [N, C] tensor with unit column stride, got {tuple(logits.shape)} {logits.dtype}")
    N, C = logits.shape
    dev = logits.device
    hard = soft = None
    if target is not None:
        if target.device != dev:
            raise L.SgbError(f"target must live on {dev}")
        if target.dim() == 1 and target.dtype == torch.int64 and target.shape[0] == N:
            hard = target.contiguous()
        elif target.dim() == 2 and tuple(target.shape) == (N, C) and target.dtype in (torch.float32, torch.bfloat16) and (C == 1 or target.stride(1) == 1):
            soft = target
        else:
            raise L.SgbError(f"target must be int64 [N] or float32 / bfloat16 [N, C], got {tuple(target.shape)} {target.dtype} for logits {tuple(logits.shape)}")
    for name, t, dt in (("counters", counters, torch.int64), ("label", label, torch.int32), ("confidence", confidence, torch.float32)):
        if t is not None and (t.dtype != dt or not t.is_contiguous() or t.device != dev or t.numel() != (4 if name == "counters" else N)):
            raise L.SgbError(f"{name} must be a contiguous {dt} tensor of {4 if name == 'counters' else N} elements on {dev}")
    _timed("sgb_classify_rows", _ptr(logits), N, C, logits.stride(0) if N > 1 else C, 1 if logits.dtype == torch.bfloat16 else 0, _ptr(hard), _ptr(soft),
           (soft.stride(0) if N > 1 else C) if soft is not None else 0, 1 if soft is not None and soft.dtype == torch.bfloat16 else 0, int(k), _ptr(counters),
           _ptr(label), _ptr(confidence), _stream())  # fmt: skip


# ------------------------------------------------------------------------------------------------ validation metrics
def match_desc(preds, targets, crowd, n_thresholds, height, width, top_k, denormalize_targets) -> L.MatchDesc:
    d = L.MatchDesc()
    d.B, d.max_preds = preds.shape[0], preds.shape[1]
    d.max_targets = targets.shape[1]
    d.max_crowd = 0 if crowd is None else crowd.shape[1]
    d.n_thresholds, d.top_k = int(n_thresholds), int(top_k)
    d.denormalize_targets = 1 if denormalize_targets else 0
    d.height, d.width = float(height), float(width)
    return d


def detection_matching(preds, pred_count, targets, target_count, crowd, crowd_count, thresholds, height, width, top_k=100, denormalize_targets=True):
    """DetectionMetrics matching of one batch.  preds [B, P, 6] f32 + pred_count [B] int32 (batched_nms' outputs), targets
    [B, M, 5] f32 rows (class, cx, cy, w, h) + target_count [B], crowd likewise or None, thresholds [T] f32 ascending.
    Returns (matched, ignore) uint8 [B, P, T]."""
    require_cuda(preds, "preds")
    for name, t, dt in (("preds", preds, torch.float32), ("targets", targets, torch.float32), ("thresholds", thresholds, torch.float32), ("pred_count", pred_count, torch.int32), ("target_count", target_count, torch.int32)):
        if t.dtype != dt or not t.is_contiguous() or t.device != preds.device:
            raise L.SgbError(f"{name} must be a contiguous {dt} tensor on {preds.device}")
    if preds.dim() != 3 or preds.shape[2] != 6 or targets.dim() != 3 or targets.shape[2] != 5 or targets.shape[0] != preds.shape[0]:
        raise L.SgbError("preds must be [B, P, 6] and targets [B, M, 5]")
    if crowd is not None and (crowd.dtype != torch.float32 or not crowd.is_contiguous() or crowd.dim() != 3 or crowd.shape[2] != 5 or crowd.shape[0] != preds.shape[0] or crowd_count.dtype != torch.int32):
        raise L.SgbError("crowd targets must be a contiguous float32 [B, C, 5] tensor with int32 counts")
    if crowd is not None and crowd.shape[1] == 0:
        crowd = crowd_count = None
    d = match_desc(preds, targets, crowd, thresholds.numel(), height, width, top_k, denormalize_targets)
    matched = torch.empty((d.B, d.max_preds, d.n_thresholds), dtype=torch.uint8, device=preds.device)
    ignore = torch.empty_like(matched)
    _timed("sgb_detection_matching", ctypes.byref(d), _ptr(preds), _ptr(pred_count), _ptr(targets), _ptr(target_count), _ptr(crowd) if crowd is not None else None,
           _ptr(crowd_count) if crowd is not None else None, _ptr(thresholds), _ptr(matched), _ptr(ignore), _stream())  # fmt: skip
    return matched, ignore


def pose_keypoint_matching(poses, scores, pred_count, gt_joints, gt_boxes, gt_areas, gt_flags, gt_count, sigmas, thresholds, top_k, oks_out=False):
    """PoseEstimationMetrics matching of one batch.  poses [B, P, J, 3] f32 (x, y, joint score), scores [B, P] f32, pred_count [B]
    int32; gt_joints [B, M, J, 3] f32 (x, y, visibility), gt_boxes [B, M, 4] f32 XYWH, gt_areas [B, M] f32, gt_flags [B, M] uint8
    (1: crowd, 2: box given, 4: area given), gt_count [B] int32; sigmas [J] f32; thresholds [T] f32.  Returns (matched, ignore
    [B, K, T] uint8, used_scores [B, K] f32, used_count [B] int32, n_targets [B] int32) with K = min(top_k, P), rows in score order,
    plus the OKS matrix [B, K, M] f32 of the used predictions against every target when `oks_out`."""
    require_cuda(poses, "poses")
    for name, t, dt in (("poses", poses, torch.float32), ("scores", scores, torch.float32), ("pred_count", pred_count, torch.int32), ("gt_joints", gt_joints, torch.float32),
                        ("gt_boxes", gt_boxes, torch.float32), ("gt_areas", gt_areas, torch.float32), ("gt_flags", gt_flags, torch.uint8), ("gt_count", gt_count, torch.int32),
                        ("sigmas", sigmas, torch.float32), ("thresholds", thresholds, torch.float32)):  # fmt: skip
        if t.dtype != dt or not t.is_contiguous() or t.device != poses.device:
            raise L.SgbError(f"{name} must be a contiguous {dt} tensor on {poses.device}")
    if poses.dim() != 4 or poses.shape[3] != 3:
        raise L.SgbError(f"poses must be [B, P, J, 3], got {tuple(poses.shape)}")
    B, P, J, _ = poses.shape
    M = gt_joints.shape[1] if gt_joints.dim() == 4 else -1
    T = thresholds.numel()
    shapes = ((scores, (B, P)), (pred_count, (B,)), (gt_joints, (B, M, J, 3)), (gt_boxes, (B, M, 4)), (gt_areas, (B, M)), (gt_flags, (B, M)), (gt_count, (B,)), (sigmas, (J,)))
    if M < 1 or any(tuple(t.shape) != s for t, s in shapes) or thresholds.dim() != 1:
        raise L.SgbError("pose matching expects scores [B, P], pred_count [B], gt_joints [B, M >= 1, J, 3], gt_boxes [B, M, 4], gt_areas / gt_flags [B, M], gt_count [B], sigmas [J], thresholds [T]")
    if not 1 <= T <= 32 or int(top_k) < 1:
        raise L.SgbError(f"pose matching needs 1..32 thresholds (got {T}) and top_k >= 1 (got {top_k})")
    K = min(int(top_k), P)
    dev = poses.device
    matched = torch.empty((B, K, T), dtype=torch.uint8, device=dev)
    ignore = torch.empty_like(matched)
    used_scores = torch.empty((B, K), dtype=torch.float32, device=dev)
    used_count = torch.empty(B, dtype=torch.int32, device=dev)
    n_targets = torch.empty(B, dtype=torch.int32, device=dev)
    oks = torch.empty((B, K, M), dtype=torch.float32, device=dev) if oks_out else None
    if oks is not None:
        oks.fill_(float("nan"))  # entries of prediction rows past the used count stay NaN
    _timed("sgb_pose_keypoint_matching", _ptr(poses), _ptr(scores), _ptr(pred_count), _ptr(gt_joints), _ptr(gt_boxes), _ptr(gt_areas), _ptr(gt_flags), _ptr(gt_count), _ptr(sigmas),
           _ptr(thresholds), B, P, M, J, T, int(top_k), _ptr(matched), _ptr(ignore), _ptr(used_scores), _ptr(used_count), _ptr(n_targets), _ptr(oks), _stream())  # fmt: skip
    out = (matched, ignore, used_scores, used_count, n_targets)
    return out + (oks,) if oks_out else out


# ------------------------------------------------------------------------------------------------ batch norm
def bn_desc(x, y, eps, momentum, act, residual=None, stats_repl=STATS_REPL, sample_scale=None) -> L.BnDesc:
    n, c, h, w = x.shape
    d = L.BnDesc()
    if sample_scale is not None:  # drop-path: fp32 [N], 0 or 1 / keep_prob per image
        if sample_scale.dtype != torch.float32 or sample_scale.numel() != n or not sample_scale.is_contiguous():
            raise L.SgbError("sample_scale must be a contiguous fp32 tensor with one entry per image")
        require_cuda(sample_scale, "sample_scale")
        d.hw, d.sample_scale = h * w, sample_scale.data_ptr()
    d.M, d.C = n * h * w, c
    d.x_pitch, d.x_off = nhwc_pitch(x), 0
    d.y_pitch, d.y_off = nhwc_pitch(y), 0
    d.r_pitch, d.r_off = (nhwc_pitch(residual), 0) if residual is not None else (0, 0)
    d.eps, d.momentum = eps, momentum
    d.act = act_code(act)
    d.stats_repl = stats_repl
    return d


# Convolutions whose epilogue keeps per-channel statistics in registers exist for 32 / 48 / 64 / 96 output channels (halo-tile, 1x1-tile
# and im2col fast paths); wider layers ran the im2col kernel's general epilogue (a 32-lane butterfly per 16 columns: 1.2-1.5 TB/s on
# 1x1 layers that move the same bytes as 4.4 TB/s ones).  Those layers now run WITHOUT epilogue statistics and their BatchNorm forward
# is one cooperative launch (sums, grid barrier, apply).  Every such layer of YOLO-NAS at batch 32 is below 40 MB, so the apply pass's
# re-read hits L2; ResNet-50's (up to 411 MB at batch 256) re-read from HBM and still win: 7819 -> 8509 img/s with the size bound
# (SGB_STATS_IN_BN_MAX_BYTES, default: none) lifted.  SGB_STATS_IN_BN=0 restores the epilogue statistics everywhere.
STATS_IN_BN = [os.environ.get("SGB_STATS_IN_BN", "1") != "0"]
STATS_IN_BN_MAX_BYTES = [int(os.environ.get("SGB_STATS_IN_BN_MAX_BYTES", str(1 << 62)))]
_EPILOGUE_STATS_CHANNELS = (32, 48, 64, 96)


def stats_in_bn(kout: int, pixels: int) -> bool:
    """True: the layer's convolution runs without epilogue statistics and bn_act_fwd(stats=None) computes them itself."""
    return STATS_IN_BN[0] and kout not in _EPILOGUE_STATS_CHANNELS and kout % 8 == 0 and 2 * kout * pixels <= STATS_IN_BN_MAX_BYTES[0]


def bn_act_fwd(x, stats, gamma, beta, running_mean, running_var, eps, momentum, act, residual=None, sample_scale=None, sync=None):
    """stats: [repl, 2, C] fp64 sums from the producing GEMM's epilogue, or None: the launch computes them itself (cooperative:
    sums, grid-wide barrier, apply).

    sync (functional.BnSync): cross-rank statistics in two passes -- the sums (epilogue sums from new_stats(count=...), or
    sgb_channel_stats) and the local count are all-reduced by ONE sync(buffer) call, then sgb_bn_act_fwd divides by the global
    count.  The reduced count is left in sync.count for the backward pass."""
    n, c, h, w = x.shape
    y = empty_nhwc(n, c, h, w, x.device)
    mean = torch.empty(c, dtype=torch.float32, device=x.device)
    rstd = torch.empty(c, dtype=torch.float32, device=x.device)
    if sync is not None:
        if stats is None:
            buf = new_sync_sums(2 * c, n * h * w, x.device)
            stats = buf[:-1].view(1, 2, c)
            _timed("sgb_channel_stats", _ptr(x), n * h * w, c, nhwc_pitch(x), 0, _ptr(stats), _stream())
        else:
            buf = _with_count(stats)
        sync(buf)
        sync.count = buf[-1:]
        d = bn_desc(x, y, eps, momentum, act, residual, stats.shape[0], sample_scale=sample_scale)
        d.count = sync.count.data_ptr()
        d.param_scale = sync.param_scale
        _timed("sgb_bn_act_fwd", ctypes.byref(d), _ptr(x), _ptr(stats), _ptr(gamma), _ptr(beta), _ptr(running_mean), _ptr(running_var), _ptr(residual), _ptr(y), _ptr(mean), _ptr(rstd), _stream())
        return y, mean, rstd
    if stats is None:
        stats = zeros((1, 2, c), torch.float64, x.device)
        d = bn_desc(x, y, eps, momentum, act, residual, 1, sample_scale=sample_scale)
        _timed("sgb_bn_act_fwd_fused", ctypes.byref(d), _ptr(x), _ptr(stats), _ptr(gamma), _ptr(beta), _ptr(running_mean), _ptr(running_var), _ptr(residual), _ptr(y), _ptr(mean), _ptr(rstd), _stream())
        return y, mean, rstd
    d = bn_desc(x, y, eps, momentum, act, residual, stats.shape[0], sample_scale=sample_scale)
    _timed("sgb_bn_act_fwd", ctypes.byref(d), _ptr(x), _ptr(stats), _ptr(gamma), _ptr(beta), _ptr(running_mean), _ptr(running_var), _ptr(residual), _ptr(y), _ptr(mean), _ptr(rstd), _stream())
    return y, mean, rstd


def bn_act_infer(x, gamma, beta, running_mean, running_var, eps, act, residual=None):
    n, c, h, w = x.shape
    y = empty_nhwc(n, c, h, w, x.device)
    d = bn_desc(x, y, eps, 0.0, act, residual, 1)
    L.call("sgb_bn_act_infer", ctypes.byref(d), _ptr(x), _ptr(gamma), _ptr(beta), _ptr(running_mean), _ptr(running_var), _ptr(residual), _ptr(y), _stream())
    return y


def bn_act_bwd(dy, x, y, gamma, mean, rstd, eps, act, want_residual_grad=False, dgamma=None, dbeta=None, beta=None, sample_scale=None, dy2=None, sync=None):
    """Returns (dx, dresidual or None, dgamma, dbeta); dgamma / dbeta are accumulated into when given.
    dy2: the gradient arrives as TWO tensors, dy for channels [0, dy.shape[1]) and dy2 for the rest (two layers that shared one GEMM,
    functional._DualConvBnAct); both are read in place (SgbBnDesc.dy2).  y may be None when the mask is recomputed from x.
    sync: the forward's functional.BnSync -- the reduction pass's sums are all-reduced by sync(sums) before the apply pass, which
    divides by sync.count and scales the parameter gradients by sync.param_scale."""
    n, c, h, w = x.shape
    dy = as_nhwc(dy)
    if act_code(act) not in (ACT_NONE, ACT_RELU):
        # the backward passes apply the ReLU mask only; SiLU exists as a forward / inference epilogue (PP-YOLOE-style heads)
        raise L.SgbError("bn_act_bwd: only identity / ReLU activations have a backward pass in super_gradients_b200")
    d = bn_desc(x, y if y is not None else x, eps, 0.0, act, None, 1, sample_scale=sample_scale)
    if dy2 is not None:
        dy2 = as_nhwc(dy2)
        if dy.shape[1] + dy2.shape[1] != c or dy.shape[1] % 8 != 0:
            raise L.SgbError("bn_act_bwd: dy and dy2 must split the layer's channels at a multiple of 8")
        if nhwc_pitch(dy) % 8 != 0 or dy.data_ptr() % 16 != 0:
            dy = dy.contiguous(memory_format=torch.channels_last)
        if nhwc_pitch(dy2) % 8 != 0 or dy2.data_ptr() % 16 != 0:
            dy2 = dy2.contiguous(memory_format=torch.channels_last)
        d.dy_pitch, d.dy_off = nhwc_pitch(dy), 0
        d.dy2_split, d.dy2_pitch, d.dy2_off, d.dy2 = dy.shape[1], nhwc_pitch(dy2), 0, dy2.data_ptr()
    elif nhwc_pitch(dy) != d.y_pitch:
        # dy is a channel slice of a wider gradient buffer (the layer's output went into a concat): the kernels read it in place
        if nhwc_pitch(dy) % 8 == 0 and dy.data_ptr() % 16 == 0:
            d.dy_pitch, d.dy_off = nhwc_pitch(dy), 0
        else:
            dy = dy.contiguous(memory_format=torch.channels_last)
            if nhwc_pitch(dy) != d.y_pitch:
                raise L.SgbError("dy pitch mismatch")
    sums = zeros((2, c), torch.float64, x.device)
    # the forward output is only read when a residual entered the activation; otherwise the mask is recomputed from x
    y_arg = y if (want_residual_grad or beta is None or sample_scale is not None) else None
    fused = FUSED_BWD[0] and nhwc_pitch(x) == c and sync is None
    if not fused:
        _timed("sgb_bn_act_bwd_reduce", ctypes.byref(d), _ptr(dy), _ptr(x), _ptr(y_arg), _ptr(gamma), _ptr(beta), _ptr(mean), _ptr(rstd), _ptr(sums), _stream())
    if sync is not None:
        sync(sums)
        d.count, d.param_scale = sync.count.data_ptr(), sync.param_scale
    dx = torch.empty_like(x, memory_format=torch.channels_last) if nhwc_pitch(x) == c else torch.zeros_like(x)
    d.x_pitch = nhwc_pitch(dx)
    # x and dx must share a pitch for the kernel: re-describe x if it is a slice
    if nhwc_pitch(x) != d.x_pitch:
        x = x.contiguous(memory_format=torch.channels_last)
    dres = None
    if want_residual_grad:
        dres = empty_nhwc(n, c, h, w, x.device)
        d.r_pitch = nhwc_pitch(dres)
    if dgamma is None:
        dgamma = zeros((c,), torch.float32, x.device)
    if dbeta is None:
        dbeta = zeros((c,), torch.float32, x.device)
    # one cooperative launch (reduction, grid barrier, apply) when every operand is dense; else the two passes
    _timed("sgb_bn_act_bwd_fused" if fused else "sgb_bn_act_bwd_apply", ctypes.byref(d), _ptr(dy), _ptr(x), _ptr(y_arg), _ptr(gamma), _ptr(beta), _ptr(mean), _ptr(rstd), _ptr(sums), _ptr(dx), _ptr(dres), _ptr(dgamma), _ptr(dbeta), _stream())
    return dx, dres, dgamma, dbeta


def channel_stats(x) -> torch.Tensor:
    n, c, h, w = x.shape
    st = zeros((1, 2, c), torch.float64, x.device)
    _timed("sgb_channel_stats", _ptr(x), n * h * w, c, nhwc_pitch(x), 0, _ptr(st), _stream())
    return st


# ------------------------------------------------------------------------------------------------ QARepVGG algebra
def qarep_desc(y3, u, out, eps3, eps_post, momentum, act, use_post_bn) -> L.QarepDesc:
    n, c, h, w = y3.shape
    d = L.QarepDesc()
    d.M, d.C = n * h * w, c
    d.pitch3, d.off3 = nhwc_pitch(y3), 0
    d.pitchu, d.offu = nhwc_pitch(u), 0
    d.pitcho, d.offo = nhwc_pitch(out), 0
    d.eps3, d.eps_post, d.momentum = eps3, eps_post, momentum
    d.act = act_code(act)
    d.use_post_bn = 1 if use_post_bn else 0
    return d


def qarep_fwd(y3, u, gamma3, beta3, bias1a, gamma_p, beta_p, rm3, rv3, rmp, rvp, eps3, eps_post, momentum, act, use_post_bn=True, residual=None, res_alpha=None, sync=None):
    """residual / res_alpha: out = act(...) + res_alpha * residual (device scalar): a bottleneck's learnable shortcut in the same pass.
    sync (functional.BnSync): the five moments and the local count are all-reduced by ONE sync(buffer) call between
    sgb_qarep_moments and sgb_qarep_fwd, which gives both BatchNorms of the block their global statistics; the reduced count is left
    in sync.count for the backward pass."""
    n, c, h, w = y3.shape
    out = empty_nhwc(n, c, h, w, y3.device)
    d = qarep_desc(y3, u, out, eps3, eps_post, momentum, act, use_post_bn)
    if residual is not None:
        residual = as_nhwc(residual)
        if tuple(residual.shape) != tuple(y3.shape) or res_alpha is None or res_alpha.dtype != torch.float32 or res_alpha.numel() != 1:
            raise L.SgbError("qarep_fwd: the shortcut must have the output's shape and a one-element fp32 device scale")
        require_cuda(res_alpha, "res_alpha")
        d.pitchr, d.offr, d.res, d.res_alpha = nhwc_pitch(residual), 0, residual.data_ptr(), res_alpha.data_ptr()
    if sync is not None:
        coef = torch.empty((9, c), dtype=torch.float32, device=y3.device)
        buf = new_sync_sums(5 * c, n * h * w, y3.device)
        mom = buf[:-1].view(5, c)
        _timed("sgb_qarep_moments", ctypes.byref(d), _ptr(y3), _ptr(u), _ptr(mom), _stream())
        sync(buf)
        sync.count = buf[-1:]
        d.count, d.param_scale = sync.count.data_ptr(), sync.param_scale
        _timed("sgb_qarep_fwd", ctypes.byref(d), _ptr(y3), _ptr(u), _ptr(mom), _ptr(gamma3), _ptr(beta3), _ptr(bias1a), _ptr(gamma_p), _ptr(beta_p), _ptr(rm3), _ptr(rv3), _ptr(rmp), _ptr(rvp), _ptr(out), _ptr(coef), _stream())
        return out, coef
    mom = zeros((5, c), torch.float64, y3.device)
    coef = torch.empty((9, c), dtype=torch.float32, device=y3.device)
    if FUSED_FWD[0]:  # moments, grid barrier, apply in one cooperative launch
        _timed("sgb_qarep_fwd_fused", ctypes.byref(d), _ptr(y3), _ptr(u), _ptr(mom), _ptr(gamma3), _ptr(beta3), _ptr(bias1a), _ptr(gamma_p), _ptr(beta_p), _ptr(rm3), _ptr(rv3), _ptr(rmp), _ptr(rvp), _ptr(out), _ptr(coef), _stream())
        return out, coef
    _timed("sgb_qarep_moments", ctypes.byref(d), _ptr(y3), _ptr(u), _ptr(mom), _stream())
    _timed("sgb_qarep_fwd", ctypes.byref(d), _ptr(y3), _ptr(u), _ptr(mom), _ptr(gamma3), _ptr(beta3), _ptr(bias1a), _ptr(gamma_p), _ptr(beta_p), _ptr(rm3), _ptr(rv3), _ptr(rmp), _ptr(rvp), _ptr(out), _ptr(coef), _stream())
    return out, coef


def qarep_bwd(dout, out, y3, u, coef, gamma3, gamma_p, eps3, eps_post, act, use_post_bn=True, acc=None, out_grads=None, sync=None):
    """Returns dy3, du, dgamma3, dbeta3, dbias1a, dgamma_p, dbeta_p.  `acc` optionally supplies existing fp32 tensors
    (dgamma3, dbeta3, dbias1a, dgamma_p, dbeta_p) to accumulate into (None entries are allocated).  The kernel writes dy3 / du
    with the channel pitch of y3 / u: `out_grads` = (dy3, du) buffers of those pitches (e.g. channel slices of one tensor when
    y3 / u are slices); by default dense tensors are allocated, which requires dense y3 / u.
    sync: the forward's functional.BnSync -- the three sums are all-reduced by sync(sums) between the two passes."""
    n, c, h, w = y3.shape
    dout = as_nhwc(dout)
    if act_code(act) not in (ACT_NONE, ACT_RELU):
        raise L.SgbError("qarep_bwd: only identity / ReLU activations have a backward pass in super_gradients_b200")
    d = qarep_desc(y3, u, out, eps3, eps_post, 0.0, act, use_post_bn)
    if nhwc_pitch(dout) != nhwc_pitch(out):
        if nhwc_pitch(dout) % 8 == 0 and dout.data_ptr() % 16 == 0:  # a concat's gradient slice: read in place
            d.pitchd, d.offd = nhwc_pitch(dout), 0
        else:
            dout = dout.contiguous(memory_format=torch.channels_last)
    sums = zeros((3, c), torch.float64, y3.device)
    fused = FUSED_BWD[0] and sync is None
    if not fused:
        _timed("sgb_qarep_bwd_reduce", ctypes.byref(d), _ptr(dout), _ptr(out), _ptr(y3), _ptr(u), _ptr(coef), _ptr(sums), _stream())
    if sync is not None:
        sync(sums)
        d.count, d.param_scale = sync.count.data_ptr(), sync.param_scale
    if out_grads is not None:
        dy3, du = out_grads
        if nhwc_pitch(dy3) != nhwc_pitch(y3) or nhwc_pitch(du) != nhwc_pitch(u):
            raise L.SgbError("qarep_bwd: dy3 / du must have the channel pitch of y3 / u")
    else:
        dy3, du = torch.empty_like(y3), torch.empty_like(u)
    z = lambda: zeros((c,), torch.float32, y3.device)  # noqa: E731
    acc = acc or (None,) * 5
    dg3, db3, dab, dgp, dbp = [a if a is not None else z() for a in acc]
    if fused:  # one cooperative launch: reduction, grid barrier, apply
        _timed("sgb_qarep_bwd_fused", ctypes.byref(d), _ptr(dout), _ptr(y3), _ptr(u), _ptr(coef), _ptr(sums), _ptr(gamma3), _ptr(gamma_p), _ptr(dy3), _ptr(du), _ptr(dg3), _ptr(db3), _ptr(dab), _ptr(dgp), _ptr(dbp), _stream())
    else:
        _timed("sgb_qarep_bwd_apply", ctypes.byref(d), _ptr(dout), _ptr(out), _ptr(y3), _ptr(u), _ptr(coef), _ptr(sums), _ptr(gamma3), _ptr(gamma_p), _ptr(dy3), _ptr(du), _ptr(dg3), _ptr(db3), _ptr(dab), _ptr(dgp), _ptr(dbp), _stream())
    return dy3, du, dg3, db3, dab, dgp, dbp


# ------------------------------------------------------------------------------------------------ pooling / misc
def maxpool_fwd(x, k, stride, pad, want_idx=True, out=None):
    n, c, h, w = x.shape
    P, Q = (h + 2 * pad - k) // stride + 1, (w + 2 * pad - k) // stride + 1
    if out is None:
        out = empty_nhwc(n, c, P, Q, x.device)
    idx = torch.empty((n, P, Q, c), dtype=torch.uint8, device=x.device) if want_idx else None
    _timed("sgb_maxpool_fwd", _ptr(x), n, h, w, c, nhwc_pitch(x), 0, k, stride, pad, _ptr(out), P, Q, nhwc_pitch(out), 0, _ptr(idx), _stream())
    return out, idx


def maxpool_bwd(dy, idx, x_shape, k, stride, pad):
    n, c, h, w = x_shape
    dy = as_nhwc(dy)
    if stride >= 2 and c % 8 == 0:  # few windows per input pixel: gather, bf16 out (no memset / atomics / conversion pass)
        dxb = empty_nhwc(n, c, h, w, dy.device)
        _timed("sgb_maxpool_bwd_bf16", _ptr(dy), n, h, w, c, k, stride, pad, dy.shape[2], dy.shape[3], nhwc_pitch(dy), 0, _ptr(idx), _ptr(dxb), nhwc_pitch(dxb), _stream())
        return dxb
    dx = torch.zeros((n, h, w, c), dtype=torch.float32, device=dy.device)
    _timed("sgb_maxpool_bwd", _ptr(dy), n, h, w, c, k, stride, pad, dy.shape[2], dy.shape[3], nhwc_pitch(dy), 0, _ptr(idx), _ptr(dx), _stream())
    return dx.permute(0, 3, 1, 2)  # NCHW-shaped view of NHWC fp32 storage


def axpby(x1, a, x2=None, b=0.0, out=None):
    n, c, h, w = x1.shape
    if out is None:
        out = empty_nhwc(n, c, h, w, x1.device)
    _timed("sgb_axpby", _ptr(x1), nhwc_pitch(x1), 0, float(a), _ptr(x2), nhwc_pitch(x2) if x2 is not None else 0, 0, float(b), _ptr(out), nhwc_pitch(out), 0, n * h * w, c, _stream())
    return out


def scale_add(x1, a_dev, x2=None, out=None):
    """(*a_dev) * x1 + x2 with the scalar read on the device (no host sync)."""
    n, c, h, w = x1.shape
    if out is None:
        out = empty_nhwc(n, c, h, w, x1.device)
    _timed("sgb_scale_add", _ptr(x1), nhwc_pitch(x1), 0, _ptr(a_dev), _ptr(x2), nhwc_pitch(x2) if x2 is not None else 0, 0, _ptr(out), nhwc_pitch(out), 0, n * h * w, c, _stream())
    return out


def scale_add_dot(x1, a_dev, xd, x2=None, out=None):
    """((*a_dev) * x1 + x2, fp64 [C] = sum over pixels of x1 * xd) in one pass over x1; `out` may be x2 (in place)."""
    n, c, h, w = x1.shape
    if out is None:
        out = empty_nhwc(n, c, h, w, x1.device)
    dot = zeros((c,), torch.float64, x1.device)
    _timed("sgb_scale_add_dot", _ptr(x1), nhwc_pitch(x1), 0, _ptr(a_dev), _ptr(x2), nhwc_pitch(x2) if x2 is not None else 0, 0, _ptr(xd), nhwc_pitch(xd), 0,
           _ptr(out), nhwc_pitch(out), 0, n * h * w, c, _ptr(dot), _stream())  # fmt: skip
    return out, dot


def channel_dot(a, b) -> torch.Tensor:
    """fp64 [C]: sum over pixels of a*b."""
    n, c, h, w = a.shape
    out = zeros((c,), torch.float64, a.device)
    _timed("sgb_channel_dot", _ptr(a), nhwc_pitch(a), 0, _ptr(b), nhwc_pitch(b), 0, n * h * w, c, _ptr(out), _stream())
    return out


def f32_to_bf16(x: torch.Tensor) -> torch.Tensor:
    y = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
    L.call("sgb_f32_to_bf16", _ptr(x.contiguous()), _ptr(y), x.numel(), _stream())
    return y


def avgpool_fwd(x):
    n, c, h, w = x.shape
    if nhwc_pitch(x) != c:
        x = x.contiguous(memory_format=torch.channels_last)
    y = torch.empty((n, c, 1, 1), dtype=torch.bfloat16, device=x.device, memory_format=torch.channels_last)
    L.call("sgb_avgpool_fwd", _ptr(x), n, h * w, c, _ptr(y), _stream())
    return y


def avgpool_bwd(dy, hw_shape):
    n, c = dy.shape[0], dy.shape[1]
    h, w = hw_shape
    dyc = dy.reshape(n, c).contiguous()
    dx = torch.empty((n, c, h, w), dtype=torch.bfloat16, device=dy.device, memory_format=torch.channels_last)
    L.call("sgb_avgpool_bwd", _ptr(dyc), n, h * w, c, _ptr(dx), _stream())
    return dx


# ------------------------------------------------------------------------------------------------ head / loss / nms
def dfl_decode(reg, cls, L_total, anchor_base, ncls, reg_max, stride, cell_offset, pred_bboxes, pred_scores, cls_logits=None, reg_distri=None):
    n, _, hf, wf = reg.shape
    _timed("sgb_dfl_decode", _ptr(reg), nhwc_pitch(reg), _ptr(cls), nhwc_pitch(cls), n, hf, wf, L_total, anchor_base, ncls, reg_max, float(stride), float(cell_offset), _ptr(pred_bboxes), _ptr(pred_scores), _ptr(cls_logits), _ptr(reg_distri), _stream())


def pose_keypoint_decode(pose, logit, logit_off, L_total, anchor_base, J, stride, cell_offset, offset_multiplier, compensate, pose_coords, pose_scores, pose_logits=None):
    """pose [N, 2J, H, W] / logit [N, >= logit_off + J, H, W] bf16 NHWC maps of one level -> rows of the fp32 [N, L, *] outputs."""
    n, _, hf, wf = pose.shape
    _timed("sgb_pose_keypoint_decode", _ptr(pose), nhwc_pitch(pose), _ptr(logit), nhwc_pitch(logit), int(logit_off), n, hf, wf, L_total, anchor_base, J, float(stride), float(cell_offset),
           float(offset_multiplier), 1 if compensate else 0, _ptr(pose_coords), _ptr(pose_scores), _ptr(pose_logits), _stream())  # fmt: skip


def head_grad_scatter(grad, n, hw, L_total, anchor_base, dy):
    gC = grad.shape[-1]
    _timed("sgb_head_grad_scatter", _ptr(grad), gC, n, hw, L_total, anchor_base, _ptr(dy), nhwc_pitch(dy), _stream())


def loss_desc(B, Lc, ncls, reg_max, n_max, topk=13, alpha=1.0, beta=6.0, w_cls=1.0, w_iou=2.5, w_dfl=0.5, iou_type=0) -> L.LossDesc:
    d = L.LossDesc()
    d.B, d.L, d.ncls, d.reg_max, d.n_max, d.topk = B, Lc, ncls, reg_max, n_max, topk
    d.alpha, d.beta, d.w_cls, d.w_iou, d.w_dfl, d.iou_type = alpha, beta, w_cls, w_iou, w_dfl, iou_type
    return d


def tal_assign(d, cls_logits, reg_distri, anchor_points, stride_tensor, gt_boxes, gt_labels, gt_valid, sums):
    dev = cls_logits.device
    al = torch.empty((d.B, d.L), dtype=torch.int32, device=dev)
    ab = torch.empty((d.B, d.L, 4), dtype=torch.float32, device=dev)
    asc = torch.empty((d.B, d.L), dtype=torch.float32, device=dev)
    nbytes = L.load().sgb_tal_workspace_bytes(ctypes.byref(d))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    _timed("sgb_tal_assign", ctypes.byref(d), _ptr(cls_logits), _ptr(reg_distri), _ptr(anchor_points), _ptr(stride_tensor), _ptr(gt_boxes), _ptr(gt_labels), _ptr(gt_valid), _ptr(al), _ptr(ab), _ptr(asc), _ptr(sums), _ptr(ws), nbytes, _stream())
    return al, ab, asc


def atss_assign(d, reg_distri, anchors, anchor_points, stride_tensor, level_sizes, gt_boxes, gt_labels, gt_valid, sums):
    """ATSS assignment with tal_assign's outputs.  anchors [L, 4] f32 anchor boxes, level_sizes = the head's num_anchors_list
    (host ints); d.topk = candidates per level (9)."""
    dev = reg_distri.device
    require_cuda(reg_distri, "reg_distri")
    if anchors.dtype != torch.float32 or not anchors.is_contiguous() or anchors.shape != (d.L, 4):
        raise L.SgbError("anchors must be a contiguous float32 [L, 4] tensor")
    al = torch.empty((d.B, d.L), dtype=torch.int32, device=dev)
    ab = torch.empty((d.B, d.L, 4), dtype=torch.float32, device=dev)
    asc = torch.empty((d.B, d.L), dtype=torch.float32, device=dev)
    nbytes = L.load().sgb_atss_workspace_bytes(ctypes.byref(d))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    lv = (ctypes.c_int32 * len(level_sizes))(*[int(v) for v in level_sizes])
    _timed("sgb_atss_assign", ctypes.byref(d), _ptr(reg_distri), _ptr(anchors), _ptr(anchor_points), _ptr(stride_tensor), lv, len(level_sizes), _ptr(gt_boxes), _ptr(gt_labels),
           _ptr(gt_valid), _ptr(al), _ptr(ab), _ptr(asc), _ptr(sums), _ptr(ws), nbytes, _stream())  # fmt: skip
    return al, ab, asc


def dfl_iou_loss(d, cls_logits, reg_distri, anchor_points, stride_tensor, al, ab, asc, sums, grad_scale=1.0, want_grad=True, focal_alpha=None):
    """focal_alpha: None = varifocal classification term (the fused kernel's); a float = focal term with that alpha (<= 0: no
    alpha_t), computed by a replacement pass after the fused kernel."""
    gc = torch.empty_like(cls_logits) if want_grad else None
    gr = torch.empty_like(reg_distri) if want_grad else None
    _timed("sgb_dfl_iou_loss_fwd_bwd", ctypes.byref(d), _ptr(cls_logits), _ptr(reg_distri), _ptr(anchor_points), _ptr(stride_tensor), _ptr(al), _ptr(ab), _ptr(asc), _ptr(sums), float(grad_scale), _ptr(gc), _ptr(gr), _stream())
    if focal_alpha is not None:
        _timed("sgb_focal_cls_fwd_bwd", ctypes.byref(d), _ptr(cls_logits), _ptr(al), _ptr(asc), _ptr(sums), float(grad_scale), float(focal_alpha), _ptr(gc), _stream())
    out = torch.empty(4, dtype=torch.float32, device=cls_logits.device)
    L.call("sgb_loss_finalize", ctypes.byref(d), _ptr(sums), _ptr(out), _stream())
    return out, gc, gr


def pose_loss_desc(B, Lc, J, reg_max, n_max, topk=13, alpha=1.0, beta=6.0, w_cls=1.0, w_iou=2.5, w_dfl=0.5, w_pose_cls=1.0, w_pose_reg=1.0, iou_type=1, cls_type=0,
                   pose_cls_type=0, multiply_by_oks=False, rescale_with_score=False) -> L.PoseLossDesc:  # fmt: skip
    """iou_type 0 giou / 1 ciou; cls_type 0 focal / 1 bce; pose_cls_type 0 bce / 1 focal."""
    d = L.PoseLossDesc()
    d.B, d.L, d.J, d.reg_max, d.n_max, d.topk = B, Lc, J, reg_max, n_max, topk
    d.alpha, d.beta, d.w_cls, d.w_iou, d.w_dfl, d.w_pose_cls, d.w_pose_reg = alpha, beta, w_cls, w_iou, w_dfl, w_pose_cls, w_pose_reg
    d.iou_type, d.cls_type, d.pose_cls_type = iou_type, cls_type, pose_cls_type
    d.multiply_by_oks, d.rescale_with_score = int(bool(multiply_by_oks)), int(bool(rescale_with_score))
    return d


def pose_tal_assign(d, cls_logits, reg_distri, pose_coords, anchor_points, stride_tensor, gt_boxes, gt_poses, gt_crowd, gt_valid, sigmas, sums):
    """-> (assigned_gt [B, L] int32: index of the assigned non-crowd instance or -1, assigned_score [B, L] f32); adds the
    normaliser into sums[3] and the number of positives into sums[6] (sums: 8 zeroed doubles)."""
    dev = cls_logits.device
    agt = torch.empty((d.B, d.L), dtype=torch.int32, device=dev)
    asc = torch.empty((d.B, d.L), dtype=torch.float32, device=dev)
    nbytes = L.load().sgb_pose_tal_workspace_bytes(ctypes.byref(d))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    _timed("sgb_pose_tal_assign", ctypes.byref(d), _ptr(cls_logits), _ptr(reg_distri), _ptr(pose_coords), _ptr(anchor_points), _ptr(stride_tensor), _ptr(gt_boxes), _ptr(gt_poses),
           _ptr(gt_crowd), _ptr(gt_valid), _ptr(sigmas), _ptr(agt), _ptr(asc), _ptr(sums), _ptr(ws), nbytes, _stream())  # fmt: skip
    return agt, asc


def pose_loss(d, cls_logits, reg_distri, pose_coords, pose_logits, anchor_points, stride_tensor, gt_boxes, gt_poses, sigmas, agt, asc, sums, grad_scale=1.0, want_grad=True):
    """-> (items [6] = cls, iou, dfl, pose_cls, pose_reg, total; grad_cls, grad_reg, grad_pose_coords, grad_pose_logits)."""
    gc, gr, gp, gl = (torch.empty_like(t) if want_grad else None for t in (cls_logits, reg_distri, pose_coords, pose_logits))
    _timed("sgb_pose_loss_fwd_bwd", ctypes.byref(d), _ptr(cls_logits), _ptr(reg_distri), _ptr(pose_coords), _ptr(pose_logits), _ptr(anchor_points), _ptr(stride_tensor), _ptr(gt_boxes),
           _ptr(gt_poses), _ptr(sigmas), _ptr(agt), _ptr(asc), _ptr(sums), float(grad_scale), _ptr(gc), _ptr(gr), _ptr(gp), _ptr(gl), _stream())  # fmt: skip
    out = torch.empty(6, dtype=torch.float32, device=cls_logits.device)
    L.call("sgb_pose_loss_finalize", ctypes.byref(d), _ptr(sums), _ptr(out), _stream())
    return out, gc, gr, gp, gl


def batched_nms(boxes, scores, score_thr, iou_thr, top_k, max_out, multi_label=True, class_agnostic=False, thr_inclusive=None):
    """boxes [B,L,4] f32, scores [B,L,C] f32 -> (out [B,max_out,6], out_idx [B,max_out] int32, count [B] int32)."""
    require_cuda(boxes, "boxes")
    B, Lc, C = scores.shape
    d = L.NmsDesc()
    d.B, d.L, d.ncls = B, Lc, C
    d.score_thr, d.iou_thr = float(score_thr), float(iou_thr)
    d.top_k, d.max_out = int(top_k), int(max_out)
    d.multi_label, d.class_agnostic = int(bool(multi_label)), int(bool(class_agnostic))
    d.thr_inclusive = int(not multi_label) if thr_inclusive is None else int(bool(thr_inclusive))
    boxes = boxes.contiguous().float()
    scores = scores.contiguous().float()
    out = torch.empty((B, max_out, 6), dtype=torch.float32, device=boxes.device)
    oidx = torch.empty((B, max_out), dtype=torch.int32, device=boxes.device)
    cnt = torch.empty((B,), dtype=torch.int32, device=boxes.device)
    nbytes = L.load().sgb_nms_workspace_bytes(ctypes.byref(d))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=boxes.device)
    _timed("sgb_batched_nms", ctypes.byref(d), _ptr(boxes), _ptr(scores), _ptr(out), _ptr(oidx), _ptr(cnt), _ptr(ws), nbytes, _stream())
    return out, oidx, cnt


# ------------------------------------------------------------------------------------------------ optimizer
def sgd_step(p, g, mom, hp):
    """hp: device float32 [5] = lr, momentum, weight_decay, grad_scale, nesterov."""
    _timed("sgb_sgd_step", _ptr(p), _ptr(g), _ptr(mom), p.numel(), _ptr(hp), _stream())


def adamw_step(p, g, m, v, hp):
    """hp: device float32 [8] = lr, beta1, beta2, eps, weight_decay, 1-beta1^t, 1-beta2^t, grad_scale."""
    _timed("sgb_adamw_step", _ptr(p), _ptr(g), _ptr(m), _ptr(v), p.numel(), _ptr(hp), _stream())


def ema_update(ema, p, decay_dev):
    _timed("sgb_ema_update", _ptr(ema), _ptr(p), p.numel(), _ptr(decay_dev), _stream())
