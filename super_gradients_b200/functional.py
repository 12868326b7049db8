"""Autograd glue: each torch.autograd.Function below is one fused hot-path block whose forward AND backward are
libsgb200 kernels (kernels.py).  torch only owns memory, streams and the autograd tape.

Activations are channels_last bf16 (NHWC); parameters stay fp32 (state-dict compatible with the reference) and are
re-laid-out to bf16 KRSC / CRSK once per optimizer step (cached on the parameter's version counter).
"""
import weakref
from types import SimpleNamespace
from typing import Optional

import torch

from . import kernels as K

__all__ = [
    "to_nhwc",
    "from_nhwc",
    "conv_bn_act",
    "conv_bias",
    "qarepvgg_block",
    "conv_transpose2x2",
    "max_pool",
    "concat",
    "add",
    "global_avg_pool",
    "dfl_decode",
    "pose_decode",
]


_WEIGHT_EPOCH = [0]
_NBT_DEFERRED = [False]  # True inside a TrainStep: it bumps every num_batches_tracked buffer with one foreach add


def bump_weight_epoch():
    """Invalidates every WeightCache.  The Trainer calls this after each optimizer step: its kernels update the flat
    parameter buffer through raw pointers, which does not advance torch's per-tensor version counters."""
    _WEIGHT_EPOCH[0] += 1


def weight_epoch() -> int:
    return _WEIGHT_EPOCH[0]


class StepContext:
    """Per-TrainStep state of the batched plumbing: the filter caches its model touched, the device work tables of the
    batched filter re-layout / gradient layout change (kept alive here because a captured CUDA graph reads them) and the
    weight gradients waiting for the batched conversion."""

    def __init__(self):
        self.caches = {}          # id(cache) -> WeightCache
        self.weight_table = None  # (device items, n, total)
        self.weight_key = None
        self.pending = []         # (dw fp32 KRSC, C, slot)
        self.wgrad_table = None
        self.wgrad_key = None
        self.alpha_pending = []   # QARepVGG alpha chain rule of every block, finished by one batched launch (flush_wgrads)
        self.stem_pending = []    # patch-stem weight gradients, unpacked into the two filters' slots after the join
        self.alpha_table = None
        self.alpha_key = None
        # Weight gradients are off the critical path of backward (nothing consumes them before the optimizer): with a side
        # stream they run concurrently with the dgrad / BatchNorm-backward chain (fork per wgrad, ONE join in flush_wgrads);
        # under stream capture the fork / join become parallel branches of the CUDA graph.
        self.side_stream = None   # torch.cuda.Stream or None (set by TrainStep)
        self.side_used = False
        self.keep = []            # operands of side-stream launches, referenced until the join


_CTX = [None]  # the StepContext of the TrainStep that is executing (None: per-layer launches everywhere)


def set_step_context(ctx: Optional["StepContext"]):
    _CTX[0] = ctx
    if ctx is not None:
        ctx.pending.clear()
        ctx.alpha_pending.clear()
        ctx.stem_pending.clear()
        ctx.keep.clear()
        ctx.side_used = False


class WeightCache:
    """bf16 KRSC / CRSK copies of an fp32 OIHW conv weight, refreshed when the parameter changes."""

    def __init__(self, batched: bool = True):
        self.key = None
        self.krsc = None
        self.crsk = None
        self.args = None  # (w, scale, add_identity, extra_key, c_pad) of the last prepare
        self.batched = batched  # False: never part of a TrainStep's batched refresh (its source is staged during the forward)

    @staticmethod
    def _key(w, scale, add_identity, extra_key, c_pad):
        return (w.data_ptr(), w._version, None if scale is None else (scale.data_ptr(), scale._version), add_identity, extra_key, c_pad, _WEIGHT_EPOCH[0])

    def get(self, w: torch.Tensor, scale: Optional[torch.Tensor] = None, add_identity=False, extra_key=None, c_pad=None):
        """c_pad: channel count of the activation the filter is applied to (>= w.shape[1]; the extra channels are zero)."""
        key = self._key(w, scale, add_identity, extra_key, c_pad)
        if key != self.key:
            self.krsc, self.crsk = K.weight_prepare(w, c_pad=c_pad, scale=scale, add_identity=add_identity, out=(self.krsc, self.crsk))
            self.key = key
            self.args = (w, scale, add_identity, extra_key, c_pad)
        if _CTX[0] is not None and self.batched:
            _CTX[0].caches.setdefault(id(self), self)
        return self.krsc, self.crsk

    # -- the train step's batched refresh (refresh_weight_caches): one work-table entry per filter
    def batch_ready(self, dev) -> bool:
        return self.args is not None and self.krsc is not None and self.args[0].device == dev and self.args[0].dtype == torch.float32 and self.args[0].is_contiguous()

    def batch_ident(self):
        a = self.args
        return (a[0].data_ptr(), self.krsc.data_ptr(), None if self.crsk is None else self.crsk.data_ptr(), None if a[1] is None else a[1].data_ptr(), a[2], a[4])

    def batch_entries(self):
        return [(self.args[0], self.args[1], self.krsc, self.crsk, self.krsc.shape[3], self.args[2])]

    def mark_current(self):
        self.key = WeightCache._key(*self.args)


def refresh_weight_caches(ctx: StepContext, device) -> int:
    """Re-prepares every filter the context's model uses with ONE batched launch (instead of one launch per layer on
    first use) and marks those caches current.  Called by the train step after the optimizer moved the weights."""
    dev = torch.device(device)
    live = [c for c in ctx.caches.values() if c.batch_ready(dev)]
    if not live:
        return 0
    ident = tuple(c.batch_ident() for c in live)
    if ctx.weight_key != ident:
        entries = [e for c in live for e in c.batch_entries()]
        ctx.weight_table = K.weight_prepare_batch(entries, device)
        ctx.weight_key = ident
    table, n, total = ctx.weight_table
    K.run_weight_prepare_batch(table, n, total)
    for c in live:
        c.mark_current()
    return n


def flush_wgrads(ctx: StepContext, device) -> int:
    """Converts every deferred fp32 KRSC weight gradient of this step into its OIHW gradient slot with one launch."""
    if ctx.side_used:  # join: every side-stream weight gradient is complete before the layout pass / optimizer read it
        ev = torch.cuda.Event()
        ev.record(ctx.side_stream)
        torch.cuda.current_stream().wait_event(ev)
        ctx.side_used = False
    ctx.keep.clear()
    for dwf, kout, cin, r, s, sw3, sw1 in ctx.stem_pending:
        _unpack_stem_wgrad(dwf, kout, cin, r, s, sw3, sw1)
    ctx.stem_pending.clear()
    if ctx.alpha_pending:
        ident = tuple(tuple(None if t is None else (t.data_ptr() if torch.is_tensor(t) else t) for t in e) for e in ctx.alpha_pending)
        if ctx.alpha_key != ident:
            ctx.alpha_table = K.qarep_alpha_finish_table(ctx.alpha_pending, device)
            ctx.alpha_key = ident
        K.run_qarep_alpha_finish(*ctx.alpha_table)
        ctx.alpha_pending.clear()
    pend = ctx.pending
    if not pend:
        return 0
    # a weight used twice in one step (shared filters) has two pending buffers for ONE gradient slot: the batched kernel
    # would race on it, so every contribution after the first goes through the per-layer kernel (stream-ordered)
    seen, first, rest = set(), [], []
    for item in pend:
        (rest if item[2].data_ptr() in seen else first).append(item)
        seen.add(item[2].data_ptr())
    if rest:
        pend[:] = first
    ident = tuple((dw.data_ptr(), g.data_ptr(), c) for dw, c, g in pend)
    if ctx.wgrad_key != ident:
        ctx.wgrad_table = K.wgrad_to_oihw_batch_table([(dw, c, g, True) for dw, c, g in pend], device)
        ctx.wgrad_key = ident
    table, n, total = ctx.wgrad_table
    K.run_wgrad_to_oihw_batch(table, n, total)
    for dw, c, g in rest:
        K.wgrad_to_oihw(dw, c, out=g, accumulate=True)
    pend.clear()
    return n + len(rest)


# Folded QARepVGG (default; SGB_QAREP_FOLD=0 restores the two-convolution form): a stride-1 block runs its 1x1 branch as the centre tap
# of ONE 3x3 convolution with 2K output channels (rows [0, K) = the 3x3 filters, rows [K, 2K) = alpha * K1 + I embedded at the centre),
# so y3 and u come out of one convolution launch that reads x once, dgrad consumes [dy3 | du] in one launch (no accumulating
# epilogue) and wgrad produces both gradients in one launch (for K <= 64 inside the M = 128 padding the 3x3 weight gradient pays
# for anyway).  The folded filters are written in place by the step's batched re-layout launch (FoldedWeightCache) and the weight
# gradient goes to the side stream.
QAREP_FOLD = [__import__("os").environ.get("SGB_QAREP_FOLD", "1") != "0"]
QAREP_FOLD_MAXPIX = [int(__import__("os").environ.get("SGB_QAREP_FOLD_MAXPIX", "0"))]  # > 0: fold only maps of at most this many pixels (N*H*W)
_FOLD_CHANNELS = (32, 48, 64, 96, 128, 192)  # channel counts of the YOLO-NAS stride-1 blocks that fold


def qarep_fold_supported(cin: int, x_channels: int, kout: int, stride: int) -> bool:
    return stride == 1 and cin == x_channels and cin in _FOLD_CHANNELS and 2 * kout in _FOLD_CHANNELS


class FoldedWeightCache:
    """bf16 KRSC [2K, 3, 3, C] / CRSK [C, 3, 3, 2K] of the folded filter (K3 ; centre(alpha * K1 + I)), written in place from the two
    fp32 parameters by two work-table entries of the batched filter re-layout (SgbWeightItem kp / koff / etaps / etap): inside a
    train step they ride in the step's ONE sgb_weight_prepare_batch launch, outside one the cache launches its own two-entry
    table.  The destination's never-written entries (the eight outer taps of rows [K, 2K)) stay zero from the allocation."""

    def __init__(self):
        self.key = None
        self.krsc = None
        self.crsk = None
        self.src = None    # (w3, w1, alpha, add_identity, c_pad)
        self.table = None  # own two-entry table (and the identity it was built for)
        self.table_ident = None

    def _key(self):
        w3, w1, alpha, add_identity, c_pad = self.src
        return (WeightCache._key(w3, None, False, None, c_pad), WeightCache._key(w1, alpha, add_identity, None, c_pad))

    def get(self, w3, w1, alpha, add_identity, c_pad):
        self.src = (w3, w1, alpha, add_identity, c_pad)
        kout, cin = w3.shape[0], w3.shape[1]
        if c_pad != cin:
            raise K.L.SgbError("folded QARepVGG filter: the input tensor must have exactly the filter's channel count")
        if self.krsc is None or tuple(self.krsc.shape) != (2 * kout, 3, 3, c_pad) or self.krsc.device != w3.device:
            self.krsc = torch.zeros((2 * kout, 3, 3, c_pad), dtype=torch.bfloat16, device=w3.device)
            self.crsk = torch.zeros((cin, 3, 3, 2 * kout), dtype=torch.bfloat16, device=w3.device)
            self.key = None
        key = self._key()
        if key != self.key:
            ident = self.batch_ident()
            if self.table_ident != ident:
                self.table = K.weight_prepare_batch(self.batch_entries(), w3.device)
                self.table_ident = ident
            K.run_weight_prepare_batch(*self.table)
            self.key = key
        if _CTX[0] is not None:
            _CTX[0].caches.setdefault(id(self), self)
        return self.krsc, self.crsk

    def batch_ready(self, dev) -> bool:
        if self.src is None or self.krsc is None:
            return False
        w3, w1 = self.src[0], self.src[1]
        return all(t.device == dev and t.dtype == torch.float32 and t.is_contiguous() for t in (w3, w1))

    def batch_ident(self):
        w3, w1, alpha, add_identity, c_pad = self.src
        return (w3.data_ptr(), w1.data_ptr(), None if alpha is None else alpha.data_ptr(), add_identity, self.krsc.data_ptr(), self.crsk.data_ptr())

    def batch_entries(self):
        w3, w1, alpha, add_identity, c_pad = self.src
        kout = w3.shape[0]
        w1_4d = w1 if w1.dim() == 4 else w1.view(w1.shape[0], w1.shape[1], 1, 1)
        return [
            (w3, None, self.krsc[:kout], self.crsk, c_pad, False, (2 * kout, 0, 0, 0)),                # rows [0, K): the 3x3 filter
            (w1_4d, alpha, self.krsc[kout:], self.crsk, c_pad, bool(add_identity), (2 * kout, kout, 9, 4)),  # rows [K, 2K): centre tap
        ]

    def mark_current(self):
        self.key = self._key()


class ConcatWeightCache:
    """bf16 KRSC [K1 + K2, R, S, C] / CRSK [C, R, S, K1 + K2] of two filters applied to the same input (the two 1x1 convolutions of a
    CSP layer as ONE GEMM), written in place from the two fp32 parameters by two entries of the batched filter re-layout, exactly like
    FoldedWeightCache (SgbWeightItem kp / koff)."""

    def __init__(self):
        self.key = None
        self.krsc = None
        self.crsk = None
        self.src = None    # (w1, w2, c_pad)
        self.table = None
        self.table_ident = None

    def _key(self):
        w1, w2, c_pad = self.src
        return (WeightCache._key(w1, None, False, None, c_pad), WeightCache._key(w2, None, False, None, c_pad))

    def get(self, w1, w2, c_pad):
        self.src = (w1, w2, c_pad)
        k1, cin, r, s_ = w1.shape
        k2 = w2.shape[0]
        if tuple(w2.shape[1:]) != (cin, r, s_) or k1 % 8 != 0 or k2 % 8 != 0:
            raise K.L.SgbError("concatenated filters need equal input channels / taps and multiples of 8 output channels")
        if self.krsc is None or tuple(self.krsc.shape) != (k1 + k2, r, s_, c_pad) or self.krsc.device != w1.device:
            self.krsc = torch.zeros((k1 + k2, r, s_, c_pad), dtype=torch.bfloat16, device=w1.device)
            self.crsk = torch.zeros((c_pad, r, s_, k1 + k2), dtype=torch.bfloat16, device=w1.device)
            self.key = None
        key = self._key()
        if key != self.key:
            ident = self.batch_ident()
            if self.table_ident != ident:
                self.table = K.weight_prepare_batch(self.batch_entries(), w1.device)
                self.table_ident = ident
            K.run_weight_prepare_batch(*self.table)
            self.key = key
        if _CTX[0] is not None:
            _CTX[0].caches.setdefault(id(self), self)
        return self.krsc, self.crsk

    def batch_ready(self, dev) -> bool:
        if self.src is None or self.krsc is None:
            return False
        return all(t.device == dev and t.dtype == torch.float32 and t.is_contiguous() for t in self.src[:2])

    def batch_ident(self):
        w1, w2, c_pad = self.src
        return (w1.data_ptr(), w2.data_ptr(), c_pad, self.krsc.data_ptr(), self.crsk.data_ptr())

    def batch_entries(self):
        w1, w2, c_pad = self.src
        k1, k2 = w1.shape[0], w2.shape[0]
        return [
            (w1, None, self.krsc[:k1], self.crsk, c_pad, False, (k1 + k2, 0, 0, 0)),
            (w2, None, self.krsc[k1:], self.crsk, c_pad, False, (k1 + k2, k1, 0, 0)),
        ]

    def mark_current(self):
        self.key = self._key()


# ------------------------------------------------------------------------------------------------ shared input gradients
# An activation consumed by several fused blocks (the two 1 x 1 convolutions of a CSP layer, a bottleneck's first block and its
# shortcut, a backbone feature feeding the next stage and the neck, a head stem feeding the cls / reg branches) receives one
# gradient per consumer, which autograd sums with an ATen add per extra consumer: 39 full-tensor read-read-write passes per
# YOLO-NAS-S step (0.78 ms at batch 32).  Every input-gradient kernel here can instead ACCUMULATE into an existing tensor in its
# epilogue (sgb_conv_dgrad's `accumulate`, sgb_scale_add's in-place form), so the consumers of one tensor object share a token:
# the first to run backward produces the gradient buffer, the others add into it and return None to autograd, the last returns
# the buffer.  Autograd's sum is unchanged whatever else consumes the tensor (non-participating consumers are added by autograd
# as before).  It relies on every registered consumer running in the same backward pass; a pass that reaches only some of them
# (part of the outputs unused) is detected by a callback at the end of the pass and raises instead of returning wrong gradients
# The ATen adds disappear, but the accumulating convolution epilogues read the residual row with dependent loads; the mechanism is
# OFF by default (SGB_SHARE_GRADS=1 turns it on) until those epilogues prefetch the residual through TMA.
SHARE_GRADS = [__import__("os").environ.get("SGB_SHARE_GRADS", "0") == "1"]


class _GradShare:
    __slots__ = ("n", "arrived", "buf", "queued")

    def __init__(self):
        self.n = 0          # consumers registered by the forward pass
        self.arrived = 0    # consumers whose backward ran in the current backward pass
        self.buf = None     # the gradient accumulated so far
        self.queued = False


def _share_pickup(x):
    """Called by a block's wrapper with the tensor object the caller passed in; returns the tensor's token (or None)."""
    if not SHARE_GRADS[0] or not torch.is_tensor(x) or not torch.is_grad_enabled() or not x.requires_grad or x.grad_fn is None:
        return None
    tok = x.__dict__.get("_sgb_share") if hasattr(x, "__dict__") else None
    if tok is None:
        tok = _GradShare()
        x._sgb_share = tok
    tok.n += 1
    return tok


def _share_check(tok):
    n, a = tok.n, tok.arrived
    tok.arrived, tok.buf, tok.queued = 0, None, False
    if a != n:
        raise RuntimeError(
            f"shared input gradient: {a} of the {n} fused blocks consuming one activation ran in this backward pass; the gradient of that "
            "activation would be incomplete.  Backward passes that reach only part of a model's outputs need SGB_SHARE_GRADS=0."
        )


def _share_dx(tok, fresh, accumulate):
    """The input gradient a backward returns to autograd.  fresh() -> new tensor; accumulate(buf) adds this consumer's gradient
    into buf in place."""
    if tok is None or tok.n <= 1:
        return fresh()
    if not tok.queued:
        tok.queued = True
        torch.autograd.Variable._execution_engine.queue_callback(lambda: _share_check(tok))
    tok.arrived += 1
    if tok.buf is None:
        buf = fresh()
    else:
        buf = tok.buf
        accumulate(buf)
    if tok.arrived == tok.n:
        tok.buf = None
        return buf
    tok.buf = buf
    return None


# ------------------------------------------------------------------------------------------------ deferred shortcut gradient
# A YOLO-NAS bottleneck computes alpha * x + cv2(cv1(x)).  Its backward used to be: scale_add_dot (reads dout, x; writes alpha * dout),
# ... cv1's dgrad (writes the main-path gradient), then autograd's ATen add of the two (reads both, writes dx): 6 tensor passes and two
# launches per bottleneck around the dgrad.  With a token the shortcut's backward only parks (dout, alpha, x); cv1's backward runs its
# dgrad as before and then ONE pass dx = alpha * dout + dx, dot = sum(dout * x) in place (reads dout, x, dx; writes dx): 4 passes, one
# launch, no ATen add (20 bottlenecks per YOLO-NAS-S step).  Unlike SGB_SHARE_GRADS nothing accumulates inside a GEMM epilogue.
DEFER_SHORTCUT = [__import__("os").environ.get("SGB_DEFER_SHORTCUT", "1") != "0"]


class _DeferTok:
    __slots__ = ("host", "pending")

    def __init__(self):
        self.host = False    # a fused block picked the token up in its forward and will finish the gradient in its backward
        self.pending = None  # (dout, alpha, x, alpha's gradient slot) parked by the shortcut's backward


def defer_shortcut_offer(x, alpha):
    """Called by the bottleneck before cv1(x): attaches a token to x for the block that consumes x next (or returns None)."""
    if not DEFER_SHORTCUT[0] or SHARE_GRADS[0] or not torch.is_grad_enabled() or not torch.is_tensor(x) or not x.requires_grad:
        return None
    if not torch.is_tensor(alpha) or getattr(alpha, "main_grad", None) is None:
        return None
    tok = _DeferTok()
    x._sgb_defer = tok
    return tok


def _defer_pickup(x):
    tok = x.__dict__.pop("_sgb_defer", None) if torch.is_tensor(x) and hasattr(x, "__dict__") else None
    if tok is not None:
        tok.host = True
    return tok


def defer_shortcut_withdraw(x, tok):
    """After cv1(x): drops an offer nobody picked up; returns the token only if a block hosts it."""
    if tok is None:
        return None
    if hasattr(x, "__dict__"):
        x.__dict__.pop("_sgb_defer", None)
    return tok if tok.host else None


def _defer_finish(tok, dx):
    """In the hosting block's backward, after its own input gradient dx exists: adds the parked shortcut gradient in place."""
    if tok is None or tok.pending is None:
        return dx
    dout, alpha, xs, slot = tok.pending
    tok.pending = None
    if dx is None:
        dx, dot = K.scale_add_dot(dout, alpha, xs)
    else:
        _, dot = K.scale_add_dot(dout, alpha, xs, dx, out=dx)
    slot.add_(dot.sum().float().reshape(slot.shape))
    return dx


# ------------------------------------------------------------------------------------------------ cross-rank BatchNorm statistics
class BnSync:
    """torch.nn.SyncBatchNorm semantics for one train-mode call of a fused block (reference: sg_trainer.py:449-456 converts the model
    under DDP): the kernel wrappers take the split path (statistics pass, sync(buffer), apply pass) and sync(buffer) sums the buffer
    over the module's process group -- one collective per layer in the forward (sums + element count) and one in the backward.

    Parameter gradients: the backward apply pass sees the all-reduced sums on every rank; it scales its gamma / beta gradients by
    param_scale = 1 / (ranks in the group), so that after the flat gradient all-reduce and the 1 / world average they equal the DDP
    average of torch's per-rank SyncBatchNorm gradients (which are computed from local sums).  `count` is the device tensor of the
    global element count the forward pass reduced; the backward pass of the same call reads it.
    A group of one rank sums nothing: the collective is skipped, the split path still runs."""

    __slots__ = ("group", "size", "param_scale", "count")

    def __init__(self, group):
        self.group = group
        self.size = torch.distributed.get_world_size(group)
        self.param_scale = 1.0 / self.size
        self.count = None

    def __call__(self, buf):
        SYNC_CALLS[0] += 1
        if self.size > 1:
            torch.distributed.all_reduce(buf, group=self.group)


SYNC_CALLS = [0]  # BnSync reductions issued so far (tools/time_sync_bn.py reports them per step)


def bn_sync(bn) -> Optional[BnSync]:
    """A BnSync when `bn` is a train-mode torch.nn.SyncBatchNorm and torch.distributed is initialised (process_group None: WORLD),
    else None: local statistics through the fused launches, exactly as for nn.BatchNorm2d."""
    if not (isinstance(bn, torch.nn.SyncBatchNorm) and bn.training and torch.distributed.is_available() and torch.distributed.is_initialized()):
        return None
    return BnSync(bn.process_group)


def _sync_kw(sync) -> dict:
    return {"sync": sync} if sync is not None else {}


def _mg(p):
    """Flat-buffer gradient slot of a parameter (training/flat_state.py) or None under plain autograd."""
    return getattr(p, "main_grad", None) if p is not None else None


def _deliver(slot, grad):
    """Adds `grad` into the parameter's flat gradient slot (returns None to autograd) or hands it to autograd."""
    if grad is None or slot is None:
        return grad
    slot.add_(grad.reshape(slot.shape))
    return None


def _side_wgrad(ctx, x, dy, r, s, stride, pad):
    """conv_wgrad on the context's side stream (after everything queued so far on the current stream); the result may only
    be read after flush_wgrads() joined the streams."""
    dw = K.zeros((dy.shape[1], r, s, x.shape[1]), torch.float32, x.device)  # arena (host-side) or a fill on the current stream
    main, side = torch.cuda.current_stream(), ctx.side_stream
    ev = torch.cuda.Event()
    ev.record(main)
    with torch.cuda.stream(side):
        side.wait_event(ev)
        K.conv_wgrad(x, dy, r, s, stride, pad, dw_krsc=dw)
    ctx.keep.append((x, dy, dw))
    ctx.side_used = True
    return dw


def _wgrad_raw(x, dy, r, s, stride, pad):
    """fp32 KRSC weight gradient; on the step's side stream when there is one (readable after flush_wgrads() joined)."""
    ctx = _CTX[0]
    if ctx is not None and ctx.side_stream is not None:
        return _side_wgrad(ctx, x, dy, r, s, stride, pad)
    return K.conv_wgrad(x, dy, r, s, stride, pad)


def _wgrad_finish(dw, cin, slot):
    """fp32 KRSC gradient (rows of dw) -> the parameter's flat gradient slot (deferred to the batched pass inside a step) or OIHW."""
    ctx = _CTX[0]
    if slot is not None and ctx is not None:
        ctx.pending.append((dw, cin, slot))  # dw (step arena or a plain tensor) stays referenced until flush_wgrads()
        return None
    if ctx is not None and ctx.side_used:  # no slot: the caller reads the result now
        torch.cuda.current_stream().wait_stream(ctx.side_stream)
    if slot is not None:
        K.wgrad_to_oihw(dw, cin, out=slot, accumulate=True)
        return None
    return K.wgrad_to_oihw(dw, cin)


def _wgrad(x, dy, r, s, stride, pad, cin, slot):
    ctx = _CTX[0]
    if slot is not None and ctx is not None:
        dw = _side_wgrad(ctx, x, dy, r, s, stride, pad) if ctx.side_stream is not None else K.conv_wgrad(x, dy, r, s, stride, pad)
        ctx.pending.append((dw, cin, slot))  # dw (step arena or a plain tensor) stays referenced until flush_wgrads()
        return None
    dw = K.conv_wgrad(x, dy, r, s, stride, pad)
    if slot is not None:
        K.wgrad_to_oihw(dw, cin, out=slot, accumulate=True)
        return None
    return K.wgrad_to_oihw(dw, cin)


def _chan_sum(dy: torch.Tensor) -> torch.Tensor:
    """Per-channel sum over pixels of an NHWC bf16 tensor (bias gradients) -> fp32 [C]."""
    n, c, h, w = dy.shape
    pitch = K.nhwc_pitch(dy)
    cp = ((c + 7) // 8) * 8
    view = dy if cp == c else torch.as_strided(dy, (n, cp, h, w), (h * w * pitch, 1, w * pitch, pitch), dy.storage_offset())
    return K.channel_stats(view)[0, 0, :c].float()


# ------------------------------------------------------------------------------------------------------------ layout
def to_nhwc(x: torch.Tensor) -> torch.Tensor:
    """fp32/bf16 NCHW image batch -> bf16 NHWC with channels zero-padded to a multiple of 8 (no gradient)."""
    K.require_cuda(x, "input")
    if x.dtype == torch.bfloat16 and x.shape[1] % 8 == 0:
        return K.as_nhwc(x)
    return K.nchw_f32_to_nhwc_bf16(x.detach(), c_align=16)


class _FromNhwc(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        return K.nhwc_bf16_to_nchw_f32(K.as_nhwc(x))

    @staticmethod
    def backward(ctx, g):
        return K.as_nhwc(g)


def from_nhwc(x: torch.Tensor) -> torch.Tensor:
    """bf16 NHWC -> fp32 contiguous NCHW (differentiable)."""
    return _FromNhwc.apply(x)


# ------------------------------------------------------------------------------------------------------------ conv + BN
class _ConvBnAct(torch.autograd.Function):
    """act(bn_train(conv(x)) + residual): GEMM with fused per-channel statistics, then one normalise+act pass."""

    @staticmethod
    def forward(ctx, x, w, gamma, beta, residual, cfg):
        x = K.as_nhwc(x)
        krsc, crsk = cfg.cache.get(w, c_pad=x.shape[1])
        kout, _, r, s = w.shape
        p_out = (x.shape[2] + 2 * cfg.pad - r) // cfg.stride + 1, (x.shape[3] + 2 * cfg.pad - s) // cfg.stride + 1
        # wide layers: no statistics in the GEMM epilogue, the BatchNorm launch computes them (kernels.stats_in_bn)
        pixels = x.shape[0] * p_out[0] * p_out[1]
        sync = getattr(cfg, "sync", None)
        stats = None if K.stats_in_bn(kout, pixels) else K.new_stats(kout, x.device, **({"count": pixels} if sync is not None else {}))
        y_raw = K.conv_fprop(x, krsc, kout, r, s, cfg.stride, cfg.pad, stats=stats)
        res = K.as_nhwc(residual) if residual is not None else None
        ss = getattr(cfg, "sample_scale", None)
        out, mean, rstd = K.bn_act_fwd(y_raw, stats, gamma, beta, cfg.running_mean, cfg.running_var, cfg.eps, cfg.momentum, cfg.act, res, **({"sample_scale": ss} if ss is not None else {}), **_sync_kw(sync))
        if cfg.num_batches_tracked is not None and not _NBT_DEFERRED[0]:
            cfg.num_batches_tracked += 1
        ctx.save_for_backward(x, y_raw, out, gamma, mean, rstd, beta)
        ctx.cfg, ctx.crsk, ctx.wshape, ctx.has_res = cfg, crsk, tuple(w.shape), residual is not None
        ctx.slots = (_mg(w), _mg(gamma), _mg(beta))
        return out

    @staticmethod
    def backward(ctx, dout):
        x, y_raw, out, gamma, mean, rstd, beta = ctx.saved_tensors
        cfg = ctx.cfg
        kout, cin, r, s = ctx.wshape
        sw, sg, sb = ctx.slots
        ss = getattr(cfg, "sample_scale", None)
        dy, dres, dgamma, dbeta = K.bn_act_bwd(dout, y_raw, out, gamma, mean, rstd, cfg.eps, cfg.act, want_residual_grad=ctx.has_res, dgamma=sg, dbeta=sb, beta=beta, **({"sample_scale": ss} if ss is not None else {}), **_sync_kw(getattr(cfg, "sync", None)))
        dx = None
        if ctx.needs_input_grad[0]:
            dx = _share_dx(
                getattr(cfg, "share", None),
                lambda: K.conv_dgrad(dy, ctx.crsk, x.shape, r, s, cfg.stride, cfg.pad),
                lambda buf: K.conv_dgrad(dy, ctx.crsk, x.shape, r, s, cfg.stride, cfg.pad, out=buf, accumulate=True),
            )
        dw = _wgrad(x, dy, r, s, cfg.stride, cfg.pad, cin, sw)
        return dx, dw, (None if sg is not None else dgamma), (None if sb is not None else dbeta), dres, None


def conv_bn_act(x, w, gamma, beta, running_mean, running_var, num_batches_tracked, *, stride, pad, eps, momentum, act, training, cache: WeightCache, residual=None, sample_scale=None, sync=None):
    """Conv2d(bias=False) -> BatchNorm2d -> (* drop-path scale per image) -> (+ residual) -> activation.   reference:
    modules/conv_bn_act_block.py:92-93, training/models/classification_models/resnet.py:53-84 (the residual form),
    training/utils/regularization_utils.py:4-15 (drop_path; `sample_scale` = bernoulli(keep) / keep per image, training only).
    sync: bn_sync(bn) -- cross-rank statistics (SyncBatchNorm)."""
    K.require_cuda(x, "x")
    if training:
        cfg = SimpleNamespace(stride=stride, pad=pad, eps=eps, momentum=momentum, act=act, cache=cache, running_mean=running_mean, running_var=running_var, num_batches_tracked=num_batches_tracked, sample_scale=sample_scale,
                              share=_share_pickup(x), sync=sync)  # fmt: skip
        return _ConvBnAct.apply(x, w, gamma, beta, residual, cfg)
    # inference: BN folded into the GEMM epilogue (one kernel)
    with torch.no_grad():
        x = K.as_nhwc(x)
        krsc, _ = cache.get(w, c_pad=x.shape[1])
        scale = gamma * torch.rsqrt(running_var + eps)
        shift = beta - running_mean * scale
        res = K.as_nhwc(residual) if residual is not None else None
        kout, _, r, s = w.shape
        return K.conv_fprop(x, krsc, kout, r, s, stride, pad, scale=scale, shift=shift, residual=res, act=act)


# Output channels that are not a multiple of 16 (the 68-channel DFL regression convolution, yolo_nas/dfl_heads.py:66) do not fit the
# wgmma kernels' N granularity and used to fall back to the mma.sync kernels for forward, input gradient and weight gradient.
# They now run as a convolution with K rounded up to 16: zero filter rows / bias entries for the padding channels (staged fp32 copy,
# refreshed when the parameter changes), the output allocated with that pitch and handed on as its first K channels, and in the
# backward the incoming gradient re-described with the padded channel count when its producer marked the padding as zero
# (`_sgb_zero_pad`, set by the head-decode backward), else copied into a zeroed buffer.
KPAD = [__import__("os").environ.get("SGB_KPAD", "1") != "0"]


# ------------------------------------------------------------------------------------------------------------ conv + BN stem on patches
# ResNet's first layer (7 x 7, stride 2, 3 input channels; training/models/classification_models/resnet.py:162 of the reference) has no wgmma
# kernel of its own: padded to 16 channels it ran on the mma.sync implicit GEMM at 130-145 TF/s -- 2.2 ms forward + 2.5 ms weight
# gradient of a 30 ms ResNet-50 step at batch 256.  Like the YOLO-NAS stem it becomes ONE 1 x 1 GEMM over gathered patches
# (3 * 7 * 7 = 147 patch channels padded to 160): the gather reads the image once, forward and weight gradient are im2col-free
# wgmma GEMMs, and there is no dgrad (the image needs no gradient).  Same products of the same bf16 operands, fp32 accumulation.
STEM_PATCH_MAX_CHANNELS = 256


def conv_stem_patches_supported(conv, bn, x, training) -> bool:
    if not (STEM_PATCHES[0] and training and bn is not None and torch.is_tensor(x) and x.dim() == 4 and x.dtype == torch.float32 and not x.requires_grad):
        return False
    w = conv.weight
    r, s = w.shape[2], w.shape[3]
    stride = conv.stride[0] if isinstance(conv.stride, (tuple, list)) else conv.stride
    if isinstance(conv.stride, (tuple, list)) and len(set(conv.stride)) != 1:
        return False
    # the gather stages C * R input rows of (128 - 1) * stride + R pixels in shared memory (sgb_stem_patches_f32: 48 KB)
    staged = w.shape[1] * r * ((128 - 1) * int(stride) + r) * 4 + (((w.shape[1] * r * s + 31) // 32) * 32) * 4
    return bool(conv.bias is None and conv.groups == 1 and r == s and r > 1 and x.shape[1] == w.shape[1] and w.shape[1] % 8 != 0
                and w.shape[1] * r * s <= STEM_PATCH_MAX_CHANNELS and w.shape[0] % 8 == 0 and staged + 64 <= 48 * 1024)  # fmt: skip


class PatchWeightCache:
    """fp32 [K, c_out, 1, 1] staging of a first-layer filter in patch-channel order (r, s, c) plus its bf16 KRSC copy."""

    def __init__(self):
        self.key = None
        self.stage = None
        self.inner = WeightCache(batched=False)

    def get(self, w, c_out):
        key = WeightCache._key(w, None, False, None, c_out)
        if key != self.key:
            kout, cin, r, s = w.shape
            with torch.no_grad():
                if self.stage is None or tuple(self.stage.shape) != (kout, c_out, 1, 1) or self.stage.device != w.device:
                    self.stage = torch.zeros((kout, c_out, 1, 1), dtype=torch.float32, device=w.device)
                self.stage.view(kout, c_out)[:, : cin * r * s].copy_(w.detach().permute(0, 2, 3, 1).reshape(kout, r * s * cin))
            self.key = key
        return self.inner.get(self.stage, c_pad=c_out, extra_key=key)


class _ConvBnActStem(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, gamma, beta, cfg):
        kout, cin, r, s = w.shape
        c_out = ((cin * r * s + 31) // 32) * 32
        xp = K.stem_patches(x, r, cfg.stride, cfg.pad, c_out)
        kf, _ = cfg.cache.get(w, c_out)
        pixels = xp.shape[0] * xp.shape[2] * xp.shape[3]
        stats = None if K.stats_in_bn(kout, pixels) else K.new_stats(kout, x.device, **({"count": pixels} if cfg.sync is not None else {}))
        y_raw = K.conv_fprop(xp, kf, kout, 1, 1, 1, 0, stats=stats)
        out, mean, rstd = K.bn_act_fwd(y_raw, stats, gamma, beta, cfg.running_mean, cfg.running_var, cfg.eps, cfg.momentum, cfg.act, **_sync_kw(cfg.sync))
        if cfg.num_batches_tracked is not None and not _NBT_DEFERRED[0]:
            cfg.num_batches_tracked += 1
        ctx.save_for_backward(xp, y_raw, gamma, mean, rstd, beta)
        ctx.cfg, ctx.geom = cfg, (kout, cin, r, s)
        ctx.slots = (_mg(w), _mg(gamma), _mg(beta))
        return out

    @staticmethod
    def backward(ctx, dout):
        xp, y_raw, gamma, mean, rstd, beta = ctx.saved_tensors
        cfg = ctx.cfg
        kout, cin, r, s = ctx.geom
        sw, sg, sb = ctx.slots
        dy, _, dgamma, dbeta = K.bn_act_bwd(dout, y_raw, None, gamma, mean, rstd, cfg.eps, cfg.act, dgamma=sg, dbeta=sb, beta=beta, **_sync_kw(cfg.sync))
        c = _CTX[0]
        if c is not None and c.side_stream is not None and sw is not None:
            dwf = _side_wgrad(c, xp, dy, 1, 1, 1, 0)
            c.stem_pending.append((dwf, kout, cin, r, s, sw, None))  # unpacked in flush_wgrads(), after the side stream joined
            dw = None
        else:
            dwf = K.conv_wgrad(xp, dy, 1, 1, 1, 0)
            dw = _deliver(sw, dwf.reshape(kout, dwf.shape[3])[:, : cin * r * s].reshape(kout, r, s, cin).permute(0, 3, 1, 2).contiguous())
        return None, dw, (None if sg is not None else dgamma), (None if sb is not None else dbeta), None


def conv_bn_act_stem(x, conv, bn, *, act, cache: PatchWeightCache):
    """act(bn_train(conv(x))) of a first layer over a raw fp32 NCHW image as a 1 x 1 GEMM over gathered patches; the caller checked
    conv_stem_patches_supported()."""
    K.require_cuda(x, "x")
    stride = conv.stride[0] if isinstance(conv.stride, (tuple, list)) else conv.stride
    pad = conv.padding[0] if isinstance(conv.padding, (tuple, list)) else conv.padding
    cfg = SimpleNamespace(stride=int(stride), pad=int(pad), eps=bn.eps, momentum=0.1 if bn.momentum is None else bn.momentum, act=act, cache=cache,
                          running_mean=bn.running_mean, running_var=bn.running_var, num_batches_tracked=bn.num_batches_tracked, sync=bn_sync(bn))  # fmt: skip
    return _ConvBnActStem.apply(x, conv.weight, bn.weight, bn.bias, cfg)


# ------------------------------------------------------------------------------------------------------------ two conv + BN on one input
# A CSP layer applies two 1x1 ConvBNAct layers to the same tensor (training/models/detection_models/yolo_nas/yolo_stages.py:134-135, 144-147 of the reference: conv1, conv2).  Separately
# that is 2 GEMMs reading x twice, 2 BatchNorm passes, and in backward 2 BatchNorm passes, 2 dgrads whose results autograd adds with an
# ATen kernel (3 more tensor passes over dx), 2 wgrads.  As ONE layer with concatenated output channels: 1 GEMM (x read once), 1
# BatchNorm launch over K1 + K2 channels (per-channel, so identical arithmetic), backward 1 BatchNorm launch reading the two incoming
# gradients in place (SgbBnDesc.dy2), 1 dgrad (no add), 1 wgrad whose rows are the two filters' gradients.  The two layers keep their
# own parameters / state-dict keys; the BatchNorm parameters, statistics and gradient slots of the pair must be adjacent in memory
# (training/flat_state.py lays them out so on request: YoloNASCSPLayer.sgb_adjacent_tensors) -- dual_conv_bn_act_ready() checks.
DUAL_CONV = [__import__("os").environ.get("SGB_DUAL_CONV", "1") != "0"]


def _follows(a, b) -> bool:
    """b starts exactly where a ends (same dtype, both contiguous)."""
    return a is not None and b is not None and a.dtype == b.dtype and a.is_contiguous() and b.is_contiguous() and b.data_ptr() == a.data_ptr() + a.numel() * a.element_size()


def dual_conv_bn_act_ready(conv1, bn1, conv2, bn2) -> bool:
    if not DUAL_CONV[0] or not torch.is_grad_enabled():
        return False
    w1, w2 = conv1.weight, conv2.weight
    if tuple(w1.shape[1:]) != tuple(w2.shape[1:]) or w1.shape[0] % 8 or w2.shape[0] % 8 or conv1.stride != conv2.stride or conv1.padding != conv2.padding:
        return False
    if bn1.eps != bn2.eps or bn1.momentum != bn2.momentum or bn1.running_mean is None or bn2.running_mean is None:
        return False
    if not (bn1.training and bn2.training):  # a frozen BatchNorm (eval() on the sub-module) normalises with its running statistics
        return False
    if type(bn1) is not type(bn2) or getattr(bn1, "process_group", None) is not getattr(bn2, "process_group", None):  # one collective serves both
        return False
    pairs = [(bn1.weight, bn2.weight), (bn1.bias, bn2.bias), (bn1.running_mean, bn2.running_mean), (bn1.running_var, bn2.running_var)]
    if not all(_follows(a, b) for a, b in pairs):
        return False
    slots = [(_mg(bn1.weight), _mg(bn2.weight)), (_mg(bn1.bias), _mg(bn2.bias))]
    return all(_follows(a, b) for a, b in slots) and _mg(w1) is not None and _mg(w2) is not None


class _DualConvBnAct(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w1, g1, b1, w2, g2, b2, cfg):
        x = K.as_nhwc(x)
        k1, cin, r, s = w1.shape
        k2 = w2.shape[0]
        krsc, crsk = cfg.cache.get(w1, w2, x.shape[1])
        kout = k1 + k2
        p_out = (x.shape[2] + 2 * cfg.pad - r) // cfg.stride + 1, (x.shape[3] + 2 * cfg.pad - s) // cfg.stride + 1
        pixels = x.shape[0] * p_out[0] * p_out[1]
        stats = None if K.stats_in_bn(kout, pixels) else K.new_stats(kout, x.device, **({"count": pixels} if cfg.sync is not None else {}))
        y_raw = K.conv_fprop(x, krsc, kout, r, s, cfg.stride, cfg.pad, stats=stats)
        # gamma / beta / running statistics of the second layer follow the first's in memory: the pointers of the first serve K1 + K2
        # channels (and one collective carries the statistics of both layers)
        out, mean, rstd = K.bn_act_fwd(y_raw, stats, g1, b1, cfg.rm1, cfg.rv1, cfg.eps, cfg.momentum, cfg.act, **_sync_kw(cfg.sync))
        if not _NBT_DEFERRED[0]:
            for nbt in cfg.nbt:
                if nbt is not None:
                    nbt += 1
        ctx.save_for_backward(x, y_raw, g1, b1, mean, rstd)
        ctx.cfg, ctx.crsk, ctx.shape = cfg, crsk, (k1, k2, cin, r, s)
        ctx.slots = (_mg(w1), _mg(w2), _mg(g1), _mg(b1))
        return out[:, :k1], out[:, k1:]

    @staticmethod
    def backward(ctx, d1, d2):
        x, y_raw, g1, b1, mean, rstd = ctx.saved_tensors
        cfg = ctx.cfg
        k1, k2, cin, r, s = ctx.shape
        sw1, sw2, sg, sb = ctx.slots
        if d1 is None or d2 is None:  # one of the two outputs unused: its gradient is zero
            n, _, h, w = y_raw.shape
            d1 = d1 if d1 is not None else torch.zeros((n, k1, h, w), dtype=torch.bfloat16, device=x.device).contiguous(memory_format=torch.channels_last)
            d2 = d2 if d2 is not None else torch.zeros((n, k2, h, w), dtype=torch.bfloat16, device=x.device).contiguous(memory_format=torch.channels_last)
        dy, _, _, _ = K.bn_act_bwd(d1, y_raw, None, g1, mean, rstd, cfg.eps, cfg.act, dgamma=sg, dbeta=sb, beta=b1, dy2=d2, **_sync_kw(cfg.sync))
        dx = K.conv_dgrad(dy, ctx.crsk, x.shape, r, s, cfg.stride, cfg.pad) if ctx.needs_input_grad[0] else None
        c = _CTX[0]
        if c is not None:
            dwf = _wgrad_raw(x, dy, r, s, cfg.stride, cfg.pad)  # fp32 [K1 + K2, R, S, C]: rows of the two filters
            c.pending.append((dwf[:k1], cin, sw1))
            c.pending.append((dwf[k1:], cin, sw2))
        else:
            dwf = K.conv_wgrad(x, dy, r, s, cfg.stride, cfg.pad)
            K.wgrad_to_oihw(dwf[:k1], cin, out=sw1, accumulate=True)
            K.wgrad_to_oihw(dwf[k1:], cin, out=sw2, accumulate=True)
        return dx, None, None, None, None, None, None, None


def dual_conv_bn_act(x, conv1, bn1, conv2, bn2, *, act, cache: ConcatWeightCache):
    """(act(bn1(conv1(x))), act(bn2(conv2(x)))) in training mode as one GEMM + one BatchNorm launch; the caller checked
    dual_conv_bn_act_ready().  Reference: modules/conv_bn_act_block.py:92-93 applied twice (training/models/detection_models/yolo_nas/yolo_stages.py:134-135, 144-147)."""
    K.require_cuda(x, "x")
    stride = conv1.stride[0] if isinstance(conv1.stride, (tuple, list)) else conv1.stride
    pad = conv1.padding[0] if isinstance(conv1.padding, (tuple, list)) else conv1.padding
    cfg = SimpleNamespace(stride=int(stride), pad=int(pad), eps=bn1.eps, momentum=0.1 if bn1.momentum is None else bn1.momentum, act=act, cache=cache,
                          rm1=bn1.running_mean, rv1=bn1.running_var, nbt=(bn1.num_batches_tracked, bn2.num_batches_tracked), sync=bn_sync(bn1))  # fmt: skip
    return _DualConvBnAct.apply(x, conv1.weight, bn1.weight, bn1.bias, conv2.weight, bn2.weight, bn2.bias, cfg)


class PaddedOutCache:
    def __init__(self):
        self.key = None
        self.stage = None
        self.bias = None
        self.inner = WeightCache(batched=False)

    def get(self, w4, b, kp, c_pad):
        key = (WeightCache._key(w4, None, False, None, c_pad), None if b is None else (b.data_ptr(), b._version), kp)
        if key != self.key:
            kout = w4.shape[0]
            with torch.no_grad():
                if self.stage is None or tuple(self.stage.shape) != (kp,) + tuple(w4.shape[1:]) or self.stage.device != w4.device:
                    self.stage = torch.zeros((kp,) + tuple(w4.shape[1:]), dtype=torch.float32, device=w4.device)
                    self.bias = torch.zeros((kp,), dtype=torch.float32, device=w4.device)
                self.stage[:kout].copy_(w4.detach())
                if b is not None:
                    self.bias[:kout].copy_(b.detach())
            self.key = key
        krsc, crsk = self.inner.get(self.stage, c_pad=c_pad, extra_key=key)
        return krsc, crsk, (self.bias if b is not None else None)


def _padded_view(t, kp):
    """The kp-channel tensor behind a channel-slice view whose buffer has pitch kp."""
    n, _c, h, w = t.shape
    return torch.as_strided(t, (n, kp, h, w), t.stride(), t.storage_offset())


class _ConvBias(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b, cfg):
        x = K.as_nhwc(x)
        # an nn.Linear weight [K, C] is the OIHW filter [K, C, 1, 1] of a 1 x 1 convolution: the PARAMETER itself is passed in (not a
        # reshaped view), so its weight gradient goes to the flat gradient slot like every filter's instead of through an autograd
        # AccumulateGrad node (whose stream bookkeeping invalidates a CUDA-graph capture of the step)
        ctx.w_orig_shape = tuple(w.shape)
        w4 = w if w.dim() == 4 else w.detach().view(w.shape[0], w.shape[1], 1, 1)
        kout, _, r, s = w4.shape
        ctx.kp = 0
        if KPAD[0] and w.dim() == 4 and kout % 16 != 0 and kout >= 32 and x.shape[1] % 16 == 0:
            kp = ((kout + 15) // 16) * 16
            pc = cfg.cache.__dict__.get("_kpad")
            if pc is None:
                pc = cfg.cache._kpad = PaddedOutCache()
            krsc, crsk, bpad = pc.get(w4, b, kp, x.shape[1])
            n, _, h, wd = x.shape
            P, Q = (h + 2 * cfg.pad - r) // cfg.stride + 1, (wd + 2 * cfg.pad - s) // cfg.stride + 1
            ybuf = K.empty_nhwc(n, kp, P, Q, x.device)
            K.conv_fprop(x, krsc, kp, r, s, cfg.stride, cfg.pad, shift=bpad, act=cfg.act, out=ybuf)
            y = ybuf[:, :kout].detach()  # a plain alias: autograd must not treat the output as a view of a tensor made inside forward
            ctx.kp = kp
        else:
            krsc, crsk = cfg.cache.get(w4, c_pad=x.shape[1])
            y = K.conv_fprop(x, krsc, kout, r, s, cfg.stride, cfg.pad, shift=b, act=cfg.act)
        ctx.save_for_backward(x)
        ctx.cfg, ctx.crsk, ctx.wshape, ctx.has_bias = cfg, crsk, tuple(w4.shape), b is not None
        ctx.slots = (_mg(w), _mg(b))
        return y

    @staticmethod
    def backward(ctx, dy):
        (x,) = ctx.saved_tensors
        cfg = ctx.cfg
        kout, cin, r, s = ctx.wshape
        zero_pad = getattr(dy, "_sgb_zero_pad", 0)
        dy = K.as_nhwc(dy)
        dyk = dy  # the gradient with the channel count the kernels see
        if ctx.kp:
            kp = ctx.kp
            if zero_pad == kp and K.nhwc_pitch(dy) == kp:
                dyk = _padded_view(dy, kp)
            else:
                n, _, h, wd = dy.shape
                dyk = _padded_view(K.empty_nhwc(n, kout, h, wd, dy.device, c_alloc=kp), kp)  # zero-initialised
                if kout % 8 == 0:
                    K.axpby(dy, 1.0, out=dyk[:, :kout])
                else:
                    dyk[:, :kout].copy_(dy)  # ragged channel count from a producer that did not mark its padding: plain strided copy
        dx = None
        if ctx.needs_input_grad[0]:
            dx = _share_dx(
                getattr(cfg, "share", None),
                lambda: K.conv_dgrad(dyk, ctx.crsk, x.shape, r, s, cfg.stride, cfg.pad),
                lambda buf: K.conv_dgrad(dyk, ctx.crsk, x.shape, r, s, cfg.stride, cfg.pad, out=buf, accumulate=True),
            )
        if ctx.kp:
            dwf = _wgrad_raw(x, dyk, r, s, cfg.stride, cfg.pad)  # fp32 [kp, r, s, c]; rows [0, kout) are the filter's gradient
            dw = _wgrad_finish(dwf[:kout], cin, ctx.slots[0])
        else:
            dw = _wgrad(x, dyk, r, s, cfg.stride, cfg.pad, cin, ctx.slots[0])
        if dw is not None:
            dw = dw.reshape(ctx.w_orig_shape)
        db = _deliver(ctx.slots[1], _chan_sum(dy)) if ctx.has_bias else None
        return dx, dw, db, None


def conv_bias(x, w, b, *, stride, pad, cache: WeightCache, act=None):
    """Plain Conv2d (+ bias), e.g. the cls/reg prediction convs (yolo_nas/dfl_heads.py:65-66) and nn.Linear as 1x1."""
    K.require_cuda(x, "x")
    cfg = SimpleNamespace(stride=stride, pad=pad, cache=cache, act=act, share=_share_pickup(x))
    return _ConvBias.apply(x, w, b, cfg)


# ------------------------------------------------------------------------------------------------------------ QARepVGG
class _QARepVGG(torch.autograd.Function):
    """Train-mode QARepVGG block (modules/qarepvgg_block.py:184-204) as
        y3 = conv3x3(x);  u = conv1x1_{alpha*K1 + I}(x);  out = act(a3*y3 + au*u + c0)
    where the per-channel coefficients fold bn(3x3 branch), the 1x1 bias, the identity and post_bn, and are derived
    from five fused moments (sum y3, y3^2, u, u^2, y3*u).  Backward is one reduction pass + one apply pass, then
    dgrad/wgrad of the two GEMMs (the identity and alpha ride inside the folded 1x1 weights)."""

    @staticmethod
    def forward(ctx, x, w3, g3, b3, w1, bias1, alpha, gp, bp, cfg):
        x = K.as_nhwc(x)
        kout = w3.shape[0]
        fold = QAREP_FOLD[0] and getattr(cfg, "cache_fold", None) is not None and qarep_fold_supported(w3.shape[1], x.shape[1], kout, cfg.stride)
        if fold and QAREP_FOLD_MAXPIX[0] > 0 and x.shape[0] * x.shape[2] * x.shape[3] > QAREP_FOLD_MAXPIX[0]:
            fold = False
        if fold:
            kf, cf = cfg.cache_fold.get(w3, w1, alpha, cfg.residual, x.shape[1])
            ycat = K.conv_fprop(x, kf, 2 * kout, 3, 3, 1, 1)
            y3, u, c3, c1 = ycat[:, :kout], ycat[:, kout:], cf, None
        else:
            k3, c3 = cfg.cache3.get(w3, c_pad=x.shape[1])
            k1, c1 = cfg.cache1.get(w1, scale=alpha, add_identity=cfg.residual, c_pad=x.shape[1])
            y3 = K.conv_fprop(x, k3, kout, 3, 3, cfg.stride, 1)
            u = K.conv_fprop(x, k1, kout, 1, 1, cfg.stride, 0)
        ab = None
        if bias1 is not None:
            ab = bias1 * alpha if alpha is not None else bias1
        sc = getattr(cfg, "shortcut", None)  # (x_s, alpha_s, token): out += alpha_s * x_s in the apply pass (a bottleneck's shortcut)
        skw = {"residual": sc[0], "res_alpha": sc[1]} if sc is not None else {}
        out, coef = K.qarep_fwd(y3, u, g3, b3, ab, gp, bp, cfg.rm3, cfg.rv3, cfg.rmp, cfg.rvp, cfg.eps, cfg.eps, cfg.momentum, cfg.act, cfg.use_post_bn, **skw, **_sync_kw(getattr(cfg, "sync", None)))
        ctx.shortcut = sc
        if not _NBT_DEFERRED[0]:
            for nbt in cfg.nbt:
                if nbt is not None:
                    nbt += 1
        ctx.save_for_backward(x, y3, u, out, coef, g3, gp if gp is not None else g3, w1, bias1 if bias1 is not None else g3, alpha if alpha is not None else g3)
        ctx.cfg, ctx.c3, ctx.c1, ctx.fold = cfg, c3, c1, fold
        ctx.share = getattr(cfg, "share_tok", None)
        ctx.defer = getattr(cfg, "defer_tok", None)
        ctx.flags = (bias1 is not None, alpha is not None, gp is not None, w3.shape[1])
        ctx.slots = (_mg(w3), _mg(g3), _mg(b3), _mg(w1), _mg(bias1), _mg(alpha), _mg(gp), _mg(bp))
        return out

    @staticmethod
    def backward(ctx, dout):
        x, y3, u, out, coef, g3, gp, w1, bias1, alpha = ctx.saved_tensors
        cfg = ctx.cfg
        has_bias, has_alpha, has_post, cin = ctx.flags
        sw3, sg3, sb3, sw1, sbias, salpha, sgp, sbp = ctx.slots
        if ctx.shortcut is not None:
            # out = act(...) + alpha_s * x_s: the shortcut's gradient (alpha_s * dout into x_s's gradient, sum(dout * x_s) into alpha_s's)
            # is finished by the block that consumes x_s, after its own dgrad (_defer_finish); nothing is launched here
            xs, alpha_s, tok_s = ctx.shortcut
            tok_s.pending = (K.as_nhwc(dout), alpha_s, K.as_nhwc(xs), alpha_s.main_grad)
        direct_bias = sbias if not has_alpha else None  # d(alpha*b1) == d(b1) when alpha is the constant 1
        dcat = None
        if ctx.fold:  # [dy3 | du] in one buffer: one dgrad and one wgrad launch consume it
            n, kout, h, w = y3.shape
            dcat = K.empty_nhwc(n, 2 * kout, h, w, y3.device)
        dy3, du, dg3, db3, dab, dgp, dbp = K.qarep_bwd(
            dout, out, y3, u, coef, g3, gp if has_post else None, cfg.eps, cfg.eps, cfg.act, cfg.use_post_bn, acc=(sg3, sb3, direct_bias, sgp, sbp),
            out_grads=(dcat[:, :kout], dcat[:, kout:]) if dcat is not None else None, **_sync_kw(getattr(cfg, "sync", None)),
        )  # fmt: skip
        dx = None
        dw1f = None
        tok = ctx.share
        if dcat is not None:
            if ctx.needs_input_grad[0]:
                dx = _share_dx(tok, lambda: K.conv_dgrad(dcat, ctx.c3, x.shape, 3, 3, 1, 1), lambda buf: K.conv_dgrad(dcat, ctx.c3, x.shape, 3, 3, 1, 1, out=buf, accumulate=True))
            dx = _defer_finish(ctx.defer, dx)
            c = _CTX[0]
            batched = c is not None and sw3 is not None and sw1 is not None and (not has_alpha or (salpha is not None and (sbias is not None or not has_bias)))
            # fp32 [2K, 3, 3, C]: rows [0, K) = dW3, rows [K, 2K) centre tap = d(alpha * K1 + I)
            dwf = _wgrad_raw(x, dcat, 3, 3, 1, 1) if batched else K.conv_wgrad(x, dcat, 3, 3, 1, 1)
            if batched:
                # inside a train step nothing reads the gradient before flush_wgrads(): the launch goes to the side stream and both
                # filters' gradients are delivered by the batched passes (the 1x1 filter's is the centre-tap view of the buffer)
                c.pending.append((dwf[:kout], cin, sw3))
                dw1v = dwf[kout:, 1:2, 1:2, :]  # [K, 1, 1, c] view, row pitch 9 * c
                if has_alpha:
                    c.alpha_pending.append((dw1v, cin, w1, alpha, dab if has_bias else None, bias1 if has_bias else None, sw1, sbias if has_bias else None, salpha))
                else:
                    c.pending.append((dw1v, cin, sw1))
                dw3 = dw1 = dbias1 = dalpha = None
                if has_bias and not has_alpha and sbias is None:
                    dbias1 = dab
                ret = lambda slot, v: None if slot is not None else v  # noqa: E731
                return dx, dw3, ret(sg3, dg3), ret(sb3, db3), dw1, dbias1, dalpha, (ret(sgp, dgp) if has_post else None), (ret(sbp, dbp) if has_post else None), None
            if sw3 is not None and _CTX[0] is not None:
                _CTX[0].pending.append((dwf[:kout], cin, sw3))
                dw3 = None
            elif sw3 is not None:
                K.wgrad_to_oihw(dwf[:kout], cin, out=sw3, accumulate=True)
                dw3 = None
            else:
                dw3 = K.wgrad_to_oihw(dwf[:kout], cin)
            dw1f = dwf[kout:, 1, 1, :cin].reshape(kout, cin, 1, 1).contiguous()
        else:
            if ctx.needs_input_grad[0]:

                def _fresh():
                    d = K.conv_dgrad(dy3, ctx.c3, x.shape, 3, 3, cfg.stride, 1)
                    return K.conv_dgrad(du, ctx.c1, x.shape, 1, 1, cfg.stride, 0, out=d, accumulate=True)

                def _acc(buf):
                    K.conv_dgrad(dy3, ctx.c3, x.shape, 3, 3, cfg.stride, 1, out=buf, accumulate=True)
                    K.conv_dgrad(du, ctx.c1, x.shape, 1, 1, cfg.stride, 0, out=buf, accumulate=True)

                dx = _share_dx(tok, _fresh, _acc)
            dx = _defer_finish(ctx.defer, dx)
            dw3 = _wgrad(x, dy3, 3, 3, cfg.stride, 1, cin, sw3)
        dalpha = None
        if has_alpha and dcat is not None and sw1 is not None and salpha is not None and (sbias is not None or not has_bias):
            # fold path with flat gradient slots: the same quantities with one launch each (dot / addcmul_) instead of mul + sum + add
            dalpha_v = torch.dot(dw1f.reshape(-1), w1.reshape(-1))
            if has_bias:
                dalpha_v = dalpha_v + torch.dot(dab, bias1)
                sbias.addcmul_(dab, alpha)
            sw1.addcmul_(dw1f, alpha)
            salpha.add_(dalpha_v)
            dw1 = dbias1 = dalpha = None
        elif has_alpha and dw1f is None and _CTX[0] is not None and sw1 is not None and salpha is not None and (sbias is not None or not has_bias):
            # batched plumbing: the 1x1 weight gradient goes to the side stream (when there is one) and the alpha chain rule of
            # every block is finished by ONE launch in flush_wgrads() instead of ~7 small launches per block
            c = _CTX[0]
            dw1k = _side_wgrad(c, x, du, 1, 1, cfg.stride, 0) if c.side_stream is not None else K.conv_wgrad(x, du, 1, 1, cfg.stride, 0)
            c.alpha_pending.append((dw1k, cin, w1, alpha, dab if has_bias else None, bias1 if has_bias else None, sw1, sbias if has_bias else None, salpha))
            dw1 = dbias1 = dalpha = None
        elif has_alpha:
            if dw1f is None:
                dw1f = K.wgrad_to_oihw(K.conv_wgrad(x, du, 1, 1, cfg.stride, 0), cin)  # grad of the folded alpha*K1 + I
            dalpha = (dw1f * w1).sum().reshape(1)
            if has_bias:
                dalpha = dalpha + (dab * bias1).sum().reshape(1)
            dw1 = _deliver(sw1, dw1f * alpha)
            dbias1 = _deliver(sbias, dab * alpha) if has_bias else None
            dalpha = _deliver(salpha, dalpha)
        else:
            dw1 = _deliver(sw1, dw1f) if dw1f is not None else _wgrad(x, du, 1, 1, cfg.stride, 0, cin, sw1)
            dbias1 = (None if sbias is not None else dab) if has_bias else None
        ret = lambda slot, v: None if slot is not None else v  # noqa: E731
        return dx, dw3, ret(sg3, dg3), ret(sb3, db3), dw1, dbias1, dalpha, (ret(sgp, dgp) if has_post else None), (ret(sbp, dbp) if has_post else None), None


FUSE_SHORTCUT = [__import__("os").environ.get("SGB_FUSE_SHORTCUT", "1") != "0"]


def qarepvgg_block(x, w3, g3, b3, w1, bias1, alpha, gp, bp, cfg):
    K.require_cuda(x, "x")
    cfg.share_tok = _share_pickup(x)  # cfg is built per call by the module
    cfg.defer_tok = _defer_pickup(x)
    return _QARepVGG.apply(x, w3, g3, b3, w1, bias1, alpha, gp, bp, cfg)


# ------------------------------------------------------------------------------------------------------------ QARepVGG stem on patches
STEM_PATCHES = [__import__("os").environ.get("SGB_STEM_PATCHES", "1") != "0"]


def stem_patch_channels(cin: int, r: int) -> int:
    return ((cin * r * r + 15) // 16) * 16


def stem_patches_supported(block, x) -> bool:
    """A train-mode, unfused QARepVGG first layer (3 x 3, stride 2, no identity, no learnable alpha) over a raw fp32 NCHW image
    with so few channels that all nine taps fit 32 patch channels: the YOLO-NAS / YOLO-NAS-POSE stem (yolo_stages.py:61-63)."""
    return bool(
        STEM_PATCHES[0] and block.training and not block.partially_fused and not block.fully_fused and torch.is_tensor(x) and x.dim() == 4
        and x.dtype == torch.float32 and not x.requires_grad and x.shape[1] == block.in_channels and block.in_channels * 9 <= 32 and block.stride == 2
        and block.identity is None and not isinstance(block.alpha, torch.Tensor) and float(block.alpha) == 1.0 and block.use_post_bn
    )  # fmt: skip


class StemPatchWeightCache:
    """fp32 [2K, c_out, 1, 1] staging of the two stem filters in patch-channel order -- rows [0, K): K3 as (r, s, c); rows [K, 2K):
    K1 at the centre tap's channels -- plus its bf16 KRSC copy, refreshed when a source changes."""

    def __init__(self):
        self.key = None
        self.stage = None
        self.inner = WeightCache(batched=False)

    def get(self, w3, w1, c_out):
        key = (WeightCache._key(w3, None, False, None, c_out), WeightCache._key(w1, None, False, None, c_out))
        if key != self.key:
            kout, cin, r, s = w3.shape
            with torch.no_grad():
                if self.stage is None or tuple(self.stage.shape) != (2 * kout, c_out, 1, 1) or self.stage.device != w3.device:
                    self.stage = torch.zeros((2 * kout, c_out, 1, 1), dtype=torch.float32, device=w3.device)
                st = self.stage.view(2 * kout, c_out)
                st[:kout, : cin * r * s].copy_(w3.detach().permute(0, 2, 3, 1).reshape(kout, r * s * cin))
                ctr = ((r // 2) * s + s // 2) * cin
                st[kout:, ctr : ctr + cin].copy_(w1.detach()[:, :, 0, 0])
            self.key = key
        return self.inner.get(self.stage, c_pad=c_out, extra_key=key)


def _unpack_stem_wgrad(dwf, kout, cin, r, s, sw3, sw1):
    """dwf fp32 [2K, 1, 1, c_out] (gradient of the staged patch filter) -> += into the two OIHW gradient slots."""
    g = dwf.reshape(dwf.shape[0], dwf.shape[3])
    sw3.add_(g[:kout, : cin * r * s].reshape(kout, r, s, cin).permute(0, 3, 1, 2))
    if sw1 is None:  # a plain conv + BN stem (functional._ConvBnActStem): one filter
        return
    ctr = ((r // 2) * s + s // 2) * cin
    sw1.add_(g[kout:, ctr : ctr + cin].reshape(kout, cin, 1, 1))


class _QARepVGGStem(torch.autograd.Function):
    """The train-mode QARepVGG stem as ONE 1 x 1 GEMM over gathered patches: y3 = conv3x3_s2(x) and u = conv1x1_s2(x) are the
    first / second K output channels of `patches(x) @ [K3 ; centre(K1)]`.  The im2col engine fetched the 16-channel-padded image
    once per tap (9 x 419 MB through L2 per pass at batch 32) for each of the four stem launches; here the image is read once by the
    gather and the two GEMMs (forward, weight gradient) read a 32-channel tensor.  Same arithmetic per output: products of the
    same bf16 operands accumulated in fp32.  The image needs no gradient, so there is no dgrad."""

    @staticmethod
    def forward(ctx, x, w3, g3, b3, w1, bias1, gp, bp, cfg):
        kout, cin, r, s = w3.shape
        c_out = stem_patch_channels(cin, r)
        xp = K.stem_patches(x, r, cfg.stride, 1, c_out)
        kf, _ = cfg.cache_stem.get(w3, w1, c_out)
        ycat = K.conv_fprop(xp, kf, 2 * kout, 1, 1, 1, 0)
        y3, u = ycat[:, :kout], ycat[:, kout:]
        out, coef = K.qarep_fwd(y3, u, g3, b3, bias1, gp, bp, cfg.rm3, cfg.rv3, cfg.rmp, cfg.rvp, cfg.eps, cfg.eps, cfg.momentum, cfg.act, True, **_sync_kw(getattr(cfg, "sync", None)))
        if not _NBT_DEFERRED[0]:
            for nbt in cfg.nbt:
                if nbt is not None:
                    nbt += 1
        ctx.save_for_backward(xp, y3, u, out, coef, g3, gp)
        ctx.cfg, ctx.geom, ctx.has_bias = cfg, (kout, cin, r, s), bias1 is not None
        ctx.slots = (_mg(w3), _mg(g3), _mg(b3), _mg(w1), _mg(bias1), _mg(gp), _mg(bp))
        return out

    @staticmethod
    def backward(ctx, dout):
        xp, y3, u, out, coef, g3, gp = ctx.saved_tensors
        cfg = ctx.cfg
        kout, cin, r, s = ctx.geom
        sw3, sg3, sb3, sw1, sbias, sgp, sbp = ctx.slots
        n, _, h, w = y3.shape
        dcat = K.empty_nhwc(n, 2 * kout, h, w, y3.device)
        _dy3, _du, dg3, db3, dab, dgp, dbp = K.qarep_bwd(dout, out, y3, u, coef, g3, gp, cfg.eps, cfg.eps, cfg.act, True, acc=(sg3, sb3, sbias, sgp, sbp),
                                                         out_grads=(dcat[:, :kout], dcat[:, kout:]), **_sync_kw(getattr(cfg, "sync", None)))  # fmt: skip
        c = _CTX[0]
        dw3 = dw1 = None
        if c is not None and sw3 is not None and sw1 is not None:
            dwf = _side_wgrad(c, xp, dcat, 1, 1, 1, 0) if c.side_stream is not None else K.conv_wgrad(xp, dcat, 1, 1, 1, 0)
            c.stem_pending.append((dwf, kout, cin, r, s, sw3, sw1))  # unpacked in flush_wgrads(), after the side stream joined
        else:
            dwf = K.conv_wgrad(xp, dcat, 1, 1, 1, 0)
            g = dwf.reshape(2 * kout, dwf.shape[3])
            dw3 = _deliver(sw3, g[:kout, : cin * r * s].reshape(kout, r, s, cin).permute(0, 3, 1, 2).contiguous())
            ctr = ((r // 2) * s + s // 2) * cin
            dw1 = _deliver(sw1, g[kout:, ctr : ctr + cin].reshape(kout, cin, 1, 1).contiguous())
        ret = lambda slot, v: None if slot is not None else v  # noqa: E731
        return None, dw3, ret(sg3, dg3), ret(sb3, db3), dw1, (ret(sbias, dab) if ctx.has_bias else None), ret(sgp, dgp), ret(sbp, dbp), None


def qarepvgg_stem_block(x, w3, g3, b3, w1, bias1, gp, bp, cfg):
    K.require_cuda(x, "x")
    return _QARepVGGStem.apply(x, w3, g3, b3, w1, bias1, gp, bp, cfg)


# ------------------------------------------------------------------------------------------------------------ ConvTranspose 2x2/s2
class _ConvT2x2(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b, cache):
        x = K.as_nhwc(x)
        cin, cout = w.shape[0], w.shape[1]
        key = (w.data_ptr(), w._version, _WEIGHT_EPOCH[0])
        if cache.get("key") != key:
            wd = w.detach()
            cache["w_up"] = wd.permute(2, 3, 1, 0).reshape(4 * cout, cin).contiguous().to(torch.bfloat16)  # [(dh,dw,co)][ci]
            cache["w_dn"] = wd.permute(0, 2, 3, 1).contiguous().to(torch.bfloat16)  # [ci][dh][dw][co]
            cache["key"] = key
        y = K.convt2x2_fprop(x, cache["w_up"], b, cout)
        ctx.save_for_backward(x)
        ctx.w_dn, ctx.shape, ctx.has_bias = cache["w_dn"], (cin, cout), b is not None
        ctx.slots = (_mg(w), _mg(b))
        return y

    @staticmethod
    def backward(ctx, dy):
        (x,) = ctx.saved_tensors
        cin, cout = ctx.shape
        dy = K.as_nhwc(dy)
        dx = K.conv_fprop(dy, ctx.w_dn, cin, 2, 2, 2, 0) if ctx.needs_input_grad[0] else None
        dwk = K.conv_wgrad(dy, x, 2, 2, 2, 0)  # [ci][dh][dw][co]
        dw = _deliver(ctx.slots[0], dwk.permute(0, 3, 1, 2))
        db = _deliver(ctx.slots[1], _chan_sum(dy)) if ctx.has_bias else None
        return dx, dw, db, None


def conv_transpose2x2(x, w, b, cache: dict):
    """nn.ConvTranspose2d(c, c, kernel_size=2, stride=2) (modules/sampling.py:72-73)."""
    K.require_cuda(x, "x")
    return _ConvT2x2.apply(x, w, b, cache)


# ------------------------------------------------------------------------------------------------------------ pooling, glue
class _MaxPool(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, k, stride, pad):
        x = K.as_nhwc(x)
        y, idx = K.maxpool_fwd(x, k, stride, pad, want_idx=x.requires_grad or torch.is_grad_enabled())
        ctx.idx, ctx.geom = idx, (tuple(x.shape), k, stride, pad)
        return y

    @staticmethod
    def backward(ctx, dy):
        shape, k, stride, pad = ctx.geom
        dx32 = K.maxpool_bwd(dy, ctx.idx, shape, k, stride, pad)  # fp32, NHWC storage
        return K.as_nhwc(dx32), None, None, None


def max_pool(x, k, stride, pad):
    return _MaxPool.apply(x, k, stride, pad)


class _Concat(torch.autograd.Function):
    """Channel concat into one NHWC buffer (each input is copied once by our axpby kernel); backward hands out views."""

    @staticmethod
    def forward(ctx, *xs):
        xs = [K.as_nhwc(x) for x in xs]
        n, _, h, w = xs[0].shape
        cs = [x.shape[1] for x in xs]
        out = K.empty_nhwc(n, sum(cs), h, w, xs[0].device)
        off = 0
        for x, c in zip(xs, cs):
            K.axpby(x, 1.0, out=out[:, off : off + c])
            off += c
        ctx.cs = cs
        return out

    @staticmethod
    def backward(ctx, dy):
        dy = K.as_nhwc(dy)
        outs, off = [], 0
        for c in ctx.cs:
            outs.append(dy[:, off : off + c])
            off += c
        return tuple(outs)


def concat(xs):
    return _Concat.apply(*xs)


class _Add(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x1, x2, a, b, tok1, tok2):
        x1, x2 = K.as_nhwc(x1), K.as_nhwc(x2)
        ctx.ab = (a, b)
        ctx.toks = (tok1, tok2)
        return K.axpby(x1, a, x2, b)

    @staticmethod
    def backward(ctx, dy):
        a, b = ctx.ab
        dy = K.as_nhwc(dy)
        # a scaled branch writes a new tensor anyway, so it can take part in the shared-gradient accumulation; an unscaled branch
        # hands dy itself to autograd (no kernel) and stays out of it
        d1 = dy if a == 1.0 else _share_dx(ctx.toks[0], lambda: K.axpby(dy, a), lambda buf: K.axpby(dy, a, buf, 1.0, out=buf))
        d2 = dy if b == 1.0 else _share_dx(ctx.toks[1], lambda: K.axpby(dy, b), lambda buf: K.axpby(dy, b, buf, 1.0, out=buf))
        return d1, d2, None, None, None, None


def add(x1, x2, a=1.0, b=1.0):
    """a*x1 + b*x2 (residual connections)."""
    a, b = float(a), float(b)
    return _Add.apply(x1, x2, a, b, _share_pickup(x1) if a != 1.0 else None, _share_pickup(x2) if b != 1.0 else None)


class _GlobalAvgPool(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        x = K.as_nhwc(x)
        ctx.hw = (x.shape[2], x.shape[3])
        return K.avgpool_fwd(x)

    @staticmethod
    def backward(ctx, dy):
        return K.avgpool_bwd(K.as_nhwc(dy), ctx.hw)


def global_avg_pool(x):
    return _GlobalAvgPool.apply(x)


# ------------------------------------------------------------------------------------------------------------ head decode
def _grad_map(shape, pitch, device):
    """Gradient buffer of a head map laid out like the forward map (same channel pitch); channels beyond the logical count are
    zero and the tensor says so (`_sgb_zero_pad`), so a K-padded prediction convolution can read it without a copy."""
    n, c, h, w = shape
    g = K.empty_nhwc(n, c, h, w, device, c_alloc=pitch if pitch > c else None)
    if pitch > c:
        g._sgb_zero_pad = pitch
    return g


class _DflDecode(torch.autograd.Function):
    """NDFLHeads decode (yolo_nas/dfl_heads.py:199-245): per-level bf16 NHWC reg/cls maps -> fp32 [B, L, *] tensors."""

    @staticmethod
    def forward(ctx, cfg, *maps):
        regs, clss = maps[0::2], maps[1::2]
        regs = [K.as_nhwc(r) for r in regs]
        clss = [K.as_nhwc(c) for c in clss]
        B = regs[0].shape[0]
        hws = [r.shape[2] * r.shape[3] for r in regs]
        Ltot = sum(hws)
        dev = regs[0].device
        nb = cfg.reg_max + 1
        pb = torch.empty((B, Ltot, 4), dtype=torch.float32, device=dev)
        ps = torch.empty((B, Ltot, cfg.num_classes), dtype=torch.float32, device=dev)
        cl = torch.empty((B, Ltot, cfg.num_classes), dtype=torch.float32, device=dev)
        rd = torch.empty((B, Ltot, 4 * nb), dtype=torch.float32, device=dev)
        base = 0
        for r, c, s, hw in zip(regs, clss, cfg.strides, hws):
            K.dfl_decode(r, c, Ltot, base, cfg.num_classes, cfg.reg_max, s, cfg.cell_offset, pb, ps, cl, rd)
            base += hw
        ctx.geom = (B, hws, Ltot, [tuple(r.shape) for r in regs], [tuple(c.shape) for c in clss])
        ctx.pitches = ([K.nhwc_pitch(r) for r in regs], [K.nhwc_pitch(c) for c in clss])
        ctx.mark_non_differentiable(pb, ps)
        return pb, ps, cl, rd

    @staticmethod
    def backward(ctx, _gpb, _gps, gcl, grd):
        B, hws, Ltot, rshapes, cshapes = ctx.geom
        outs = [None]
        base = 0
        for hw, rs, cs, rp, cp in zip(hws, rshapes, cshapes, ctx.pitches[0], ctx.pitches[1]):
            dr = dc = None
            if grd is not None:
                dr = _grad_map(rs, rp, grd.device)
                K.head_grad_scatter(grd.contiguous(), B, hw, Ltot, base, dr)
            if gcl is not None:
                dc = _grad_map(cs, cp, gcl.device)
                K.head_grad_scatter(gcl.contiguous(), B, hw, Ltot, base, dc)
            outs += [dr, dc]
            base += hw
        return tuple(outs)


class _PoseDecode(torch.autograd.Function):
    """YoloNASPoseNDFLHeads decode (yolo_nas_pose_ndfl_heads.py:126-206): per-level bf16 NHWC maps reg [B, 4*(reg_max+1), H, W],
    cls [B, 1 + J, H, W] (channel 0 person logit, 1..J joint logits), pose [B, 2J, H, W] -> the fp32 [B, L, *] tensors.
    Backward scatters the gradients of the raw outputs (cls_logits, reg_distri, pose_coords, pose_logits) back into the
    per-level maps; d(pose_coords)/d(offset) = pose_offset_multiplier * stride."""

    @staticmethod
    def forward(ctx, cfg, *maps):
        regs, clss, poses = [[K.as_nhwc(t) for t in maps[k::3]] for k in range(3)]
        B, dev, J = regs[0].shape[0], regs[0].device, cfg.num_joints
        hws = [r.shape[2] * r.shape[3] for r in regs]
        Ltot = sum(hws)
        nb = cfg.reg_max + 1
        pb = torch.empty((B, Ltot, 4), dtype=torch.float32, device=dev)
        ps = torch.empty((B, Ltot, 1), dtype=torch.float32, device=dev)
        cl = torch.empty((B, Ltot, 1), dtype=torch.float32, device=dev)
        rd = torch.empty((B, Ltot, 4 * nb), dtype=torch.float32, device=dev)
        pc = torch.empty((B, Ltot, J, 2), dtype=torch.float32, device=dev)
        pj = torch.empty((B, Ltot, J), dtype=torch.float32, device=dev)
        pl = torch.empty((B, Ltot, J), dtype=torch.float32, device=dev)
        base = 0
        for r, c, p, s, hw in zip(regs, clss, poses, cfg.strides, hws):
            K.dfl_decode(r, c, Ltot, base, 1, cfg.reg_max, s, cfg.cell_offset, pb, ps, cl, rd)  # class head channel 0 = person logit
            K.pose_keypoint_decode(p, c, 1, Ltot, base, J, s, cfg.cell_offset, cfg.pose_offset_multiplier, cfg.compensate, pc, pj, pl)
            base += hw
        ctx.cfg = cfg
        ctx.geom = (B, hws, Ltot, [tuple(t.shape) for t in regs], [tuple(t.shape) for t in clss], [tuple(t.shape) for t in poses])
        ctx.pitches = [[K.nhwc_pitch(t) for t in ts] for ts in (regs, clss, poses)]
        ctx.mark_non_differentiable(pb, ps, pj)
        return pb, ps, pc, pj, cl, rd, pl

    @staticmethod
    def backward(ctx, _gpb, _gps, gpc, _gpj, gcl, grd, gpl):
        cfg = ctx.cfg
        B, hws, Ltot, rshapes, cshapes, pshapes = ctx.geom
        J = cfg.num_joints
        some = next(g for g in (gpc, gcl, grd, gpl) if g is not None)
        g_cls = g_pose = None
        if gcl is not None or gpl is not None:  # one [B, L, 1 + J] gradient for the class head: person logit, then joint logits
            zc = gcl if gcl is not None else torch.zeros((B, Ltot, 1), dtype=torch.float32, device=some.device)
            zl = gpl if gpl is not None else torch.zeros((B, Ltot, J), dtype=torch.float32, device=some.device)
            g_cls = torch.cat([zc.reshape(B, Ltot, 1), zl], -1).contiguous()
        if gpc is not None:
            g_pose = gpc.reshape(B, Ltot, 2 * J).clone()
            base = 0
            for s, hw in zip(cfg.strides, hws):
                g_pose[:, base : base + hw] *= float(cfg.pose_offset_multiplier) * float(s)
                base += hw
        outs = [None]
        base = 0
        for lvl, (hw, rs, cs, psh) in enumerate(zip(hws, rshapes, cshapes, pshapes)):
            dr = dc = dp = None
            if grd is not None:
                dr = _grad_map(rs, ctx.pitches[0][lvl], some.device)
                K.head_grad_scatter(grd.contiguous(), B, hw, Ltot, base, dr)
            if g_cls is not None:
                dc = _grad_map(cs, ctx.pitches[1][lvl], some.device)
                K.head_grad_scatter(g_cls, B, hw, Ltot, base, dc)
            if g_pose is not None:
                dp = _grad_map(psh, ctx.pitches[2][lvl], some.device)
                K.head_grad_scatter(g_pose, B, hw, Ltot, base, dp)
            outs += [dr, dc, dp]
            base += hw
        return tuple(outs)


def pose_decode(regs, clss, poses, strides, num_joints, reg_max, cell_offset, pose_offset_multiplier=1.0, compensate_grid_cell_offset=True):
    """-> pred_bboxes [B, L, 4], pred_scores [B, L, 1], pose_coords [B, L, J, 2] (pixels), pose_scores [B, L, J] and the raw
    cls_logits [B, L, 1], reg_distri [B, L, 4*(reg_max+1)], pose_logits [B, L, J]; differentiable w.r.t. the maps through
    pose_coords and the three raw tensors."""
    cfg = SimpleNamespace(strides=tuple(strides), num_joints=num_joints, reg_max=reg_max, cell_offset=cell_offset, pose_offset_multiplier=pose_offset_multiplier,
                          compensate=compensate_grid_cell_offset)  # fmt: skip
    maps = []
    for r, c, p in zip(regs, clss, poses):
        maps += [r, c, p]
    pb, ps, pc, pj, cl, rd, pl = _PoseDecode.apply(cfg, *maps)
    return pb, ps, pc, pj, cl, rd, pl


def dfl_decode(regs, clss, strides, num_classes, reg_max, cell_offset):
    cfg = SimpleNamespace(strides=tuple(strides), num_classes=num_classes, reg_max=reg_max, cell_offset=cell_offset)
    maps = []
    for r, c in zip(regs, clss):
        maps += [r, c]
    return _DflDecode.apply(cfg, *maps)
