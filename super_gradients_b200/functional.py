"""Autograd glue: each torch.autograd.Function below is one fused hot-path block whose forward AND backward are
libsgb200 kernels (kernels.py).  torch only owns memory, streams and the autograd tape.

Activations are channels_last bf16 (NHWC); parameters stay fp32 (state-dict compatible with the reference) and are
re-laid-out to bf16 KRSC / CRSK once per optimizer step (cached on the parameter's version counter).
"""
import functools
import inspect
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
        self.stem_pending = []    # patch-stem weight gradients, unpacked into the filters' slots after the join
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


def _tensor_key(t):
    return None if t is None else (t.data_ptr(), t._version)


class WeightCache:
    """bf16 KRSC / CRSK copies of fp32 OIHW filters, refreshed when a source changes.

    get(): one filter, re-laid-out by sgb_weight_prepare.  get_blocks(): several filters applied to the same input, written in
    place as row blocks of ONE destination by entries of the batched filter re-layout (SgbWeightItem kp / koff / etaps / etap);
    outside a train step the cache launches its own table.  Inside a train step every cache the model touched contributes its
    entries to the step's ONE sgb_weight_prepare_batch launch (refresh_weight_caches)."""

    def __init__(self, batched: bool = True):
        self.key = None
        self.krsc = None
        self.crsk = None
        # (sources, c_pad) of the last get: (w fp32 OIHW, scale or None, add_identity, rows or None, (etaps, etap)) per source
        self.args = ((), None)
        self.table = None   # own work table of a multi-source cache, and the batch_ident() it was built for
        self.table_ident = None
        self.batched = batched  # False: never part of a TrainStep's batched refresh (its source is staged during the forward)

    @staticmethod
    def _key(srcs, c_pad):
        return tuple((w.data_ptr(), w._version, _tensor_key(scale), add_identity) for w, scale, add_identity, _, _ in srcs) + (c_pad, _WEIGHT_EPOCH[0])

    def get(self, w: torch.Tensor, scale: Optional[torch.Tensor] = None, add_identity=False, c_pad=None):
        """c_pad: channel count of the activation the filter is applied to (>= w.shape[1]; the extra channels are zero)."""
        self.args = (((w, scale, add_identity, None, None),), c_pad)
        key = self._key(*self.args)
        if key != self.key:
            self.krsc, self.crsk = K.weight_prepare(w, c_pad=c_pad, scale=scale, add_identity=add_identity, out=(self.krsc, self.crsk))
            self.key = key
        return self._enrol()

    def get_blocks(self, srcs, r, s, c_pad):
        """srcs: (w, scale, add_identity, rows, (etaps, etap)) per filter.  The filter is written into rows `rows` (a slice) of the
        destination KRSC [K, r, s, c_pad] / CRSK [c_pad, r, s, K] (K: the filters' output channels together); etaps > 0 places a 1x1
        filter at tap `etap` of the destination's etaps taps.  Entries no source writes stay zero from the allocation."""
        kout, dev = sum(src[0].shape[0] for src in srcs), srcs[0][0].device
        self.args = (srcs, c_pad)
        if self.krsc is None or tuple(self.krsc.shape) != (kout, r, s, c_pad) or self.krsc.device != dev:
            self.krsc = torch.zeros((kout, r, s, c_pad), dtype=torch.bfloat16, device=dev)
            self.crsk = torch.zeros((c_pad, r, s, kout), dtype=torch.bfloat16, device=dev)
            self.key = None
        key = self._key(*self.args)
        if key != self.key:
            ident = self.batch_ident()
            if self.table_ident != ident:
                self.table = K.weight_prepare_batch(self.batch_entries(), dev)
                self.table_ident = ident
            K.run_weight_prepare_batch(*self.table)
            self.key = key
        return self._enrol()

    def _enrol(self):
        if _CTX[0] is not None and self.batched:
            _CTX[0].caches.setdefault(id(self), self)
        return self.krsc, self.crsk

    # -- the train step's batched refresh (refresh_weight_caches)
    def batch_ready(self, dev) -> bool:
        return self.krsc is not None and all(w.device == dev and w.dtype == torch.float32 and w.is_contiguous() for w, *_ in self.args[0])

    def batch_ident(self):
        srcs, c_pad = self.args
        srcs = tuple((w.data_ptr(), None if scale is None else scale.data_ptr(), add_identity) for w, scale, add_identity, _, _ in srcs)
        return (srcs, c_pad, self.krsc.data_ptr(), None if self.crsk is None else self.crsk.data_ptr())

    def batch_entries(self):
        """The sources as weight_prepare_batch entries, one per filter."""
        srcs, c_pad = self.args
        if srcs[0][3] is None:  # one filter: the whole destination
            w, scale, add_identity, _, _ = srcs[0]
            return [(w, scale, self.krsc, self.crsk, self.krsc.shape[3], add_identity)]
        kout = self.krsc.shape[0]
        return [(w, scale, self.krsc[rows], self.crsk, c_pad, bool(add_identity), (kout, rows.start or 0) + taps)
                for w, scale, add_identity, rows, taps in srcs]  # fmt: skip


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
        c.key = c._key(*c.args)
    return n


def flush_wgrads(ctx: StepContext, device) -> int:
    """Converts every deferred fp32 KRSC weight gradient of this step into its OIHW gradient slot with one launch."""
    if ctx.side_used:  # join: every side-stream weight gradient is complete before the layout pass / optimizer read it
        ev = torch.cuda.Event()
        ev.record(ctx.side_stream)
        torch.cuda.current_stream().wait_event(ev)
        ctx.side_used = False
    ctx.keep.clear()
    for dwf, cin, kout, r, s, slots in ctx.stem_pending:
        for slot, g in zip(slots, _stem_filter_grads(dwf, cin, kout, r, s, len(slots))):
            slot.add_(g)
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


class StagedWeightCache:
    """A filter the kernels cannot take as it is, staged by torch copies into an fp32 filter they can (patch-channel order, output
    channels padded), plus the bf16 copies of that stage (an inner WeightCache outside the step's batched refresh: the stage is
    written during the forward).  The stage is rewritten when a source changes."""

    def __init__(self):
        self.key = None
        self.stages = None  # fp32 staging tensors, zero-initialised: what fill() does not write stays zero
        self.inner = WeightCache(batched=False)

    def get(self, srcs, shapes, c_pad, fill):
        """srcs: the tensors the stage is computed from (None entries allowed); shapes: of the staging tensors; fill(*stages) writes
        them.  Returns the inner cache's (KRSC, CRSK) of the first stage."""
        key = tuple(_tensor_key(t) for t in srcs) + (tuple(shapes), c_pad, _WEIGHT_EPOCH[0])
        if key != self.key:
            dev = srcs[0].device
            with torch.no_grad():
                if self.stages is None or [tuple(t.shape) for t in self.stages] != list(shapes) or self.stages[0].device != dev:
                    self.stages = [torch.zeros(shape, dtype=torch.float32, device=dev) for shape in shapes]
                    self.inner.key = None  # a new stage may sit at the old one's address with the same version
                fill(*self.stages)
            self.key = key
        return self.inner.get(self.stages[0], c_pad=c_pad)


# ------------------------------------------------------------------------------------------------ deferred shortcut gradient
# A YOLO-NAS bottleneck computes alpha * x + cv2(cv1(x)).  Its backward used to be: scale_add_dot (reads dout, x; writes alpha * dout),
# ... cv1's dgrad (writes the main-path gradient), then autograd's ATen add of the two (reads both, writes dx): 6 tensor passes and two
# launches per bottleneck around the dgrad.  With a token the shortcut's backward only parks (dout, alpha, x); cv1's backward runs its
# dgrad as before and then ONE pass dx = alpha * dout + dx, dot = sum(dout * x) in place (reads dout, x, dx; writes dx): 4 passes, one
# launch, no ATen add (20 bottlenecks per YOLO-NAS-S step).
DEFER_SHORTCUT = [True]  # False: the plain shortcut backward, which test_dual_conv_and_deferred_shortcut_are_the_same_csp_layer compares against


class _DeferTok:
    __slots__ = ("host", "pending")

    def __init__(self):
        self.host = False    # a fused block picked the token up in its forward and will finish the gradient in its backward
        self.pending = None  # (dout, alpha, x, alpha's gradient slot) parked by the shortcut's backward


def defer_shortcut_offer(x, alpha):
    """Called by the bottleneck before cv1(x): attaches a token to x for the block that consumes x next (or returns None)."""
    if not DEFER_SHORTCUT[0] or not torch.is_grad_enabled() or not torch.is_tensor(x) or not x.requires_grad:
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


def _kw(**kw) -> dict:
    """The optional keyword arguments that are set (a wrapper's default stands for the others)."""
    return {k: v for k, v in kw.items() if v is not None}


def _mg(p):
    """Flat-buffer gradient slot of a parameter (training/flat_state.py) or None under plain autograd."""
    return getattr(p, "main_grad", None) if p is not None else None


def _deliver(slot, grad):
    """Adds `grad` into the parameter's flat gradient slot (returns None to autograd) or hands it to autograd."""
    if grad is None or slot is None:
        return grad
    slot.add_(grad.reshape(slot.shape))
    return None


def _unless_slot(slot, grad):
    """A gradient a kernel has already accumulated into the parameter's slot when there is one: autograd gets it only without."""
    return None if slot is not None else grad


def _scalar(v) -> int:
    """A conv module's stride / padding as one int (the callers checked that it is symmetric)."""
    return int(v[0]) if isinstance(v, (tuple, list)) else int(v)


def _gemm_stats(kout, pixels, device, sync):
    """BatchNorm statistics buffer for the producing GEMM's epilogue, or None for wide layers: the BatchNorm launch computes them
    (kernels.stats_in_bn).  With cross-rank statistics the buffer carries the local element count too."""
    return None if K.stats_in_bn(kout) else K.new_stats(kout, device, **({"count": pixels} if sync is not None else {}))


def _bump_batches_tracked(*nbts):
    """num_batches_tracked += 1 per BatchNorm, unless a TrainStep bumps every counter at once after the step."""
    if not _NBT_DEFERRED[0]:
        for nbt in nbts:
            if nbt is not None:
                nbt += 1


def _stem_filter_grads(dwf, cin, kout, r, s, n):
    """Gradient of a staged patch filter (fp32 [n * K, 1, 1, c_out], StagedWeightCache) -> OIHW views of the gradients of its n
    filters: K3 from the patch channels (r, s, c), then K1 from the centre tap's channels."""
    g = dwf.reshape(dwf.shape[0], dwf.shape[3])
    out = [g[:kout, : cin * r * s].reshape(kout, r, s, cin).permute(0, 3, 1, 2)]
    if n > 1:
        ctr = ((r // 2) * s + s // 2) * cin
        out.append(g[kout:, ctr : ctr + cin].reshape(kout, cin, 1, 1))
    return out


def _has_slots(dest) -> bool:
    kind, slot = dest[0], dest[2]
    if kind == "stem":
        return all(t is not None for t in slot)
    if kind == "alpha":
        _w1, _alpha, dab, _bias1, sbias, salpha = dest[3]
        return slot is not None and salpha is not None and (dab is None or sbias is not None)
    return slot is not None


def _wgrad(x, dy, r, s, stride, pad, cin, *dests, centre_from=0):
    """The weight gradient of one convolution, dw = fp32 KRSC conv_wgrad(x, dy), delivered to `dests`:
      ("oihw", rows, slot)                 dw[rows] -> that filter's OIHW gradient
      ("alpha", rows, slot, chain)         dw[rows] is the gradient of a QARepVGG block's alpha * K1 + I; chain = (w1, alpha, dab, bias1,
                                           bias1's slot, alpha's slot) (dab, bias1 None without a 1x1 bias): the chain rule through alpha
                                           gives the gradients of K1, the bias and alpha
      ("stem", (kout, r, s), slots)        dw is the gradient of a staged patch filter: the gradients of its len(slots) filters
    A slot is the parameter's flat gradient slot, or None: the gradient goes to autograd.  Inside a train step, when every
    destination has its slots, nothing reads the result before flush_wgrads(): the launch goes to the step's side stream (when it
    has one) and the deliveries wait for the batched passes there.  Otherwise the gradient is computed and delivered now.
    Returns per destination what autograd receives: a tensor or None ("oihw"), (dK1, dbias, dalpha) ("alpha"), a list ("stem").
    centre_from (a folded QARepVGG filter): rows from there on get only their centre tap, the only one the destinations read."""
    ctx = _CTX[0]
    ckw = _centre_kw(K.conv_wgrad, centre_from) if centre_from else {}
    if ctx is not None and all(_has_slots(d) for d in dests):
        if ctx.side_stream is not None:
            dw = K.zeros((dy.shape[1], r, s, x.shape[1]), torch.float32, x.device)  # arena (host-side) or a fill on the current stream
            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream())
            with torch.cuda.stream(ctx.side_stream):
                ctx.side_stream.wait_event(ev)
                K.conv_wgrad(x, dy, r, s, stride, pad, dw_krsc=dw, **ckw)
            ctx.keep.append((x, dy, dw))
            ctx.side_used = True
        else:
            dw = K.conv_wgrad(x, dy, r, s, stride, pad, **ckw)
        out = []
        for kind, rows, slot, *chain in dests:  # the queued tensors (step arena or plain) stay referenced until flush_wgrads()
            if kind == "oihw":
                ctx.pending.append((dw[rows], cin, slot))
                out.append(None)
            elif kind == "alpha":
                w1, alpha, dab, bias1, sbias, salpha = chain[0]
                ctx.alpha_pending.append((dw[rows], cin, w1, alpha, dab, bias1, slot, sbias, salpha))
                out.append((None, None, None))
            else:
                ctx.stem_pending.append((dw, cin, *rows, slot))
                out.append([None] * len(slot))
        return out
    dw = K.conv_wgrad(x, dy, r, s, stride, pad, **ckw)
    out = []
    for kind, rows, slot, *chain in dests:
        if kind == "stem":
            out.append([_deliver(sl, g.contiguous()) for sl, g in zip(slot, _stem_filter_grads(dw, cin, *rows, len(slot)))])
            continue
        v = dw[rows]
        if not v.is_contiguous():  # one tap of a wider filter (a folded QARepVGG's centre tap): [K, C, 1, 1] by a torch copy
            g = v[:, 0, 0, :cin].reshape(v.shape[0], cin, 1, 1).contiguous()
        elif kind == "oihw" and slot is not None:
            K.wgrad_to_oihw(v, cin, out=slot, accumulate=True)
            out.append(None)
            continue
        else:
            g = K.wgrad_to_oihw(v, cin)
        if kind == "oihw":
            out.append(_deliver(slot, g))
            continue
        w1, alpha, dab, bias1, sbias, salpha = chain[0]
        dalpha = (g * w1).sum().reshape(1)
        if dab is not None:
            dalpha = dalpha + (dab * bias1).sum().reshape(1)
        out.append((_deliver(slot, g * alpha), _deliver(sbias, dab * alpha) if dab is not None else None, _deliver(salpha, dalpha)))
    return out


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
        stats = _gemm_stats(kout, x.shape[0] * p_out[0] * p_out[1], x.device, cfg.sync)
        y_raw = K.conv_fprop(x, krsc, kout, r, s, cfg.stride, cfg.pad, stats=stats)
        res = K.as_nhwc(residual) if residual is not None else None
        out, mean, rstd = K.bn_act_fwd(y_raw, stats, gamma, beta, cfg.running_mean, cfg.running_var, cfg.eps, cfg.momentum, cfg.act, res, **_kw(sample_scale=cfg.sample_scale, sync=cfg.sync))
        _bump_batches_tracked(cfg.num_batches_tracked)
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
        dy, dres, dgamma, dbeta = K.bn_act_bwd(dout, y_raw, out, gamma, mean, rstd, cfg.eps, cfg.act, want_residual_grad=ctx.has_res, dgamma=sg, dbeta=sb, beta=beta, **_kw(sample_scale=cfg.sample_scale, sync=cfg.sync))
        dx = K.conv_dgrad(dy, ctx.crsk, x.shape, r, s, cfg.stride, cfg.pad) if ctx.needs_input_grad[0] else None
        (dw,) = _wgrad(x, dy, r, s, cfg.stride, cfg.pad, cin, ("oihw", ..., sw))
        return dx, dw, _unless_slot(sg, dgamma), _unless_slot(sb, dbeta), dres, None


def conv_bn_act(x, w, gamma, beta, running_mean, running_var, num_batches_tracked, *, stride, pad, eps, momentum, act, training, cache: WeightCache, residual=None, sample_scale=None, sync=None):
    """Conv2d(bias=False) -> BatchNorm2d -> (* drop-path scale per image) -> (+ residual) -> activation.   reference:
    modules/conv_bn_act_block.py:92-93, training/models/classification_models/resnet.py:53-84 (the residual form),
    training/utils/regularization_utils.py:4-15 (drop_path; `sample_scale` = bernoulli(keep) / keep per image, training only).
    sync: bn_sync(bn) -- cross-rank statistics (SyncBatchNorm)."""
    K.require_cuda(x, "x")
    if training:
        cfg = SimpleNamespace(stride=stride, pad=pad, eps=eps, momentum=momentum, act=act, cache=cache, running_mean=running_mean, running_var=running_var, num_batches_tracked=num_batches_tracked, sample_scale=sample_scale,
                              sync=sync)  # fmt: skip
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
KPAD = [True]  # False: the unpadded convolution, which test_k_padded_prediction_conv_is_the_same_conv compares against


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
    if isinstance(conv.stride, (tuple, list)) and len(set(conv.stride)) != 1:
        return False
    stride = _scalar(conv.stride)
    # the gather stages C * R input rows of (128 - 1) * stride + R pixels in shared memory (sgb_stem_patches_f32: 48 KB)
    staged = w.shape[1] * r * ((128 - 1) * stride + r) * 4 + (((w.shape[1] * r * s + 31) // 32) * 32) * 4
    return bool(conv.bias is None and conv.groups == 1 and r == s and r > 1 and x.shape[1] == w.shape[1] and w.shape[1] % 8 != 0
                and w.shape[1] * r * s <= STEM_PATCH_MAX_CHANNELS and w.shape[0] % 8 == 0 and staged + 64 <= 48 * 1024)  # fmt: skip


class _ConvBnActStem(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, gamma, beta, cfg):
        kout, cin, r, s = w.shape
        c_out = ((cin * r * s + 31) // 32) * 32
        xp = K.stem_patches(x, r, cfg.stride, cfg.pad, c_out)
        # the staged filter [K, c_out, 1, 1]: w in patch-channel order (r, s, c)
        kf, _ = cfg.cache.get((w,), [(kout, c_out, 1, 1)], c_out, lambda st: st.view(kout, c_out)[:, : cin * r * s].copy_(w.detach().permute(0, 2, 3, 1).reshape(kout, r * s * cin)))
        stats = _gemm_stats(kout, xp.shape[0] * xp.shape[2] * xp.shape[3], x.device, cfg.sync)
        y_raw = K.conv_fprop(xp, kf, kout, 1, 1, 1, 0, stats=stats)
        out, mean, rstd = K.bn_act_fwd(y_raw, stats, gamma, beta, cfg.running_mean, cfg.running_var, cfg.eps, cfg.momentum, cfg.act, **_kw(sync=cfg.sync))
        _bump_batches_tracked(cfg.num_batches_tracked)
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
        dy, _, dgamma, dbeta = K.bn_act_bwd(dout, y_raw, None, gamma, mean, rstd, cfg.eps, cfg.act, dgamma=sg, dbeta=sb, beta=beta, **_kw(sync=cfg.sync))
        ((dw,),) = _wgrad(xp, dy, 1, 1, 1, 0, cin, ("stem", (kout, r, s), (sw,)))
        return None, dw, _unless_slot(sg, dgamma), _unless_slot(sb, dbeta), None


def conv_bn_act_stem(x, conv, bn, *, act, cache: StagedWeightCache):
    """act(bn_train(conv(x))) of a first layer over a raw fp32 NCHW image as a 1 x 1 GEMM over gathered patches; the caller checked
    conv_stem_patches_supported()."""
    K.require_cuda(x, "x")
    cfg = SimpleNamespace(stride=_scalar(conv.stride), pad=_scalar(conv.padding), eps=bn.eps, momentum=0.1 if bn.momentum is None else bn.momentum, act=act, cache=cache,
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
DUAL_CONV = [True]  # False: two separate layers, which test_dual_conv_and_deferred_shortcut_are_the_same_csp_layer compares against


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
        if tuple(w2.shape[1:]) != (cin, r, s) or k1 % 8 != 0 or k2 % 8 != 0:
            raise K.L.SgbError("concatenated filters need equal input channels / taps and multiples of 8 output channels")
        # one filter [K1 + K2, R, S, C]: rows [0, K1) = w1, rows [K1, K1 + K2) = w2
        krsc, crsk = cfg.cache.get_blocks([(w1, None, False, slice(None, k1), (0, 0)), (w2, None, False, slice(k1, None), (0, 0))], r, s, x.shape[1])
        kout = k1 + k2
        p_out = (x.shape[2] + 2 * cfg.pad - r) // cfg.stride + 1, (x.shape[3] + 2 * cfg.pad - s) // cfg.stride + 1
        stats = _gemm_stats(kout, x.shape[0] * p_out[0] * p_out[1], x.device, cfg.sync)
        y_raw = K.conv_fprop(x, krsc, kout, r, s, cfg.stride, cfg.pad, stats=stats)
        # gamma / beta / running statistics of the second layer follow the first's in memory: the pointers of the first serve K1 + K2
        # channels (and one collective carries the statistics of both layers)
        out, mean, rstd = K.bn_act_fwd(y_raw, stats, g1, b1, cfg.rm1, cfg.rv1, cfg.eps, cfg.momentum, cfg.act, **_kw(sync=cfg.sync))
        _bump_batches_tracked(*cfg.nbt)
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
        dy, _, _, _ = K.bn_act_bwd(d1, y_raw, None, g1, mean, rstd, cfg.eps, cfg.act, dgamma=sg, dbeta=sb, beta=b1, dy2=d2, **_kw(sync=cfg.sync))
        dx = K.conv_dgrad(dy, ctx.crsk, x.shape, r, s, cfg.stride, cfg.pad) if ctx.needs_input_grad[0] else None
        _wgrad(x, dy, r, s, cfg.stride, cfg.pad, cin, ("oihw", slice(None, k1), sw1), ("oihw", slice(k1, None), sw2))  # both slots exist (dual_conv_bn_act_ready)
        return dx, None, None, None, None, None, None, None


def dual_conv_bn_act(x, conv1, bn1, conv2, bn2, *, act, cache: WeightCache):
    """(act(bn1(conv1(x))), act(bn2(conv2(x)))) in training mode as one GEMM + one BatchNorm launch; the caller checked
    dual_conv_bn_act_ready().  Reference: modules/conv_bn_act_block.py:92-93 applied twice (training/models/detection_models/yolo_nas/yolo_stages.py:134-135, 144-147)."""
    K.require_cuda(x, "x")
    cfg = SimpleNamespace(stride=_scalar(conv1.stride), pad=_scalar(conv1.padding), eps=bn1.eps, momentum=0.1 if bn1.momentum is None else bn1.momentum, act=act, cache=cache,
                          rm1=bn1.running_mean, rv1=bn1.running_var, nbt=(bn1.num_batches_tracked, bn2.num_batches_tracked), sync=bn_sync(bn1))  # fmt: skip
    return _DualConvBnAct.apply(x, conv1.weight, bn1.weight, bn1.bias, conv2.weight, bn2.weight, bn2.bias, cfg)


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
                pc = cfg.cache._kpad = StagedWeightCache()

            def fill(stage, bias):  # the filter and bias with zero rows / entries for the padding channels
                stage[:kout].copy_(w4.detach())
                if b is not None:
                    bias[:kout].copy_(b.detach())

            krsc, crsk = pc.get((w4, b), [(kp,) + tuple(w4.shape[1:]), (kp,)], x.shape[1], fill)
            n, _, h, wd = x.shape
            P, Q = (h + 2 * cfg.pad - r) // cfg.stride + 1, (wd + 2 * cfg.pad - s) // cfg.stride + 1
            ybuf = K.empty_nhwc(n, kp, P, Q, x.device)
            K.conv_fprop(x, krsc, kp, r, s, cfg.stride, cfg.pad, shift=pc.stages[1] if b is not None else None, act=cfg.act, out=ybuf)
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
        dx = K.conv_dgrad(dyk, ctx.crsk, x.shape, r, s, cfg.stride, cfg.pad) if ctx.needs_input_grad[0] else None
        # with K padded, rows [0, kout) of the fp32 [kp, r, s, c] gradient are the filter's
        (dw,) = _wgrad(x, dyk, r, s, cfg.stride, cfg.pad, cin, ("oihw", slice(None, kout) if ctx.kp else ..., ctx.slots[0]))
        if dw is not None:
            dw = dw.reshape(ctx.w_orig_shape)
        db = _deliver(ctx.slots[1], _chan_sum(dy)) if ctx.has_bias else None
        return dx, dw, db, None


def conv_bias(x, w, b, *, stride, pad, cache: WeightCache, act=None):
    """Plain Conv2d (+ bias), e.g. the cls/reg prediction convs (yolo_nas/dfl_heads.py:65-66) and nn.Linear as 1x1."""
    K.require_cuda(x, "x")
    cfg = SimpleNamespace(stride=stride, pad=pad, cache=cache, act=act)
    return _ConvBias.apply(x, w, b, cfg)


# ------------------------------------------------------------------------------------------------------------ QARepVGG
# Folded QARepVGG (QAREP_FOLD; test_folded_qarepvgg_path_is_the_same_block holds the two-convolution form): a stride-1 block runs its 1x1 branch as the centre tap
# of ONE 3x3 convolution with 2K output channels (rows [0, K) = the 3x3 filters, rows [K, 2K) = alpha * K1 + I embedded at the centre),
# so y3 and u come out of one convolution launch that reads x once, dgrad consumes [dy3 | du] in one launch (no accumulating
# epilogue) and wgrad produces both gradients in one launch.  The eight off-centre taps of rows [K, 2K) are zeros: the three calls
# pass centre_from=K, and the kernels skip the products with those zeros (and, in wgrad, the off-centre gradients of those rows,
# which nobody reads).  The folded filters are written in place by the step's batched re-layout launch (WeightCache.get_blocks) and
# the weight gradient goes to the side stream.
QAREP_FOLD = [True]
_FOLD_CHANNELS = (32, 48, 64, 96, 128, 192)  # channel counts of the YOLO-NAS stride-1 blocks that fold


def qarep_fold_supported(cin: int, x_channels: int, kout: int, stride: int) -> bool:
    return stride == 1 and cin == x_channels and cin in _FOLD_CHANNELS and 2 * kout in _FOLD_CHANNELS


@functools.lru_cache(maxsize=None)
def _takes_centre_from(fn) -> bool:
    return "centre_from" in inspect.signature(fn).parameters


def _centre_kw(fn, kout: int) -> dict:
    """centre_from=kout for a folded filter's convolution `fn` (kernels.conv_fprop / conv_dgrad / conv_wgrad) when the kernels
    accept it (a multiple of 16).  Skipping the zero taps changes no result, so a substitute of `fn` without the keyword is called
    without it."""
    return {"centre_from": kout} if kout % 16 == 0 and _takes_centre_from(fn) else {}


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
        fold = QAREP_FOLD[0] and qarep_fold_supported(w3.shape[1], x.shape[1], kout, cfg.stride)
        if fold:
            # one filter [2K, 3, 3, C]: rows [0, K) = K3, rows [K, 2K) = alpha * K1 + I at the centre tap (tap 4 of 9)
            srcs = [(w3, None, False, slice(None, kout), (0, 0)), (w1, alpha, cfg.residual, slice(kout, None), (9, 4))]
            kf, cf = cfg.cache_fold.get_blocks(srcs, 3, 3, x.shape[1])
            ycat = K.conv_fprop(x, kf, 2 * kout, 3, 3, 1, 1, **_centre_kw(K.conv_fprop, kout))
            y3, u, c3, c1 = ycat[:, :kout], ycat[:, kout:], cf, None
        else:
            k3, c3 = cfg.cache3.get(w3, c_pad=x.shape[1])
            k1, c1 = cfg.cache1.get(w1, scale=alpha, add_identity=cfg.residual, c_pad=x.shape[1])
            y3 = K.conv_fprop(x, k3, kout, 3, 3, cfg.stride, 1)
            u = K.conv_fprop(x, k1, kout, 1, 1, cfg.stride, 0)
        ab = None
        if bias1 is not None:
            ab = bias1 * alpha if alpha is not None else bias1
        sc = cfg.shortcut  # (x_s, alpha_s, token): out += alpha_s * x_s in the apply pass (a bottleneck's shortcut)
        skw = {"residual": sc[0], "res_alpha": sc[1]} if sc is not None else {}
        out, coef = K.qarep_fwd(y3, u, g3, b3, ab, gp, bp, cfg.rm3, cfg.rv3, cfg.rmp, cfg.rvp, cfg.eps, cfg.eps, cfg.momentum, cfg.act, cfg.use_post_bn, **skw, **_kw(sync=cfg.sync))
        ctx.shortcut = sc
        _bump_batches_tracked(*cfg.nbt)
        ctx.save_for_backward(x, y3, u, out, coef, g3, gp if gp is not None else g3, w1, bias1 if bias1 is not None else g3, alpha if alpha is not None else g3)
        ctx.cfg, ctx.c3, ctx.c1, ctx.fold = cfg, c3, c1, fold
        ctx.defer = cfg.defer_tok
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
            out_grads=(dcat[:, :kout], dcat[:, kout:]) if dcat is not None else None, **_kw(sync=cfg.sync),
        )  # fmt: skip
        # the gradient of the 1x1 filter alpha * K1 + I: with a learnable alpha the chain rule gives those of K1, its bias and alpha
        chain = (w1, alpha, dab if has_bias else None, bias1 if has_bias else None, sbias if has_bias else None, salpha)
        dest1 = lambda rows: ("alpha", rows, sw1, chain) if has_alpha else ("oihw", rows, sw1)  # noqa: E731
        dx = None
        if ctx.fold:
            if ctx.needs_input_grad[0]:
                dx = K.conv_dgrad(dcat, ctx.c3, x.shape, 3, 3, 1, 1, **_centre_kw(K.conv_dgrad, kout))
            dx = _defer_finish(ctx.defer, dx)
            # fp32 [2K, 3, 3, C]: rows [0, K) = dW3, the centre tap of rows [K, 2K) = d(alpha * K1 + I) (their other taps are not computed)
            dw3, d1 = _wgrad(x, dcat, 3, 3, 1, 1, cin, ("oihw", slice(None, kout), sw3), dest1((slice(kout, None), slice(1, 2), slice(1, 2))),
                             centre_from=kout)
        else:
            if ctx.needs_input_grad[0]:
                dx = K.conv_dgrad(dy3, ctx.c3, x.shape, 3, 3, cfg.stride, 1)
                K.conv_dgrad(du, ctx.c1, x.shape, 1, 1, cfg.stride, 0, out=dx, accumulate=True)
            dx = _defer_finish(ctx.defer, dx)
            (dw3,) = _wgrad(x, dy3, 3, 3, cfg.stride, 1, cin, ("oihw", ..., sw3))
            (d1,) = _wgrad(x, du, 1, 1, cfg.stride, 0, cin, dest1(...))
        if has_alpha:
            dw1, dbias1, dalpha = d1
        else:
            dw1, dbias1, dalpha = d1, (_unless_slot(sbias, dab) if has_bias else None), None
        post = (_unless_slot(sgp, dgp), _unless_slot(sbp, dbp)) if has_post else (None, None)
        return dx, dw3, _unless_slot(sg3, dg3), _unless_slot(sb3, db3), dw1, dbias1, dalpha, *post, None


FUSE_SHORTCUT = [True]  # False: the separate shortcut add, which test_csp_layer_merged_launches_match_the_separate_layers compares against


def qarepvgg_block(x, w3, g3, b3, w1, bias1, alpha, gp, bp, cfg):
    K.require_cuda(x, "x")
    cfg.defer_tok = _defer_pickup(x)  # cfg is built per call by the module
    return _QARepVGG.apply(x, w3, g3, b3, w1, bias1, alpha, gp, bp, cfg)


# ------------------------------------------------------------------------------------------------------------ QARepVGG stem on patches
STEM_PATCHES = [True]  # False: the direct convolution, which test_patch_stem_is_the_same_block compares against
STEM_RECOMPUTE = [True]  # False: [y3 | u] stored by the patch GEMM and read by the passes, which test_stem_recompute_gpu.py compares against


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

        def fill(stage):  # [2K, c_out, 1, 1]: rows [0, K) = K3 in patch-channel order (r, s, c), rows [K, 2K) = K1 at the centre tap's channels
            st = stage.view(2 * kout, c_out)
            st[:kout, : cin * r * s].copy_(w3.detach().permute(0, 2, 3, 1).reshape(kout, r * s * cin))
            ctr = ((r // 2) * s + s // 2) * cin
            st[kout:, ctr : ctr + cin].copy_(w1.detach()[:, :, 0, 0])

        kf, _ = cfg.cache_stem.get((w3, w1), [(2 * kout, c_out, 1, 1)], c_out, fill)
        # the recompute kernels have no stand-in in the tests' CPU backend, which runs this Function on host tensors
        recompute = STEM_RECOMPUTE[0] and xp.is_cuda and c_out == 32 and kout in (32, 48, 64)
        if recompute:  # [y3 | u] is never stored: the four passes recompute it from xp
            out, coef = K.stem_qarep_fwd(xp, kf, kout, g3, b3, bias1, gp, bp, cfg.rm3, cfg.rv3, cfg.rmp, cfg.rvp, cfg.eps, cfg.momentum, cfg.act, **_kw(sync=cfg.sync))
            saved = (xp, kf, coef, g3, gp)
        else:
            ycat = K.conv_fprop(xp, kf, 2 * kout, 1, 1, 1, 0)
            y3, u = ycat[:, :kout], ycat[:, kout:]
            out, coef = K.qarep_fwd(y3, u, g3, b3, bias1, gp, bp, cfg.rm3, cfg.rv3, cfg.rmp, cfg.rvp, cfg.eps, cfg.eps, cfg.momentum, cfg.act, True, **_kw(sync=cfg.sync))
            saved = (xp, y3, u, out, coef, g3, gp)
        _bump_batches_tracked(*cfg.nbt)
        ctx.save_for_backward(*saved)
        ctx.cfg, ctx.geom, ctx.has_bias, ctx.recompute = cfg, (kout, cin, r, s), bias1 is not None, recompute
        ctx.slots = (_mg(w3), _mg(g3), _mg(b3), _mg(w1), _mg(bias1), _mg(gp), _mg(bp))
        return out

    @staticmethod
    def backward(ctx, dout):
        cfg = ctx.cfg
        kout, cin, r, s = ctx.geom
        sw3, sg3, sb3, sw1, sbias, sgp, sbp = ctx.slots
        acc = (sg3, sb3, sbias, sgp, sbp)
        if ctx.recompute:
            xp, kf, coef, g3, gp = ctx.saved_tensors
            n, _, h, w = xp.shape
            dcat = K.empty_nhwc(n, 2 * kout, h, w, xp.device)
            dg3, db3, dab, dgp, dbp = K.stem_qarep_bwd(dout, xp, kf, kout, coef, g3, gp, cfg.eps, cfg.act, dcat, acc=acc, **_kw(sync=cfg.sync))
        else:
            xp, y3, u, out, coef, g3, gp = ctx.saved_tensors
            n, _, h, w = y3.shape
            dcat = K.empty_nhwc(n, 2 * kout, h, w, y3.device)
            _dy3, _du, dg3, db3, dab, dgp, dbp = K.qarep_bwd(dout, out, y3, u, coef, g3, gp, cfg.eps, cfg.eps, cfg.act, True, acc=acc,
                                                             out_grads=(dcat[:, :kout], dcat[:, kout:]), **_kw(sync=cfg.sync))  # fmt: skip
        ((dw3, dw1),) = _wgrad(xp, dcat, 1, 1, 1, 0, cin, ("stem", (kout, r, s), (sw3, sw1)))
        return None, dw3, _unless_slot(sg3, dg3), _unless_slot(sb3, db3), dw1, (_unless_slot(sbias, dab) if ctx.has_bias else None), _unless_slot(sgp, dgp), _unless_slot(sbp, dbp), None


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
    def forward(ctx, x1, x2, a, b):
        x1, x2 = K.as_nhwc(x1), K.as_nhwc(x2)
        ctx.ab = (a, b)
        return K.axpby(x1, a, x2, b)

    @staticmethod
    def backward(ctx, dy):
        a, b = ctx.ab
        dy = K.as_nhwc(dy)
        return (dy if a == 1.0 else K.axpby(dy, a)), (dy if b == 1.0 else K.axpby(dy, b)), None, None


def add(x1, x2, a=1.0, b=1.0):
    """a*x1 + b*x2 (residual connections)."""
    return _Add.apply(x1, x2, float(a), float(b))


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
