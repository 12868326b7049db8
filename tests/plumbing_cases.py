"""Exact oracles and launch recorders for the per-step plumbing kernels of csrc/elementwise.cu: the batched filter re-layout, the batched
gradient re-layout, the QARepVGG alpha chain rule, the deferred-shortcut scale-add-dot, max / average pooling and the stem patch gather.

The oracles are written from the kernels' documented semantics (include/sgb200.h) in fp64 / numpy and import no kernel code.
`record_plumbing()` monkeypatches the kernel front ends in super_gradients_b200.kernels (functional.py and the models call them as
`K.<name>`, so every launch of a train step passes through the wrappers) and keeps what each launch read and wrote.

`maxpool_transcribed` is a plain transcription of the two max-pool forward kernels' selection logic, before and after they were made
to select the way torch does, so the CPU suite can show the old selection's out-of-bounds tap without running it on a GPU.
"""
import contextlib
import math

import numpy as np
import torch

SENTINEL_BITS = 0x7FA5  # a bf16 NaN with a payload no kernel writes: marks destination elements nothing should touch


# ------------------------------------------------------------------------------------------------ rounding
def bf16_ulp(x):
    """Spacing of bf16 numbers at |x| (fp64 ndarray): 2^(e - 8) for 2^(e-1) <= |x| < 2^e, 2^-133 among the subnormals."""
    _, e = np.frexp(np.abs(np.where(np.isfinite(x), x, 0.0)))
    return np.ldexp(1.0, np.maximum(e, -125) - 8)


def round_bf16(x):
    """fp64 -> fp64 holding the bf16 nearest to x (ties to even), rounded once from fp64; overflow to +-inf, NaN stays NaN."""
    x = np.asarray(x, dtype=np.float64)
    u = bf16_ulp(x)
    with np.errstate(invalid="ignore", over="ignore"):
        r = np.round(x / u) * u  # x / u is exact (a power-of-two scale); np.round rounds halves to even
        r = np.where(np.abs(r) >= 2.0**128, np.copysign(np.inf, x), r)
    return np.where(np.isfinite(x), r, x)


def bf16_bits(x64):
    """int16 bit patterns of fp64 values that are bf16 numbers (round_bf16 output)."""
    return torch.from_numpy(np.ascontiguousarray(x64, dtype=np.float64)).float().bfloat16().view(torch.int16).numpy()


def bits_to_f64(bits):
    return torch.from_numpy(np.ascontiguousarray(bits, dtype=np.int16)).view(torch.bfloat16).double().numpy()


def bf16_neighbours(x):
    """(lower, upper) bf16 neighbours of fp64 x (equal when x is a bf16 number)."""
    u = bf16_ulp(x)
    return np.floor(x / u) * u, np.ceil(x / u) * u


def near_bf16_midpoint(x, rel=2.0**-23):
    """True where fp64 x lies within `rel` (relative) of the midpoint between two bf16 neighbours: the band in which an fp32
    intermediate may round the other way (double rounding)."""
    u = bf16_ulp(x)
    with np.errstate(invalid="ignore"):
        mid = (np.floor(x / u) + 0.5) * u
        return np.abs(x - mid) <= rel * np.abs(x)


def f32_ulp(x):
    x = np.abs(np.asarray(x, dtype=np.float64))
    _, e = np.frexp(x)
    return np.ldexp(1.0, np.maximum(e, -125) - 24)


# ------------------------------------------------------------------------------------------------ filter re-layout
def weight_prepare_writes(w, sc, K, C, R, S, c_pad, add_identity, has_crsk, kp=0, koff=0, etaps=0, etap=0):
    """What one SgbWeightItem writes: [(part, element offsets from the part's pointer, fp64 values before rounding)], part 'krsc' or
    'crsk'.  KRSC: every (k, r, s, c < c_pad), channels [C, c_pad) as zero; with etaps > 0 the 1 x 1 source lands at tap etap of
    etaps-tap rows.  CRSK [C, R, S, Kp] (Kp = K rounded up to 8): columns [K, Kp) as zero; with kp > 0 or etaps > 0 the rows are kp (or
    Kp) wide, this filter's columns start at koff, and only k < K is written."""
    w = np.asarray(w, dtype=np.float64).reshape(K, C, R, S)
    Kp = (K + 7) // 8 * 8
    val = w * float(sc)
    if add_identity:
        n = min(K, C)
        val[np.arange(n), np.arange(n), R // 2, S // 2] += 1.0
    out = []
    # KRSC part
    k, r, s, c = np.meshgrid(np.arange(K), np.arange(R), np.arange(S), np.arange(c_pad), indexing="ij")
    v = np.zeros((K, R, S, c_pad))
    v[..., :C] = val.transpose(0, 2, 3, 1)
    if etaps > 0:
        off = (k * etaps + etap) * c_pad + c
    else:
        off = ((k * R + r) * S + s) * c_pad + c
    out.append(("krsc", off.ravel(), v.ravel()))
    if has_crsk:
        c, r, s, k = np.meshgrid(np.arange(C), np.arange(R), np.arange(S), np.arange(Kp), indexing="ij")
        v = np.zeros((C, R, S, Kp))
        v[..., :K] = val.transpose(1, 2, 3, 0)
        if kp > 0 or etaps > 0:
            row = c * etaps + etap if etaps > 0 else (c * R + r) * S + s
            keep = k < K
            off = row * (kp if kp > 0 else Kp) + koff + k
            out.append(("crsk", off[keep], v[keep]))
        else:
            out.append(("crsk", (((c * R + r) * S + s) * Kp + k).ravel(), v.ravel()))
    return out


def weight_item_elements(K, C, R, S, c_pad, has_crsk):
    """Length of one item's index space (the kernel walks the SOURCE-shaped KRSC + CRSK spaces)."""
    return K * R * S * c_pad + (C * R * S * ((K + 7) // 8 * 8) if has_crsk else 0)


# ------------------------------------------------------------------------------------------------ max-pool
def maxpool_transcribed(x, k, stride, pad, fixed=True, separable=False):
    """Transcription of maxpool_fwd_kernel (separable=False) / maxpool_s1_smem_kernel (separable=True, stride 1) for one channel of one
    image: x [H, W] float -> (values [P, Q], taps [P, Q]).  fixed=False: the selection before the fix (strict >, tap 0 to start);
    fixed=True: v > best or v is NaN, starting at the first in-bounds tap."""
    x = np.asarray(x, dtype=np.float32)
    H, W = x.shape
    P, Q = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    better = (lambda v, b: v > b or v != v) if fixed else (lambda v, b: v > b)
    y = np.zeros((P, Q), np.float32)
    taps = np.zeros((P, Q), np.int64)
    if not separable:
        for p in range(P):
            for q in range(Q):
                best, bi = -np.inf, (max(0, pad - p * stride) * k + max(0, pad - q * stride)) if fixed else 0
                for r in range(k):
                    h = p * stride - pad + r
                    if not 0 <= h < H:
                        continue
                    for s in range(k):
                        w = q * stride - pad + s
                        if 0 <= w < W and better(x[h, w], best):
                            best, bi = x[h, w], r * k + s
                y[p, q], taps[p, q] = best, bi
        return y, taps
    assert stride == 1
    rmax = np.zeros((H, Q), np.float32)
    rarg = np.zeros((H, Q), np.int64)
    for h in range(H):
        for q in range(Q):
            best, bi = -np.inf, max(0, pad - q) if fixed else 0
            for s in range(k):
                w = q - pad + s
                if 0 <= w < W and better(x[h, w], best):
                    best, bi = x[h, w], s
            rmax[h, q], rarg[h, q] = best, bi
    for p in range(P):
        for q in range(Q):
            r0 = max(0, pad - p)
            best, bi = -np.inf, (r0 * k + rarg[p - pad + r0, q]) if fixed else 0
            for r in range(k):
                h = p - pad + r
                if 0 <= h < H and better(rmax[h, q], best):
                    best, bi = rmax[h, q], r * k + rarg[h, q]
            y[p, q], taps[p, q] = best, bi
    return y, taps


def torch_maxpool_taps(x, k, stride, pad):
    """torch CPU max_pool2d of x [N, C, H, W] (any float dtype, taken as fp32 NCHW): (values fp32, arg-max as the window tap r * k + s)."""
    x = x.detach().float().cpu().contiguous()
    H, W = x.shape[-2:]
    y, flat = torch.nn.functional.max_pool2d(x, k, stride, pad, return_indices=True)
    P, Q = y.shape[-2:]
    h, w = flat // W, flat % W
    r = h - (torch.arange(P).view(P, 1) * stride - pad)
    s = w - (torch.arange(Q).view(1, Q) * stride - pad)
    return y, r * k + s, flat


def maxpool_bwd_oracle(dy, flat, x_shape):
    """fp64 gradient routed the way torch routes it (dy of every window to its arg-max input element), with the number of terms
    and the sum of their magnitudes per input element: (sum64, n_terms, sum_abs), all [N, C, H, W]."""
    N, C, H, W = x_shape
    d = dy.detach().double().cpu().reshape(N, C, -1)
    f = flat.reshape(N, C, -1)
    s = torch.zeros(N, C, H * W, dtype=torch.float64).scatter_add_(2, f, d)
    n = torch.zeros(N, C, H * W, dtype=torch.float64).scatter_add_(2, f, torch.ones_like(d))
    a = torch.zeros(N, C, H * W, dtype=torch.float64).scatter_add_(2, f, d.abs())
    return s.view(N, C, H, W), n.view(N, C, H, W), a.view(N, C, H, W)


# ------------------------------------------------------------------------------------------------ stem patches, dot bound
def stem_patches_oracle(x, R, stride, pad, c_out):
    """fp32 NCHW image -> bf16 [N, c_out, P, Q]: channel (r * R + s) * C + c of pixel (p, q) is x[n, c, p * stride - pad + r,
    q * stride - pad + s] (0 outside the image), channels >= C * R * R zero."""
    x = x.detach().float().cpu()
    N, C, H, W = x.shape
    P, Q = (H + 2 * pad - R) // stride + 1, (W + 2 * pad - R) // stride + 1
    u = torch.nn.functional.unfold(x, R, padding=pad, stride=stride)  # [N, C * R * R, P * Q], channel c * R * R + r * R + s
    u = u.view(N, C, R * R, P * Q).transpose(1, 2).reshape(N, R * R * C, P, Q)
    out = torch.zeros(N, c_out, P, Q)
    out[:, : R * R * C] = u
    return out.bfloat16()


def chan_reduce_terms_bound(M, C, tpb=256, sms=132):
    """Number of fp32 roundings one output of chan_reduce_kernel can see: ceil(M / (grid * lanes)) per-thread accumulations, then
    `lanes` in the cross-lane sum.  lanes = TPB / min(C / 8, TPB); grid = min(ceil(M / 256), cap) with cap at least one CTA per SM, and
    a smaller grid only lengthens the per-thread runs, so the smallest cap gives the bound."""
    cvb = min(C // 8, tpb)
    lanes = tpb // cvb
    grid = max(1, min(math.ceil(M / 256), sms))
    per_cta = math.ceil(M / grid)
    return math.ceil(per_cta / lanes) + lanes + 1


# ------------------------------------------------------------------------------------------------ recorders
def _storage_base(t):
    """A 1-d tensor over the whole storage of t (same dtype), and t's element offset in it."""
    st = t.untyped_storage()
    base = torch.empty(0, dtype=t.dtype, device=t.device).set_(st, 0, (st.nbytes() // t.element_size(),), (1,))
    return base, t.storage_offset()


def _clone_storages(ts):
    out = {}
    for t in ts:
        if t is not None:
            key = t.untyped_storage().data_ptr()
            if key not in out:
                out[key] = _storage_base(t)[0].clone()
    return out


class PlumbingRecord:
    def __init__(self):
        self.weight_tables = {}  # id(table) -> (table, entries)
        self.weight_runs = []    # {"entries", "before", "after"} (storages keyed by data_ptr)
        self.wgrad_tables = {}
        self.wgrad_runs = []
        self.alpha_tables = {}
        self.alpha_runs = []
        self.scale_add_dot = []
        self.maxpool_fwd = []
        self.maxpool_bwd = []


@contextlib.contextmanager
def record_plumbing():
    """Patches the kernel front ends for the duration of the block and yields a PlumbingRecord of every launch made in it."""
    from super_gradients_b200 import kernels as K

    rec = PlumbingRecord()
    orig = {n: getattr(K, n) for n in ("weight_prepare_batch", "run_weight_prepare_batch", "wgrad_to_oihw_batch_table", "run_wgrad_to_oihw_batch",
                                         "qarep_alpha_finish_table", "run_qarep_alpha_finish", "scale_add_dot", "maxpool_fwd", "maxpool_bwd")}  # fmt: skip
    sync = torch.cuda.synchronize
    cl = lambda t: None if t is None else t.detach().clone()  # noqa: E731

    def weight_prepare_batch(entries, device):
        out = orig["weight_prepare_batch"](entries, device)
        rec.weight_tables[id(out[0])] = (out[0], [tuple(e) for e in entries])
        return out

    def run_weight_prepare_batch(table, n, total):
        entries = rec.weight_tables[id(table)][1]
        sync()
        src = [(cl(e[0]), cl(e[1])) for e in entries]
        dst = [t for e in entries for t in (e[2], e[3])]
        before = _clone_storages(dst)
        orig["run_weight_prepare_batch"](table, n, total)
        sync()
        rec.weight_runs.append({"entries": entries, "src": src, "before": before, "after": _clone_storages(dst)})

    def wgrad_to_oihw_batch_table(entries, device):
        out = orig["wgrad_to_oihw_batch_table"](entries, device)
        rec.wgrad_tables[id(out[0])] = (out[0], [tuple(e) for e in entries])
        return out

    def run_wgrad_to_oihw_batch(table, n, total):
        entries = rec.wgrad_tables[id(table)][1]
        sync()
        src = [cl(e[0]) for e in entries]
        before = _clone_storages([e[2] for e in entries])
        orig["run_wgrad_to_oihw_batch"](table, n, total)
        sync()
        rec.wgrad_runs.append({"entries": entries, "src": src, "before": before, "after": _clone_storages([e[2] for e in entries])})

    def qarep_alpha_finish_table(entries, device):
        out = orig["qarep_alpha_finish_table"](entries, device)
        rec.alpha_tables[id(out[0])] = (out[0], [tuple(e) for e in entries])
        return out

    def run_qarep_alpha_finish(table, n):
        entries = rec.alpha_tables[id(table)][1]
        sync()
        before = [tuple(cl(t) if torch.is_tensor(t) else t for t in e) for e in entries]
        orig["run_qarep_alpha_finish"](table, n)
        sync()
        after = [tuple(cl(t) for t in (e[6], e[7], e[8])) for e in entries]
        rec.alpha_runs.append({"entries": entries, "before": before, "after": after})

    def scale_add_dot(x1, a_dev, xd, x2=None, out=None):
        sync()
        args = (cl(x1), cl(a_dev), cl(xd), cl(x2), out is not None and x2 is not None and out.data_ptr() == x2.data_ptr())
        y, dot = orig["scale_add_dot"](x1, a_dev, xd, x2, out=out)
        sync()
        rec.scale_add_dot.append({"x1": args[0], "a": args[1], "xd": args[2], "x2": args[3], "in_place": args[4], "y": cl(y), "dot": cl(dot)})
        return y, dot

    def maxpool_fwd(x, k, stride, pad, want_idx=True, out=None):
        sync()
        xc = cl(x)
        y, idx = orig["maxpool_fwd"](x, k, stride, pad, want_idx=want_idx, out=out)
        sync()
        rec.maxpool_fwd.append({"x": xc, "k": k, "stride": stride, "pad": pad, "y": cl(y), "idx": cl(idx), "idx_ptr": None if idx is None else idx.data_ptr()})
        return y, idx

    def maxpool_bwd(dy, idx, x_shape, k, stride, pad):
        sync()
        dyc, idxc = cl(dy), cl(idx)
        fwd = next((f for f in reversed(rec.maxpool_fwd) if f["idx_ptr"] == idx.data_ptr()), None)
        dx = orig["maxpool_bwd"](dy, idx, x_shape, k, stride, pad)
        sync()
        rec.maxpool_bwd.append({"dy": dyc, "idx": idxc, "x_shape": tuple(x_shape), "k": k, "stride": stride, "pad": pad, "dx": cl(dx), "fwd": fwd})
        return dx

    for n in orig:
        setattr(K, n, locals()[n])
    try:
        yield rec
    finally:
        for n, f in orig.items():
            setattr(K, n, f)


# ------------------------------------------------------------------------------------------------ recorded train steps
def yolo_nas_s_step_record(steps=2, batch=2, img=640, seed=0):
    """`steps` eager TrainSteps of YOLO-NAS-S (80 classes) on random images with detection targets, recorded."""
    from super_gradients_b200.training import models
    from super_gradients_b200.training.losses import PPYoloELoss, pad_targets_host
    from super_gradients_b200.training.sg_trainer import TrainStep

    torch.manual_seed(seed)
    m = models.get("yolo_nas_s", num_classes=80).cuda().train()
    st = TrainStep(m, PPYoloELoss(num_classes=80, use_static_assigner=False), "SGD", {"weight_decay": 1e-5, "momentum": 0.9}, zero_wd_on_bias_and_bn=True)
    g = torch.Generator().manual_seed(seed + 1)
    x = torch.randn(batch, 3, img, img, generator=g).cuda()
    rows = []
    for b in range(batch):
        for _ in range(6):
            cx, cy = (torch.rand(2, generator=g) * (img - 200) + 100).tolist()
            w, h = (torch.rand(2, generator=g) * 150 + 30).tolist()
            rows.append([b, int(torch.randint(0, 80, (1,), generator=g)), cx, cy, w, h])
    t = tuple(a.cuda() for a in pad_targets_host(torch.tensor(rows), batch, 16))
    with record_plumbing() as rec:
        for _ in range(steps):
            st.set_hyper_params(1e-3)
            st.run(x, t)
        torch.cuda.synchronize()
    return rec


def resnet50_step_record(steps=2, batch=2, img=224, seed=0):
    from super_gradients_b200.training import models
    from super_gradients_b200.training.losses import CrossEntropyLoss
    from super_gradients_b200.training.sg_trainer import TrainStep

    torch.manual_seed(seed)
    m = models.get("resnet50", num_classes=1000).cuda().train()
    st = TrainStep(m, CrossEntropyLoss(), "SGD", {"weight_decay": 1e-4, "momentum": 0.9}, zero_wd_on_bias_and_bn=True)
    g = torch.Generator().manual_seed(seed + 1)
    x, y = torch.randn(batch, 3, img, img, generator=g).cuda(), torch.randint(0, 1000, (batch,), generator=g).cuda()
    with record_plumbing() as rec:
        for _ in range(steps):
            st.set_hyper_params(0.1)
            st.run(x, y)
        torch.cuda.synchronize()
    return rec


def _linear_loss(out, wt):
    loss = (out.float() * wt).sum() / out.shape[0]
    return loss, loss.detach().reshape(1)


def qarep_alpha_step_record(steps=2, batch=2, seed=0):
    """YOLO-NAS-S's QARepVGG blocks have no learnable alpha: `steps` eager TrainSteps of a stack of QARepVGG blocks with use_alpha=True
    (folded stride-1 blocks with and without a 1 x 1 bias, a stride-2 block, a channel change), recorded."""
    import torch.nn as nn

    from super_gradients_b200.modules.qarepvgg_block import QARepVGGBlock
    from super_gradients_b200.training.sg_trainer import TrainStep

    torch.manual_seed(seed)
    m = nn.Sequential(
        QARepVGGBlock(32, 32, use_alpha=True),
        QARepVGGBlock(32, 64, stride=2, use_alpha=True, use_residual_connection=False),
        QARepVGGBlock(64, 64, use_alpha=True, use_1x1_bias=False),
        QARepVGGBlock(64, 48, use_alpha=True, use_residual_connection=False),
    ).cuda().train()
    st = TrainStep(m, _linear_loss, "SGD", {"momentum": 0.9}, zero_wd_on_bias_and_bn=True)
    g = torch.Generator().manual_seed(seed + 1)
    x, wt = torch.randn(batch, 32, 24, 24, generator=g).cuda(), torch.randn(batch, 48, 12, 12, generator=g).cuda()
    with record_plumbing() as rec:
        for _ in range(steps):
            st.set_hyper_params(1e-3)
            st.run(x, wt)
        torch.cuda.synchronize()
    return rec
