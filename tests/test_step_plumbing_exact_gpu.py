"""The per-step plumbing kernels of csrc/elementwise.cu element by element against the exact oracles of tests/plumbing_cases.py, on the
work lists that two eager train steps of YOLO-NAS-S (2 x 3 x 640 x 640, detection targets) and ResNet-50 (2 x 3 x 224 x 224) build,
and on synthetic shapes at the launch-path boundaries: the batched filter and gradient re-layouts, the QARepVGG alpha chain rule,
the deferred-shortcut scale-add-dot and the channel dot, max-pool forward / backward on every kernel (with ties, NaN and -inf),
the global average pool and the stem patch gather.  Every test prints its worst error next to its bound."""
import numpy as np
import pytest
import torch

import plumbing_cases as PC

pytestmark = pytest.mark.gpu
DEV = "cuda"
EPS = 2.0**-24


@pytest.fixture(scope="module")
def yolo_rec():
    return PC.yolo_nas_s_step_record()


@pytest.fixture(scope="module")
def resnet_rec():
    return PC.resnet50_step_record()


@pytest.fixture(scope="module")
def alpha_rec():
    return PC.qarep_alpha_step_record()


def _nhwc(x):
    return x.to(DEV).bfloat16().contiguous(memory_format=torch.channels_last)


def _unique(runs):
    seen, out = set(), []
    for r in runs:
        if id(r["entries"]) not in seen:
            seen.add(id(r["entries"]))
            out.append(r)
    return out


# ------------------------------------------------------------------------------------------------ a. filter re-layout
def _check_weight_list(entries, src):
    """Runs the list through the real table builder and kernel into sentinel-filled copies of the destination storages and compares
    every element with the oracle: written elements round(w * scale + identity), the rest untouched.  Returns (the copies as the
    re-pointed entries saw them, number of double-rounding cases)."""
    from super_gradients_b200 import kernels as K

    copies, offs, vals = {}, {}, {}

    def repoint(t):
        if t is None:
            return None
        key = t.untyped_storage().data_ptr()
        if key not in copies:
            n = t.untyped_storage().nbytes() // 2
            copies[key] = torch.full((n,), PC.SENTINEL_BITS, dtype=torch.int16, device=DEV).view(torch.bfloat16)
            offs[key], vals[key] = [], []
        return copies[key].as_strided(t.shape, t.stride(), t.storage_offset())

    new = []
    for e, (w, sc) in zip(entries, src):
        _, _, krsc, crsk, c_pad, add_identity, *extra = e
        new.append((w, sc, repoint(krsc), repoint(crsk), c_pad, add_identity, *extra))
        Kk, C, R, S = w.shape
        kp, koff, etaps, etap = extra[0] if extra else (0, 0, 0, 0)
        scv = 1.0 if sc is None else float(sc.double().cpu().reshape(-1)[0])
        for part, off, val in PC.weight_prepare_writes(w.double().cpu().numpy(), scv, Kk, C, R, S, c_pad, add_identity, crsk is not None, kp, koff, etaps, etap):
            t = krsc if part == "krsc" else crsk
            key = t.untyped_storage().data_ptr()
            offs[key].append(t.storage_offset() + off)
            vals[key].append(val)
    table = K.weight_prepare_batch(new, DEV)
    K.run_weight_prepare_batch(*table)
    torch.cuda.synchronize()
    band_cases = 0
    for key, buf in copies.items():
        got = buf.view(torch.int16).cpu().numpy()
        o = np.concatenate(offs[key])
        c = np.bincount(o, minlength=got.size)
        assert c.size == got.size, "an item writes past the end of its destination"
        e = np.zeros(got.size)
        e[o] = np.concatenate(vals[key])
        assert c.max() <= 1, "an element is written by two items"
        assert (got[c == 0] == PC.SENTINEL_BITS).all(), f"{int((got[c == 0] != PC.SENTINEL_BITS).sum())} elements outside every item were written"
        v = e[c == 1]
        want = PC.bf16_bits(PC.round_bf16(v))
        g = got[c == 1]
        bad = g != want
        if bad.any():
            gv, vb = PC.bits_to_f64(g[bad]), v[bad]
            lo, hi = PC.bf16_neighbours(vb)
            ok = PC.near_bf16_midpoint(vb) & ((gv == lo) | (gv == hi))
            assert ok.all(), f"{int((~ok).sum())} written elements differ from round_bf16(w * scale + identity), e.g. got {gv[~ok][:4]} want {vb[~ok][:4]}"
            band_cases += int(bad.sum())
    return new, band_cases


def test_weight_prepare_batch_writes_exactly_what_the_items_describe(yolo_rec, resnet_rec):
    from super_gradients_b200 import kernels as K

    for name, rec in (("yolo_nas_s", yolo_rec), ("resnet50", resnet_rec)):
        runs = _unique(rec.weight_runs)
        assert runs, f"{name}: no batched filter re-layout was recorded"
        n_items = n_band = n_elem = 0
        for run in runs:
            new, band = _check_weight_list(run["entries"], run["src"])
            n_items += len(new)
            n_band += band
            n_elem += sum(PC.weight_item_elements(w.shape[0], w.shape[1], w.shape[2], w.shape[3], e[4], e[3] is not None) for e, (w, _) in zip(run["entries"], run["src"]))
            # the single-filter kernel gives the same bytes as the batch for a filter in the plain layout
            for (w, sc, krsc, crsk, c_pad, add_identity, *extra) in new:
                if extra:
                    continue
                k1, c1 = K.weight_prepare(w, c_pad=c_pad, want_crsk=crsk is not None, scale=sc, add_identity=add_identity)
                assert torch.equal(k1.view(torch.int16), krsc.contiguous().view(torch.int16))
                if crsk is not None and c1 is not None:
                    assert torch.equal(c1.view(torch.int16), crsk.contiguous().view(torch.int16))
        print(f"{name}: {len(runs)} lists, {n_items} items, {n_elem} elements; worst error 0 outside the double-rounding band (bound: bit-equal), "
              f"{n_band} double-rounding cases (bound: either bf16 neighbour within 2^-23 of a midpoint)")
    # the YOLO-NAS step's lists hold the folded QARepVGG placements and items that start off a chunk boundary
    items = [e for run in _unique(yolo_rec.weight_runs) for e in run["entries"]]
    assert any(e[6:] and e[6][2] == 9 for e in items), "no etaps = 9 item"
    assert any(e[6:] and e[6][0] > 0 for e in items), "no kp > 0 item"
    big = max(_unique(yolo_rec.weight_runs), key=lambda r: len(r["entries"]))
    starts = np.cumsum([0] + [PC.weight_item_elements(*e[0].shape, e[4], e[3] is not None) for e in big["entries"]])[1:-1]
    assert (starts % 2048 != 0).any()


# ------------------------------------------------------------------------------------------------ b. gradient re-layout
def _gather(dw, C):
    """OIHW [K, C, R, S] from a KRSC [K, R, S, c_pad] (possibly one-tap view) gradient: g[k, c, r, s] = dw[k, r, s, c]."""
    return dw.permute(0, 3, 1, 2)[:, :C].contiguous()


def test_wgrad_to_oihw_batch_recorded_lists(yolo_rec, resnet_rec):
    one_tap = 0
    for name, rec in (("yolo_nas_s", yolo_rec), ("resnet50", resnet_rec)):
        assert rec.wgrad_runs, f"{name}: no batched gradient re-layout was recorded"
        n = 0
        for run in rec.wgrad_runs:
            mask = {k: torch.zeros(v.numel(), dtype=torch.bool, device=DEV) for k, v in run["before"].items()}
            for (dw, C, g, acc), dwc in zip(run["entries"], run["src"]):
                key = g.untyped_storage().data_ptr()
                view = lambda b: b.as_strided(g.shape, g.stride(), g.storage_offset())  # noqa: E731
                gathered = _gather(dwc, C).reshape(g.shape)  # a linear layer's slot is [K, C]: the kernel sees the same memory
                want = view(run["before"][key]) + gathered if acc else gathered
                assert torch.equal(view(run["after"][key]).view(torch.int32), want.view(torch.int32)), (name, tuple(dw.shape), C)
                mask[key].as_strided(g.shape, g.stride(), g.storage_offset()).fill_(True)
                one_tap += dw.shape[1] == dw.shape[2] == 1 and dw.stride(0) > dw.shape[3]
                n += 1
            for key, m in mask.items():  # nothing outside the slots moved
                assert torch.equal(run["after"][key][~m].view(torch.int32), run["before"][key][~m].view(torch.int32))
        print(f"{name}: {len(rec.wgrad_runs)} launches, {n} items bit-equal to g + gather(dw) (worst error 0, bound 0)")
    assert one_tap > 0, "no one-tap view with a wider row pitch in the recorded lists"


def _synthetic_wgrad_entries(g, accumulate):
    """Items of mixed sizes (none a multiple of the 2048-element chunk) including one-tap views of wider buffers."""
    out = []
    for K_, C, R, S, cp in ((64, 32, 3, 3, 32), (7, 5, 3, 3, 8), (200, 130, 1, 1, 136), (48, 24, 1, 1, 24), (3, 3, 7, 7, 8), (96, 64, 1, 1, 64)):
        if R == 1 and K_ in (200, 48):  # tap (1, 2) of a [K, 3, 3, cp] buffer: rows 9 * cp apart
            base = torch.randn(K_, 3, 3, cp, generator=g).to(DEV)
            dw = base[:, 1:2, 2:3, :]
        else:
            dw = torch.randn(K_, R, S, cp, generator=g).to(DEV)
        slot = (torch.randn(K_, C, R, S, generator=g) if accumulate else torch.full((K_, C, R, S), float("nan"))).to(DEV)
        out.append((dw, C, slot, accumulate))
    return out


@pytest.mark.parametrize("accumulate", [False, True])
def test_wgrad_to_oihw_batch_synthetic(accumulate):
    from super_gradients_b200 import kernels as K

    g = torch.Generator().manual_seed(5)
    entries = _synthetic_wgrad_entries(g, accumulate)
    before = [e[2].clone() for e in entries]
    K.run_wgrad_to_oihw_batch(*K.wgrad_to_oihw_batch_table(entries, DEV))
    torch.cuda.synchronize()
    for (dw, C, slot, _), b in zip(entries, before):
        want = b + _gather(dw, C) if accumulate else _gather(dw, C)
        assert torch.equal(slot.view(torch.int32), want.view(torch.int32)), (tuple(dw.shape), C)
    print(f"accumulate={accumulate}: {len(entries)} items bit-equal (worst error 0, bound 0)")


def test_flush_wgrads_two_gradients_on_one_slot():
    """A filter used twice in one step: the first contribution goes through the batched kernel, the second through the per-layer
    kernel after it; the slot ends as (g + dw1) + dw2."""
    from super_gradients_b200 import functional as SF

    g = torch.Generator().manual_seed(6)
    dw1, dw2 = (torch.randn(40, 3, 3, 24, generator=g).to(DEV) for _ in range(2))
    other = torch.randn(16, 1, 1, 8, generator=g).to(DEV)
    slot, slot2 = torch.randn(40, 20, 3, 3, generator=g).to(DEV), torch.randn(16, 8, 1, 1, generator=g).to(DEV)
    s0, s20 = slot.clone(), slot2.clone()
    ctx = SF.StepContext()
    ctx.pending = [(dw1, 20, slot), (other, 8, slot2), (dw2, 20, slot)]
    assert SF.flush_wgrads(ctx, DEV) == 3
    torch.cuda.synchronize()
    assert torch.equal(slot.view(torch.int32), ((s0 + _gather(dw1, 20)) + _gather(dw2, 20)).view(torch.int32))
    assert torch.equal(slot2.view(torch.int32), (s20 + _gather(other, 8)).view(torch.int32))
    print("flush_wgrads: (g + dw1) + dw2 bit-equal (worst error 0, bound 0)")


# ------------------------------------------------------------------------------------------------ c. QARepVGG alpha
def _check_alpha(before, after):
    """Worst (|err| / bound) over the g_w1 / g_bias increments and g_alpha of one item."""
    dw1, C, w1, alpha, dab, bias1, g_w1, g_bias, g_alpha = before
    a_w1, a_bias, a_alpha = after
    a = float(alpha.double().cpu().reshape(-1)[0])
    gk = dw1[:, 0, 0, :C].double().cpu().numpy()
    worst = 0.0
    pairs = [(g_w1, a_w1, gk)] + ([(g_bias, a_bias, dab.double().cpu().numpy())] if dab is not None and g_bias is not None else [])
    for b, af, gg in pairs:
        b, af = b.double().cpu().numpy().reshape(gg.shape), af.double().cpu().numpy().reshape(gg.shape)
        err = np.abs(af - (b + a * gg))
        bound = 0.5 * PC.f32_ulp(a * gg) + 0.5 * PC.f32_ulp(af)  # one rounding of the product, one of the sum
        assert (err <= bound).all(), f"g_w1 / g_bias: err {err.max():.3e}"
        worst = max(worst, float((err / np.maximum(bound, 1e-300)).max()))
    terms = [(gk * w1.double().cpu().numpy().reshape(gk.shape)).ravel()]
    if dab is not None and bias1 is not None:
        terms.append(dab.double().cpu().numpy() * bias1.double().cpu().numpy())
    t = np.concatenate(terms)
    n = t.size
    ga_b, ga_a = float(g_alpha.double().cpu().reshape(-1)[0]), float(a_alpha.double().cpu().reshape(-1)[0])
    err = abs(ga_a - (ga_b + t.sum()))
    bound = (-(-n // 256) + 9) * EPS * np.abs(t).sum() + float(PC.f32_ulp(ga_a))
    assert err <= bound, f"g_alpha: err {err:.3e} bound {bound:.3e} (n = {n})"
    return max(worst, err / bound)


def test_qarep_alpha_finish_recorded_lists(alpha_rec):
    assert alpha_rec.alpha_runs, "no QARepVGG alpha launch was recorded"
    assert any(b[4] is None for run in alpha_rec.alpha_runs for b in run["before"]) and any(b[4] is not None for run in alpha_rec.alpha_runs for b in run["before"])
    worst, n = 0.0, 0
    for run in alpha_rec.alpha_runs:
        for b, a in zip(run["before"], run["after"]):
            worst = max(worst, _check_alpha(b, a))
            n += 1
    print(f"{len(alpha_rec.alpha_runs)} launches, {n} blocks: worst |err| / bound {worst:.3f} (bound 1)")


def test_qarep_alpha_finish_synthetic():
    from super_gradients_b200 import kernels as K

    g = torch.Generator().manual_seed(7)
    entries = []
    for Kk, C, cp, with_bias in ((48, 40, 48, True), (130, 96, 96, False), (8, 300, 304, True)):
        base = torch.randn(Kk, 3, 3, cp, generator=g).to(DEV)
        dw1 = base[:, 1:2, 1:2, :]  # the centre tap of the folded filter's gradient: rows 9 * cp apart
        r = lambda *s: torch.randn(*s, generator=g).to(DEV)  # noqa: E731
        entries.append((dw1, C, r(Kk, C, 1, 1), torch.tensor([0.37]).to(DEV), r(Kk) if with_bias else None, r(Kk) if with_bias else None,
                        r(Kk, C, 1, 1), r(Kk) if with_bias else None, r(1)))  # fmt: skip
    before = [tuple(t.clone() if torch.is_tensor(t) else t for t in e) for e in entries]
    K.run_qarep_alpha_finish(*K.qarep_alpha_finish_table(entries, DEV))
    torch.cuda.synchronize()
    worst = max(_check_alpha(b, (e[6], e[7], e[8])) for b, e in zip(before, entries))
    print(f"synthetic blocks with / without a bias: worst |err| / bound {worst:.3f} (bound 1)")


# ------------------------------------------------------------------------------------------------ d / e. max-pool
def _pool_inputs(kind, N, C, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    if kind == "randn":
        return torch.randn(N, C, H, W, generator=g)
    if kind == "ties":
        return torch.randint(-3, 4, (N, C, H, W), generator=g).float().relu()
    if kind == "const":
        return torch.full((N, C, H, W), 0.75)
    x = torch.randn(N, C, H, W, generator=g)
    if kind == "nan":
        x[torch.rand(x.shape, generator=g) < 0.05] = float("nan")
        x[:, 0, :3, :3] = float("nan")  # all-NaN border windows
        x[:, 1] = float("nan")
    elif kind == "ninf":
        x[:, 0, :4, :4] = -float("inf")
        x[:, 2, -3:, :] = -float("inf")
        x[:, 3] = -float("inf")
    return x


def _check_fwd(x, y, idx, k, stride, pad):
    """The kernel's values and arg-max taps against torch CPU max_pool2d; returns (torch's flat indices, number of outputs)."""
    ref, taps, flat = PC.torch_maxpool_taps(x, k, stride, pad)
    yc = y.detach().cpu()
    assert torch.equal(yc.isnan(), ref.isnan()), "NaN outputs differ from torch"
    fin = ~ref.isnan()
    assert torch.equal(yc[fin].view(torch.int16), ref.bfloat16()[fin].view(torch.int16)), "max-pool values are not bit-equal to torch"
    assert torch.equal(idx.permute(0, 3, 1, 2).long().cpu(), taps), "arg-max taps differ from torch's indices"
    return flat, ref.numel()


def _check_bwd(dx, dy, flat, x_shape, stride):
    s64, n, a = PC.maxpool_bwd_oracle(dy, flat, x_shape)
    d = dx.detach().double().cpu()
    assert (d[n == 0] == 0).all(), "gradient routed to an element torch routes nothing to"
    if dx.dtype == torch.float32:  # scatter: fp32 atomics in any order
        err, bound = (d - s64).abs(), n * EPS * a
        assert bool((err <= bound).all()), f"scatter max-pool backward: err {float((err - bound).max()):.3e} over the bound"
        return float((err / bound.clamp_min(1e-300))[n > 0].max()) if bool((n > 0).any()) else 0.0
    lo, hi = PC.bf16_neighbours(s64.numpy())  # gather: one bf16 rounding of the exact sum
    dn = d.numpy()
    assert ((dn == lo) | (dn == hi)).all(), "gather max-pool backward is not a bf16 neighbour of the exact sum"
    return float((np.abs(dn - s64.numpy()) / np.maximum(PC.bf16_ulp(s64.numpy()), 1e-300)).max())


def _run_pool(xcpu, k, stride, pad, x_slice=None, out_slice=None, seed=0):
    """Max-pool forward / backward of xcpu [N, C, H, W] through the kernels, with optional channel offsets of wider input / output
    buffers (x_slice / out_slice: (offset, total channels)); returns (worst backward error over bound, outputs checked)."""
    from super_gradients_b200 import kernels as K

    N, C, H, W = xcpu.shape
    if x_slice:
        buf = torch.randn(N, x_slice[1], H, W)
        buf[:, x_slice[0] : x_slice[0] + C] = xcpu
        x = _nhwc(buf)[:, x_slice[0] : x_slice[0] + C]
    else:
        x = _nhwc(xcpu)
    P, Q = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    out, obuf = None, None
    if out_slice:
        obuf = torch.full((N, P, Q, out_slice[1]), PC.SENTINEL_BITS, dtype=torch.int16, device=DEV).view(torch.bfloat16).permute(0, 3, 1, 2)
        out = obuf[:, out_slice[0] : out_slice[0] + C]
    y, idx = K.maxpool_fwd(x, k, stride, pad, out=out)
    torch.cuda.synchronize()
    flat, n_out = _check_fwd(xcpu.bfloat16().float(), y, idx, k, stride, pad)
    if obuf is not None:
        rest = torch.cat([obuf[:, : out_slice[0]], obuf[:, out_slice[0] + C :]], 1)
        assert bool((rest.contiguous().view(torch.int16) == PC.SENTINEL_BITS).all()), "max-pool wrote outside its output slice"
    dy = torch.randn(N, C, P, Q, generator=torch.Generator().manual_seed(seed + 1)).bfloat16()
    dx = K.maxpool_bwd(_nhwc(dy), idx, (N, C, H, W), k, stride, pad)
    torch.cuda.synchronize()
    return _check_bwd(dx, dy, flat, (N, C, H, W), stride), n_out


KINDS = ["randn", "ties", "const", "nan", "ninf"]
POOL_CASES = [  # (k, stride, H, W, C): the shared-memory kernel (SPP), the direct stride-1 kernel (plane over 96 KB), stride 2 (ResNet)
    (5, 1, 20, 20, 32), (9, 1, 20, 20, 16), (13, 1, 20, 20, 16), (5, 1, 40, 40, 16), (13, 1, 40, 40, 16),
    (5, 1, 80, 80, 16), (3, 1, 81, 80, 8),
    (3, 2, 112, 112, 64), (3, 2, 57, 57, 16),
]  # fmt: skip


@pytest.mark.parametrize("kind", KINDS)
def test_maxpool_matches_torch(kind):
    worst, n = 0.0, 0
    for i, (k, stride, H, W, C) in enumerate(POOL_CASES):
        x = _pool_inputs(kind, 2, C, H, W, seed=10 * i)
        e, m = _run_pool(x, k, stride, k // 2, seed=i)
        worst, n = max(worst, e), n + m
    # channel slices of wider input / output buffers, on each kernel
    for i, (k, stride, H, W) in enumerate(((5, 1, 20, 20), (5, 1, 80, 80), (3, 2, 57, 57))):
        x = _pool_inputs(kind, 2, 16, H, W, seed=100 + i)
        e, m = _run_pool(x, k, stride, k // 2, x_slice=(16, 48), out_slice=(8, 40), seed=100 + i)
        worst, n = max(worst, e), n + m
    print(f"{kind}: {n} outputs, values and arg-max bit-equal to torch (bound: equal); backward worst err / bound {worst:.3f} (bound 1)")


def test_maxpool_recorded_calls(yolo_rec, resnet_rec):
    n_f = n_b = 0
    worst = 0.0
    for name, rec in (("yolo_nas_s", yolo_rec), ("resnet50", resnet_rec)):
        assert rec.maxpool_fwd and rec.maxpool_bwd, f"{name}: no max-pool launch recorded"
        for f in rec.maxpool_fwd:
            _check_fwd(f["x"].float(), f["y"], f["idx"], f["k"], f["stride"], f["pad"])
            n_f += 1
        for b in rec.maxpool_bwd:
            f = b["fwd"]
            _, _, flat = PC.torch_maxpool_taps(f["x"].float(), f["k"], f["stride"], f["pad"])
            worst = max(worst, _check_bwd(b["dx"], b["dy"], flat, b["x_shape"], b["stride"]))
            n_b += 1
    assert {f["stride"] for f in yolo_rec.maxpool_fwd} == {1} and {f["stride"] for f in resnet_rec.maxpool_fwd} == {2}
    print(f"{n_f} recorded forwards bit-equal to torch, {n_b} backwards: worst err / bound {worst:.3f} (bound 1)")


# ------------------------------------------------------------------------------------------------ f. scale-add-dot, channel dot
def _rows(t):
    """[N, C, H, W] -> fp64 [pixels, C] ndarray."""
    return t.double().cpu().permute(0, 2, 3, 1).reshape(-1, t.shape[1]).numpy()


def _check_dot(u, xd, dot):
    """fp64 sum over pixels of u * xd within the chan_reduce bound; returns the worst err / bound."""
    M, C = u.shape
    p = u * _rows(xd)
    s, sa = p.sum(0), np.abs(p).sum(0)
    err, bound = np.abs(dot.double().cpu().numpy() - s), PC.chan_reduce_terms_bound(M, C) * EPS * sa + 1e-300
    assert (err <= bound).all(), f"dot: err {err.max():.3e} over the bound (M {M}, C {C})"
    return float((err / bound).max())


def _check_sad(x1, a, xd, x2, y, dot):
    """y within 1 bf16 ulp of round_bf16(a * x1 + x2); dot within the chan_reduce bound.  Returns (worst y err in ulps, worst dot
    err / bound)."""
    av = float(a.double().cpu().reshape(-1)[0])
    u = _rows(x1)
    r = PC.round_bf16(av * u + (_rows(x2) if x2 is not None else 0.0))
    ulps = np.abs(_rows(y) - r) / PC.bf16_ulp(r)
    assert (ulps <= 1).all(), f"y: {ulps.max():.2f} bf16 ulp from round_bf16(a * x1 + x2)"
    return float(ulps.max()), _check_dot(u, xd, dot)


SAD_SHAPES = [(2, 200, 40, 40), (2, 2048, 8, 8), (1, 4096, 16, 16), (1, 200, 1, 1), (1, 200, 1, 7), (1, 2048, 1, 1), (4, 64, 80, 80)]


@pytest.mark.parametrize("shape", SAD_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_scale_add_dot_and_channel_dot(shape):
    from super_gradients_b200 import kernels as K

    g = torch.Generator().manual_seed(sum(shape))
    x1, xd, x2 = (_nhwc(torch.randn(*shape, generator=g)) for _ in range(3))
    a = torch.tensor([-0.73]).to(DEV)
    y, dot = K.scale_add_dot(x1, a, xd, x2)
    y0, dot0 = K.scale_add_dot(x1, a, xd)  # no x2
    x2c = x2.clone()
    yi, doti = K.scale_add_dot(x1, a, xd, x2c, out=x2c)  # in place
    cd = K.channel_dot(x1, xd)
    torch.cuda.synchronize()
    w1 = _check_sad(x1, a, xd, x2, y, dot)
    w2 = _check_sad(x1, a, xd, None, y0, dot0)
    assert torch.equal(yi.view(torch.int16), y.view(torch.int16)) and torch.equal(doti, dot), "in-place result differs from out-of-place"
    w3 = _check_dot(_rows(x1), xd, cd)
    print(f"{shape}: y worst {max(w1[0], w2[0]):.2f} bf16 ulp (bound 1); dot worst err / bound {max(w1[1], w2[1]):.3f}, channel_dot {w3:.3f} (bound 1)")


def test_scale_add_dot_recorded_calls(yolo_rec):
    assert yolo_rec.scale_add_dot, "no deferred-shortcut launch recorded"
    wy = wd = 0.0
    for r in yolo_rec.scale_add_dot:
        e = _check_sad(r["x1"], r["a"], r["xd"], r["x2"], r["y"], r["dot"])
        wy, wd = max(wy, e[0]), max(wd, e[1])
    assert any(r["in_place"] for r in yolo_rec.scale_add_dot)
    print(f"{len(yolo_rec.scale_add_dot)} recorded calls: y worst {wy:.2f} bf16 ulp (bound 1), dot worst err / bound {wd:.3f} (bound 1)")


# ------------------------------------------------------------------------------------------------ g. average pool
@pytest.mark.parametrize("shape", [(256, 2048, 7, 7), (3, 12, 1, 1), (3, 12, 7, 7)], ids=lambda s: "x".join(map(str, s)))
def test_avgpool(shape):
    from super_gradients_b200 import kernels as K

    N, C, H, W = shape
    HW = H * W
    g = torch.Generator().manual_seed(HW + C)
    xc = torch.randn(*shape, generator=g).bfloat16()
    y = K.avgpool_fwd(_nhwc(xc))
    dyc = torch.randn(N, C, 1, 1, generator=g).bfloat16()
    dx = K.avgpool_bwd(_nhwc(dyc), (H, W))
    torch.cuda.synchronize()
    x64 = xc.double()
    m = x64.mean((2, 3)).numpy()
    e32 = (HW + 1) * EPS * x64.abs().mean((2, 3)).numpy()  # fp32 running sum of HW terms and the division
    err = np.abs(y.double().cpu().reshape(N, C).numpy() - m)
    bound = 0.5 * PC.bf16_ulp(np.abs(m) + e32) + e32
    assert (err <= bound).all(), f"forward: err {err.max():.3e} over the bound"
    want = (dyc.float() / HW).bfloat16().expand(N, C, H, W)
    assert torch.equal(dx.cpu().view(torch.int16), want.contiguous().view(torch.int16))
    print(f"{shape}: forward worst err / bound {float((err / bound).max()):.3f} (bound 1); backward bit-equal")


# ------------------------------------------------------------------------------------------------ h. stem patches
@pytest.mark.parametrize("shape,R,stride,pad,c_out", [
    ((2, 3, 640, 640), 3, 2, 1, 32),  # YOLO-NAS: the c3r3s2 kernel
    ((2, 3, 65, 96), 3, 2, 1, 32),    # odd H: the generic kernel
    ((1, 3, 64, 81), 3, 2, 1, 32),    # odd W
    ((2, 3, 224, 224), 7, 2, 3, 160), # ResNet's 7 x 7 / 2 / 3 stem
    ((2, 3, 201, 173), 7, 2, 3, 160),
], ids=["yolo640", "oddH", "oddW", "resnet224", "resnet201x173"])  # fmt: skip
def test_stem_patches(shape, R, stride, pad, c_out):
    from super_gradients_b200 import kernels as K

    x = torch.randn(*shape, generator=torch.Generator().manual_seed(R * shape[2]))
    y = K.stem_patches(x.to(DEV), R, stride, pad, c_out)
    torch.cuda.synchronize()
    want = PC.stem_patches_oracle(x, R, stride, pad, c_out)
    assert torch.equal(y.cpu().view(torch.int16), want.view(torch.int16))
    print(f"{shape} R{R}/s{stride}/p{pad} -> {c_out} channels: bit-equal to F.unfold (worst error 0, bound 0)")
