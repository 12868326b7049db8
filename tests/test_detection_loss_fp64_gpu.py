"""The PP-YOLOE / YOLO-NAS loss and head-decode kernels (csrc/loss.cu, csrc/focal_cls.cu) element by element against float64.

Gradients are bounded per anchor row (one anchor's 4 * (reg_max + 1) bins, or its ncls classes), never by the largest value of the
whole tensor:  |g - g64| <= r |g64| + a max_row |g64| with r = a = 1e-4 (detection_loss_cases.row_errors).  Each test prints the
worst error it saw, relative to the row maximum and relative to the element itself.

Assignment decisions (labels, assigned gt) must equal those of the fp32 oracle with the kernel's top-k order; a decision that
differs is accepted only as a near-tie of the competing fp64 metrics or IoUs (<= 1e-6 relative), and is counted and printed."""
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import detection_loss_cases as DC  # noqa: E402
from oracle import sg_oracle as O  # noqa: E402

DEV = "cuda"


def K():
    from super_gradients_b200 import kernels

    return kernels


def _loss(c, iou_type, focal_alpha, grad_scale=1.0, want_grad=True):
    """dfl_iou_loss on a given assignment; sums[3] (the normaliser the assigner accumulates) is set to sum(asc)."""
    k = K()
    B, Lc, C = c["cls"].shape
    d = k.loss_desc(B, Lc, C, c["reg_max"], 1, iou_type=iou_type)
    sums = torch.zeros(4, dtype=torch.float64, device=DEV)
    sums[3] = c["asc"].double().sum()
    dev = {n: c[n].to(DEV).contiguous() for n in ("cls", "reg", "ap", "st", "al", "ab", "asc")}
    items, gc, gr = k.dfl_iou_loss(d, dev["cls"], dev["reg"], dev["ap"], dev["st"], dev["al"], dev["ab"], dev["asc"], sums, grad_scale, want_grad, focal_alpha)
    torch.cuda.synchronize()
    return items.cpu(), None if gc is None else gc.cpu(), None if gr is None else gr.cpu()


def _check_loss(tag, items, gc, gr, i64, gc64, gr64, r=1e-4, a=1e-4):
    item_err = float(((items.double() - i64).abs() / i64.abs().clamp_min(1e-30)).max())
    ok_c, row_c, rel_c = DC.row_errors(gc, gc64, r, a)
    ok_r, row_r, rel_r = DC.row_errors(gr, gr64, r, a)
    print(f"{tag}: items rel {item_err:.2e} | cls row {row_c:.2e} elem {rel_c:.2e} | reg row {row_r:.2e} elem {rel_r:.2e}")
    assert bool((items.double() - i64).abs().le(r * i64.abs() + 1e-6 * float(i64[3].abs())).all()), (items, i64)
    assert ok_c, f"cls gradient outside the per-row bound: {row_c:.3e}"
    assert ok_r, f"reg gradient outside the per-row bound: {row_r:.3e}"


# ------------------------------------------------------------------------------------------------ a. loss on constructed assignments
@pytest.mark.parametrize("ncls,reg_max,norm_above_1", [(1, 7, False), (80, 16, True), (365, 31, True)])
@pytest.mark.parametrize("focal_alpha", [None, -1.0, 0.25])
@pytest.mark.parametrize("iou_type", [0, 1])
def test_loss_on_constructed_assignments(iou_type, focal_alpha, ncls, reg_max, norm_above_1):
    """Every branch of loss_kernel (box inside / enclosing / crossing one side / disjoint, CIoU extreme aspect ratios, v ~ 0, iou -> 1,
    DFL targets negative / on a bin / below reg_max - 0.01 / above reg_max, saturated logits, asc = 0 positives), varifocal or focal
    classification, normaliser below or above 1.  grad_scale = 0.5 halves every gradient bit for bit; want_grad = False gives the
    same items."""
    c = DC.constructed_case(ncls, reg_max, seed=ncls + reg_max, norm_above_1=norm_above_1)
    assert (float(c["asc"].sum()) > 1) == norm_above_1
    i64, gc64, gr64 = DC.loss_given_assignment(c["cls"], c["reg"], c["ap"], c["st"], c["al"], c["ab"], c["asc"], ncls, reg_max, iou_type=iou_type, focal_alpha=focal_alpha)
    items, gc, gr = _loss(c, iou_type, focal_alpha)
    _check_loss(f"constructed iou_type={iou_type} focal={focal_alpha} ncls={ncls} reg_max={reg_max}", items, gc, gr, i64, gc64, gr64)
    items_h, gc_h, gr_h = _loss(c, iou_type, focal_alpha, grad_scale=0.5)
    assert torch.equal(2 * gc_h, gc) and torch.equal(2 * gr_h, gr)
    torch.testing.assert_close(items_h, items, rtol=1e-6, atol=0)
    items_n, gc_n, gr_n = _loss(c, iou_type, focal_alpha, want_grad=False)
    assert gc_n is None and gr_n is None
    torch.testing.assert_close(items_n, items, rtol=1e-6, atol=0)


def test_coincident_boxes_pin_the_tie_convention():
    """At exact coordinate ties (predicted box == gt box) the kernel's strict comparisons give the predicted coordinate no share of
    min / max: the CIoU gradient equals the fp64 restatement's with min / max taking the gt operand, and differs from the one with
    torch's own min / max, which split the gradient between equal operands.  (GIoU's gradient there is 0 under either convention:
    its IoU and enclosing-area terms cancel.)"""
    c = DC.coincident_case()
    items, gc, gr = _loss(c, 1, None)
    with DC.strict_minmax():
        i64, gc64, gr64 = DC.loss_given_assignment(c["cls"], c["reg"], c["ap"], c["st"], c["al"], c["ab"], c["asc"], 3, 16, iou_type=1)
    _check_loss("coincident boxes, CIoU", items, gc, gr, i64, gc64, gr64)
    _, _, gr_split = DC.loss_given_assignment(c["cls"], c["reg"], c["ap"], c["st"], c["al"], c["ab"], c["asc"], 3, 16, iou_type=1)
    assert not DC.row_errors(gr, gr_split)[0]


# ------------------------------------------------------------------------------------------------ b / c. assignment
def _assign(c, topk, alpha, beta):
    k = K()
    B = c["cls"].shape[0]
    n_max = c["n"]
    d = k.loss_desc(B, c["L"], c["ncls"], c["reg_max"], n_max, topk=topk, alpha=alpha, beta=beta)
    sums = torch.zeros(4, dtype=torch.float64, device=DEV)
    al, ab, asc = k.tal_assign(d, c["cls"].to(DEV), c["reg"].to(DEV), c["ap"].to(DEV), c["st"].to(DEV), c["gb"].to(DEV), c["gl"].to(DEV), c["gv"].to(DEV), sums)
    return al.cpu().long(), ab.cpu(), asc.cpu(), float(sums[3])


def _check_assignment(c, topk, alpha, beta, tag, exact=False):
    """exact: the metrics tie exactly in both implementations, so the documented order alone decides and no difference is allowed."""
    al, ab, asc, nrm = _assign(c, topk, alpha, beta)
    B, ncls = c["cls"].shape[0], c["ncls"]
    pbox = DC.decode_fp32(c["reg"], c["ap"], c["st"])
    ties, unexplained, worst_asc, npos = [], [], 0.0, 0
    for b in range(B):
        gb, gl, gv = c["gb"][b], c["gl"][b], c["gv"][b]
        lab_o, g_o = DC.tal_assign_stable(c["cls"][b], pbox[b], c["ap"], gb, gl, gv, ncls, topk, alpha, beta)
        g_k = DC.kernel_gt_index(al[b], ab[b], gb, gl, ncls)
        assert bool(((al[b] == ncls) | (g_k >= 0)).all()), "an assigned label / box pair that is no gt row"
        differ = (lab_o != al[b]) | (g_o != g_k)
        for l in differ.nonzero().flatten().tolist():
            why = None if exact else DC.explain_difference(l, int(g_k[l]), int(g_o[l]), c["cls"][b], pbox[b], c["ap"], gb, gl, topk, alpha, beta)
            (ties if why else unexplained).append((b, l, int(g_k[l]), int(g_o[l]), why))
        # c. continuous outputs on the kernel's own assignment
        assert torch.equal(ab[b], gb[g_k.clamp_min(0)]), "assigned boxes are not copies of the assigned (or, unassigned: the first) gt row"
        asc64 = DC.assigned_scores_fp64(c["cls"][b], pbox[b], gb, gl, g_k, alpha, beta)
        err = (asc[b].double() - asc64).abs()
        scale = float(asc64.abs().max()) if bool((asc64 != 0).any()) else 1.0
        assert bool((err <= 1e-5 * asc64.abs() + 1e-6 * scale).all()), float(err.max())
        assert bool((asc[b][g_k < 0] == 0).all())
        worst_asc = max(worst_asc, float((err / (asc64.abs() + 1e-6 * scale)).max()))
        npos += int((g_k >= 0).sum())
    assert abs(nrm - float(asc.double().sum())) <= 1e-6 * max(nrm, 1.0)
    print(f"{tag}: {npos} positives, {len(ties)} near-tie differences, asc worst rel {worst_asc:.2e}" + "".join(f"\n  image {t[0]} anchor {t[1]}: kernel gt {t[2]}, oracle gt {t[3]}: {t[4]}" for t in ties[:10]))
    assert not unexplained, f"{len(unexplained)} assignment decisions differ without a near-tie: {unexplained[:5]}"
    return npos


@pytest.mark.parametrize("beta", [6.0, 2.0])
@pytest.mark.parametrize("alpha", [1.0, 0.5])
@pytest.mark.parametrize("topk", [1, 13, 64])
def test_tal_decisions_parameter_sweep(topk, alpha, beta):
    """150 crowded gts (duplicates, nested, sub-cell, whole-image, border-crossing, invalid rows between valid ones) on 640 x 384."""
    c = DC.decision_case(1, 384, 640, 150, seed=topk * 7 + int(alpha * 2) + int(beta), n_invalid=6)
    assert _check_assignment(c, topk, alpha, beta, f"640x384 topk={topk} alpha={alpha} beta={beta}") > 0


@pytest.mark.parametrize("B,H,W,n,topk", [(8, 640, 640, 120, 13), (8, 384, 640, 200, 64), (2, 480, 1248, 150, 13), (1, 1024, 1024, 200, 13), (8, 1024, 1024, 100, 64)])
def test_tal_decisions_image_sizes(B, H, W, n, topk):
    """L = 8400 (640^2), 5040 (640 x 384), 12285 (1248 x 480: a 49140 B row, under 48 KB alone but not with the kernel's static
    shared memory) and 21504 (1024^2: the top-k metric row takes 84 KB of shared memory, above 48 KB)."""
    c = DC.decision_case(B, H, W, n, seed=B + H + n, n_invalid=4)
    assert _check_assignment(c, topk, 1.0, 6.0, f"B={B} {W}x{H} n={n} topk={topk}") > 0


@pytest.mark.parametrize("beta", [6.0, 2.0])
@pytest.mark.parametrize("alpha", [1.0, 0.5])
@pytest.mark.parametrize("topk", [1, 13, 64])
def test_tal_decisions_at_exact_metric_ties(topk, alpha, beta):
    """Many anchors inside a gt with exactly equal metrics: the top-k takes the lowest anchor indices first, as the stable oracle
    does (the highest-index order changes about one positive in seven here), and no difference is excused."""
    c = DC.decision_case(2, 640, 640, 60, seed=topk, n_invalid=2, exact_ties=True)
    assert _check_assignment(c, topk, alpha, beta, f"exact ties 640x640 topk={topk} alpha={alpha} beta={beta}", exact=True) > 0


@pytest.mark.parametrize("case", ["n_max_0", "all_invalid"])
def test_tal_without_valid_gts(case):
    """n_max = 0 and a batch whose gt rows are all invalid: every anchor is background with score 0 (box: gt row 0, as the reference
    gathers it), the normaliser stays 0, and the loss has no box terms."""
    c = DC.decision_case(2, 256, 256, 0 if case == "n_max_0" else 5)
    if case == "all_invalid":
        c["gv"].zero_()
    al, ab, asc, nrm = _assign(c, 13, 1.0, 6.0)
    assert bool((al == c["ncls"]).all()) and bool((asc == 0).all()) and nrm == 0.0
    assert torch.equal(ab, c["gb"][:, :1].expand_as(ab)) if case == "all_invalid" else bool((ab == 0).all())
    c.update(al=al.int(), ab=ab, asc=asc)
    i64, gc64, gr64 = DC.loss_given_assignment(c["cls"], c["reg"], c["ap"], c["st"], al, ab, asc, c["ncls"], c["reg_max"])
    items, gc, gr = _loss(c, 0, None)
    assert float(items[1]) == 0.0 and float(items[2]) == 0.0 and bool((gr == 0).all())
    _check_loss(f"no valid gts ({case})", items, gc, torch.zeros(1, 1), i64, gc64, torch.zeros(1, 1))


# ------------------------------------------------------------------------------------------------ d. end to end
@pytest.mark.parametrize("iou_type", [0, 1])
def test_end_to_end_config2_crowded(iou_type):
    """tal_assign + dfl_iou_loss at the config-2 anchor set (B = 8, 640^2, C = 80) with 150 crowded gts per image and random reg
    logits (kept off the gt corners' 1/2 px grid, where fp32 would round a corner pair to an exact tie), against the fp64 loss on
    the kernel's own assignment."""
    g = torch.Generator().manual_seed(40 + iou_type)
    c = DC.decision_case(8, 640, 640, 150, seed=40 + iou_type, n_invalid=5)
    c["reg"] = DC.off_grid_reg(torch.randn(c["reg"].shape, generator=g) * 1.5, c["ap"], c["st"], g)
    al, ab, asc, _ = _assign(c, 13, 1.0, 6.0)
    assert int((al != 80).sum()) > 3000
    c.update(al=al.int(), ab=ab, asc=asc)
    i64, gc64, gr64 = DC.loss_given_assignment(c["cls"], c["reg"], c["ap"], c["st"], al, ab, asc, 80, 16, iou_type=iou_type)
    items, gc, gr = _loss(c, iou_type, None)
    _check_loss(f"end to end config 2 iou_type={iou_type}", items, gc, gr, i64, gc64, gr64)


# ------------------------------------------------------------------------------------------------ e. head kernels
def _nhwc(x, pitch=None, off=0):
    """CPU NCHW fp32 -> CUDA NHWC bf16 view, a channel slice at `off` of a buffer with channel pitch `pitch`."""
    n, c, h, w = x.shape
    pitch = pitch or ((c + 7) // 8) * 8
    buf = torch.zeros(n, pitch, h, w, dtype=torch.bfloat16, device=DEV).contiguous(memory_format=torch.channels_last)
    view = buf[:, off : off + c]
    view.copy_(x.to(DEV))
    return view


# (ncls, reg_max, reg pitch, reg channel offset, Hf, Wf, anchor_base, cell_offset, optional outputs); the host serves the tile kernel
# when both pitches are multiples of 8 covering the 16-byte rounded rows, both bases are 16-byte aligned and the tile fits 48 KB
DECODE_CASES = [
    (80, 16, None, 0, 9, 7, 37, 0.5, True),  # tile
    (1, 7, None, 0, 13, 11, 0, 0.0, False),  # tile
    (80, 31, None, 0, 5, 13, 5, 0.5, True),  # tile
    (365, 16, None, 0, 9, 7, 11, 0.5, True),  # generic: 365 classes need a 56 KB tile
    (80, 16, 68, 0, 7, 9, 3, 0.0, False),  # generic: pitch 68
    (80, 16, 80, 4, 9, 7, 20, 0.5, True),  # generic: channel slice 8 bytes into the row
    (365, 31, None, 0, 3, 21, 1, 0.0, False),  # generic
    (17, 7, 40, 8, 11, 6, 2, 0.5, True),  # tile: a 16-byte aligned channel slice
]


@pytest.mark.parametrize("ncls,reg_max,rpitch,roff,Hf,Wf,base,cell,opts", DECODE_CASES)
def test_dfl_decode(ncls, reg_max, rpitch, roff, Hf, Wf, base, cell, opts):
    k = K()
    g = torch.Generator().manual_seed(ncls + reg_max + Hf)
    B, s, HW = 2, 16.0, Hf * Wf
    nb = reg_max + 1
    Lt = base + HW + 5
    reg = (torch.randn(B, 4 * nb, Hf, Wf, generator=g) * 2).bfloat16().float()
    cls = (torch.randn(B, ncls, Hf, Wf, generator=g) * 3).bfloat16().float()
    (pb64, ps64), raw = O.ndfl_decode([reg.double()], [cls.double()], [s], reg_max=reg_max, cell_offset=cell)
    nan = lambda *shape: torch.full(shape, float("nan"), device=DEV)  # noqa: E731
    pb, ps = nan(B, Lt, 4), nan(B, Lt, ncls)
    cl, rd = (nan(B, Lt, ncls), nan(B, Lt, 4 * nb)) if opts else (None, None)
    k.dfl_decode(_nhwc(reg, rpitch, roff), _nhwc(cls), Lt, base, ncls, reg_max, s, cell, pb, ps, cl, rd)
    rows = slice(base, base + HW)
    outside = torch.ones(Lt, dtype=torch.bool)
    outside[rows] = False
    for t in (pb, ps) + ((cl, rd) if opts else ()):
        t = t.cpu()
        assert bool(t[:, outside].isnan().all()), "rows outside [anchor_base, anchor_base + HW) were written"
    err_b = (pb.cpu()[:, rows].double() - pb64).abs()
    bound_b = 4e-7 * s * (max(Hf, Wf) + nb)  # a few fp32 ulp of (grid + distance) * stride
    print(f"dfl_decode ncls={ncls} reg_max={reg_max}: box err {float(err_b.max()) / bound_b:.2f} of bound, score rel {float(((ps.cpu()[:, rows].double() - ps64).abs() / ps64).max()):.2e}")
    assert float(err_b.max()) <= bound_b
    torch.testing.assert_close(ps.cpu()[:, rows].double(), ps64, rtol=1e-6, atol=0)
    if opts:
        assert torch.equal(cl.cpu()[:, rows], raw[0].float()) and torch.equal(rd.cpu()[:, rows], raw[1].float())


@pytest.mark.parametrize("logit_off", [0, 1])
@pytest.mark.parametrize("compensate", [True, False])
@pytest.mark.parametrize("mult", [1.0, 2.0])
@pytest.mark.parametrize("J", [1, 17])
def test_pose_keypoint_decode(J, mult, compensate, logit_off):
    k = K()
    g = torch.Generator().manual_seed(J * 4 + int(mult) * 2 + int(compensate))
    B, Hf, Wf, s, base, cell = 2, 7, 9, 32.0, 19, 0.5
    HW, Lt = Hf * Wf, 19 + 63 + 3
    pose = (torch.randn(B, 2 * J, Hf, Wf, generator=g) * 3).bfloat16().float()
    logit = (torch.randn(B, logit_off + J, Hf, Wf, generator=g) * 3).bfloat16().float()
    decoded, raw = O.pose_ndfl_decode([torch.zeros(B, 68, Hf, Wf, dtype=torch.float64)], [torch.zeros(B, 1, Hf, Wf, dtype=torch.float64)], [pose.double().reshape(B, J, 2, Hf, Wf)],
                                      [logit[:, logit_off:].double()], [s], cell_offset=cell, pose_offset_multiplier=mult, compensate_grid_cell_offset=compensate)  # fmt: skip
    pc, pj, pl = (torch.full(sh, float("nan"), device=DEV) for sh in ((B, Lt, J, 2), (B, Lt, J), (B, Lt, J)))
    k.pose_keypoint_decode(_nhwc(pose), _nhwc(logit), logit_off, Lt, base, J, s, cell, mult, compensate, pc, pj, pl)
    rows = slice(base, base + HW)
    pc, pj, pl = pc.cpu(), pj.cpu(), pl.cpu()
    assert bool(pc[:, :base].isnan().all() and pc[:, base + HW :].isnan().all() and pj[:, :base].isnan().all() and pl[:, base + HW :].isnan().all())
    err = float((pc[:, rows].double() - decoded[2]).abs().max())
    bound = 4e-7 * s * (max(Hf, Wf) + 3 * 4 * mult)
    print(f"pose_keypoint_decode J={J} mult={mult} compensate={compensate} logit_off={logit_off}: coord err {err / bound:.2f} of bound")
    assert err <= bound
    torch.testing.assert_close(pj[:, rows].double(), decoded[3], rtol=1e-6, atol=0)
    assert torch.equal(pl[:, rows], raw[3].float())


@pytest.mark.parametrize("path", ["v8", "generic"])
@pytest.mark.parametrize("gC", [1, 17, 18, 34, 68, 80, 365])
def test_head_grad_scatter(gC, path):
    """fp32 [B, L, gC] rows [anchor_base, anchor_base + HW) -> bf16 NHWC map, bit-exact with .bfloat16() (round to nearest even, ties
    included).  v8: 16-byte aligned source and map, pitch = gC rounded up to 8, plus 8 channels the kernel must not touch;
    generic: a source 4 bytes off 16-byte alignment, pitch = gC.  Pad channels up to the next multiple of 8 (inside the pitch) are
    zero; nothing past the map is written."""
    k = K()
    g = torch.Generator().manual_seed(gC)
    B, H, W, base = 2, 5, 7, 13
    HW, Lt = H * W, 13 + 35 + 9
    src = torch.randn(B, Lt, gC, generator=g) * 10.0 ** torch.randint(-6, 6, (B, Lt, gC), generator=g).float()
    src.view(-1)[::7] = 1.0 + 2.0**-8  # halfway between two bf16 values: ties round to even
    src.view(-1)[3::7] = 1.0 + 3 * 2.0**-8
    pitch = ((gC + 7) // 8) * 8 + 8 if path == "v8" else gC
    cpad = min(((gC + 7) // 8) * 8, pitch)
    sentinel = -7.5
    buf = torch.full((B * HW * pitch + 64,), sentinel, dtype=torch.bfloat16, device=DEV)
    dy = buf[: B * HW * pitch].view(B, H, W, pitch)[..., :gC].permute(0, 3, 1, 2)
    if path == "v8":
        grad = src.to(DEV)
    else:
        flat = torch.zeros(src.numel() + 1, device=DEV)
        flat[1:] = src.flatten().to(DEV)
        grad = flat[1:].view(B, Lt, gC)
        assert grad.data_ptr() % 16 != 0
    k.head_grad_scatter(grad, B, HW, Lt, base, dy)
    out = buf.cpu()
    maps = out[: B * HW * pitch].view(B, HW, pitch)
    want = src[:, base : base + HW].bfloat16()
    assert torch.equal(maps[..., :gC].view(torch.int16), want.view(torch.int16))
    assert bool((maps[..., gC:cpad] == 0).all()), "pad channels are not zero"
    assert bool((maps[..., cpad:] == sentinel).all()) and bool((out[B * HW * pitch :] == sentinel).all()), "written past the pad / the map"
