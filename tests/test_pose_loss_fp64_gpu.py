"""The YOLO-NAS-POSE assigner and loss kernels (csrc/pose_loss.cu) element by element against float64, at training size.

Gradients are bounded per anchor row, never by the largest value of the whole tensor:  |g - g64| <= r |g64| + a max_row |g64| with
r = a = 1e-4, a row being one anchor's 4 * (reg_max + 1) bins, its J x 2 coordinates, its J joint logits or its person logit
(pose_loss_cases.check_loss).  The person and joint logits add the fp32 rounding of sigmoid before p - q (`logit_slacks`).  Each test
prints the worst error it saw, relative to the row maximum and relative to the element itself.

Assignment decisions must equal those of the fp32 oracle with the kernel's top-k order (`pose_assign_stable`); a decision that
differs is accepted only as a near-tie of the competing fp64 metrics or pair IoUs (<= 1e-6 relative), and is counted and printed."""
import ctypes

import pytest
import torch

import detection_loss_cases as DC
import pose_loss_cases as PC

pytestmark = pytest.mark.gpu

DEV = "cuda"


def K():
    from super_gradients_b200 import kernels

    return kernels


def _dev(t):
    return t.contiguous().to(DEV)


# ------------------------------------------------------------------------------------------------ a. loss on constructed assignments
def _loss(c, sw, grad_scale=1.0, want_grad=True):
    """pose_loss on a given assignment; sums[3] (the normaliser) and sums[6] (the positive count), which the assigner accumulates,
    are set here."""
    k = K()
    B, L = c["agt"].shape
    d = k.pose_loss_desc(B, L, c["J"], c["reg_max"], c["gb"].shape[1], **sw)
    sums = torch.zeros(8, dtype=torch.float64, device=DEV)
    sums[3] = c["asc"].double().sum()
    sums[6] = float(c["n_pos"])
    items, *grads = k.pose_loss(d, _dev(c["cls"].reshape(B, L, 1)), _dev(c["reg"]), _dev(c["pose"]), _dev(c["plog"]), _dev(c["ap"]), _dev(c["st"].reshape(-1)), _dev(c["gb"]),
                                _dev(c["gp"]), _dev(c["sigmas"]), _dev(c["agt"].int()), _dev(c["asc"]), sums, grad_scale, want_grad)  # fmt: skip
    torch.cuda.synchronize()
    return items.cpu(), [None if g is None else g.cpu() for g in grads]


def _fp64(c, sw):
    i64, *g64 = PC.pose_loss_given_assignment(c["cls"], c["reg"], c["pose"], c["plog"], c["ap"], c["st"], c["gb"], c["gp"], c["agt"], c["asc"], c["n_pos"], c["sigmas"],
                                              c["reg_max"], **sw)  # fmt: skip
    return i64, g64, PC.logit_slacks(c["cls"], c["plog"], c["gp"], c["agt"], c["asc"], c["n_pos"], **sw)


RECIPE_WEIGHTS = dict(w_dfl=0.01, w_pose_reg=34.0)


@pytest.mark.parametrize("J,reg_max", [(1, 7), (17, 16), (64, 31)])
@pytest.mark.parametrize("rescale", [False, True])
@pytest.mark.parametrize("pose_cls_type", [0, 1])
@pytest.mark.parametrize("cls_type", [0, 1])
@pytest.mark.parametrize("iou_type", [0, 1])
def test_loss_on_constructed_assignments(iou_type, cls_type, pose_cls_type, rescale, J, reg_max):
    """Every branch of anchor_loss: the box scenarios of the detection cases, crowd instances, positives without a visible joint,
    all-visible positives (visibility 1 and 2), joints on target, joints whose exp(-e) underflows, a gt area next to the 1e-9 eps,
    the smallest and largest COCO sigmas, normaliser below (J = 1) and above 1; the recipe's weights with the focal joint term.
    grad_scale = 0.5 halves every gradient bit for bit; want_grad = False gives the same items."""
    c = PC.constructed_case(J, reg_max, seed=J + reg_max + 3 * iou_type + cls_type, norm_above_1=J != 1)
    sw = dict(iou_type=iou_type, cls_type=cls_type, pose_cls_type=pose_cls_type, rescale_with_score=rescale, **(RECIPE_WEIGHTS if pose_cls_type else {}))
    i64, g64, slacks = _fp64(c, sw)
    items, grads = _loss(c, sw)
    PC.check_loss(f"constructed J={J} reg_max={reg_max} {sw}", items, grads, i64, g64, slacks)
    items_h, grads_h = _loss(c, sw, grad_scale=0.5)
    for name, g, gh in zip(PC.GRAD_NAMES, grads, grads_h):
        assert torch.equal(2 * gh, g), f"{name}: grad_scale 0.5 is not an exact halving"
    torch.testing.assert_close(items_h, items, rtol=1e-6, atol=0)
    items_n, grads_n = _loss(c, sw, want_grad=False)
    assert all(g is None for g in grads_n)
    torch.testing.assert_close(items_n, items, rtol=1e-6, atol=0)


# ------------------------------------------------------------------------------------------------ b / c. assignment
def _assign(c, topk, alpha, beta, oks):
    k = K()
    B = c["cls"].shape[0]
    d = k.pose_loss_desc(B, c["L"], c["J"], c["reg_max"], c["n_max"], topk=topk, alpha=alpha, beta=beta, multiply_by_oks=oks)
    sums = torch.zeros(8, dtype=torch.float64, device=DEV)
    agt, asc = k.pose_tal_assign(d, _dev(c["cls"].reshape(B, -1)), _dev(c["reg"]), _dev(c["pose"]), _dev(c["ap"]), _dev(c["st"].reshape(-1)), _dev(c["gb"]), _dev(c["gp"]),
                                 _dev(c["gc"]), _dev(c["gv"]), _dev(c["sigmas"]), sums)  # fmt: skip
    torch.cuda.synchronize()
    return agt.cpu().long(), asc.cpu(), sums.cpu()


def _check_assignment(c, topk, alpha, beta, oks, tag, exact=False):
    """exact: many anchors share one metric exactly, in the kernel and in the oracle alike, so the documented order alone decides
    among them: a difference at an anchor whose fp32 metric is exactly tied with another anchor of its gt is never excused.  Any
    other difference still needs an fp64 near-tie, as without exact ties: untied metrics carry OKS sums that the kernel and the
    oracle round differently."""
    agt, asc, sums = _assign(c, topk, alpha, beta, oks)
    B = c["cls"].shape[0]
    pbox = DC.decode_fp32(c["reg"], c["ap"], c["st"])
    ties, unexplained, worst_asc, npos = [], [], 0.0, 0
    for b in range(B):
        args = (c["cls"][b], pbox[b], c["pose"][b], c["ap"], c["gb"][b], c["gp"][b])
        _, pos = PC.pose_assign_stable(*args, c["gc"][b], c["gv"][b], c["sigmas"], topk, alpha, beta, oks)
        for l in (pos != agt[b]).nonzero().flatten().tolist():
            cands = [g for g in (int(agt[b, l]), int(pos[l])) if g >= 0]
            if exact and any(PC.exactly_tied(l, g, *args, c["sigmas"], alpha, beta, oks) for g in cands):
                why = None
            else:
                why = PC.explain_difference(l, int(agt[b, l]), int(pos[l]), *args, c["sigmas"], topk, alpha, beta, oks)
            (ties if why else unexplained).append((b, l, int(agt[b, l]), int(pos[l]), why))
        # assigned scores on the kernel's own assignment
        asc64 = PC.assigned_scores_fp64(c["cls"][b], pbox[b], c["pose"][b], c["gb"][b], c["gp"][b], c["sigmas"], agt[b], alpha, beta, oks)
        err = (asc[b].double() - asc64).abs()
        scale = float(asc64.abs().max()) if bool((asc64 != 0).any()) else 1.0
        assert bool((err <= 1e-5 * asc64.abs() + 1e-6 * scale).all()), float(err.max())
        assert bool((asc[b][agt[b] < 0] == 0).all())
        assert bool((agt[b] < c["n_max"]).all()) and not bool(c["gc"][b].bool()[agt[b].clamp_min(0)][agt[b] >= 0].any()), "a positive on a crowd instance"
        worst_asc = max(worst_asc, float((err / (asc64.abs() + 1e-6 * scale)).max()))
        npos += int((agt[b] >= 0).sum())
    assert abs(float(sums[3]) - float(asc.double().sum())) <= 1e-6 * max(float(sums[3]), 1.0)
    assert float(sums[6]) == npos
    print(f"{tag}: {npos} positives, {len(ties)} near-tie differences, asc worst rel {worst_asc:.2e}" + "".join(f"\n  image {t[0]} anchor {t[1]}: kernel gt {t[2]}, oracle gt {t[3]}: {t[4]}" for t in ties[:10]))
    assert not unexplained, f"{len(unexplained)} assignment decisions differ without a near-tie: {unexplained[:5]}"
    return agt


@pytest.mark.parametrize("alpha,beta", [(1.0, 6.0), (0.5, 2.0)])
@pytest.mark.parametrize("topk", [1, 13, 64])
@pytest.mark.parametrize("oks", [False, True])
def test_pose_decisions_parameter_sweep(oks, topk, alpha, beta):
    """60 crowded persons (duplicates, nested, sub-cell, whole-image, border-crossing, invalid rows between valid ones, trailing
    padding to n_max = 72, one in four a crowd) on 640 x 384."""
    c = PC.pose_decision_case(1, 384, 640, 60, seed=topk * 7 + int(alpha * 2) + int(beta) + oks, n_invalid=4, n_max=72)
    agt = _check_assignment(c, topk, alpha, beta, oks, f"640x384 oks={oks} topk={topk} alpha={alpha} beta={beta}")
    assert int((agt >= 0).sum()) > 0


@pytest.mark.parametrize("B,H,W,n,n_max,topk,oks", [(8, 640, 640, 30, 40, 13, True), (2, 384, 640, 30, 40, 64, False), (2, 768, 768, 30, 36, 13, True), (1, 1024, 1024, 40, 48, 64, True),
                                                     (2, 1536, 1536, 30, 36, 13, True), (16, 1024, 1024, 20, 24, 13, True)])  # fmt: skip
def test_pose_decisions_image_sizes(B, H, W, n, n_max, topk, oks):
    """L = 8400 (640^2), 5040 (640 x 384), 12096 (768^2: a 48384 B row, under 48 KB alone but not with the kernel's static shared
    memory), 21504 (1024^2: the top-k metric row takes 84 KB of dynamic shared memory, above 48 KB),
    48384 (1536^2: 189 KB, just under the 200 KB cap) and B = 16 at 1024^2 (344064 anchors: the capped grid of 1056 x 256 threads
    takes more than one anchor per thread)."""
    c = PC.pose_decision_case(B, H, W, n, seed=B + H + n, n_invalid=3, n_max=n_max)
    assert c["L"] * 4 <= 200 * 1024 and (B * c["L"] > 1056 * 256) == (B == 16)
    agt = _check_assignment(c, topk, 1.0, 6.0, oks, f"B={B} {W}x{H} L={c['L']} n={n} topk={topk} oks={oks}")
    assert int((agt >= 0).sum()) > 0


@pytest.mark.parametrize("topk", [1, 13, 64])
@pytest.mark.parametrize("oks", [False, True])
def test_pose_decisions_at_exact_metric_ties(oks, topk):
    """Many anchors inside an instance with exactly equal metrics (integer logits, one-bin distances, one pose for all of them), and
    per image an instance whose joints are all invisible, so that under multiply_by_oks each of its metrics is 0: the top-k takes the
    lowest anchor indices first, as the stable oracle does, and no difference is excused."""
    c = PC.pose_decision_case(2, 640, 640, 40, seed=topk + 10 * oks, n_invalid=2, n_max=44, exact_ties=True)
    agt = _check_assignment(c, topk, 1.0, 6.0, oks, f"exact ties 640x640 oks={oks} topk={topk}", exact=True)
    assert int((agt >= 0).sum()) > 0
    if oks:  # the all-invisible instance still takes its lowest-index anchors
        dark = c["gv"].bool() & (c["gp"][..., 2] == 0).all(-1)
        rows = dark.nonzero().tolist()
        assert any(bool((agt[b] == r).any()) for b, r in rows), "the all-invisible instance took no anchor"


@pytest.mark.parametrize("case", ["n_max_0", "all_invalid", "all_crowd"])
def test_pose_without_valid_gts(case):
    """n_max = 0, a batch whose instances are all invalid, and one whose instances are all crowds: no positives, normaliser 0 (clamped
    to 1 by the loss), box and keypoint items exactly 0 and zero box and keypoint gradients; the person logits against fp64."""
    c = PC.pose_decision_case(2, 256, 256, 0 if case == "n_max_0" else 6)
    if case == "all_invalid":
        c["gv"].zero_()
    if case == "all_crowd":
        c["gc"].copy_(c["gv"])
    agt, asc, sums = _assign(c, 13, 1.0, 6.0, True)
    assert bool((agt == -1).all()) and bool((asc == 0).all()) and float(sums[3]) == 0.0 and float(sums[6]) == 0.0
    g = torch.Generator().manual_seed(3)
    c.update(agt=agt, asc=asc, n_pos=0, plog=torch.randn(c["pose"].shape[:3], generator=g))
    if c["gb"].shape[1] == 0:
        c.update(gb=torch.zeros(2, 1, 4), gp=torch.zeros(2, 1, c["J"], 3))
    sw = dict(iou_type=1, cls_type=0, pose_cls_type=0)
    i64, g64, slacks = _fp64(c, sw)
    items, grads = _loss(c, sw)
    assert all(float(items[k]) == 0.0 for k in (1, 2, 3, 4)), items
    assert all(bool((g == 0).all()) for g in grads[1:])
    PC.check_loss(f"no valid gts ({case})", items, grads, i64, g64, slacks)


# ------------------------------------------------------------------------------------------------ d. end to end
@pytest.mark.parametrize("oks", [False, True])
def test_end_to_end_training_size(oks):
    """pose_tal_assign + pose_loss at training size (B = 8, 640^2, J = 17, reg_max = 16, 30 persons per image with crowds, invalid
    rows and padding to 36, random reg logits), against the fp64 loss on the kernel's own assignment.  Run twice: the assignment
    and every gradient are bit-identical (they are written per element, without atomics; CUDA-graph replays rely on it), the items
    differ at most by the order of the fp64 atomics."""
    k = K()
    g = torch.Generator().manual_seed(70 + oks)
    c = PC.pose_decision_case(8, 640, 640, 30, seed=70 + oks, n_invalid=3, n_max=36)
    c["reg"] = DC.off_grid_reg(torch.randn(c["reg"].shape, generator=g) * 1.5, c["ap"], c["st"], g)
    c["plog"] = torch.randn(c["pose"].shape[:3], generator=g) * 2.0
    B, L = 8, c["L"]
    sw = dict(iou_type=1, cls_type=0, pose_cls_type=1, rescale_with_score=oks, **RECIPE_WEIGHTS)
    d = k.pose_loss_desc(B, L, 17, 16, c["n_max"], multiply_by_oks=oks, **sw)
    dev = {n: _dev(c[n]) for n in ("reg", "pose", "plog", "ap", "gb", "gp", "gc", "gv", "sigmas")}
    cls, st = _dev(c["cls"].reshape(B, L, 1)), _dev(c["st"].reshape(-1))

    def run():
        sums = torch.zeros(8, dtype=torch.float64, device=DEV)
        agt, asc = k.pose_tal_assign(d, cls, dev["reg"], dev["pose"], dev["ap"], st, dev["gb"], dev["gp"], dev["gc"], dev["gv"], dev["sigmas"], sums)
        items, *grads = k.pose_loss(d, cls, dev["reg"], dev["pose"], dev["plog"], dev["ap"], st, dev["gb"], dev["gp"], dev["sigmas"], agt, asc, sums)
        torch.cuda.synchronize()
        return agt.cpu(), asc.cpu(), items.cpu(), [t.cpu() for t in grads]

    agt, asc, items, grads = run()
    agt2, asc2, items2, grads2 = run()
    assert torch.equal(agt, agt2) and torch.equal(asc, asc2)
    for name, a, b in zip(PC.GRAD_NAMES, grads, grads2):
        assert torch.equal(a, b), f"{name} differs between two runs"
    torch.testing.assert_close(items2, items, rtol=1e-6, atol=0)
    n_pos = int((agt >= 0).sum())
    assert n_pos > 1000
    c.update(agt=agt.long(), asc=asc, n_pos=n_pos)
    i64, g64, slacks = _fp64(c, sw)
    PC.check_loss(f"end to end B=8 640x640 oks={oks}", items, grads, i64, g64, slacks)


# ------------------------------------------------------------------------------------------------ host validation
def test_refused_metric_row_launches_nothing():
    """1600^2 (L = 52500: a 205 KB metric row) is refused before any launch: the caller's sentinel-filled workspace and outputs are
    untouched."""
    from super_gradients_b200 import lib as L

    k = K()
    Lc = sum(h * w for h, w in DC.level_shapes(1600, 1600))
    B, n, J = 1, 2, 17
    d = k.pose_loss_desc(B, Lc, J, 16, n)
    lib = L.load()
    nbytes = lib.sgb_pose_tal_workspace_bytes(ctypes.byref(d))
    ws = torch.full((nbytes,), 0xA5, dtype=torch.uint8, device=DEV)
    agt = torch.full((B, Lc), -7, dtype=torch.int32, device=DEV)
    asc = torch.full((B, Lc), -7.0, device=DEV)
    sums = torch.full((8,), -7.0, dtype=torch.float64, device=DEV)
    ins = [torch.zeros(s, device=DEV) for s in ((B, Lc), (B, Lc, 68), (B, Lc, J, 2), (Lc, 2), (Lc,), (B, n, 4), (B, n, J, 3))]
    flags = [torch.ones(B, n, dtype=torch.uint8, device=DEV) for _ in range(2)]
    sig = PC.sigmas_for(J).to(DEV)
    p = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    torch.cuda.synchronize()
    rc = lib.sgb_pose_tal_assign(ctypes.byref(d), *[p(t) for t in ins], *[p(t) for t in flags], p(sig), p(agt), p(asc), p(sums), p(ws), nbytes,
                                 ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))  # fmt: skip
    torch.cuda.synchronize()
    assert rc == -1 and b"too many anchors" in lib.sgb_last_error()
    assert bool((ws == 0xA5).all()) and bool((agt == -7).all()) and bool((asc == -7.0).all()) and bool((sums == -7.0).all())
