"""Cases and fp64 restatements for the YOLO-NAS-POSE assigner and loss kernels (csrc/pose_loss.cu, csrc/pose_loss_math.cuh).

`pose_loss_given_assignment` restates YoloNASPoseLoss.forward after the assigner in float64 from the oracle's dtype-generic term
functions (O.yolo_nas_pose_loss itself is pinned to fp32) and returns the six loss items and d(total)/d(cls, reg, pose coords,
pose logits) by autograd.  `pose_assign_stable` is the oracle's OKS-aware task-aligned assigner for one image in fp32 with the
kernel's documented top-k order (metric descending, then anchor index ascending); `O.yolo_nas_pose_loss`'s torch.topk leaves the
order of ties unspecified.

The decision cases reuse the detection cases' grid (detection_loss_cases.py): decoded distances are k or k + 1/2 bins and gt
corners multiples of 1/2 px, so box IoUs are exact in fp32.  The OKS factor of the pair IoU is not: it sums exp() terms, and the
kernel and the oracle round them differently by a few ulp.  A decision that differs is therefore excused only by an fp64 near-tie
(`explain_difference`)."""
import torch
import torch.nn.functional as F

from detection_loss_cases import FLT_TINY, constructed_case as det_constructed_case, decision_case as det_decision_case, decode_fp32, iou_matrix, near_tie, row_errors
from oracle import sg_oracle as O

# COCO keypoint sigmas: the smallest is 0.025, the largest 0.107
COCO_SIGMAS = [0.026, 0.025, 0.025, 0.035, 0.035, 0.079, 0.079, 0.072, 0.072, 0.062, 0.062, 0.107, 0.107, 0.087, 0.087, 0.089, 0.089]


def sigmas_for(J):
    """J sigmas cycling through COCO's (J = 1: the largest)."""
    return torch.tensor([0.107] if J == 1 else [COCO_SIGMAS[j % 17] for j in range(J)], dtype=torch.float32)


# ------------------------------------------------------------------------------------------------ fp64 loss restatement
def pose_loss_given_assignment(cls, reg, pose, plog, ap, st, gb, gp, agt, asc, n_pos, sigmas, reg_max, iou_type=1, cls_type=0, pose_cls_type=0, rescale_with_score=False,
                               w_cls=1.0, w_iou=2.5, w_dfl=0.5, w_pose_cls=1.0, w_pose_reg=1.0):  # fmt: skip
    """YoloNASPoseLoss.forward after the assigner, in float64.  cls [B, L] or [B, L, 1], reg [B, L, 4*(reg_max+1)], pose [B, L, J, 2]
    px, plog [B, L, J], ap [L, 2] px, st [L] or [L, 1], gb [B, n, 4] px, gp [B, n, J, 3] (x, y, visibility), agt [B, L] the positive
    (non-crowd) instance of each anchor or -1, asc [B, L] its assigned score (a constant), n_pos the number of positives.
    iou_type 0 GIoU / 1 CIoU, cls_type 0 focal / 1 BCE, pose_cls_type 0 BCE / 1 focal.  Returns (items [cls, iou, dfl, pose_cls,
    pose_reg, total] float64, d total / d cls [B, L, 1], / d reg, / d pose, / d plog)."""
    dd = lambda t: t.detach().cpu().double()  # noqa: E731
    B, L = agt.shape
    cls = dd(cls).reshape(B, L, 1).requires_grad_(True)
    reg, pose, plog = dd(reg).requires_grad_(True), dd(pose).requires_grad_(True), dd(plog).requires_grad_(True)
    ap, st, gb, gp, asc, sig = dd(ap), dd(st).reshape(-1), dd(gb), dd(gp), dd(asc), dd(sigmas)
    agt = agt.detach().cpu().long()
    score = asc.unsqueeze(-1)
    cls_sum = O.focal_loss(cls, score, alpha=-1) if cls_type == 0 else F.binary_cross_entropy_with_logits(cls, score, reduction="sum")
    norm = asc.sum().clamp_min(1.0)
    zero = torch.zeros([], dtype=torch.float64)
    iou_l = dfl_l = pc_l = pr_l = zero
    pos = agt >= 0
    if bool(pos.any()):
        bi, li = pos.nonzero(as_tuple=True)
        gi = agt[pos]
        box, s = gb[bi, gi], st[li].unsqueeze(-1)  # [P, 4] px, [P, 1]
        w = asc[pos].unsqueeze(-1)
        pts_s = ap / st.unsqueeze(-1)
        pred = O.bbox_decode(pts_s, reg)[pos]
        gbs = box / s
        iou_fn = O.giou_loss if iou_type == 0 else O.ciou_loss
        iou_l = (iou_fn(pred, gbs) * w).sum() / norm
        pts = pts_s[li]
        ltrb = torch.cat([pts - gbs[:, :2], gbs[:, 2:] - pts], -1).clip(0, reg_max - 0.01)
        dfl_l = (O.df_loss(reg[pos].reshape(-1, 4, reg_max + 1), ltrb) * w).sum() / norm
        kp, pc, pl = gp[bi, gi], pose[pos], plog[pos]  # [P, J, 3], [P, J, 2], [P, J]
        area = ((box[:, 2] - box[:, 0]) * (box[:, 3] - box[:, 1]) * 0.53).unsqueeze(-1)
        vis = (kp[..., 2] > 0).double()
        e = ((pc - kp[..., :2]) ** 2).sum(-1) / (2 * sig) ** 2 / (area + 1e-9) / 2
        reg_red = ((1 - torch.exp(-e)) * vis).sum(1) / (vis.sum(1) + 1e-9)
        if pose_cls_type == 0:
            pcls = F.binary_cross_entropy_with_logits(pl, vis, reduction="none").mean(1)
        else:
            pcls = O.focal_loss(pl, vis, alpha=0.25, gamma=2.0, reduction="none").mean(1)
        if rescale_with_score:
            pc_l, pr_l = (pcls * w[:, 0]).sum() / norm, (reg_red * w[:, 0]).sum() / norm
        else:
            pc_l, pr_l = pcls.sum() / max(n_pos, 1), reg_red.sum() / max(n_pos, 1)
    terms = [w_cls * cls_sum / norm, w_iou * iou_l, w_dfl * dfl_l, w_pose_cls * pc_l, w_pose_reg * pr_l]
    total = sum(terms)
    total.backward()
    items = torch.stack([t.detach() for t in terms + [total]])
    grads = [t.grad if t.grad is not None else torch.zeros_like(t) for t in (cls, reg, pose, plog)]
    return (items, *grads)


def logit_slacks(cls, plog, gp, agt, asc, n_pos, cls_type=0, pose_cls_type=0, rescale_with_score=False, w_cls=1.0, w_pose_cls=1.0, **_):
    """Per-element slack of the person-logit and joint-logit gradients for the one error an fp32 kernel cannot avoid: it rounds
    p = sigmoid(x) (expf, 1 + e and the division: at most 2 ulp) before p - q, so dq is off by up to 2^-22 max(p, q), which the
    gradient passes on times |d grad / d dq| = 1 (BCE) or at (2 p (1 - p) bce + 3 dq^2) (focal), times the term's factor.  Where
    p ~ q (a soft person target met by the prediction, a saturated joint logit on its target) that is no longer small against the
    gradient itself, and a person-logit row, or a joint-logit row at J = 1, has no other element to measure it against.  Twice the
    rounding bound is allowed.  Returns (slack [B, L, 1], slack [B, L, J])."""
    def one(x, q, focal, alpha, factor):
        p = torch.sigmoid(x)
        dq = p - q
        d = torch.ones_like(x)
        if focal:
            at = alpha * q + (1 - alpha) * (1 - q) if alpha > 0 else torch.ones_like(q)
            bce = F.softplus(x) - x * q
            d = at * (2 * p * (1 - p) * bce.abs() + 3 * dq * dq)
        return factor * 2 * 2.0**-22 * torch.maximum(p, q) * d

    B, L = agt.shape
    x, plog, asc = cls.detach().double().reshape(B, L), plog.detach().double(), asc.detach().double()
    norm = max(float(asc.sum()), 1.0)
    s_cls = one(x, asc, cls_type == 0, -1.0, w_cls / norm).unsqueeze(-1)
    agt = agt.long()
    kp = gp.double()[torch.arange(B).unsqueeze(-1), agt.clamp_min(0)]  # [B, L, J, 3]
    vis = (kp[..., 2] > 0).double()
    kf = (asc / norm) if rescale_with_score else torch.full_like(asc, 1.0 / max(n_pos, 1))
    factor = (w_pose_cls * kf / plog.shape[-1] * (agt >= 0)).unsqueeze(-1)
    return s_cls, one(plog, vis, pose_cls_type == 1, 0.25, factor)


def row_errors_with_slack(g, g64, slack, r=1e-4, a=1e-4):
    """detection_loss_cases.row_errors with a per-element slack added to the bound."""
    g, g64 = g.detach().cpu().double(), g64.detach().cpu().double()
    rowmax = g64.abs().amax(-1, keepdim=True)
    err = (g - g64).abs()
    ok = bool((err <= r * g64.abs() + a * rowmax + slack + FLT_TINY).all())
    return ok, float((err / (rowmax + slack).clamp_min(FLT_TINY)).max())


GRAD_NAMES = ("cls_logits", "reg_distri", "pose_coords", "pose_logits")


def check_loss(tag, items, grads, i64, g64, slacks, r=1e-4, a=1e-4):
    """Items within r relative (+ 1e-6 of the total); every gradient within the per-row bound (pose coordinates as rows of J x 2, the
    person and joint logits with `logit_slacks`).  Prints the worst items error and, per gradient, the worst error relative to the
    row maximum (for the logits: plus the slack) and to the element itself."""
    item_err = float(((items.double() - i64).abs() / i64.abs().clamp_min(1e-30)).max())
    msg, bad = [f"{tag}: items rel {item_err:.2e}"], []
    for k, (name, g, ref) in enumerate(zip(GRAD_NAMES, grads, g64)):
        if g.dim() == 4:
            g, ref = g.reshape(*g.shape[:2], -1), ref.reshape(*ref.shape[:2], -1)
        ok, row, rel = row_errors(g, ref, r, a)
        if k in (0, 3):  # logits: the row maximum plus the slack
            ok, row = row_errors_with_slack(g, ref, slacks[0] if k == 0 else slacks[1], r, a)
        msg.append(f"{name} row {row:.2e} elem {rel:.2e}")
        if not ok:
            bad.append(f"{name} outside the per-row bound: {row:.3e}")
    print(" | ".join(msg))
    assert bool((items.double() - i64).abs().le(r * i64.abs() + 1e-6 * float(i64[5].abs())).all()), (items, i64)
    assert not bad, bad


# ------------------------------------------------------------------------------------------------ assignment
def pair_iou(gb, pbox, gp, pose, sigmas, multiply_by_oks, eps=1e-9):
    """The assigner's pair IoU of one image: [n, 4] x [L, 4] -> [n, L] box IoU, times the OKS of the instance's visible joints
    (gp [n, J, 3]) with each anchor's predicted pose (pose [L, J, 2]) when multiply_by_oks.  In the inputs' dtype."""
    iou = iou_matrix(gb, pbox, eps)
    if multiply_by_oks:
        iou = iou * O.pose_oks(gp.unsqueeze(0), pose.unsqueeze(0), gb.unsqueeze(0), sigmas.to(gp.dtype))[0]
    return iou


def _in_gts(ap, gb, eps=1e-9):
    delta = torch.cat([ap.unsqueeze(0) - gb[:, None, :2], gb[:, None, 2:] - ap.unsqueeze(0)], -1)
    return delta.min(-1).values > eps


def pose_assign_stable(cls, pbox, pose, ap, gb, gp, gc, gv, sigmas, topk, alpha, beta, multiply_by_oks, eps=1e-9):
    """The oracle's assigner for one image, in fp32, with the kernel's top-k order.  cls [L] or [L, 1] logits, pbox [L, 4] px,
    pose [L, J, 2], gb [n, 4], gp [n, J, 3], gc [n] crowd, gv [n] valid.  Several claimants: the anchor goes to the row of highest
    pair IoU over ALL rows, padded ones included (first maximum).  Returns (claim [L]: the instance, crowd included, or -1;
    pos [L]: the claim unless it is a crowd instance, else -1)."""
    L, n = pbox.shape[0], gb.shape[0]
    ious = pair_iou(gb, pbox, gp, pose, sigmas, multiply_by_oks, eps)
    metrics = torch.sigmoid(cls.reshape(-1)).pow(alpha).unsqueeze(0) * ious.pow(beta)
    in_gts = _in_gts(ap, gb, eps).float()
    idx = torch.sort(metrics * in_gts, dim=-1, descending=True, stable=True).indices[:, :topk]
    pad = gv.float().unsqueeze(-1)
    mask_pos = torch.zeros(n, L).scatter_(1, idx, 1.0) * in_gts * pad
    pos_sum = mask_pos.sum(0)
    if pos_sum.max() > 1:
        is_max = F.one_hot(ious.argmax(0), n).t().float()
        mask_pos = torch.where((pos_sum > 1).unsqueeze(0), is_max, mask_pos)
        pos_sum = mask_pos.sum(0)
    claim = torch.where(pos_sum > 0, mask_pos.argmax(0), -1)
    crowd = gc.bool()[claim.clamp_min(0)] & (claim >= 0)
    return claim, torch.where(crowd, -1, claim)


def _metrics64(gi, cls, pbox, pose, ap, gb, gp, sigmas, alpha, beta, multiply_by_oks, eps=1e-9):
    """fp64 metric of gt row gi with every anchor (zero outside the gt)."""
    g = gb[gi : gi + 1].double()
    iou = pair_iou(g, pbox.double(), gp[gi : gi + 1].double(), pose.double(), sigmas, multiply_by_oks, eps)[0]
    m = torch.sigmoid(cls.reshape(-1).double()).pow(alpha) * iou.pow(beta)
    return m * _in_gts(ap.double(), g, eps)[0].double()


def exactly_tied(l, gi, cls, pbox, pose, ap, gb, gp, sigmas, alpha, beta, multiply_by_oks, eps=1e-9):
    """Whether anchor l's fp32 metric for gt row gi equals that of another anchor inside the gt: an exact tie, which the top-k order
    alone decides, the same in the kernel and the oracle (identical inputs give identical fp32 metrics in each)."""
    g = gb[gi : gi + 1]
    m = torch.sigmoid(cls.reshape(-1)).pow(alpha) * pair_iou(g, pbox, gp[gi : gi + 1], pose, sigmas, multiply_by_oks, eps)[0].pow(beta)
    inside = _in_gts(ap, g, eps)[0]
    return bool(inside[l]) and int(((m == m[l]) & inside).sum()) > 1


def explain_difference(l, g_ker, g_ora, cls, pbox, pose, ap, gb, gp, sigmas, topk, alpha, beta, multiply_by_oks, eps=1e-9):
    """Why anchor l of one image may be assigned differently: at a candidate gt's top-k boundary the last anchor taken and the first
    one left have fp64 metrics within 1e-6 of each other and l's metric is one of them, or the two candidate gts' fp64 pair IoUs
    with l's prediction agree to 1e-6.  Returns a reason, or None when the difference is a real disagreement."""
    cands = [g for g in dict.fromkeys((g_ker, g_ora)) if g >= 0]
    for gi in cands:
        m = _metrics64(gi, cls, pbox, pose, ap, gb, gp, sigmas, alpha, beta, multiply_by_oks, eps)
        srt = torch.sort(m, descending=True).values
        last, first_left, ml = float(srt[topk - 1]), float(srt[topk]), float(m[l])
        if near_tie(last, first_left) and (near_tie(ml, last) or near_tie(ml, first_left)):
            return f"top-k boundary of gt {gi}: last taken {last:.9g}, first left {first_left:.9g}, anchor {ml:.9g}"
    if len(cands) == 2:
        i2 = pair_iou(gb[cands].double(), pbox[l : l + 1].double(), gp[cands].double(), pose[l : l + 1].double(), sigmas, multiply_by_oks, eps)[:, 0].tolist()
        if near_tie(i2[0], i2[1]):
            return f"pair IoU tie between gts {cands}: {i2[0]:.9g} vs {i2[1]:.9g}"
    return None


def assigned_scores_fp64(cls, pbox, pose, gb, gp, sigmas, gidx, alpha, beta, multiply_by_oks, eps=1e-9):
    """assigned_score of one image in fp64 for a given instance per anchor (-1 = none): metric / (max metric of that instance's
    anchors + eps) * max pair IoU of that instance's anchors.  Exact for non-crowd instances when gidx is the positive assignment
    (a non-crowd instance's anchors are all positives)."""
    L = pbox.shape[0]
    out = torch.zeros(L, dtype=torch.float64)
    posm = gidx >= 0
    if not bool(posm.any()):
        return out
    gi = gidx[posm]
    iou = iou_matrix(gb.double()[gi], pbox.double()[posm], eps).diagonal()
    if multiply_by_oks:
        d = ((gp.double()[gi, :, :2] - pose.double()[posm]) ** 2).sum(-1)  # [P, J]
        g = gb.double()[gi]
        area = ((g[:, 2] - g[:, 0]) * (g[:, 3] - g[:, 1]) * 0.53).unsqueeze(-1)
        e = d / (2 * sigmas.double()) ** 2 / (area + eps) / 2
        vis = (gp.double()[gi, :, 2] > 0).double()
        iou = iou * (torch.exp(-e) * vis).sum(-1) / (vis.sum(-1) + eps)
    met = torch.sigmoid(cls.reshape(-1).double()[posm]).pow(alpha) * iou.pow(beta)
    n = gb.shape[0]
    mm = torch.zeros(n, dtype=torch.float64).scatter_reduce(0, gi, met, "amax")
    mi = torch.zeros(n, dtype=torch.float64).scatter_reduce(0, gi, iou, "amax")
    out[posm] = met / (mm[gi] + eps) * mi[gi]
    return out


# ------------------------------------------------------------------------------------------------ constructed assignments
KP_SCENARIOS = ["mixed", "all_visible", "nvis_0", "far", "degenerate"]


def constructed_case(J, reg_max, seed=0, B=2, norm_above_1=True):
    """A hand-built assignment on one stride-8 level of 16 x 16 anchors: the detection file's constructed case (every IoU and DFL
    scenario of the box terms, saturated reg logits, person logits at +-20 / +-100, asc = 0 positives) with one instance row per
    anchor (n = L) and keypoints on top.  Each positive gets a keypoint scenario:
      mixed        visibilities 0 / 1 / 2, predictions with OKS exponents e in [0, 4], every fifth joint exactly on target
      all_visible  every joint visible (1 or 2), e in [0, 4]
      nvis_0       no visible joint: inv_vis = 1e9, no regression term, visibility targets all 0
      far          visible joints with e in [120, 200]: exp(-e) underflows to 0 in fp32
      degenerate   a 6e-5 px square gt box (0.53 * area = 2e-9, next to the 1e-9 eps) with joints within 2e-5 px
    About one positive in four is a crowd instance: it keeps nothing (agt = -1, score 0), as the assigner leaves it.  Joint logits are
    N(0, 2) with some at +-15 (saturated, and still clear of fp32's subnormal range in the focal gradient).  Strides are powers of
    two, so gt boxes in stride units are exact."""
    c = det_constructed_case(1, reg_max, seed=seed, B=B, norm_above_1=norm_above_1)
    g = torch.Generator().manual_seed(1000 + seed)
    L = c["cls"].shape[1]
    sig = sigmas_for(J)
    gb = c["ab"].clone()  # [B, L, 4]: instance row l belongs to anchor l
    pos = c["al"] == 0
    agt = torch.where(pos, torch.arange(L).expand(B, L), -1).int()
    asc = c["asc"].clone()
    gp = torch.zeros(B, L, J, 3)
    pose = torch.rand(B, L, J, 2, generator=g) * 128.0
    plog = torch.randn(B, L, J, generator=g) * 2.0
    plog.view(-1)[::11] = 15.0
    plog.view(-1)[5::11] = -15.0
    scen = torch.full((B, L), -1, dtype=torch.long)
    crowd = torch.zeros(B, L, dtype=torch.bool)
    for b in range(B):
        for l in range(L):
            if not bool(pos[b, l]):
                continue
            s = KP_SCENARIOS[(l * 3 + b) % len(KP_SCENARIOS)]
            scen[b, l] = KP_SCENARIOS.index(s)
            crowd[b, l] = float(torch.rand(1, generator=g)) < 0.25
            if s == "degenerate":
                x0, y0 = float(gb[b, l, 0]), float(gb[b, l, 1])
                gb[b, l] = torch.tensor([x0, y0, x0 + 6e-5, y0 + 6e-5])
            x1, y1, x2, y2 = gb[b, l].tolist()
            jx = x1 + torch.rand(J, generator=g, dtype=torch.float64) * (x2 - x1)
            jy = y1 + torch.rand(J, generator=g, dtype=torch.float64) * (y2 - y1)
            if s == "mixed":
                vis = torch.randint(0, 3, (J,), generator=g).float()
            elif s == "nvis_0":
                vis = torch.zeros(J)
            else:
                vis = torch.randint(1, 3, (J,), generator=g).float()
            gp[b, l, :, 0], gp[b, l, :, 1], gp[b, l, :, 2] = jx.float(), jy.float(), vis
            # distance for a target exponent e: e = d / (2 sigma)^2 / (0.53 area + 1e-9) / 2
            area = float(gb[b, l, 2] - gb[b, l, 0]) * float(gb[b, l, 3] - gb[b, l, 1]) * 0.53
            e = torch.rand(J, generator=g, dtype=torch.float64) * 4.0
            if s == "far":
                e = 120.0 + torch.rand(J, generator=g, dtype=torch.float64) * 80.0
            dist = (e * 8.0 * sig.double() ** 2 * (area + 1e-9)).sqrt()
            ang = torch.rand(J, generator=g, dtype=torch.float64) * 6.283185307179586
            px, py = gp[b, l, :, 0].double() + dist * ang.cos(), gp[b, l, :, 1].double() + dist * ang.sin()
            if s == "mixed":
                px[::5], py[::5] = gp[b, l, ::5, 0].double(), gp[b, l, ::5, 1].double()  # exactly on target
            pose[b, l, :, 0], pose[b, l, :, 1] = px.float(), py.float()
    agt = torch.where(crowd, -1, agt)
    asc = torch.where(crowd, 0.0, asc)
    if not norm_above_1:
        asc = asc * (0.6 / float(asc.sum()))
    # premises: every keypoint scenario among positives and among crowds, the far joints underflow in fp32, the degenerate areas sit
    # next to the eps, both sigma extremes (J >= 17), visibilities 0 and 2, asc = 0 positives, the normaliser on the asked side of 1
    for k, name in enumerate(KP_SCENARIOS):
        assert bool(((agt >= 0) & (scen == k)).any()) and bool((crowd & (scen == k)).any()), name
    far = (scen == KP_SCENARIOS.index("far")).nonzero().tolist()
    for b, l in far:
        box = gb[b, l]
        area = (box[2] - box[0]) * (box[3] - box[1]) * 0.53
        e = ((pose[b, l] - gp[b, l, :, :2]) ** 2).sum(-1) / (2 * sig) ** 2 / (area + 1e-9) / 2
        assert bool((torch.exp(-e) == 0).all()), "a far joint does not underflow"
    deg = gb[scen == KP_SCENARIOS.index("degenerate")].double()
    area = (deg[:, 2] - deg[:, 0]) * (deg[:, 3] - deg[:, 1]) * 0.53
    assert bool(((area > 1e-9) & (area < 4e-9)).all())
    if J >= 17:
        assert float(sig.min()) == float(torch.tensor(0.025)) and float(sig.max()) == float(torch.tensor(0.107))
    mixed = gp[(scen == 0)][..., 2]
    assert bool((mixed == 0).any() and (mixed == 2).any())
    assert bool((asc[agt >= 0] == 0).any()) and bool((asc[agt < 0] == 0).all())
    assert (float(asc.sum()) > 1) == norm_above_1
    return dict(cls=c["cls"], reg=c["reg"], pose=pose, plog=plog, ap=c["ap"], st=c["st"], gb=gb, gp=gp, agt=agt, asc=asc.float(), crowd=crowd, scen=scen,
                n_pos=int((agt >= 0).sum()), sigmas=sig, J=J, reg_max=reg_max)  # fmt: skip


# ------------------------------------------------------------------------------------------------ assignment decisions
def pose_decision_case(B, H, W, n, J=17, reg_max=16, seed=0, n_invalid=0, n_max=None, crowd_every=4, exact_ties=False, dark=True):
    """Crowded persons on the 3-level anchor set of an H x W input: the detection file's crowded gts (nested, duplicate, sub-cell,
    whole-image and border-crossing boxes on a 1/2 px grid, `n_invalid` invalid rows between valid ones), trailing padding up to
    n_max, every `crowd_every`-th valid row a crowd instance, and per image one instance in the top-left corner whose joints are all
    invisible (`dark`: under multiply_by_oks its pair IoU and every metric are 0, so the top-k order alone decides).  Joints lie in their
    box (visibility 0 / 1 / 2); each anchor inside a box predicts that instance's joints jittered by about one OKS scale, so OKS is
    not ~0.  exact_ties: the detection case's exact ties (integer logits, one-bin distances) and a pose that is the same for every
    anchor inside an instance, so many anchors share one metric exactly."""
    c = det_decision_case(B, H, W, n, ncls=1, reg_max=reg_max, seed=seed, n_invalid=n_invalid, exact_ties=exact_ties)
    g = torch.Generator().manual_seed(500 + seed)
    n_max = n if n_max is None else n_max
    assert n_max >= n
    L = c["L"]
    gb = torch.zeros(B, n_max, 4)
    gv = torch.zeros(B, n_max, dtype=torch.uint8)
    gb[:, :n], gv[:, :n] = c["gb"][:, :n], c["gv"][:, :n]
    gc = torch.zeros(B, n_max, dtype=torch.uint8)
    gp = torch.zeros(B, n_max, J, 3)
    sig = sigmas_for(J)
    pose = torch.rand(B, L, J, 2, generator=g) * torch.tensor([float(W), float(H)])
    ap = c["ap"]
    owner = torch.full((B, L), -1, dtype=torch.long)  # the instance whose joints an anchor predicts
    dark_rows = []
    for b in range(B):
        valid = gv[b].nonzero().flatten().tolist()
        if not valid:
            continue
        gc[b, valid[crowd_every - 1 :: crowd_every]] = 1
        dark_row = (valid[1] if len(valid) > 1 else valid[0]) if dark else -1  # the all-invisible instance, kept out of the crowd
        if dark:
            gc[b, dark_row] = 0
            gb[b, dark_row] = torch.tensor([0.0, 0.0, 44.5, 20.5])
            dark_rows.append((b, dark_row))
        for r in valid:
            x1, y1, x2, y2 = gb[b, r].tolist()
            gp[b, r, :, 0] = x1 + torch.rand(J, generator=g) * (x2 - x1)
            gp[b, r, :, 1] = y1 + torch.rand(J, generator=g) * (y2 - y1)
            gp[b, r, :, 2] = 0.0 if r == dark_row else torch.randint(0, 3, (J,), generator=g).float()
        # predictions: anchors inside an instance predict its joints; later rows overwrite earlier ones
        inside = _in_gts(ap, gb[b])  # [n_max, L]
        for r in valid:
            m = inside[r]
            k = int(m.sum())
            if not k:
                continue
            owner[b, m] = r
            x1, y1, x2, y2 = gb[b, r].tolist()
            scale = (8.0 * (x2 - x1) * (y2 - y1) * 0.53) ** 0.5 * sig  # one OKS scale per joint: e ~ (jitter / scale)^2
            if exact_ties:
                off = torch.randn(1, J, 2, generator=g) * scale.reshape(1, J, 1) * 0.5
                pose[b, m] = (gp[b, r, :, :2].unsqueeze(0) + off).expand(k, J, 2)
            else:
                pose[b, m] = gp[b, r, :, :2].unsqueeze(0) + torch.randn(k, J, 2, generator=g) * scale.reshape(1, J, 1) * 0.7
    out = dict(cls=c["cls"], reg=c["reg"], pose=pose, ap=ap, st=c["st"], gb=gb, gp=gp, gc=gc, gv=gv, n=n, n_max=n_max, sigmas=sig, J=J, reg_max=reg_max, L=L)
    _decision_case_premises(out, n_invalid, crowd_every, dark_rows, owner, exact_ties)
    return out


def _decision_case_premises(c, n_invalid, crowd_every, dark_rows, owner, exact_ties):
    """The premises pose_decision_case promises, asserted at the size it was built."""
    gb, gp, gc, gv, n, sig = c["gb"], c["gp"], c["gc"], c["gv"], c["n"], c["sigmas"]
    B = gv.shape[0]
    if n == 0:
        return
    assert int(gv[:, n:].sum()) == 0, "trailing padding"
    assert bool((gv[:, :n] == 0).sum(1).eq(n_invalid).all()), "interleaved invalid rows"
    assert bool((gc.bool() <= gv.bool()).all()) and bool(((gv.sum(1) < crowd_every) | gc.bool().any(1)).all()), "crowds"
    for b, r in dark_rows:
        assert bool(gv[b, r]) and not bool(gc[b, r]) and bool((gp[b, r, :, 2] == 0).all()), "the all-invisible instance"
    # OKS of each anchor with the instance whose joints it predicts is away from 0
    bi, li = (owner >= 0).nonzero(as_tuple=True)
    ri = owner[bi, li]
    lit = gp[bi, ri, :, 2] > 0
    box = gb[bi, ri]
    area = ((box[:, 2] - box[:, 0]) * (box[:, 3] - box[:, 1]) * 0.53).unsqueeze(-1)
    e = ((c["pose"][bi, li] - gp[bi, ri, :, :2]) ** 2).sum(-1) / (2 * sig) ** 2 / (area + 1e-9) / 2
    oks = (torch.exp(-e) * lit).sum(-1) / (lit.sum(-1) + 1e-9)
    assert float(oks[lit.any(-1)].mean()) > 0.2, "predicted poses far from their instances"
    if exact_ties:  # most instances with several anchors inside hold exactly tied metrics, with and without OKS
        pbox = decode_fp32(c["reg"], c["ap"], c["st"])
        for oks_on in (False, True):
            tied = rows = 0
            for b in range(B):
                m = torch.sigmoid(c["cls"][b].reshape(-1)).unsqueeze(0) * pair_iou(gb[b], pbox[b], gp[b], c["pose"][b], sig, oks_on).pow(6.0)
                inside = _in_gts(c["ap"], gb[b])
                for r in gv[b].nonzero().flatten().tolist():
                    mr = m[r][inside[r] & (m[r] > 0)]
                    if mr.numel() > 1:
                        rows += 1
                        tied += int(mr.unique().numel() < mr.numel())
            assert tied * 2 >= rows > 0, f"only {tied} of {rows} instances hold exactly tied metrics (multiply_by_oks={oks_on})"
