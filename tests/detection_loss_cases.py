"""Cases and fp64 restatements for the PP-YOLOE / YOLO-NAS loss kernels (csrc/loss.cu, csrc/focal_cls.cu).

`loss_given_assignment` restates the fused varifocal / focal + GIoU / CIoU + DFL loss around a GIVEN assignment in float64, from
the oracle's own term functions, and returns the four loss items and d(total)/d(cls), d(total)/d(reg) by autograd.
`tal_assign_stable` is the oracle's task-aligned assigner in fp32 with the kernel's documented top-k order (metric descending, then
anchor index ascending); `O.tal_assign`'s torch.topk leaves the order of ties unspecified.

The assignment cases put every decoded box and every gt corner on a grid (decoded distances are k or k + 1/2 bins, gt corners are
multiples of 1/2 px), so that areas and intersections are exact in fp32 and the kernel and the oracle compute bit-identical IoUs:
a decision that differs then comes from the assigner, not from rounding of the boxes."""
import contextlib
from unittest import mock

import torch
import torch.nn.functional as F

from oracle import sg_oracle as O

FLT_TINY = torch.finfo(torch.float32).tiny  # gradients below fp32's normal range cannot be resolved by an fp32 kernel


# ------------------------------------------------------------------------------------------------ fp64 loss restatement
def loss_given_assignment(cls, reg, ap, st, al, ab, asc, ncls, reg_max, w_cls=1.0, w_iou=2.5, w_dfl=0.5, iou_type=0, focal_alpha=None):
    """PPYoloELoss.forward (the oracle's ppyoloe_loss) after the assigner, in float64.  cls [B, L, ncls], reg [B, L, 4*(reg_max+1)],
    ap [L, 2] px, st [L] or [L, 1], al [B, L] (ncls = background), ab [B, L, 4] px, asc [B, L] (the assigned score, a constant).
    Returns (items [cls, iou, dfl, total] float64, d total / d cls, d total / d reg), normalised by max(sum(asc), 1)."""
    cls = cls.detach().cpu().double().requires_grad_(True)
    reg = reg.detach().cpu().double().requires_grad_(True)
    st = st.detach().cpu().double().reshape(-1, 1)
    ap, ab, asc, al = ap.detach().cpu().double(), ab.detach().cpu().double(), asc.detach().cpu().double(), al.detach().cpu().long()
    B, L, _ = cls.shape
    onehot = F.one_hot(al, ncls + 1)[..., :ncls].double()
    score = onehot * asc.unsqueeze(-1)
    cls_sum = O.varifocal_loss(cls, score, onehot) if focal_alpha is None else O.focal_loss(cls, score, alpha=focal_alpha)
    pts_s = ap / st
    pred = O.bbox_decode(pts_s, reg)
    pos = al != ncls
    if bool(pos.any()):
        w = asc[pos].unsqueeze(-1)
        gb = (ab / st)[pos]
        iou_fn = O.giou_loss if iou_type == 0 else O.ciou_loss
        iou_sum = (iou_fn(pred[pos], gb) * w).sum()
        pts = pts_s.unsqueeze(0).expand(B, L, 2)[pos]
        ltrb = torch.cat([pts - gb[:, :2], gb[:, 2:] - pts], -1).clip(0, reg_max - 0.01)
        dfl_sum = (O.df_loss(reg[pos].reshape(-1, 4, reg_max + 1), ltrb) * w).sum()
    else:
        iou_sum = dfl_sum = torch.zeros([], dtype=torch.float64)
    norm = asc.sum().clamp_min(1.0)
    lc, li, ld = w_cls * cls_sum / norm, w_iou * iou_sum / norm, w_dfl * dfl_sum / norm
    total = lc + li + ld
    total.backward()
    items = torch.stack([lc, li, ld, total]).detach()
    return items, cls.grad, reg.grad if reg.grad is not None else torch.zeros_like(reg)


@contextlib.contextmanager
def strict_minmax():
    """torch.maximum / minimum with the kernel's convention at exact ties: the second operand (the gt coordinate) is taken, so the
    predicted coordinate gets no gradient.  torch's own maximum / minimum split the gradient between equal operands."""
    with mock.patch.object(torch, "maximum", lambda a, b: torch.where(a > b, a, b)), mock.patch.object(torch, "minimum", lambda a, b: torch.where(a < b, a, b)):
        yield


def row_errors(g, g64, r=1e-4, a=1e-4):
    """Per-element bound |g - g64| <= r |g64| + a max_row |g64| (+ fp32's smallest normal), a row being the last dimension (one
    anchor's classes or bins).  Returns (ok, worst |g - g64| / max_row |g64|, worst |g - g64| / |g64| over elements above 1e-3 of
    their row's maximum)."""
    g, g64 = g.detach().cpu().double(), g64.detach().cpu().double()
    rowmax = g64.abs().amax(-1, keepdim=True)
    err = (g - g64).abs()
    ok = bool((err <= r * g64.abs() + a * rowmax + FLT_TINY).all())
    big = (g64.abs() > 1e-3 * rowmax) & (g64.abs() > FLT_TINY)
    worst_row = float((err / rowmax.clamp_min(FLT_TINY)).max())
    worst_rel = float((err[big] / g64.abs()[big]).max()) if bool(big.any()) else 0.0
    return ok, worst_row, worst_rel


# ------------------------------------------------------------------------------------------------ constructed assignments
IOU_SCENARIOS = ["inside", "encloses", "side_x1", "side_y1", "side_x2", "side_y2", "disjoint", "disjoint_x", "tall", "wide", "same_ratio", "iou_to_1"]
DFL_SCENARIOS = ["negative", "on_bin", "below_top", "above_top"]


def constructed_case(ncls, reg_max, seed=0, B=2, hw=(16, 16), stride=8.0, norm_above_1=True):
    """Hand-built assignment on one stride-8 level: every anchor gets a scenario that drives one branch of the loss kernel.
    IoU scenarios place the gt relative to the fp64-decoded predicted box (margins >= 0.3 stride units, so no coordinate ties);
    DFL scenarios place the gt relative to the anchor point.  Some rows carry saturated logits (reg one-hot at +-30 on bin 0 or
    bin reg_max, cls +-20 / +-100), some positives have asc = 0, and the assigned scores sum above or below 1."""
    g = torch.Generator().manual_seed(seed)
    h, w = hw
    _, ap, _, st = O.anchors_for_levels([(h, w)], (int(stride),))
    st = st.flatten()
    L, nb = h * w, reg_max + 1
    cls = torch.randn(B, L, ncls, generator=g) * 2.0 - 1.0
    reg = torch.randn(B, L, 4 * nb, generator=g) * 1.5
    # saturated rows
    for b in range(B):
        for l in range(3, L, 17):
            # bin 0 on two sides, bin reg_max on the other two (bin 0 on all four would decode to a point box, whose CIoU
            # aspect term is 0 / 0 in the reference as well)
            z = torch.full((4, nb), -30.0)
            lo = (l // 17) % 2
            z[[0, 1], 0 if lo else reg_max] = 30.0
            z[[2, 3], reg_max if lo else 0] = 30.0
            reg[b, l] = z.flatten()
        for l in range(5, L, 13):
            c = int(torch.randint(0, ncls, (1,), generator=g))
            cls[b, l, c] = [20.0, -20.0, 100.0, -100.0][(l // 13) % 4]
    pts = (ap / st[:, None]).double()
    pred = O.bbox_decode(pts, reg.double())  # [B, L, 4] stride units
    al = torch.full((B, L), ncls, dtype=torch.int32)
    ab = torch.zeros(B, L, 4, dtype=torch.float64)
    asc = torch.zeros(B, L)
    scen = IOU_SCENARIOS + DFL_SCENARIOS
    for b in range(B):
        for l in range(L):
            if (l + b) % 5 == 4:
                continue  # background anchor
            m = 0.3 + torch.rand(4, generator=g, dtype=torch.float64) * 1.7
            px1, py1, px2, py2 = pred[b, l].tolist()
            pw, ph = px2 - px1, py2 - py1
            cx, cy = (px1 + px2) / 2, (py1 + py2) / 2
            ax, ay = pts[l].tolist()
            s = scen[(l * 7 + b) % len(scen)]
            if min(pw, ph) < 1.0 and s not in ("inside", "disjoint", "negative", "above_top"):
                s = "inside"  # a (near-)point box from saturated bins: no margin-free placement relative to it
            if s == "inside":
                box = [px1 - m[0], py1 - m[1], px2 + m[2], py2 + m[3]]
            elif s == "encloses":
                f = 0.2 + 0.25 * torch.rand(4, generator=g, dtype=torch.float64)
                box = [px1 + f[0] * pw, py1 + f[1] * ph, px2 - f[2] * pw, py2 - f[3] * ph]
            elif s.startswith("side_"):
                # the predicted box crosses the gt on this one side only
                k = ["side_x1", "side_y1", "side_x2", "side_y2"].index(s)
                box = [px1 - m[0], py1 - m[1], px2 + m[2], py2 + m[3]]
                box[k] = [px1, py1, px2, py2][k] + (m[k] if k < 2 else -m[k]) * 0.5 * min(1.0, (pw if k % 2 == 0 else ph) / 2)
            elif s == "disjoint":
                box = [px2 + m[0], py2 + m[1], px2 + m[0] + 1 + m[2], py2 + m[1] + 1 + m[3]]
            elif s == "disjoint_x":
                box = [px2 + m[0], py1 - m[1], px2 + m[0] + 1 + m[2], py2 + m[3]]
            elif s == "tall":
                box = [cx - 0.02, py1 - m[1], cx + 0.02, py2 + m[3]]
            elif s == "wide":
                box = [px1 - m[0], cy - 0.02, px2 + m[2], cy + 0.02]
            elif s == "same_ratio":
                f = 1.3 + 0.2 * float(torch.rand(1, generator=g))
                box = [cx - f * pw / 2 + 0.3, cy - f * ph / 2 + 0.3, cx + f * pw / 2 + 0.3, cy + f * ph / 2 + 0.3]
            elif s == "iou_to_1":
                e = 1e-3 * m * torch.where(torch.rand(4, generator=g) < 0.5, -1.0, 1.0).double()
                box = [px1 + e[0], py1 + e[1], px2 + e[2], py2 + e[3]]
            elif s == "negative":
                box = [ax + 0.4 + m[0], ay + 0.4 + m[1], ax + 3 + m[2], ay + 3 + m[3]]  # anchor left of / above the gt
            elif s == "on_bin":
                t = torch.randint(0, reg_max, (4,), generator=g).double()
                box = [ax - t[0], ay - t[1], ax + t[2], ay + t[3]]  # exact: ax = i + 1/2, t integral
            elif s == "below_top":
                t = reg_max - 0.0101
                box = [ax - t, ay - m[1], ax + t, ay + m[3]]
            else:  # above_top
                box = [ax - reg_max - 2 - m[0], ay - m[1], ax + reg_max + 1.5, ay + m[3]]
            ab[b, l] = torch.tensor(box, dtype=torch.float64) * stride
            al[b, l] = int(torch.randint(0, ncls, (1,), generator=g))
            q = float(torch.rand(1, generator=g)) if (l % 11) else 0.0  # positives with asc = 0
            asc[b, l] = q
    if not norm_above_1:
        asc = asc * (0.6 / float(asc.sum()))
    # keep label logits off p == q, where the kernel's p - q cancels to fp32's rounding (a one-class row has no other entry to
    # measure that error against)
    pos = al != ncls
    lab = al.clamp_max(ncls - 1).long().unsqueeze(-1)
    x = cls.gather(-1, lab)
    near = (pos & ((torch.sigmoid(x.squeeze(-1)) - asc).abs() < 0.02) & (asc > 0)).unsqueeze(-1)
    cls.scatter_(-1, lab, torch.where(near, x + 1.5, x))
    return dict(cls=cls, reg=reg, ap=ap, st=st, al=al, ab=ab.float(), asc=asc.float(), ncls=ncls, reg_max=reg_max)


def coincident_case(reg_max=16):
    """Predicted boxes that coincide exactly with their gt: two bins k, k + 1 at logit 0 and the rest at -200 decode to exactly
    k + 1/2 in fp32 (exp(-200) is 0) and in fp64 (exp(-200) is below half an ulp), and the gt is that box.  Every min / max of GIoU
    and CIoU is then an exact tie, while the softmax still passes a gradient to the two bins."""
    _, ap, _, st = O.anchors_for_levels([(4, 4)], (8,))
    st = st.flatten()
    L, nb = 16, reg_max + 1
    reg = torch.full((1, L, 4, nb), -200.0)
    ab = torch.zeros(1, L, 4)
    g = torch.Generator().manual_seed(5)
    for l in range(L):
        ks = torch.randint(1, reg_max - 1, (4,), generator=g)
        for s in range(4):
            reg[0, l, s, ks[s] : ks[s] + 2] = 0.0
        d = ks.float() + 0.5
        ax, ay = (ap[l] / st[l]).tolist()
        ab[0, l] = torch.stack([ax - d[0], ay - d[1], ax + d[2], ay + d[3]]) * st[l]
    cls = torch.randn(1, L, 3, generator=g)
    al = torch.randint(0, 3, (1, L), generator=g, dtype=torch.int32)
    asc = torch.rand(1, L, generator=g) * 0.5 + 0.25
    return dict(cls=cls, reg=reg.reshape(1, L, 4 * nb), ap=ap, st=st, al=al, ab=ab, asc=asc, ncls=3, reg_max=reg_max)


# ------------------------------------------------------------------------------------------------ assignment decisions
def level_shapes(H, W, strides=(8, 16, 32)):
    return [(H // s, W // s) for s in strides]


def grid_reg(B, L, reg_max, g, halves=True):
    """reg logits whose fp32 softmax expectation is exactly k or k + 1/2 (one or two bins at +30, the rest at -30)."""
    nb = reg_max + 1
    k = torch.randint(0 if halves else 1, reg_max, (B, L, 4), generator=g)
    two = (torch.rand(B, L, 4, generator=g) < 0.5) & halves
    z = torch.full((B, L, 4, nb), -30.0)
    z.scatter_(-1, k.unsqueeze(-1), 30.0)
    z.scatter_(-1, (k + 1).unsqueeze(-1), torch.where(two, 30.0, -30.0).unsqueeze(-1))
    return z.reshape(B, L, 4 * nb), k.double() + two.double() * 0.5


def crowded_gts(B, H, W, n, ncls, g, n_invalid=0):
    """n gt rows per image on a 1/2 px grid: clusters of heavily overlapping boxes, exact duplicates (with a different label, so the
    winner is visible), nested boxes, boxes smaller than a stride-8 cell, the whole image, boxes touching and crossing the border,
    and `n_invalid` invalid (zero) rows between the valid ones.  Returns gt_boxes [B, n, 4], gt_labels [B, n] int32, gt_valid
    [B, n] uint8."""
    h2 = lambda t: torch.round(t * 2) / 2  # noqa: E731
    boxes = torch.zeros(B, n, 4)
    labels = torch.randint(0, ncls, (B, n), generator=g, dtype=torch.int32)
    valid = torch.ones(B, n, dtype=torch.uint8)
    for b in range(B):
        centres = torch.rand(6, 2, generator=g) * torch.tensor([W, H])
        rows, dups = [], []
        while len(rows) < n:
            kind = len(rows) % 10
            if kind == 0 and rows:  # exact duplicate of an earlier row
                src = int(torch.randint(0, len(rows), (1,), generator=g))
                dups.append((len(rows), src))
                rows.append(list(rows[src]))
                continue
            if kind == 1 and rows:  # nested inside an earlier row
                x1, y1, x2, y2 = rows[-1]
                f = torch.rand(4, generator=g) * 0.3
                rows.append([x1 + f[0].item() * (x2 - x1), y1 + f[1].item() * (y2 - y1), x2 - f[2].item() * (x2 - x1), y2 - f[3].item() * (y2 - y1)])
                continue
            if kind == 2:  # smaller than a stride-8 cell
                c = torch.rand(2, generator=g) * torch.tensor([W, H])
                s = 1.0 + torch.rand(2, generator=g) * 5
                rows.append([c[0] - s[0] / 2, c[1] - s[1] / 2, c[0] + s[0] / 2, c[1] + s[1] / 2])
                continue
            if kind == 3 and len(rows) % 40 == 3:  # the whole image
                rows.append([0.0, 0.0, float(W), float(H)])
                continue
            if kind == 4:  # touching or crossing the border
                s = 10 + torch.rand(2, generator=g) * 120
                over = float(torch.rand(1, generator=g)) < 0.5
                x1 = -s[0].item() / 3 if over else 0.0
                y1 = float(torch.rand(1, generator=g)) * (H - s[1].item())
                row = [x1, y1, x1 + s[0].item(), y1 + s[1].item()]
                if len(rows) % 20 == 4:  # right / bottom border
                    row = [W - s[0].item() + (s[0].item() / 3 if over else 0.0), H - s[1].item(), W + (s[0].item() / 3 if over else 0.0), float(H)]
                rows.append(row)
                continue
            c = centres[int(torch.randint(0, 6, (1,), generator=g))] + torch.randn(2, generator=g) * 25
            s = 8 + torch.rand(2, generator=g) * 150
            rows.append([c[0] - s[0] / 2, c[1] - s[1] / 2, c[0] + s[0] / 2, c[1] + s[1] / 2])
        t = h2(torch.tensor(rows, dtype=torch.float32))
        t[:, 2:] = torch.maximum(t[:, 2:], t[:, :2] + 0.5)
        boxes[b] = t
        # a duplicate keeps its box but gets the next label: which one wins the tie is then visible in the assigned label
        for i, src in dups:
            labels[b, i] = (labels[b, src] + 1) % ncls
        if n_invalid:
            inv = torch.randperm(n - 2, generator=g)[:n_invalid] + 1
            valid[b, inv] = 0
            boxes[b, inv] = 0.0
    return boxes, labels, valid


def decision_case(B, H, W, n, ncls=80, reg_max=16, seed=0, n_invalid=0, exact_ties=False):
    """exact_ties: every decoded distance is exactly one bin and the class logits are integers, so that many anchors inside a gt
    share one metric exactly (equal boxes inside the gt give equal IoUs) and the top-k order among equal metrics decides."""
    g = torch.Generator().manual_seed(seed)
    _, ap, nums, st = O.anchors_for_levels(level_shapes(H, W), (8, 16, 32))
    L = sum(nums)
    reg, dist = grid_reg(B, L, 2 if exact_ties else reg_max, g, halves=not exact_ties)
    if exact_ties:
        reg = torch.cat([reg.reshape(B, L, 4, 3), torch.full((B, L, 4, reg_max - 2), -30.0)], -1).reshape(B, L, -1)
    cls = torch.randint(-2, 3, (B, L, ncls), generator=g).float() if exact_ties else torch.randn(B, L, ncls, generator=g) * 2.0 - 1.0
    gb, gl, gv = crowded_gts(B, H, W, n, ncls, g, n_invalid) if n else (torch.zeros(B, 1, 4), torch.zeros(B, 1, dtype=torch.int32), torch.zeros(B, 1, dtype=torch.uint8))
    return dict(cls=cls, reg=reg, dist=dist, ap=ap, st=st.flatten(), gb=gb, gl=gl, gv=gv, n=n, ncls=ncls, reg_max=reg_max, L=L)


def off_grid_reg(reg, ap, st, g, tol_px=1e-3):
    """Random reg logits nudged until no decoded corner lies within tol_px of the 1/2 px grid the gt corners sit on: there fp32
    rounds the two coordinates to an exact tie, where the kernel's min / max convention departs from torch's."""
    reg = reg.clone()
    B, L, C = reg.shape
    for _ in range(10):
        px = O.bbox_decode((ap / st.reshape(-1, 1)).double(), reg.double()) * st.reshape(-1, 1).double()
        near = ((px * 2 - torch.round(px * 2)).abs() < 2 * tol_px).any(-1)  # [B, L]
        if not bool(near.any()):
            return reg
        reg[near] += torch.randn(int(near.sum()), C, generator=g) * 0.1
    raise AssertionError("could not move the decoded boxes off the gt grid")


def iou_matrix(gb, pb, eps=1e-9):
    """[n, 4] x [L, 4] -> [n, L]: O.iou_similarity for one image."""
    return O.iou_similarity(gb.unsqueeze(0), pb.unsqueeze(0), eps)[0]


def tal_assign_stable(cls, pbox, ap, gb, gl, gv, ncls, topk, alpha, beta, eps=1e-9):
    """O.tal_assign for one image with the kernel's top-k order.  cls [L, C] logits, pbox [L, 4] px, gb [n, 4], gl [n], gv [n].
    Returns (labels [L] int64 with ncls = background, gt index [L] int64 with -1 = background)."""
    L = pbox.shape[0]
    n = gb.shape[0]
    ious = iou_matrix(gb, pbox, eps)
    scores = torch.sigmoid(cls).t()[gl.long()]  # [n, L]
    metrics = scores.pow(alpha) * ious.pow(beta)
    delta = torch.cat([ap.unsqueeze(0) - gb[:, None, :2], gb[:, None, 2:] - ap.unsqueeze(0)], -1)
    in_gts = (delta.min(-1).values > eps).float()
    idx = torch.sort(metrics * in_gts, dim=-1, descending=True, stable=True).indices[:, :topk]
    pad = gv.float().unsqueeze(-1)
    in_topk = torch.zeros(n, L).scatter_(1, idx, 1.0) * pad
    mask_pos = in_topk * in_gts * pad
    pos_sum = mask_pos.sum(0)
    if pos_sum.max() > 1:
        is_max = F.one_hot(ious.argmax(0), n).t().float()
        mask_pos = torch.where((pos_sum > 1).unsqueeze(0), is_max, mask_pos)
        pos_sum = mask_pos.sum(0)
    gidx = mask_pos.argmax(0)
    assigned = pos_sum > 0
    labels = torch.where(assigned, gl.long()[gidx], torch.full_like(gidx, ncls))
    return labels, torch.where(assigned, gidx, torch.full_like(gidx, -1))


def kernel_gt_index(al, ab, gb, gl, ncls):
    """The gt row behind each of one image's kernel decisions: the first row with the assigned label and box (-1 = background)."""
    match = (gb.unsqueeze(1) == ab.unsqueeze(0)).all(-1) & (gl.long().unsqueeze(1) == al.long().unsqueeze(0))  # [n, L]
    first = torch.where(match.any(0), match.float().argmax(0), torch.full((ab.shape[0],), -1, dtype=torch.long))
    return torch.where(al.long() == ncls, torch.full_like(first, -1), first)


def near_tie(a, b, rel=1e-6):
    return abs(a - b) <= rel * max(abs(a), abs(b)) + FLT_TINY


def explain_difference(l, g_ker, g_ora, cls, pbox, ap, gb, gl, topk, alpha, beta, eps=1e-9):
    """Why anchor l of one image may be assigned differently: at a gt's top-k boundary the last anchor taken and the first one left
    have fp64 metrics within 1e-6 of each other and l's metric is one of them, or the two candidate gts' fp64 IoUs with l's
    predicted box agree to 1e-6.  Returns a reason, or None when the difference is a real disagreement."""
    pb64 = pbox.double()
    cands = [g for g in (g_ker, g_ora) if g >= 0]
    for gi in cands:
        gbox = gb[gi].double()
        iou = iou_matrix(gbox.unsqueeze(0), pb64, eps)[0]
        score = torch.sigmoid(cls[:, int(gl[gi])].double())
        delta = torch.cat([ap.double() - gbox[:2], gbox[2:] - ap.double()], -1)
        m = score.pow(alpha) * iou.pow(beta) * (delta.min(-1).values > eps).double()
        srt = torch.sort(m, descending=True).values
        last, first_left, ml = float(srt[topk - 1]), float(srt[topk]), float(m[l])
        if near_tie(last, first_left) and (near_tie(ml, last) or near_tie(ml, first_left)):
            return f"top-k boundary of gt {gi}: last taken {last:.9g}, first left {first_left:.9g}, anchor {ml:.9g}"
    if len(cands) == 2:
        i2 = iou_matrix(gb[cands].double(), pb64[l : l + 1], eps)[:, 0].tolist()
        if near_tie(i2[0], i2[1]):
            return f"IoU tie between gts {cands}: {i2[0]:.9g} vs {i2[1]:.9g}"
    return None


def assigned_scores_fp64(cls, pbox, gb, gl, gidx, alpha, beta, eps=1e-9):
    """assigned_score of one image in fp64 for a given gt index per anchor (-1 = background): metric / (max metric of that gt's
    anchors + eps) * max IoU of that gt's anchors."""
    L = pbox.shape[0]
    out = torch.zeros(L, dtype=torch.float64)
    posm = gidx >= 0
    if not bool(posm.any()):
        return out
    gi = gidx[posm]
    g = gb.double()[gi]
    p = pbox.double()[posm]
    lt, rb = torch.maximum(g[:, :2], p[:, :2]), torch.minimum(g[:, 2:], p[:, 2:])
    ov = (rb - lt).clip(0).prod(-1)
    iou = ov / ((g[:, 2:] - g[:, :2]).clip(0).prod(-1) + (p[:, 2:] - p[:, :2]).clip(0).prod(-1) - ov + eps)
    score = torch.sigmoid(cls.double()[posm, gl.long()[gi]])
    met = score.pow(alpha) * iou.pow(beta)
    n = gb.shape[0]
    mm = torch.zeros(n, dtype=torch.float64).scatter_reduce(0, gi, met, "amax")
    mi = torch.zeros(n, dtype=torch.float64).scatter_reduce(0, gi, iou, "amax")
    out[posm] = met / (mm[gi] + eps) * mi[gi]
    return out


def decode_fp32(reg, ap, st):
    """The oracle's decode in fp32 (pixels): O.bbox_decode(anchor_points / stride, reg) * stride."""
    st = st.reshape(-1, 1)
    return O.bbox_decode(ap / st, reg) * st
