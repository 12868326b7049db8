"""CPU checks of the fp64 pose-loss restatement and the fp32 stable assigner in pose_loss_cases.py, of the case builders, and of the
host build of the kernels' arithmetic (csrc/pose_loss_math.cuh through tests/host_pose_loss.py) against them.

The restatement is what the GPU tests of csrc/pose_loss.cu compare against element by element, so here it is pinned to the oracle's
full YoloNASPoseLoss for every loss switch and to the reference's own outputs in tests/golden/pose.pt.  Gradients are bounded per
row (one anchor's bins, its J x 2 coordinates, its J joint logits or its person logit): |g - g64| <= r |g64| + a max_row |g64|."""
import ctypes
import shutil

import pytest
import torch

import detection_loss_cases as DC
import host_pose_loss
import pose_loss_cases as PC
from oracle import sg_oracle as O
from super_gradients_b200 import kernels as K
from super_gradients_b200 import lib as L
from test_pose_loss_host import KWS, _random_case

GRAD_NAMES = PC.GRAD_NAMES


def _rows(g):
    """A gradient as [..., row]: pose coordinates [B, L, J, 2] -> [B, L, 2J]; the others already end in their row."""
    return g.reshape(*g.shape[:2], -1) if g.dim() == 4 else g


def _desc_kw(kw):
    return dict(iou_type=0 if kw.get("regression_iou_loss_type", "ciou") == "giou" else 1, cls_type=0 if kw.get("classification_loss_type", "focal") == "focal" else 1,
                pose_cls_type=1 if kw.get("pose_classification_loss_type", "bce") == "focal" else 0, rescale_with_score=kw.get("rescale_pose_loss_with_assigned_score", False),
                w_cls=kw.get("classification_loss_weight", 1.0), w_iou=kw.get("iou_loss_weight", 2.5), w_dfl=kw.get("dfl_loss_weight", 0.5),
                w_pose_cls=kw.get("pose_cls_loss_weight", 1.0), w_pose_reg=kw.get("pose_reg_loss_weight", 1.0))  # fmt: skip


def _oracle_with_assignment(raw, targets, sigmas, kw):
    names = dict(classification_loss_weight="w_cls", iou_loss_weight="w_iou", dfl_loss_weight="w_dfl", pose_cls_loss_weight="w_pose_cls", pose_reg_loss_weight="w_pose_reg",
                 bbox_assigner_topk="topk", bbox_assigned_alpha="alpha", bbox_assigned_beta="beta")  # fmt: skip
    okw = {names.get(k, k): v for k, v in kw.items()}
    leaves = [t.detach().clone().requires_grad_(True) for t in raw[:4]]
    loss, items, (a_gt, a_score, a_crowd) = O.yolo_nas_pose_loss((*leaves, *raw[4:]), targets, sigmas, return_assignment=True, **okw)
    loss.backward()
    return items, [t.grad if t.grad is not None else torch.zeros_like(t) for t in leaves], a_gt, a_score, a_crowd


def _padded(targets, B):
    from super_gradients_b200.training.losses import max_pose_targets_host, pad_pose_targets_host

    return pad_pose_targets_host(targets, B, max(max_pose_targets_host(targets), 1))


def _restate(raw, targets, sigmas, kw, agt, asc):
    cl, rd, pc, pl, _a, ap, _n, st = raw
    gb, gp, _gc, _gv = _padded(targets, cl.shape[0])
    reg_max = rd.shape[-1] // 4 - 1
    return PC.pose_loss_given_assignment(cl, rd, pc, pl, ap, st, gb, gp, agt, asc, int((agt >= 0).sum()), torch.tensor(sigmas), reg_max, **_desc_kw(kw))


@pytest.mark.parametrize("kw_i", range(len(KWS)))
@pytest.mark.parametrize("seed,n_inst", [(0, (3, 0, 2)), (1, (1, 4, 1))])
def test_restatement_reproduces_the_oracle(kw_i, seed, n_inst):
    """Around the oracle's own assignment (crowd instances dropped from the positives, as the assigner leaves them), the fp64
    restatement gives the fp32 oracle's items and all four gradients."""
    kw = KWS[kw_i]
    raw, targets, sigmas = _random_case(seed, n_inst=n_inst)
    items, grads, a_gt, a_score, a_crowd = _oracle_with_assignment(raw, targets, sigmas, kw)
    agt = torch.where(a_crowd, -1, a_gt)
    assert int((agt >= 0).sum()) > 0 and bool(a_crowd.any())
    i64, *g64 = _restate(raw, targets, sigmas, kw, agt, a_score)
    torch.testing.assert_close(i64, items.double(), rtol=2e-5, atol=1e-7)
    for name, g, ref in zip(GRAD_NAMES, grads, g64):
        ok, worst, _ = DC.row_errors(_rows(g), _rows(ref), r=1e-4, a=1e-5)
        assert ok, f"{name}: {worst:.3e}"


@pytest.mark.parametrize("case", ["loss_default", "loss_oks_rescale_bce_giou", "loss_recipe"])
def test_restatement_reproduces_the_reference_golden(golden, case):
    """Around the stable fp32 assignment, the fp64 restatement gives the reference's recorded fp32 items and gradients
    (tests/golden/pose.pt).  The stable assigner first reproduces the oracle's assignment there."""
    g = golden("pose")[case]
    kw = g["kw"]
    _items, _grads, a_gt, a_score, a_crowd = _oracle_with_assignment(g["raw"], g["targets"], g["sigmas"], kw)
    cl, rd, pc, _pl, _a, ap, _n, st = g["raw"]
    B = cl.shape[0]
    gb, gp, gc, gv = _padded(g["targets"], B)
    pbox = DC.decode_fp32(rd, ap, st)
    for b in range(B):
        claim, pos = PC.pose_assign_stable(cl[b], pbox[b], pc[b], ap, gb[b], gp[b], gc[b], gv[b], torch.tensor(g["sigmas"]), kw.get("bbox_assigner_topk", 13), 1.0, 6.0,
                                           kw.get("assigner_multiply_by_pose_oks", False))  # fmt: skip
        assert torch.equal(claim, a_gt[b])
    agt = torch.where(a_crowd, -1, a_gt)
    i64, *g64 = _restate(g["raw"], g["targets"], g["sigmas"], kw, agt, a_score)
    torch.testing.assert_close(i64.float(), g["items"], rtol=2e-5, atol=1e-7)
    for name, got, ref in zip(GRAD_NAMES, g["grads"], g64):
        ok, worst, _ = DC.row_errors(_rows(got), _rows(ref), r=1e-4, a=1e-5)
        assert ok, f"{name}: {worst:.3e}"


def _flat_targets(c):
    """A padded decision case as the flat (boxes, joints, crowd) targets the oracle unpacks, every row (invalid ones too) in order."""
    B, n = c["gv"].shape
    img = torch.arange(B, dtype=torch.float32).repeat_interleave(n)
    boxes = torch.cat([img[:, None], c["gb"].reshape(-1, 4)], 1)
    joints = torch.cat([img[:, None, None].expand(-1, c["J"], 1), c["gp"].reshape(B * n, c["J"], 3)], 2)
    return boxes, joints, torch.stack([img, c["gc"].reshape(-1).float()], 1)


@pytest.mark.parametrize("oks", [False, True])
@pytest.mark.parametrize("seed", [6, 7])
def test_stable_assigner_matches_the_oracle(seed, oks):
    """On a crowded case with random boxes whose in-gt metrics leave no tie for torch.topk to order (positive metrics distinct in fp32,
    and zero ones only below the top 5), the stable
    fp32 assigner makes the oracle's decisions: the instance of every anchor, crowd instances included."""
    c = PC.pose_decision_case(2, 96, 128, 12, n_invalid=2, seed=seed, dark=False)
    g = torch.Generator().manual_seed(seed)
    c["reg"] = DC.off_grid_reg(torch.randn(c["reg"].shape, generator=g), c["ap"], c["st"], g)
    pbox = DC.decode_fp32(c["reg"], c["ap"], c["st"])
    for b in range(2):
        m = PC.pair_iou(c["gb"][b], pbox[b], c["gp"][b], c["pose"][b], c["sigmas"], oks).pow(6.0) * torch.sigmoid(c["cls"][b, :, 0])
        for r in c["gv"][b].nonzero().flatten().tolist():
            mr = m[r][PC._in_gts(c["ap"], c["gb"][b, r : r + 1])[0]]
            npos = int((mr > 0).sum())
            assert mr[mr > 0].unique().numel() == npos and (npos >= 5 or npos == mr.numel()), f"tied metrics in gt {r}"
    plog = torch.zeros(c["pose"].shape[:3])
    raw = (c["cls"], c["reg"], c["pose"], plog, None, c["ap"], None, c["st"].reshape(-1, 1))
    _items, _grads, a_gt, _a_score, _a_crowd = _oracle_with_assignment(raw, _flat_targets(c), c["sigmas"].tolist(), dict(assigner_multiply_by_pose_oks=oks, bbox_assigner_topk=5))
    for b in range(2):
        claim, _ = PC.pose_assign_stable(c["cls"][b], pbox[b], c["pose"][b], c["ap"], c["gb"][b], c["gp"][b], c["gc"][b], c["gv"][b], c["sigmas"], 5, 1.0, 6.0, oks)
        assert torch.equal(claim, a_gt[b]), b
    assert int((a_gt >= 0).sum()) > 20 and bool(c["gc"].bool()[torch.arange(2)[:, None], a_gt.clamp_min(0)][a_gt >= 0].any())


def test_constructed_and_decision_cases_hold_their_premises():
    """The builders assert their own premises (keypoint scenarios with and without crowd, far joints that underflow, degenerate areas
    next to the eps, crowds, invalid rows, padding, the all-invisible instance, OKS away from 0, exact ties).  They hold at every
    J / reg_max of the GPU tests, and the decision-case check refuses a broken case: the all-invisible instance made a crowd."""
    for J, reg_max in ((1, 7), (17, 16), (64, 31)):
        for above in (True, False):
            PC.constructed_case(J, reg_max, seed=J, norm_above_1=above)
    PC.pose_decision_case(2, 128, 160, 24, exact_ties=True)
    d = PC.pose_decision_case(2, 128, 160, 24, n_invalid=3, n_max=30)
    dark = (d["gv"].bool() & (d["gp"][..., 2] == 0).all(-1)).nonzero().tolist()
    assert len(dark) == 2
    with pytest.raises(AssertionError, match="all-invisible"):
        PC._decision_case_premises(dict(d, gc=d["gv"].clone()), 3, 4, dark, torch.full((2, d["L"]), -1), False)


def test_near_tie_excuse_needs_a_tie_at_the_boundary():
    """A differing decision is excused only when the last anchor taken and the first one left agree to 1e-6 in fp64 and the anchor is
    one of them: a top-1 that takes the runner-up of a clear winner is a real disagreement, with OKS in the pair IoU or without."""
    gb = torch.tensor([[0.0, 0.0, 64.0, 64.0]])
    gp = torch.tensor([[[20.0, 20.0, 2.0], [40.0, 30.0, 1.0]]])
    ap = torch.tensor([[12.0, 12.0], [20.0, 20.0], [28.0, 28.0]])
    pbox = torch.tensor([[1.0, 1.0, 63.0, 63.0], [16.0, 16.0, 24.0, 24.0], [26.0, 26.0, 30.0, 30.0]])
    pose = torch.tensor([[[21.0, 20.0], [40.0, 31.0]], [[25.0, 20.0], [40.0, 36.0]], [[30.0, 20.0], [45.0, 30.0]]])
    sig, cls = torch.tensor([0.025, 0.107]), torch.zeros(3, 1)
    for oks in (False, True):
        assert PC.explain_difference(0, -1, 0, cls, pbox, pose, ap, gb, gp, sig, 1, 1.0, 6.0, oks) is None
        assert PC.explain_difference(1, 0, -1, cls, pbox, pose, ap, gb, gp, sig, 1, 1.0, 6.0, oks) is None
    # anchors 0 and 1 with the same box and pose and logits 1e-7 apart: a near-tie either way round
    pbox[1], pose[1], cls[1, 0] = pbox[0], pose[0], 1e-7
    for oks in (False, True):
        assert PC.explain_difference(0, -1, 0, cls, pbox, pose, ap, gb, gp, sig, 1, 1.0, 6.0, oks) is not None
        assert PC.explain_difference(1, 0, -1, cls, pbox, pose, ap, gb, gp, sig, 1, 1.0, 6.0, oks) is not None
    # two instances over one anchor: a clear pair-IoU winner is no tie, equal boxes and poses are
    gb2, gp2 = torch.cat([gb, gb + 5.0]), torch.cat([gp, gp])
    assert PC.explain_difference(0, 0, 1, cls, pbox, pose, ap, gb2, gp2, sig, 2, 1.0, 6.0, True) is None
    gb2[1] = gb2[0]
    assert "pair IoU tie" in PC.explain_difference(0, 0, 1, cls, pbox, pose, ap, gb2, gp2, sig, 2, 1.0, 6.0, True)


# ------------------------------------------------------------------------------------------------ the host build of the arithmetic
LOSS_SWITCHES = [dict(iou_type=1, cls_type=0, pose_cls_type=0, rescale_with_score=False), dict(iou_type=0, cls_type=1, pose_cls_type=1, rescale_with_score=True),
                 dict(iou_type=1, cls_type=0, pose_cls_type=1, rescale_with_score=True, w_dfl=0.01, w_pose_reg=34.0)]  # fmt: skip


def _host_vs_fp64(tmp_path, c, gc, gv, n_max, J, reg_max, sw, oks, topk=13):
    d = K.pose_loss_desc(c["cls"].shape[0], c["cls"].shape[1], J, reg_max, n_max, topk=topk, multiply_by_oks=oks, **sw)
    h = host_pose_loss.run(host_pose_loss.build(str(tmp_path)), d, c["cls"], c["reg"], c["pose"], c["plog"], c["ap"], c["st"], c["gb"], c["gp"], gc, gv, c["sigmas"])
    agt = h["assigned_gt"].long()
    i64, *g64 = PC.pose_loss_given_assignment(c["cls"], c["reg"], c["pose"], c["plog"], c["ap"], c["st"], c["gb"], c["gp"], agt, h["assigned_score"], int((agt >= 0).sum()), c["sigmas"],
                                              reg_max, **sw)  # fmt: skip
    slacks = PC.logit_slacks(c["cls"], c["plog"], c["gp"], agt, h["assigned_score"], int((agt >= 0).sum()), **sw)
    return h, agt, i64, g64, slacks


@pytest.mark.skipif(shutil.which("g++") is None, reason="g++ not available")
@pytest.mark.parametrize("sw_i", range(len(LOSS_SWITCHES)))
@pytest.mark.parametrize("J,reg_max", [(1, 7), (17, 16), (64, 31)])
def test_host_build_on_constructed_cases(tmp_path, J, reg_max, sw_i):
    """The host build assigns the constructed case's instances (one per anchor, crowds among them) itself; its loss on that
    assignment is the fp64 restatement's within the per-row bound."""
    c = PC.constructed_case(J, reg_max, seed=J + reg_max)
    gv = (c["gb"].sum(-1) > 0).to(torch.uint8)
    h, agt, i64, g64, slacks = _host_vs_fp64(tmp_path, c, c["crowd"].to(torch.uint8), gv, c["gb"].shape[1], J, reg_max, LOSS_SWITCHES[sw_i], oks=sw_i == 2)
    assert int((agt >= 0).sum()) > 20
    PC.check_loss(f"host constructed J={J} reg_max={reg_max} {LOSS_SWITCHES[sw_i]}", h["items"], h["grads"], i64, g64, slacks)


@pytest.mark.skipif(shutil.which("g++") is None, reason="g++ not available")
@pytest.mark.parametrize("oks", [False, True])
def test_host_build_on_decision_cases(tmp_path, oks):
    """The host build on a crowded 256 x 192 case: its decisions are the stable assigner's (up to counted fp64 near-ties), its
    positives and normaliser are its assignment's, and its loss is the fp64 restatement's within the per-row bound."""
    c = PC.pose_decision_case(2, 192, 256, 40, n_invalid=3, n_max=48, seed=3 + oks)
    g = torch.Generator().manual_seed(9)
    c["plog"] = torch.randn(c["pose"].shape[:3], generator=g) * 2.0
    c["reg"] = DC.off_grid_reg(torch.randn(c["reg"].shape, generator=g) * 1.5, c["ap"], c["st"], g)
    sw = LOSS_SWITCHES[1 if oks else 0]
    h, agt, i64, g64, slacks = _host_vs_fp64(tmp_path, c, c["gc"], c["gv"], c["n_max"], c["J"], c["reg_max"], sw, oks)
    assert int((agt >= 0).sum()) > 50
    assert float(h["sums"][6]) == int((agt >= 0).sum())
    assert abs(float(h["sums"][3]) - float(h["assigned_score"].double().sum())) <= 1e-6 * max(float(h["sums"][3]), 1.0)
    PC.check_loss(f"host decision oks={oks}", h["items"], h["grads"], i64, g64, slacks)
    pbox = DC.decode_fp32(c["reg"], c["ap"], c["st"])
    ties = []
    for b in range(2):
        _, pos = PC.pose_assign_stable(c["cls"][b], pbox[b], c["pose"][b], c["ap"], c["gb"][b], c["gp"][b], c["gc"][b], c["gv"][b], c["sigmas"], 13, 1.0, 6.0, oks)
        for l in (pos != agt[b]).nonzero().flatten().tolist():
            why = PC.explain_difference(l, int(agt[b, l]), int(pos[l]), c["cls"][b], pbox[b], c["pose"][b], c["ap"], c["gb"][b], c["gp"][b], c["sigmas"], 13, 1.0, 6.0, oks)
            assert why, f"image {b} anchor {l}: host {int(agt[b, l])}, oracle {int(pos[l])}"
            ties.append(why)
    print(f"host decision oks={oks}: {int((agt >= 0).sum())} positives, {len(ties)} near-tie differences")


# ------------------------------------------------------------------------------------------------ host validation
def test_assigners_refuse_a_metric_row_above_200_KB(monkeypatch):
    """A 1600 x 1600 input has L = 52500 anchors: the top-k's shared-memory metric row would take 205 KB.  Both task-aligned
    assigners refuse that in host validation, before any launch (host tensors only: no kernel runs here)."""
    monkeypatch.setattr(K, "_stream", lambda: None)
    Lc = sum(h * w for h, w in DC.level_shapes(1600, 1600))
    assert Lc == 52500
    B, n, J = 1, 2, 17
    cls, reg, pose = torch.zeros(B, Lc), torch.zeros(B, Lc, 68), torch.zeros(B, Lc, J, 2)
    ap, st = torch.zeros(Lc, 2), torch.ones(Lc)
    gb, gp, gc, gv = torch.zeros(B, n, 4), torch.zeros(B, n, J, 3), torch.zeros(B, n, dtype=torch.uint8), torch.ones(B, n, dtype=torch.uint8)
    for call in (lambda: K.pose_tal_assign(K.pose_loss_desc(B, Lc, J, 16, n), cls, reg, pose, ap, st, gb, gp, gc, gv, PC.sigmas_for(J), torch.zeros(8, dtype=torch.float64)),
                 lambda: K.tal_assign(K.loss_desc(B, Lc, 80, 16, n), torch.zeros(B, Lc, 80), reg, ap, st, gb, torch.zeros(B, n, dtype=torch.int32), gv, torch.zeros(4, dtype=torch.float64))):  # fmt: skip
        with pytest.raises(L.SgbError) as e:
            call()
        assert "code -1" in str(e.value) and "too many anchors" in str(e.value), str(e.value)
    lib = L.load()
    rc = lib.sgb_pose_tal_assign(ctypes.byref(K.pose_loss_desc(B, Lc, J, 16, n)), *([None] * 14), 0, None)
    assert rc == -1 and b"too many anchors" in lib.sgb_last_error()
