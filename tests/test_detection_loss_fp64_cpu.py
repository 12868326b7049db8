"""CPU checks of the fp64 loss restatement in detection_loss_cases.py, and of the host validation of the loss entry points.

The restatement (`loss_given_assignment`) is what the GPU tests of csrc/loss.cu compare against element by element, so here it is
pinned to the oracle's full PPYoloELoss (GIoU and CIoU) and to the reference's own fp32 outputs in tests/golden/loss.pt."""
import ctypes
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import detection_loss_cases as DC  # noqa: E402
from oracle import sg_oracle as O  # noqa: E402
from super_gradients_b200 import kernels as K  # noqa: E402
from super_gradients_b200 import lib as L  # noqa: E402


def _random_batch(seed, B=3, C=6):
    g = torch.Generator().manual_seed(seed)
    _, ap, nums, st = O.anchors_for_levels([(12, 12), (6, 6), (3, 3)], (8, 16, 32))
    Lc = sum(nums)
    cls = torch.randn(B, Lc, C, generator=g, dtype=torch.float64) * 1.5 - 1.0
    reg = torch.randn(B, Lc, 68, generator=g, dtype=torch.float64)
    rows = []
    for b in range(B):
        for _ in range(2 + 2 * b):
            cx, cy = (torch.rand(2, generator=g) * 60 + 18).tolist()
            w, h = (torch.rand(2, generator=g) * 40 + 6).tolist()
            rows.append([b, int(torch.randint(0, C, (1,), generator=g)), cx, cy, w, h])
    return cls, reg, ap, nums, st, torch.tensor(rows), C


@pytest.mark.parametrize("iou_type", ["giou", "ciou"])
def test_restatement_reproduces_oracle_loss(iou_type):
    """Around the oracle's own assignment, loss_given_assignment gives the oracle's items and gradients (both in fp64)."""
    cls, reg, ap, nums, st, targets, C = _random_batch(1)
    cls_r, reg_r = cls.clone().requires_grad_(True), reg.clone().requires_grad_(True)
    loss, items, (al, ab, asc) = O.ppyoloe_loss((cls_r, reg_r, None, ap.double(), nums, st.double()), targets, C, iou_type=iou_type, return_assignment=True)
    loss.backward()
    assert int((al != C).sum()) > 20
    i64, gc, gr = DC.loss_given_assignment(cls, reg, ap, st, al, ab, asc.sum(-1), C, 16, iou_type=0 if iou_type == "giou" else 1)
    torch.testing.assert_close(i64, items.double(), rtol=1e-12, atol=1e-14)
    torch.testing.assert_close(gc, cls_r.grad, rtol=1e-10, atol=1e-14)
    torch.testing.assert_close(gr, reg_r.grad, rtol=1e-10, atol=1e-14)


@pytest.mark.parametrize("case", ["regular", "ragged_with_empty", "no_targets"])
def test_restatement_reproduces_reference_golden(golden, case):
    """Around the reference's assignment, the fp64 restatement gives the reference's fp32 items and gradients (tests/golden/loss.pt)."""
    G = golden("loss")
    g = G[case]
    C = g["cls_logits"].shape[2]
    i64, gc, gr = DC.loss_given_assignment(g["cls_logits"], g["reg_distri"], G["anchor_points"], G["stride_tensor"], g["assigned_labels"], g["assigned_bboxes"], g["assigned_scores"].sum(-1), C, 16)
    torch.testing.assert_close(i64.float(), g["items"], rtol=1e-5, atol=1e-7)
    for got, ref in ((g["g_cls"], gc), (g["g_reg"], gr)):
        ok, worst_row, _ = DC.row_errors(got, ref, r=1e-4, a=1e-5)
        assert ok, worst_row


def test_constructed_and_decision_cases_hold_their_premises():
    """The constructed assignment hits every scenario with a finite fp64 loss; the decision cases' reg logits decode exactly to the
    intended k or k + 1/2 bins in fp32, so kernel and oracle see the same boxes."""
    c = DC.constructed_case(80, 16)
    pos = c["al"] != 80
    assert int(pos.sum()) > 300 and bool((c["asc"][pos] == 0).any()) and float(c["asc"].sum()) > 1
    assert float(DC.constructed_case(1, 7, norm_above_1=False)["asc"].sum()) < 1
    for iou_type in (0, 1):
        items, gc, gr = DC.loss_given_assignment(c["cls"], c["reg"], c["ap"], c["st"], c["al"], c["ab"], c["asc"], 80, 16, iou_type=iou_type)
        assert bool(torch.isfinite(items).all() and torch.isfinite(gc).all() and torch.isfinite(gr).all())
    d = DC.decision_case(2, 128, 96, 40, n_invalid=3)
    ap, st = d["ap"], d["st"].reshape(-1, 1)
    want = torch.cat([ap / st - d["dist"][..., :2], ap / st + d["dist"][..., 2:]], -1) * st
    assert torch.equal(DC.decode_fp32(d["reg"], d["ap"], d["st"]).double(), want)
    assert bool((d["gb"] * 2 == torch.round(d["gb"] * 2)).all()) and int((d["gv"] == 0).sum()) == 6


def test_near_tie_excuse_needs_a_tie_at_the_boundary():
    """A decision that differs is excused only when the last anchor taken and the first one left have fp64 metrics within 1e-6 and
    the anchor is one of them: a top-1 that takes the runner-up of a clear winner is a real disagreement, for both anchors."""
    gb, gl = torch.tensor([[0.0, 0.0, 64.0, 64.0]]), torch.tensor([0], dtype=torch.int32)
    ap = torch.tensor([[12.0, 12.0], [20.0, 20.0], [28.0, 28.0]])
    pbox = torch.tensor([[1.0, 1.0, 63.0, 63.0], [16.0, 16.0, 24.0, 24.0], [26.0, 26.0, 30.0, 30.0]])
    cls = torch.zeros(3, 1)
    # oracle takes anchor 0, a kernel taking anchor 1 instead would differ on both
    assert DC.explain_difference(0, -1, 0, cls, pbox, ap, gb, gl, 1, 1.0, 6.0) is None
    assert DC.explain_difference(1, 0, -1, cls, pbox, ap, gb, gl, 1, 1.0, 6.0) is None
    # anchors 0 and 1 with the same box and logits 1e-7 apart: their metrics agree to ~3e-8, a near-tie either way round
    pbox[1], cls[1, 0] = pbox[0], 1e-7
    assert DC.explain_difference(0, -1, 0, cls, pbox, ap, gb, gl, 1, 1.0, 6.0) is not None
    assert DC.explain_difference(1, 0, -1, cls, pbox, ap, gb, gl, 1, 1.0, 6.0) is not None


def _host_loss_inputs(monkeypatch):
    monkeypatch.setattr(K, "_stream", lambda: None)
    B, Lc, C, n = 1, 21, 3, 2
    cls, reg = torch.zeros(B, Lc, C), torch.zeros(B, Lc, 68)
    ap, st = torch.zeros(Lc, 2), torch.ones(Lc)
    gb, gl, gv = torch.zeros(B, n, 4), torch.zeros(B, n, dtype=torch.int32), torch.ones(B, n, dtype=torch.uint8)
    return B, Lc, C, n, cls, reg, ap, st, gb, gl, gv, torch.zeros(4, dtype=torch.float64)


def _error_text(fn):
    with pytest.raises(L.SgbError) as e:
        fn()
    return str(e.value)


def test_loss_entry_points_refuse_topk_above_L(monkeypatch):
    """topk > L is refused before any launch (torch.topk raises in the reference).  Host tensors only: no kernel runs here."""
    B, Lc, C, n, cls, reg, ap, st, gb, gl, gv, sums = _host_loss_inputs(monkeypatch)
    msg = _error_text(lambda: K.tal_assign(K.loss_desc(B, Lc, C, 16, n, topk=Lc + 1), cls, reg, ap, st, gb, gl, gv, sums))
    assert "code -1" in msg and "topk" in msg
    al, ab, asc = torch.full((B, Lc), C, dtype=torch.int32), torch.zeros(B, Lc, 4), torch.zeros(B, Lc)
    d = K.loss_desc(B, Lc, C, 16, n, topk=Lc + 1)
    rc = L.load().sgb_dfl_iou_loss_fwd_bwd(ctypes.byref(d), cls.data_ptr(), reg.data_ptr(), ap.data_ptr(), st.data_ptr(), al.data_ptr(), ab.data_ptr(), asc.data_ptr(), sums.data_ptr(), 1.0, None, None, None)
    assert rc == -1
    # the pose assigner runs the same top-k loop; its descriptor check comes before any pointer is looked at
    lib = L.load()
    rc = lib.sgb_pose_tal_assign(ctypes.byref(K.pose_loss_desc(B, Lc, 17, 16, n, topk=Lc + 1)), *([None] * 14), 0, None)
    assert rc == -1 and b"topk" in lib.sgb_last_error()


@pytest.mark.skipif(torch.cuda.is_available(), reason="with a device the call would launch the assigner on host addresses")
def test_tal_assign_accepts_topk_equal_to_L(monkeypatch):
    """topk == L passes the host validation and gets as far as the first CUDA call (SGB_E_CUDA without a device)."""
    B, Lc, C, n, cls, reg, ap, st, gb, gl, gv, sums = _host_loss_inputs(monkeypatch)
    assert "code -3" in _error_text(lambda: K.tal_assign(K.loss_desc(B, Lc, C, 16, n, topk=Lc), cls, reg, ap, st, gb, gl, gv, sums))
