"""The batched NMS kernel (csrc/nms.cu) on every edge case of tests/nms_cases.py, bit for bit against the oracle (which
tests/test_nms_edges_cpu.py pins to the unmodified reference): every launch path the host can pick, checked to be covered, the
one-launch direct path against the pre-filter / split launches, and the public callers."""
import ctypes

import numpy as np
import pytest
import torch

import nms_cases as N
from oracle import sg_oracle as O
from super_gradients_b200 import kernels as K
from super_gradients_b200 import lib as L

pytestmark = pytest.mark.gpu

DEV = "cuda"
PP = [n for n in N.CASES if N.build(n)["kind"] == "ppyoloe"]
MULTI = [n for n in PP if N.build(n)["params"]["multi_label_per_box"]]


def _bits(x):
    return np.ascontiguousarray(np.asarray(x, np.float32)).view(np.int32)


def _desc(case):
    p = case["params"]
    B, Lc, C = case["scores"].shape
    d = L.NmsDesc()
    d.B, d.L, d.ncls = B, Lc, C
    d.score_thr, d.iou_thr = float(p["score_threshold"]), float(p["nms_threshold"])
    d.top_k, d.max_out = int(p["nms_top_k"]), int(p["max_predictions"])
    d.multi_label, d.class_agnostic = int(p["multi_label_per_box"]), int(p["class_agnostic_nms"])
    d.thr_inclusive = int(not p["multi_label_per_box"])
    return d


def _kernel(case):
    p = case["params"]
    out, oidx, cnt = K.batched_nms(case["boxes"].to(DEV), case["scores"].to(DEV), p["score_threshold"], p["nms_threshold"], p["nms_top_k"], p["max_predictions"],
                                   p["multi_label_per_box"], p["class_agnostic_nms"])  # fmt: skip
    return out.cpu().numpy(), oidx.cpu().numpy(), cnt.cpu().numpy()


def _assert_matches_oracle(case, out, oidx, cnt, what):
    ref_rows, ref_idx = O.ppyoloe_postprocess(case["boxes"], case["scores"], **case["params"])
    for b in range(len(ref_rows)):
        n = ref_rows[b].shape[0]
        assert cnt[b] == n, (what, b, cnt[b], n)
        np.testing.assert_array_equal(oidx[b, :n], ref_idx[b], err_msg=f"{what} image {b}: selected candidates")
        np.testing.assert_array_equal(_bits(out[b, :n]), _bits(ref_rows[b]), err_msg=f"{what} image {b}: rows")  # NaN and -0.0 included
        assert (oidx[b, n:] == -1).all() and (out[b, n:] == 0).all()


@pytest.mark.parametrize("name", PP)
def test_kernel_bit_exact_vs_oracle(name):
    case = N.build(name)
    _assert_matches_oracle(case, *_kernel(case), name)


# ------------------------------------------------------------------------------------------------------------ path coverage
_STAGE_BYTES = 4 * 1024 * 4 + 1024 * 4 * 3 + 16  # sizeof(NmsStage)


def _a256(v):
    return (v + 255) // 256 * 256


def _expected_ws(d, prefilter, split):
    """sgb_nms_workspace_bytes' layout: [conf / labels | pre-filter candidates] [stages] [masks]."""
    head = d.B * d.L * 8
    if prefilter:
        n = d.L * d.ncls
        ns = -(-n // N.PF_SLICE)
        sl = (-(-n // ns) + 3) // 4 * 4
        head = max(head, d.B * (-(-n // sl)) * min(d.top_k, N.KMAX) * 8)
    ws = _a256(head) + 256
    if split:
        ws += _a256(d.B * _STAGE_BYTES) + d.B * N.KMAX * (N.KMAX // 64) * 8
    return ws


def launch_path(case):
    """(pre-filter, split) of a case: the host's rules (pre-filter: multi-label rows longer than 4 slices with a finite threshold;
    split: top_k > 512), checked against the workspace the host asks for -- the stages and IoU masks appear with the split, and the
    head grows with the pre-filter's candidate lists wherever those outgrow the single-label buffers."""
    d = _desc(case)
    pf = bool(d.multi_label and d.L * d.ncls > 4 * N.PF_SLICE and np.isfinite(d.score_thr))
    sp = d.top_k > 512
    ws = L.load().sgb_nms_workspace_bytes(ctypes.byref(d))
    assert ws == _expected_ws(d, pf, sp), (ws, pf, sp)
    assert ws != _expected_ws(d, pf, not sp)
    return pf, sp


def cells(case):
    """Per image with candidates: (pre-filter, split, NMS branch, radix select or take everything)."""
    pf, sp = launch_path(case)
    k = case["params"]["nms_top_k"]
    out = set()
    for s in N.candidate_scores(case):
        if s.size:
            out.add((pf, sp, N.nms_mode(case, min(s.size, k)), "radix" if s.size > k else "all"))
    return out


def test_cases_cover_every_reachable_path():
    covered = set()
    for name in PP:
        covered |= cells(N.build(name))
    # per-class NMS needs more than 1000 candidates, so top_k > 512: it only runs in the split form
    reachable = {(pf, sp, mode, sel) for pf in (False, True) for sp in (False, True) for mode in ("trick", "per_class", "agnostic") for sel in ("all", "radix")
                 if not (mode == "per_class" and not sp)}  # fmt: skip
    print("covered:", sorted(covered))
    assert covered == reachable, sorted(reachable - covered)


# ----------------------------------------------------------------------------------------------------------- path agreement
@pytest.mark.parametrize("name", MULTI)
def test_one_launch_direct_path_agrees(name):
    """A null workspace forces the one-launch direct scan (multi-label needs no workspace otherwise): bit-identical to the
    pre-filter / split launches K.batched_nms takes."""
    case = N.build(name)
    ref = _kernel(case)
    d = _desc(case)
    B, mo = d.B, d.max_out
    boxes, scores = case["boxes"].to(DEV).contiguous(), case["scores"].to(DEV).contiguous()
    out = torch.full((B, mo, 6), 7.0, device=DEV)
    oidx = torch.full((B, mo), 7, dtype=torch.int32, device=DEV)
    cnt = torch.full((B,), 7, dtype=torch.int32, device=DEV)
    L.call("sgb_batched_nms", ctypes.byref(d), K._ptr(boxes), K._ptr(scores), K._ptr(out), K._ptr(oidx), K._ptr(cnt), None, 0, K._stream())
    got = out.cpu().numpy(), oidx.cpu().numpy(), cnt.cpu().numpy()
    np.testing.assert_array_equal(got[2], ref[2])
    np.testing.assert_array_equal(got[1], ref[1])
    np.testing.assert_array_equal(_bits(got[0]), _bits(ref[0]))


# ------------------------------------------------------------------------------------------------------------ public callers
@pytest.mark.parametrize("name", ["direct_k1024", "prefilter_unaligned_k1010", "single_k1024", "tied_prefilter", "nan_box_trick", "nan_score_single", "signed_zero_single", "mixed_batch"])
def test_ppyoloe_callback(name):
    from super_gradients_b200.training.models.detection_models.pp_yolo_e import PPYoloEPostPredictionCallback

    case = N.build(name)
    ref_rows, _ = O.ppyoloe_postprocess(case["boxes"], case["scores"], **case["params"])
    got = PPYoloEPostPredictionCallback(**case["params"])(((case["boxes"].to(DEV), case["scores"].to(DEV)), None))
    assert len(got) == len(ref_rows)
    for g, r in zip(got, ref_rows):
        np.testing.assert_array_equal(_bits(g.cpu().numpy()), _bits(r))


@pytest.mark.parametrize("name", [n for n in N.CASES if N.build(n)["kind"] == "yolox"])
def test_yolox_non_max_suppression(name):
    """detection_utils.non_max_suppression asks the kernel for top_k = max_out = 1 024: exactly 1 024 candidates per image, on the
    pre-filter and the direct path, multi- and single-label (`>` given explicitly as thr_inclusive)."""
    from super_gradients_b200.training.utils.detection_utils import non_max_suppression

    case = N.build(name)
    ref = O.yolox_non_max_suppression(case["pred"], **case["params"])
    got = non_max_suppression(case["pred"].to(DEV), **case["params"])
    for g, r in zip(got, ref):
        assert (g is None) == (r is None)
        if r is not None:
            np.testing.assert_array_equal(_bits(g.cpu().numpy()), _bits(r))


def test_yolox_non_max_suppression_refuses_1025_candidates():
    from super_gradients_b200.training.utils.detection_utils import non_max_suppression

    case = N._yolox(175, 8400, 80, [3, 1025])
    with pytest.raises(L.SgbError):
        non_max_suppression(case["pred"].to(DEV), **case["params"])
    case = N._yolox(176, 3000, 6, [1025], multi=False)
    with pytest.raises(L.SgbError):
        non_max_suppression(case["pred"].to(DEV), **case["params"])


@pytest.mark.parametrize("name", [n for n in N.CASES if N.build(n)["kind"] == "pose"])
def test_pose_callback(name):
    from super_gradients_b200.training.models.pose_estimation_models import YoloNASPosePostPredictionCallback

    case = N.build(name)
    p = case["params"]
    ref, ref_idx = O.yolo_nas_pose_postprocess(case["boxes"], case["conf"], case["coords"], case["jscores"], **p)
    cb = YoloNASPosePostPredictionCallback(**p)
    dev = tuple(case[k].to(DEV) for k in ("boxes", "conf", "coords", "jscores"))
    _, _, idx, cnt = cb.forward_batched((dev, None))
    preds = cb((dev, None))
    for b, ((rposes, rscores, rboxes), kept) in enumerate(zip(ref, ref_idx)):
        n = int(cnt[b])
        assert n == kept.shape[0]
        np.testing.assert_array_equal(idx[b, :n].cpu().numpy(), kept)
        np.testing.assert_array_equal(_bits(preds[b].scores.cpu().numpy()), _bits(rscores))
        np.testing.assert_array_equal(_bits(preds[b].bboxes_xyxy.cpu().numpy()), _bits(rboxes))
        np.testing.assert_array_equal(_bits(preds[b].poses.cpu().numpy()), _bits(rposes))
