"""The oracle's NMS post-processing (oracle/sg_oracle.py) against the unmodified reference's outputs on every edge case of
tests/nms_cases.py (tests/golden/nms_edges.pt), so that the GPU test's bit-exact comparison with the oracle rests on a validated
contract.

The oracle is exact except where the reference itself is not determined: torch.topk orders (and, at a cut inside a run of equal
scores, chooses) tied entries in an implementation-defined way, and torchvision's per-class path ends with an unstable sort.  Where
the cut falls inside a run of equal scores, both sides must select the same number of candidates with the same score multiset
before NMS; where only the order of equal scores is open, both must keep the same rows in the same score order."""
import contextlib

import numpy as np
import pytest
import torch

import nms_cases as N
from oracle import sg_oracle as O


@contextlib.contextmanager
def _capture_pre_nms():
    """Records the scores of every outermost NMS call the oracle makes (batched_nms_numpy calls nms_numpy)."""
    calls, depth = [], [0]
    orig = {k: getattr(O, k) for k in ("nms_numpy", "batched_nms_numpy")}

    def wrap(f):
        def g(boxes, scores, *a):
            if depth[0] == 0:
                calls.append(np.asarray(scores, np.float32).copy())
            depth[0] += 1
            try:
                return f(boxes, scores, *a)
            finally:
                depth[0] -= 1

        return g

    for k, f in orig.items():
        setattr(O, k, wrap(f))
    try:
        yield calls
    finally:
        for k, f in orig.items():
            setattr(O, k, f)


def oracle_outputs(case):
    """Per image: rows [N, 6] (ppyoloe, yolox; yolox None when nothing survives) or (poses, scores, boxes) (pose); and the scores
    handed to NMS per image."""
    p = case["params"]
    with _capture_pre_nms() as calls:
        if case["kind"] == "ppyoloe":
            rows, _ = O.ppyoloe_postprocess(case["boxes"], case["scores"], **p)
        elif case["kind"] == "yolox":
            rows = O.yolox_non_max_suppression(case["pred"], **p)
        else:
            rows, _ = O.yolo_nas_pose_postprocess(case["boxes"], case["conf"], case["coords"], case["jscores"], **p)
    it = iter(calls)
    pre = [next(it) if s.size else np.zeros(0, np.float32) for s in N.candidate_scores(case)]
    return rows, pre


def _bits(x):
    return np.ascontiguousarray(np.asarray(x, np.float32)).view(np.int32)


def _canon(rows):
    """Rows sorted by (score desc, then every column's bits): the order inside runs of equal scores no longer matters."""
    b = _bits(rows)
    return b[np.lexsort(tuple(b[:, c] for c in (5, 3, 2, 1, 0)) + (-rows[:, 4],))]


@pytest.mark.parametrize("name", list(N.CASES))
def test_oracle_reproduces_reference(golden, name):
    case = N.build(name)
    ref, ref_pre = N.reference_outputs(case, golden("nms_edges")[name])
    got, got_pre = oracle_outputs(case)
    tied, exact = N.tied_cut(case), N.order_defined(case)
    assert len(got) == len(ref)
    for b in range(len(ref)):
        if tied[b]:
            # the reference's choice among the tied entries is implementation defined: same count, same score multiset (by value:
            # which of the equal +0.0 / -0.0 scores are chosen is open too)
            assert np.array_equal(np.sort(got_pre[b])[::-1], ref_pre[b].numpy()), (name, b)
            continue
        r, g = ref[b], got[b]
        if case["kind"] == "pose":
            r, g = torch.cat([r[2], r[1][:, None], r[0].flatten(1)], 1).numpy(), np.concatenate([g[2], g[1][:, None], g[0].reshape(len(g[0]), -1)], 1)
            # (boxes, score, poses) as one row per detection; the score sits in column 4 as in the detection rows
        elif case["kind"] == "yolox" and (r is None or g is None):
            assert r is None and g is None, (name, b)
            continue
        else:
            r = r.numpy()
        assert g.shape == r.shape, (name, b, g.shape, r.shape)
        if exact[b]:
            np.testing.assert_array_equal(_bits(g), _bits(r), err_msg=f"{name} image {b}")
        else:
            np.testing.assert_array_equal(_canon(g), _canon(r), err_msg=f"{name} image {b}")
            np.testing.assert_array_equal(_bits(g[:, 4]), _bits(r[:, 4]))


def test_cases_reach_their_edges():
    """The inputs do what their names say: the planted candidate counts sit at top_k and top_k + 1, the tie and threshold cases
    have their runs and ulp neighbours, the IoU pairs sit on and beside the threshold, and the unaligned rows are unaligned."""
    for name in ("direct_k512", "direct_k1001", "prefilter_k1024", "prefilter_unaligned_k1010"):
        c = N.build(name)
        k = N.top_k_of(c)
        assert [s.size for s in N.candidate_scores(c)][:2] == [k, k + 1], name
    c = N.build("prefilter_unaligned_k1010")
    n = c["scores"].shape[1] * c["scores"].shape[2]
    assert n > 4 * N.PF_SLICE and n % 4 != 0
    for name in ("tied_prefilter", "tied_direct", "all_equal_multi", "signed_zero_topk", "pose_tied_topk"):
        assert all(N.tied_cut(N.build(name))), name
    c = N.build("tied_prefilter")
    s = np.sort(N.candidate_scores(c)[0])[::-1]
    assert (s == s[999]).sum() > 128  # the run at the cut is longer than a warp's 4 x 32 items
    t = np.float32(0.3)
    for name in ("thr_ulps_multi", "thr_ulps_single"):
        v = set(N.build(name)["scores"].numpy().ravel().tolist())
        assert {float(np.nextafter(t, np.float32(0))), float(t), float(np.nextafter(t, np.float32(1)))} <= v
    for target in (0.5, 0.65):
        for where, pairs in N.iou_pairs(target).items():
            f = np.float32(target)
            want = {"below": np.nextafter(f, np.float32(0)), "at": f, "above": np.nextafter(f, np.float32(1))}[where]
            assert all(N._ovr32(a, b) == want for a, b in pairs)
    # fp32(0.65) < 0.65 < its upper neighbour, so exactly the "above" pairs suppress; at 0.5 the fp32 value is exact and ">" keeps it
    assert float(np.float32(0.65)) < 0.65 < float(np.nextafter(np.float32(0.65), np.float32(1)))
    z = N.build("signed_zero_single")["scores"][..., 0]
    assert bool(((z == 0) & torch.signbit(z)).any()) and bool(((z == 0) & ~torch.signbit(z)).any())
