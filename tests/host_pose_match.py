"""Test infrastructure: builds tests/host_kernels/pose_match_host.cpp (serial host driver around the product header
super_gradients_b200/csrc/pose_match_math.cuh) with g++ and exposes it with the signature of kernels.pose_keypoint_matching."""
import ctypes
import os
import subprocess
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_LIB = {}


def _handle():
    if "h" not in _LIB:
        d = tempfile.mkdtemp(prefix="sgb_pose_match_host_")
        so = os.path.join(d, "pose_match_host.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", os.path.join(ROOT, "tests", "host_kernels", "pose_match_host.cpp"), "-I", os.path.join(ROOT, "include"),
                        "-I", os.path.join(ROOT, "super_gradients_b200", "csrc"), "-o", so], check=True)  # fmt: skip
        h = ctypes.CDLL(so)
        h.pose_match_host.argtypes = [ctypes.c_void_p] * 10 + [ctypes.c_int] * 6 + [ctypes.c_void_p] * 6
        h.pose_best_free_target_lanes.argtypes = [ctypes.c_void_p, ctypes.c_float, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
        _LIB["h"] = h
    return _LIB["h"]


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def pose_keypoint_matching(poses, scores, pred_count, gt_joints, gt_boxes, gt_areas, gt_flags, gt_count, sigmas, thresholds, top_k, oks_out=False):
    poses, scores, gt_joints, gt_boxes, gt_areas = (t.contiguous().float() for t in (poses, scores, gt_joints, gt_boxes, gt_areas))
    pred_count, gt_count = pred_count.contiguous().to(torch.int32), gt_count.contiguous().to(torch.int32)
    gt_flags, sigmas, thresholds = gt_flags.contiguous().to(torch.uint8), sigmas.contiguous().float(), thresholds.contiguous().float()
    B, P, J, _ = poses.shape
    M, T = gt_joints.shape[1], thresholds.numel()
    K = min(int(top_k), P)
    matched = torch.empty((B, K, T), dtype=torch.uint8)
    ignore = torch.empty_like(matched)
    used_scores = torch.empty((B, K))
    used_count = torch.empty(B, dtype=torch.int32)
    n_targets = torch.empty(B, dtype=torch.int32)
    oks = torch.full((B, K, M), float("nan")) if oks_out else None
    rc = _handle().pose_match_host(_p(poses), _p(scores), _p(pred_count), _p(gt_joints), _p(gt_boxes), _p(gt_areas), _p(gt_flags), _p(gt_count), _p(sigmas), _p(thresholds),
                                   B, P, M, J, T, int(top_k), _p(matched), _p(ignore), _p(used_scores), _p(used_count), _p(n_targets), _p(oks))  # fmt: skip
    assert rc == 0
    out = (matched, ignore, used_scores, used_count, n_targets)
    return out + (oks,) if oks_out else out


def best_free_target_lanes(oks_row, floor, taken):
    v = torch.zeros(1)
    t = _handle().pose_best_free_target_lanes(_p(oks_row), float(floor), _p(taken), oks_row.numel(), _p(v))
    return t, float(v)


def pad_golden_batch(images, J, no_areas=False):
    """A batch of tests/golden/pose_metrics.pt (per-image dicts of numpy arrays) -> the padded host tensors of the kernel's
    arguments (poses, scores, pred_count, gt_joints, gt_boxes, gt_areas, gt_flags, gt_count)."""
    B = len(images)
    P = max(max(len(im["scores"]) for im in images), 1)
    M = max(max(len(im["joints"]) for im in images), 1)
    poses, scores = torch.zeros(B, P, J, 3), torch.zeros(B, P)
    joints, boxes, areas = torch.zeros(B, M, J, 3), torch.zeros(B, M, 4), torch.zeros(B, M)
    flags = torch.zeros(B, M, dtype=torch.uint8)
    pc = torch.tensor([len(im["scores"]) for im in images], dtype=torch.int32)
    gc = torch.tensor([len(im["joints"]) for im in images], dtype=torch.int32)
    for b, im in enumerate(images):
        n, m = int(pc[b]), int(gc[b])
        poses[b, :n], scores[b, :n] = torch.from_numpy(im["poses"]).reshape(n, J, 3), torch.from_numpy(im["scores"])
        if m:
            joints[b, :m], boxes[b, :m] = torch.from_numpy(im["joints"]), torch.from_numpy(im["bboxes"])
            areas[b, :m] = torch.from_numpy(im["areas"])
            flags[b, :m] = torch.from_numpy(im["is_crowd"].astype("uint8")) | 2 | (0 if no_areas else 4)
    return poses, scores, pc, joints, boxes, areas, flags, gc


def assert_matches_golden(case, batch, out, oks_atol=2e-6):
    """(matched, ignore, used_scores, used_count, n_targets, oks) of one golden batch against the reference's per-image
    ImageKeypointMatchingResult (flags, scores and target counts exactly) and compute_oks matrices (within oks_atol)."""
    import numpy as np

    matched, ignore, used_scores, used_count, n_targets, oks = (t.cpu() for t in out)
    for b, (im, ref) in enumerate(zip(batch["images"], batch["results"])):
        if ref is None:
            assert int(used_count[b]) == 0 and len(im["joints"]) == 0
            continue
        n = len(ref[0])
        assert int(used_count[b]) == n, (b, int(used_count[b]), n)
        assert torch.equal(matched[b, :n].bool(), ref[0]), b
        assert torch.equal(ignore[b, :n].bool(), ref[1]), b
        assert torch.equal(used_scores[b, :n], ref[2].float()), b
        assert int(n_targets[b]) == int(ref[3]), b
        assert not matched[b, n:].any() and not ignore[b, n:].any() and not used_scores[b, n:].any()
        ign = (im["joints"][:, :, 2] == 0).all(1) | im["is_crowd"].astype(bool)
        m = len(im["joints"])
        for cols, want in ((np.nonzero(~ign)[0], batch["oks"][b]), (np.nonzero(ign)[0], batch["oks_crowd"][b])):
            got = oks[b, :n, :m][:, torch.from_numpy(cols)]
            assert got.shape == want.shape, (b, got.shape, want.shape)
            torch.testing.assert_close(got, want.float(), rtol=0, atol=oks_atol)


def install(monkeypatch, training=False):
    """cpu_backend's stand-in backend (install / install_training) plus this host driver in place of
    kernels.pose_keypoint_matching."""
    import cpu_backend

    from super_gradients_b200 import kernels as K

    (cpu_backend.install_training if training else cpu_backend.install)(monkeypatch)
    monkeypatch.setattr(K, "pose_keypoint_matching", pose_keypoint_matching)
