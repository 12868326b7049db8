"""Test infrastructure: builds tests/host_kernels/distance_match_host.cpp (serial host driver around the distance matching of
super_gradients_b200/csrc/detection_match_math.cuh) with g++ and exposes it with the signature of
kernels.detection_distance_matching -- the CPU stand-in of the distance matching kernel."""
import ctypes
import os
import subprocess
import tempfile

import torch

from super_gradients_b200 import kernels as K

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_LIB = {}


def _handle():
    if "h" not in _LIB:
        d = tempfile.mkdtemp(prefix="sgb_distance_host_")
        so = os.path.join(d, "distance_match_host.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", os.path.join(ROOT, "tests", "host_kernels", "distance_match_host.cpp"), "-I", os.path.join(ROOT, "include"),
                        "-I", os.path.join(ROOT, "super_gradients_b200", "csrc"), "-o", so], check=True)  # fmt: skip
        _LIB["h"] = ctypes.CDLL(so)
    return _LIB["h"]


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def detection_distance_matching(preds, pred_count, targets, target_count, crowd, crowd_count, thresholds, metric, height, width, top_k=100, denormalize_targets=True):
    if crowd is not None and crowd.shape[1] == 0:
        crowd = crowd_count = None
    thresholds = torch.as_tensor(thresholds, dtype=torch.float32).reshape(-1).contiguous()
    preds, targets = preds.contiguous().float(), targets.contiguous().float()
    d = K.match_desc(preds, targets, crowd, thresholds.numel(), height, width, top_k, denormalize_targets)
    matched = torch.empty((d.B, d.max_preds, d.n_thresholds), dtype=torch.uint8)
    ignore = torch.empty_like(matched)
    rc = _handle().distance_match_host(ctypes.byref(d), K.DISTANCE_METRICS[metric], _p(preds), _p(pred_count), _p(targets), _p(target_count), _p(crowd), _p(crowd_count), _p(thresholds),
                                       _p(matched), _p(ignore))  # fmt: skip
    assert rc == 0
    return matched, ignore


def nearest_free_target_lanes(metric, pbox, cls_p, thr, tbox, tcls, taken):
    h = _handle()
    h.nearest_free_target_lanes.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_float, ctypes.c_float, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
    v = torch.zeros(1)
    t = h.nearest_free_target_lanes(K.DISTANCE_METRICS[metric], _p(pbox), float(cls_p), float(thr), _p(tbox), _p(tcls), _p(taken), tbox.shape[0], _p(v))
    return t, float(v)
