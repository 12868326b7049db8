"""Test infrastructure: builds tests/host_kernels/classification_host.cpp (serial host drivers around the product headers
super_gradients_b200/csrc/resample_math.cuh and classify_math.cuh) with g++ and exposes them with the signatures of
kernels.resample_crop_u8 / kernels.classify_rows, so that the product's processing, metrics and predict() run on the kernels'
arithmetic without a GPU (`install()`)."""
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
        d = tempfile.mkdtemp(prefix="sgb_classification_host_")
        so = os.path.join(d, "classification_host.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", os.path.join(ROOT, "tests", "host_kernels", "classification_host.cpp"), "-I", os.path.join(ROOT, "include"),
                        "-I", os.path.join(ROOT, "super_gradients_b200", "csrc"), "-o", so], check=True)  # fmt: skip
        h = ctypes.CDLL(so)
        P, I = ctypes.c_void_p, ctypes.c_int
        h.resample_crop_host.argtypes = [P, P, I, I, I, I, I, I, ctypes.c_double, P, P, P]
        h.classify_rows_host.argtypes = [P, I, ctypes.c_int64, I, P, P, I, P, P, P]
        _LIB["h"] = h
    return _LIB["h"]


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def resample_crop_u8(table_host, table, src, out, max_value=255.0, reverse_channels=False, mean=None, std=None):
    B, pitch, oh, ow = out.shape[0], out.shape[1], out.shape[2], out.shape[3]
    buf = torch.empty((B, oh, ow, pitch), dtype=torch.int16)
    m = s = None
    if mean is not None:
        m, s = (ctypes.c_float * 4)(*[float(v) for v in mean][:4]), (ctypes.c_float * 4)(*[float(v) for v in std][:4])
    rc = _handle().resample_crop_host(_p(table_host.contiguous()), _p(src.contiguous()), B, 3, oh, ow, pitch, 1 if reverse_channels else 0, float(max_value) if max_value else 0.0, m, s, _p(buf))
    assert rc == 0
    out.copy_(buf.view(torch.bfloat16).permute(0, 3, 1, 2))
    return out


def classify_rows(logits, target=None, k=1, counters=None, label=None, confidence=None):
    logits = logits.contiguous()
    N, C = logits.shape
    hard = soft = None
    if target is not None:
        if target.dim() == 1:
            hard = target.contiguous().to(torch.int64)
        else:
            soft = target.float().contiguous()
    host_counters = torch.zeros(4, dtype=torch.int64) if counters is not None else None
    lab = torch.empty(N, dtype=torch.int32) if label is not None else None
    conf = torch.empty(N, dtype=torch.float32) if confidence is not None else None
    lg = logits.view(torch.int16) if logits.dtype == torch.bfloat16 else logits.float()
    rc = _handle().classify_rows_host(_p(lg), 1 if logits.dtype == torch.bfloat16 else 0, N, C, _p(hard), _p(soft), int(k), _p(host_counters), _p(lab), _p(conf))
    assert rc == 0
    if counters is not None:
        counters += host_counters.to(counters.device)
    if label is not None:
        label.copy_(lab)
    if confidence is not None:
        confidence.copy_(conf)


def install(monkeypatch):
    """Routes the two classification kernels to the host build (on top of cpu_backend.install / install_training)."""
    monkeypatch.setattr(K, "resample_crop_u8", resample_crop_u8)
    monkeypatch.setattr(K, "classify_rows", classify_rows)
