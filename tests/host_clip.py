"""g++ build of tests/host_kernels/clip_host.cpp (the clip_grad_norm arithmetic of csrc/optim_math.cuh) behind the call signature
of kernels.clip_grad_norm, on host tensors.  -ffp-contract=off keeps every separate multiply and add rounded on its own, as the
device intrinsics do."""
import ctypes
import os
import subprocess
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_LIB = {}
_P, _I = ctypes.c_void_p, ctypes.c_int32


def install(monkeypatch):
    """Routes kernels.clip_grad_norm to this host build (on top of tests/cpu_backend.install_training)."""
    from super_gradients_b200 import kernels as K

    monkeypatch.setattr(K, "clip_grad_norm", clip_grad_norm)


def lib():
    if "h" not in _LIB:
        d = tempfile.mkdtemp(prefix="sgb_clip_host_")
        so = os.path.join(d, "clip_host.so")
        subprocess.run(["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-shared", "-fPIC", "-x", "c++", os.path.join(ROOT, "tests", "host_kernels", "clip_host.cpp"),
                        "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "super_gradients_b200", "csrc"), "-o", so], check=True)  # fmt: skip
        h = ctypes.CDLL(so)
        h.clip_total_norm_host.argtypes, h.clip_total_norm_host.restype = [ctypes.c_double], ctypes.c_float
        h.clip_coef_host.argtypes, h.clip_coef_host.restype = [ctypes.c_float, ctypes.c_float], ctypes.c_float
        h.clip_grad_norm_host.argtypes = [_P, _P, _I, _P, _I, _I, ctypes.c_float, _P, _P]
        _LIB["h"] = h
    return _LIB["h"]


def _p(t):
    assert t.is_contiguous() and not t.is_cuda
    return ctypes.c_void_p(t.data_ptr())


def clip_grad_norm(g, chunks, hp, gs_col, max_norm, partials, norm_coef):
    assert hp.dim() == 2 and hp.shape[0] == 2
    lib().clip_grad_norm_host(_p(g), _p(chunks), chunks.shape[0], _p(hp), hp.shape[1], int(gs_col), float(max_norm), _p(partials), _p(norm_coef))


def total_norm(grad_sqsum: float) -> float:
    return lib().clip_total_norm_host(grad_sqsum)


def coef(total: float, max_norm: float) -> float:
    return lib().clip_coef_host(total, max_norm)
