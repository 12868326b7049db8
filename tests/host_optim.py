"""g++ build of tests/host_kernels/optim_host.cpp (csrc/optim_math.cuh, the kernels' per-element arithmetic) behind the call
signatures of kernels.adam_step / rmsprop_step / rmsprop_tf_step / lion_step / lamb_grad_sqnorm / lamb_step, on host tensors.
-ffp-contract=off keeps every separate multiply and add rounded on its own, as the device intrinsics do."""
import ctypes
import os
import subprocess
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_LIB = {}
_P, _L, _I = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int32


KERNELS = ("adam_step", "rmsprop_step", "rmsprop_tf_step", "lion_step", "lamb_grad_sqnorm", "lamb_step")


def install(monkeypatch):
    """Routes the optimizer wrappers of kernels.py to this host build (on top of tests/cpu_backend.install_training, which covers the
    rest of the train step)."""
    from super_gradients_b200 import kernels as K

    for name in KERNELS:
        monkeypatch.setattr(K, name, globals()[name])


def lib():
    if "h" not in _LIB:
        d = tempfile.mkdtemp(prefix="sgb_optim_host_")
        so = os.path.join(d, "optim_host.so")
        subprocess.run(["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-shared", "-fPIC", "-x", "c++", os.path.join(ROOT, "tests", "host_kernels", "optim_host.cpp"),
                        "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "super_gradients_b200", "csrc"), "-o", so], check=True)  # fmt: skip
        h = ctypes.CDLL(so)
        h.adam_host.argtypes = [_P, _P, _P, _P, _L, _P]
        h.rmsprop_host.argtypes = [_P, _P, _P, _P, _P, _L, _P]
        h.rmsprop_tf_host.argtypes = [_P, _P, _P, _P, _P, _L, _P]
        h.lion_host.argtypes = [_P, _P, _P, _L, _P]
        h.lamb_grad_sqnorm_host.argtypes = [_P, _P, _I, _P, _P]
        h.lamb_step_host.argtypes = [_P, _P, _P, _P, _P, _L, _P, _I, _P, _P]
        _LIB["h"] = h
    return _LIB["h"]


def _p(t):
    if t is None:
        return None
    assert t.is_contiguous() and not t.is_cuda
    return ctypes.c_void_p(t.data_ptr())


def adam_step(p, g, m, v, hp):
    lib().adam_host(_p(p), _p(g), _p(m), _p(v), p.numel(), _p(hp))


def rmsprop_step(p, g, square_avg, buf, grad_avg, hp):
    lib().rmsprop_host(_p(p), _p(g), _p(square_avg), _p(buf), _p(grad_avg), p.numel(), _p(hp))


def rmsprop_tf_step(p, g, square_avg, buf, grad_avg, hp):
    lib().rmsprop_tf_host(_p(p), _p(g), _p(square_avg), _p(buf), _p(grad_avg), p.numel(), _p(hp))


def lion_step(p, g, m, hp):
    lib().lion_host(_p(p), _p(g), _p(m), p.numel(), _p(hp))


def lamb_grad_sqnorm(g, chunks, hp, partials):
    lib().lamb_grad_sqnorm_host(_p(g), _p(chunks), chunks.shape[0], _p(hp), _p(partials))


def lamb_step(p, g, m, v, update, n_decay, chunks, hp, partials):
    lib().lamb_step_host(_p(p), _p(g), _p(m), _p(v), _p(update), int(n_decay), _p(chunks), chunks.shape[0], _p(hp), _p(partials))
