"""SgbConvDesc.centre_from at the C ABI, without a GPU: its place in the struct, and the host-side rules that refuse it
(SGB_E_INVALID) before any CUDA call.  An accepted descriptor gets past the validation to the first CUDA call, which fails here."""
import ctypes

import pytest
import torch

from super_gradients_b200 import lib as L

E_INVALID = -1


def _desc(c=32, k=64, r=3, stride=1, pad=1, centre_from=0, h=16):
    d = L.ConvDesc()
    d.N, d.H, d.W, d.C = 2, h, h, c
    d.K, d.R, d.S = k, r, r
    d.P = d.Q = (h + 2 * pad - r) // stride + 1
    d.stride, d.pad = stride, pad
    d.x_pitch, d.y_pitch = c, k
    d.centre_from = centre_from
    return d


def _calls(d):
    """rc of fprop, dgrad and wgrad on host buffers (validation only: nothing is read through them without a device)."""
    lib = L.load()
    buf = torch.zeros(1 << 16, dtype=torch.float32)
    p = ctypes.c_void_p(buf.data_ptr())
    ep = L.Epilogue()
    ep.stats_repl = 1
    return (lib.sgb_conv_fprop(ctypes.byref(d), p, p, p, ctypes.byref(ep), None),
            lib.sgb_conv_dgrad(ctypes.byref(d), p, p, p, 0, None),
            lib.sgb_conv_wgrad(ctypes.byref(d), p, p, p, None))  # fmt: skip


def test_centre_from_is_the_last_field():
    assert [f for f, _ in L.ConvDesc._fields_][-2:] == ["up2", "centre_from"]
    assert L.ConvDesc.centre_from.offset == 16 * 4 and ctypes.sizeof(L.ConvDesc) == 17 * 4
    assert L.ConvDesc().centre_from == 0  # a zeroed descriptor means: every tap


@pytest.mark.parametrize(
    "kw",
    [dict(centre_from=8), dict(centre_from=40), dict(centre_from=64), dict(centre_from=96), dict(centre_from=-16),
     dict(r=1, pad=0, centre_from=32), dict(stride=2, centre_from=32), dict(pad=0, centre_from=32)],
    ids=["not_16", "not_16b", "equals_K", "past_K", "negative", "1x1", "stride2", "pad0"],
)  # fmt: skip
def test_refused(kw):
    assert _calls(_desc(**kw)) == (E_INVALID,) * 3


@pytest.mark.parametrize("cf", [0, 16, 32, 48])
def test_accepted_up_to_the_device(cf):
    assert E_INVALID not in _calls(_desc(centre_from=cf))
