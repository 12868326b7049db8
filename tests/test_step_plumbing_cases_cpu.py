"""The oracles of tests/plumbing_cases.py against torch on the CPU, and the max-pool selection before and after it was made to match
torch's: the old selection records a padding tap for a border window that holds only NaN or -inf, which the stride-1 backward
then scatters to outside the image."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import plumbing_cases as PC


def test_round_bf16_matches_torch_away_from_the_double_rounding_band():
    g = np.random.default_rng(0)
    x = g.standard_normal(200_000) * np.exp2(g.integers(-140, 120, 200_000))
    x = np.concatenate([x, [0.0, -0.0, 1.0 + 2.0**-8, 1.0 + 3 * 2.0**-8, 2.0**-133, 1.5 * 2.0**127, np.inf, -np.inf]])
    r = PC.round_bf16(x)
    via32 = torch.from_numpy(x).float().bfloat16().double().numpy()  # fp64 -> fp32 -> bf16: rounds twice
    differ = r != via32
    assert not differ[~PC.near_bf16_midpoint(x)].any()
    # exact halves go to the even neighbour; the largest bf16 plus half an ulp overflows
    assert PC.round_bf16(1.0 + 2.0**-8) == 1.0 and PC.round_bf16(1.0 + 3 * 2.0**-8) == 1.0 + 2.0**-6
    assert PC.round_bf16(1.5 * 2.0**127) == 1.5 * 2.0**127 and np.isinf(PC.round_bf16((2 - 2.0**-8) * 2.0**127))
    # fp64 values that fp32 rounds onto a bf16 midpoint: one rounding from fp64 differs from two
    y = np.array([1.0 + 2.0**-8 + 2.0**-40, 1.0 + 2.0**-8 - 2.0**-40])
    assert list(PC.round_bf16(y)) == [1.0 + 2.0**-7, 1.0]
    assert np.isnan(PC.round_bf16(np.nan))
    b = PC.bf16_bits(r[np.isfinite(r)])
    assert (PC.bits_to_f64(b) == r[np.isfinite(r)]).all()


def _planes():
    g = torch.Generator().manual_seed(3)
    ties = torch.randint(-2, 3, (2, 3, 9, 11), generator=g).float().relu()
    nan = torch.randn(2, 3, 9, 11, generator=g)
    nan[torch.rand(nan.shape, generator=g) < 0.15] = float("nan")
    nan[0, 0, :2, :2] = float("nan")  # an all-NaN border window
    ninf = torch.randn(2, 3, 9, 11, generator=g)
    ninf[0, 1, :3, :3] = -float("inf")
    ninf[1, 2] = -float("inf")
    return {"ties": ties, "nan": nan, "ninf": ninf, "const": torch.full((1, 2, 7, 7), 0.5)}


@pytest.mark.parametrize("k,stride,pad", [(3, 1, 1), (5, 1, 2), (3, 2, 1), (9, 1, 4)])
def test_torch_taps_and_the_fixed_transcription_agree(k, stride, pad):
    for name, x in _planes().items():
        y, taps, flat = PC.torch_maxpool_taps(x, k, stride, pad)
        assert torch.equal(y.isnan(), F.max_pool2d(x, k, stride, pad).isnan())
        P, Q = y.shape[-2:]
        for n in range(x.shape[0]):
            for c in range(x.shape[1]):
                for sep in ([False, True] if stride == 1 else [False]):
                    yt, tt = PC.maxpool_transcribed(x[n, c].numpy(), k, stride, pad, fixed=True, separable=sep)
                    assert (tt == taps[n, c].numpy()).all(), (name, n, c, sep)
                    assert np.array_equal(yt, y[n, c].numpy(), equal_nan=True), (name, n, c, sep)
        # every tap lies inside the image
        r, s = taps // k, taps % k
        h = r + torch.arange(P).view(P, 1) * stride - pad
        w = s + torch.arange(Q).view(1, Q) * stride - pad
        assert bool(((h >= 0) & (h < x.shape[2]) & (w >= 0) & (w < x.shape[3])).all())


def test_torch_selection_rules():
    """The rules the kernels follow: ties to the first maximum in row-major order, NaN to the last NaN, all -inf to the first
    in-bounds element."""
    x = torch.tensor([[[[1.0, 2.0, 2.0], [2.0, 0.0, 1.0], [0.0, 2.0, 0.0]]]])
    assert PC.torch_maxpool_taps(x, 3, 1, 0)[1].item() == 1
    x = torch.tensor([[[[1.0, float("nan"), 2.0], [float("nan"), 5.0, 1.0], [0.0, 2.0, 0.0]]]])
    assert PC.torch_maxpool_taps(x, 3, 1, 0)[1].item() == 3
    x = torch.full((1, 1, 3, 3), -float("inf"))
    assert PC.torch_maxpool_taps(x, 3, 1, 1)[1][0, 0, 0, 0].item() == 4  # window (0, 0): first in-bounds tap is (1, 1)


@pytest.mark.parametrize("separable", [False, True])
def test_old_selection_records_a_padding_tap_for_non_finite_border_windows(separable):
    """Before the fix both forward kernels kept tap 0 for a window with nothing above -inf (a border window's tap 0 is padding, and
    the stride-1 backward adds at that tap: row -1 of the image) and never selected a NaN; after it they return torch's tap."""
    k, pad = 3, 1
    for fill, want_tap in ((float("nan"), 8), (-float("inf"), 4)):
        x = np.ones((5, 5), np.float32)
        x[:2, :2] = fill
        y_old, t_old = PC.maxpool_transcribed(x, k, 1, pad, fixed=False, separable=separable)
        y_new, t_new = PC.maxpool_transcribed(x, k, 1, pad, fixed=True, separable=separable)
        _, t_torch, _ = PC.torch_maxpool_taps(torch.from_numpy(x)[None, None], k, 1, pad)
        assert t_old[0, 0] == 0 and y_old[0, 0] == -np.inf  # tap (0, 0) = pixel (-1, -1)
        assert t_new[0, 0] == want_tap == t_torch[0, 0, 0, 0].item()
        assert np.isnan(y_new[0, 0]) == np.isnan(fill)
    # a NaN among finite values: the old selection returned the finite maximum, torch returns NaN
    x = np.arange(25, dtype=np.float32).reshape(5, 5)
    x[2, 2] = np.nan
    y_old, _ = PC.maxpool_transcribed(x, k, 1, pad, fixed=False, separable=separable)
    y_new, t_new = PC.maxpool_transcribed(x, k, 1, pad, fixed=True, separable=separable)
    assert y_old[2, 2] == 18 and np.isnan(y_new[2, 2]) and t_new[2, 2] == 4


def test_stem_patch_order_and_padding():
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 3, 7, 9, generator=g)
    out = PC.stem_patches_oracle(x, 3, 2, 1, 32).float()
    P, Q = out.shape[-2:]
    xp = F.pad(x, (1, 1, 1, 1))
    for p in range(P):
        for q in range(Q):
            for r in range(3):
                for s in range(3):
                    for c in range(3):
                        assert out[1, (r * 3 + s) * 3 + c, p, q] == xp[1, c, 2 * p + r, 2 * q + s].bfloat16().float()
    assert (out[:, 27:] == 0).all()


def test_weight_prepare_writes_cover_the_documented_layout():
    g = np.random.default_rng(2)
    K, C, R, S = 12, 5, 3, 3
    w = g.standard_normal((K, C, R, S))
    parts = dict((p, (o, v)) for p, o, v in PC.weight_prepare_writes(w, 0.5, K, C, R, S, 8, True, True))
    krsc = np.full(K * R * S * 8, np.nan)
    krsc[parts["krsc"][0]] = parts["krsc"][1]
    krsc = krsc.reshape(K, R, S, 8)
    want = w * 0.5
    want[np.arange(5), np.arange(5), 1, 1] += 1
    assert np.array_equal(krsc[..., :C], want.transpose(0, 2, 3, 1)) and (krsc[..., C:] == 0).all()
    crsk = np.full(C * R * S * 16, np.nan)
    crsk[parts["crsk"][0]] = parts["crsk"][1]
    crsk = crsk.reshape(C, R, S, 16)
    assert np.array_equal(crsk[..., :K], want.transpose(1, 2, 3, 0)) and (crsk[..., K:] == 0).all()
    # a 1 x 1 filter at tap 4 of 9-tap rows, columns from koff in kp-wide CRSK rows: nothing else written
    w1 = g.standard_normal((K, C, 1, 1))
    (_, ok, vk), (_, oc, vc) = PC.weight_prepare_writes(w1, 1.0, K, C, 1, 1, 8, False, True, kp=2 * K, koff=K, etaps=9, etap=4)
    assert sorted(ok) == sorted(k * 72 + 32 + c for k in range(K) for c in range(8))
    assert sorted(oc) == sorted((c * 9 + 4) * 2 * K + K + k for c in range(C) for k in range(K))
    assert PC.weight_item_elements(K, C, R, S, 8, True) == K * R * S * 8 + C * R * S * 16
