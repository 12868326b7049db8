"""The convolution entry points on every route of the wgmma / TMA engine (conv_sm100.cu) and the mma.sync engine (conv_mma.cu) against
the fp64 oracles of tests/conv_cases.py: every case of the matrix with exact integer operands (bit-exact results), a subset again
with real-valued operands against the derived bounds, and the route of every call (engine, kernel and the number of launches)
against the route mirror through the library's launch counters.  Operands are channel slices with poisoned neighbours where a
case says so: input channels outside the slice hold bf16 NaN, output channels outside it a sentinel that must survive.  Then a
replay of one train step of YOLO-NAS-S and of ResNet-50 and one YOLO-NAS-POSE inference forward, every convolution call checked
against the oracle and the mirror."""
import re
import zlib

import pytest
import torch

import conv_cases as CC
from bn_qarep_cases import resnet_step_record, yolo_nas_s_step_record

pytestmark = pytest.mark.gpu

DEV = "cuda"
CASES = CC.all_cases()
REAL = [c for c in CASES if c["real"]]


def K():
    from super_gradients_b200 import kernels

    return kernels


def L():
    from super_gradients_b200 import lib

    return lib.load()


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def dev_slice(t, pitch, off, fill, zero_to=None):
    """fp64 NCHW values -> bf16 NHWC view, channel slice [off, off + C) of a `pitch`-wide buffer whose other channels hold the bit
    pattern `fill` (channels [off + C, off + zero_to) hold zero: dy's padding, which the kernels read).  Returns (view, buffer)."""
    N, C, H, W = t.shape
    pitch = pitch or -(-C // 8) * 8
    buf = torch.full((N, H, W, pitch), fill, dtype=torch.int16, device=DEV).view(torch.bfloat16)
    if zero_to:
        buf[..., off + C : off + zero_to] = 0
    buf[..., off : off + C] = t.permute(0, 2, 3, 1).to(DEV).bfloat16()
    return buf.permute(0, 3, 1, 2)[:, off : off + C], buf


def outside(buf, off, C):
    return torch.cat([buf[..., :off], buf[..., off + C :]], -1)


def run_case(c, o):
    """Runs case c on operands o through the kernels' front ends; returns (outputs for verify_*, launch-counter deltas)."""
    k, lib = K(), L()
    op = c["op"]
    N, C, H, W, Kc, R, st, pad = (c[key] for key in ("N", "C", "H", "W", "K", "R", "stride", "pad"))
    d = CC.desc_of(c)
    guards = []
    if op == "fprop":
        xv, _ = dev_slice(o["x"], c["x_pitch"], c["x_off"], CC.BF16_NAN)
        krsc, _ = k.weight_prepare(o["w"].float().to(DEV))
        out = None
        if not c["out_f32"]:
            out, ybuf = dev_slice(torch.zeros(N, Kc, d["P"], d["Q"], dtype=CC.F64), c["y_pitch"], c["y_off"], CC.SENTINEL)
            out.view(torch.int16).fill_(CC.SENTINEL)
            guards.append(("y neighbours", ybuf, c["y_off"], Kc, outside(ybuf, c["y_off"], Kc).clone()))
        res = dev_slice(o["residual"], c["y_pitch"], c["y_off"], CC.BF16_NAN)[0] if c["residual"] else None
        stats = torch.zeros(c["stats"], 2, Kc, dtype=torch.float64, device=DEV) if c["stats"] else None
        f32 = lambda key: None if o.get(key) is None else o[key].float().to(DEV)  # noqa: E731
        args = (xv, krsc, Kc, R, R, st, pad)
        kw = dict(scale=f32("scale"), shift=f32("shift"), residual=res, stats=stats, act=c["act"], out=out, out_f32=c["out_f32"], centre_from=c["centre_from"])
        fn = k.conv_fprop
    elif op == "dgrad":
        kp = -(-Kc // 8) * 8
        dyv, _ = dev_slice(o["dy"], c["y_pitch"], c["y_off"], CC.BF16_NAN, zero_to=kp)
        _, crsk = k.weight_prepare(o["w"].float().to(DEV))
        old = o["dx_old"] if c["accumulate"] else torch.zeros(N, C, H, W, dtype=CC.F64)
        out, xbuf = dev_slice(old, c["x_pitch"], c["x_off"], CC.SENTINEL)
        if not c["accumulate"]:
            out.view(torch.int16).fill_(CC.SENTINEL)  # every element must be written (zero where no tap reaches it)
        guards.append(("dx neighbours", xbuf, c["x_off"], C, outside(xbuf, c["x_off"], C).clone()))
        args = (dyv, crsk, (N, C, H, W), R, R, st, pad)
        kw = dict(out=out, accumulate=c["accumulate"], centre_from=c["centre_from"])
        fn = k.conv_dgrad
    elif op == "wgrad":
        kp = -(-Kc // 8) * 8
        xv, _ = dev_slice(o["x"], c["x_pitch"], c["x_off"], CC.BF16_NAN)
        dyv, _ = dev_slice(o["dy"], c["y_pitch"], c["y_off"], CC.BF16_NAN, zero_to=kp)
        out = o["dw_old"].float().to(DEV).contiguous()
        args = (xv, dyv, R, R, st, pad)
        kw = dict(dw_krsc=out, centre_from=c["centre_from"])
        fn = k.conv_wgrad
    else:
        xv, _ = dev_slice(o["x"], c["x_pitch"], 0, CC.BF16_NAN)
        w_up = o["w"].permute(2, 3, 1, 0).reshape(4 * C, Kc).to(DEV).bfloat16().contiguous()  # [(dh, dw, co)][ci]
        args = (xv, w_up, None if o.get("bias") is None else o["bias"].float().to(DEV), C)
        kw = {}
        fn = k.convt2x2_fprop
    force = "sgb_conv_wgrad_force_im2col" if op == "wgrad" else "sgb_conv_force_im2col"
    if c["force"]:
        getattr(lib, force)(1)
    try:
        torch.cuda.synchronize()
        n0 = CC._counters()
        res_t = fn(*args, **kw)
        torch.cuda.synchronize()
        deltas = tuple(b - a for a, b in zip(n0, CC._counters()))
    finally:
        if c["force"]:
            getattr(lib, force)(0)
    for name, buf, off, ch, before in guards:
        CC.expect_bits(name, outside(buf, off, ch), before)
    if op == "fprop":
        got = {"y": res_t.double(), "stats": stats.sum(0) if stats is not None else None}
    elif op == "dgrad":
        got = {"dx": out.double()}
    elif op == "wgrad":
        got = {"dw": out.double()}
    else:
        got = {"y": res_t.double()}
    return got, deltas


def _check(c, real):
    r = CC.case_route(c, sms())
    g = torch.Generator().manual_seed(zlib.crc32(c["id"].encode()))
    o = CC.case_operands(c, real, g, DEV)
    got, deltas = run_case(c, o)
    assert deltas == (r.launches, r.halo, r.whalo), f"{c['id']}: launch counters {deltas}, the route mirror says {r}"
    CC.VERIFY[c["op"]](c, o, got, exact=not real, chain=r.chain)


@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_conv_exact_integer(case):
    _check(case, real=False)


@pytest.mark.parametrize("case", REAL, ids=[c["id"] for c in REAL])
def test_conv_real_within_bounds(case):
    _check(case, real=True)


def _require(seen, patterns, what):
    missing = [p for p in patterns if not any(re.fullmatch(p, t) for t in seen)]
    assert not missing, f"{what} did not reach {missing}; seen: {sorted(t for t in seen if t.count(':') == 2)}"


def test_replay_yolo_nas_s_train_step():
    seen = CC.replay_conv(yolo_nas_s_step_record(batch=2, img=640, recorder=CC.record_conv), sms())
    print(sorted(seen))
    # the ConvTranspose2d backward receives dy as a slice of the concatenated gradient: its 2 x 2 / stride-2 calls go to mma.sync, not
    # to the row-pair path (which only a dense x takes)
    _require(seen, [r"fprop:conv3x3_halo_kernel:bn\d+.*", r"fprop:.*:stats_repl8", r"dgrad:conv3x3_halo_kernel:bn\d+_skip.*",
                    r"dgrad:conv_wgmma_kernel:parity4_.*", r"dgrad:conv_wgmma_kernel:s2_1x1_acc_.*", r"wgrad:wgrad3x3_halo_kernel:nb\d+_cf",
                    r"wgrad:wgrad3x3_halo_kernel:centre_from_inside_row_block", r"convt2x2:conv_wgmma_kernel:parity4_.*",
                    r"fprop:igemm_conv_kernel:x_slice", r"wgrad:wgrad_kernel:bmw\d+"], "YOLO-NAS-S")


def test_replay_resnet50_train_step():
    seen = CC.replay_conv(resnet_step_record("resnet50", batch=2, img=224, recorder=CC.record_conv), sms())
    print(sorted(seen))
    _require(seen, [r"dgrad:conv_wgmma_kernel:s2_1x1_memset_.*", r"dgrad:conv_wgmma_kernel:parity4_.*", r"wgrad:wgrad_wgmma_kernel:.*_split"], "ResNet-50")


def test_replay_yolo_nas_pose_inference():
    seen = CC.replay_conv(CC.pose_infer_record("yolo_nas_pose_s", batch=2, img=640), sms())
    print(sorted(seen))
    _require(seen, [r"fprop:conv3x3_halo_kernel:scale", r"fprop:conv3x3_halo_kernel:act_relu", r"fprop:conv_wgmma_kernel:act_relu",
                    r"convt2x2:conv_wgmma_kernel:parity4_.*"], "YOLO-NAS-POSE inference")
