"""ctypes binding of libsgb200.so (the C ABI declared in include/sgb200.h).

The library is the product: there is NO Python/PyTorch fallback for any function bound here.  If the shared object
is missing or an entry point fails, we raise.
"""
import ctypes
import os
from ctypes import POINTER, Structure, c_char_p, c_double, c_float, c_int, c_int32, c_int64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libsgb200.so")

ACT_NONE, ACT_RELU, ACT_SILU = 0, 1, 2


class SgbError(RuntimeError):
    pass


class ConvDesc(Structure):
    _fields_ = [(n, c_int32) for n in ("N", "H", "W", "C", "K", "R", "S", "P", "Q", "stride", "pad", "x_pitch", "x_off", "y_pitch", "y_off", "up2", "centre_from")]


class Epilogue(Structure):
    _fields_ = [
        ("scale", c_void_p),
        ("shift", c_void_p),
        ("residual", c_void_p),
        ("stats", c_void_p),
        ("stats_repl", c_int32),
        ("act", c_int32),
        ("out_f32", c_int32),
    ]


class WeightItem(Structure):  # SgbWeightItem
    _fields_ = [("w", c_void_p), ("scale", c_void_p), ("krsc", c_void_p), ("crsk", c_void_p)] + [(n, c_int32) for n in ("K", "C", "R", "S", "c_pad", "add_identity", "kp", "koff", "etaps", "etap")] + [("start", c_int64)]


class WgradItem(Structure):  # SgbWgradItem
    _fields_ = [("dw", c_void_p), ("g", c_void_p)] + [(n, c_int32) for n in ("K", "C", "R", "S", "c_pad", "accumulate")] + [("start", c_int64)]


class AlphaItem(Structure):  # SgbAlphaItem
    _fields_ = [(n, c_void_p) for n in ("dw1", "w1", "alpha", "dab", "bias1", "g_w1", "g_bias", "g_alpha")] + [(n, c_int32) for n in ("K", "C", "c_pad", "pad_")]


class BnDesc(Structure):
    _fields_ = [
        ("M", c_int64),
        ("C", c_int32),
        ("x_pitch", c_int32),
        ("x_off", c_int32),
        ("y_pitch", c_int32),
        ("y_off", c_int32),
        ("r_pitch", c_int32),
        ("r_off", c_int32),
        ("eps", c_float),
        ("momentum", c_float),
        ("act", c_int32),
        ("stats_repl", c_int32),
        ("dy_pitch", c_int32),
        ("dy_off", c_int32),
        ("hw", c_int64),
        ("sample_scale", c_void_p),
        ("dy2_split", c_int32),
        ("dy2_pitch", c_int32),
        ("dy2_off", c_int32),
        ("dy2_reserved", c_int32),
        ("dy2", c_void_p),
        ("count", c_void_p),
        ("param_scale", c_float),
        ("count_reserved", c_int32),
    ]


class QarepDesc(Structure):
    _fields_ = [
        ("M", c_int64),
        ("C", c_int32),
        ("pitch3", c_int32),
        ("off3", c_int32),
        ("pitchu", c_int32),
        ("offu", c_int32),
        ("pitcho", c_int32),
        ("offo", c_int32),
        ("eps3", c_float),
        ("eps_post", c_float),
        ("momentum", c_float),
        ("act", c_int32),
        ("use_post_bn", c_int32),
        ("pitchd", c_int32),
        ("offd", c_int32),
        ("pitchr", c_int32),
        ("offr", c_int32),
        ("res", c_void_p),
        ("res_alpha", c_void_p),
        ("count", c_void_p),
        ("param_scale", c_float),
        ("count_reserved", c_int32),
    ]


class PoseLossDesc(Structure):  # SgbPoseLossDesc
    _fields_ = (
        [(n, c_int32) for n in ("B", "L", "J", "reg_max", "n_max", "topk")]
        + [(n, c_float) for n in ("alpha", "beta", "w_cls", "w_iou", "w_dfl", "w_pose_cls", "w_pose_reg")]
        + [(n, c_int32) for n in ("iou_type", "cls_type", "pose_cls_type", "multiply_by_oks", "rescale_with_score")]
    )


class PreprocDesc(Structure):  # SgbPreprocDesc
    _fields_ = (
        [(n, c_int32) for n in ("src_h", "src_w", "src_c", "src_pitch", "dst_h", "dst_w", "out_h", "out_w", "pad_top", "pad_left", "out_pitch", "reverse_channels", "normalize")]
        + [("pad_value", c_float), ("max_value", c_double), ("mean", c_float * 4), ("std", c_float * 4)]
    )


class MatchDesc(Structure):  # SgbMatchDesc
    _fields_ = [(n, c_int32) for n in ("B", "max_preds", "max_targets", "max_crowd", "n_thresholds", "top_k", "denormalize_targets")] + [("height", c_float), ("width", c_float)]


class LossDesc(Structure):
    _fields_ = [
        ("B", c_int32),
        ("L", c_int32),
        ("ncls", c_int32),
        ("reg_max", c_int32),
        ("n_max", c_int32),
        ("topk", c_int32),
        ("alpha", c_float),
        ("beta", c_float),
        ("w_cls", c_float),
        ("w_iou", c_float),
        ("w_dfl", c_float),
        ("iou_type", c_int32),
    ]


class NmsDesc(Structure):
    _fields_ = [
        ("B", c_int32),
        ("L", c_int32),
        ("ncls", c_int32),
        ("score_thr", c_float),
        ("iou_thr", c_double),
        ("top_k", c_int32),
        ("max_out", c_int32),
        ("multi_label", c_int32),
        ("class_agnostic", c_int32),
        ("thr_inclusive", c_int32),
    ]


P = c_void_p
_I, _F, _L = c_int, c_float, c_int64

# name -> (restype, argtypes).  Mirrors include/sgb200.h one to one (tests/test_cabi.py checks the set of names).
_SIGNATURES = {
    "sgb_last_error": (c_char_p, []),
    "sgb_version": (c_int, []),
    "sgb_check_device": (c_int, []),
    "sgb_sm100_launches": (c_int64, []),
    "sgb_conv_halo_launches": (c_int64, []),
    "sgb_conv_force_im2col": (None, [_I]),
    "sgb_conv_wgrad_halo_launches": (c_int64, []),
    "sgb_conv_wgrad_force_im2col": (None, [_I]),
    "sgb_conv_fprop": (c_int, [POINTER(ConvDesc), P, P, P, POINTER(Epilogue), P]),
    "sgb_conv_dgrad": (c_int, [POINTER(ConvDesc), P, P, P, _I, P]),
    "sgb_conv_wgrad": (c_int, [POINTER(ConvDesc), P, P, P, P]),
    "sgb_weight_prepare": (c_int, [P, _I, _I, _I, _I, _I, P, P, P, _I, P]),
    "sgb_wgrad_to_oihw": (c_int, [P, _I, _I, _I, _I, _I, P, _I, P]),
    "sgb_weight_prepare_batch": (c_int, [P, _I, c_int64, P]),
    "sgb_wgrad_to_oihw_batch": (c_int, [P, _I, c_int64, P]),
    "sgb_qarep_alpha_finish_batch": (c_int, [P, _I, P]),
    "sgb_convt2x2_fprop": (c_int, [POINTER(ConvDesc), P, P, P, P, P]),
    "sgb_nchw_f32_to_nhwc_bf16": (c_int, [P, _I, _I, _I, _I, P, _I, _I, _I, P]),
    "sgb_stem_patches_f32": (c_int, [P, _I, _I, _I, _I, _I, _I, _I, P, _I, _I, _I, P]),
    "sgb_nhwc_bf16_to_nchw_f32": (c_int, [P, _I, _I, _I, _I, _I, _I, P, P]),
    "sgb_bn_act_fwd": (c_int, [POINTER(BnDesc), P, P, P, P, P, P, P, P, P, P, P]),
    "sgb_bn_act_fwd_fused": (c_int, [POINTER(BnDesc), P, P, P, P, P, P, P, P, P, P, P]),
    "sgb_bn_act_infer": (c_int, [POINTER(BnDesc), P, P, P, P, P, P, P, P]),
    "sgb_bn_act_bwd_reduce": (c_int, [POINTER(BnDesc), P, P, P, P, P, P, P, P, P]),
    "sgb_bn_act_bwd_apply": (c_int, [POINTER(BnDesc), P, P, P, P, P, P, P, P, P, P, P, P, P]),
    "sgb_bn_act_bwd_fused": (c_int, [POINTER(BnDesc), P, P, P, P, P, P, P, P, P, P, P, P, P]),
    "sgb_channel_stats": (c_int, [P, _L, _I, _I, _I, P, P]),
    "sgb_qarep_moments": (c_int, [POINTER(QarepDesc), P, P, P, P]),
    "sgb_qarep_fwd": (c_int, [POINTER(QarepDesc)] + [P] * 15),
    "sgb_qarep_fwd_fused": (c_int, [POINTER(QarepDesc)] + [P] * 15),
    "sgb_qarep_bwd_reduce": (c_int, [POINTER(QarepDesc), P, P, P, P, P, P, P]),
    "sgb_qarep_bwd_apply": (c_int, [POINTER(QarepDesc)] + [P] * 16),
    "sgb_qarep_bwd_fused": (c_int, [POINTER(QarepDesc)] + [P] * 15),
    "sgb_stem_gemm": (c_int, [POINTER(QarepDesc), P, P, P, P]),
    "sgb_stem_qarep_moments": (c_int, [POINTER(QarepDesc), P, P, P, P]),
    "sgb_stem_qarep_fwd": (c_int, [POINTER(QarepDesc)] + [P] * 15),
    "sgb_stem_qarep_bwd_reduce": (c_int, [POINTER(QarepDesc)] + [P] * 6),
    "sgb_stem_qarep_bwd_apply": (c_int, [POINTER(QarepDesc)] + [P] * 15),
    "sgb_stem_recompute_launches": (c_int64, []),
    "sgb_maxpool_fwd": (c_int, [P, _I, _I, _I, _I, _I, _I, _I, _I, _I, P, _I, _I, _I, _I, P, P]),
    "sgb_maxpool_bwd": (c_int, [P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, P, P, P]),
    "sgb_maxpool_bwd_bf16": (c_int, [P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, P, P, _I, P]),
    "sgb_axpby": (c_int, [P, _I, _I, _F, P, _I, _I, _F, P, _I, _I, _L, _I, P]),
    "sgb_scale_add": (c_int, [P, _I, _I, P, P, _I, _I, P, _I, _I, _L, _I, P]),
    "sgb_channel_dot": (c_int, [P, _I, _I, P, _I, _I, _L, _I, P, P]),
    "sgb_scale_add_dot": (c_int, [P, _I, _I, P, P, _I, _I, P, _I, _I, P, _I, _I, _L, _I, P, P]),
    "sgb_f32_to_bf16": (c_int, [P, P, _L, P]),
    "sgb_avgpool_fwd": (c_int, [P, _I, _I, _I, P, P]),
    "sgb_avgpool_bwd": (c_int, [P, _I, _I, _I, P, P]),
    "sgb_dfl_decode": (c_int, [P, _I, P, _I, _I, _I, _I, _I, _I, _I, _I, _F, _F, P, P, P, P, P]),
    "sgb_pose_keypoint_decode": (c_int, [P, _I, P, _I, _I, _I, _I, _I, _I, _I, _I, _F, _F, _F, _I, P, P, P, P]),
    "sgb_tal_assign": (c_int, [POINTER(LossDesc)] + [P] * 12 + [_L, P]),
    "sgb_tal_workspace_bytes": (c_int64, [POINTER(LossDesc)]),
    "sgb_atss_assign": (c_int, [POINTER(LossDesc)] + [P] * 5 + [c_int32] + [P] * 7 + [P, _L, P]),
    "sgb_atss_workspace_bytes": (c_int64, [POINTER(LossDesc)]),
    "sgb_dfl_iou_loss_fwd_bwd": (c_int, [POINTER(LossDesc)] + [P] * 8 + [_F, P, P, P]),
    "sgb_focal_cls_fwd_bwd": (c_int, [POINTER(LossDesc), P, P, P, P, c_float, c_float, P, P]),
    "sgb_loss_finalize": (c_int, [POINTER(LossDesc), P, P, P]),
    "sgb_preprocess_u8": (c_int, [POINTER(PreprocDesc), P, P, P]),
    "sgb_resample_crop_u8": (c_int, [P, P, P, _L, _I, _I, _I, _I, _I, _I, c_double, P, P, P, P]),
    "sgb_classify_rows": (c_int, [P, _L, _I, _L, _I, P, P, _L, _I, _I, P, P, P, P]),
    "sgb_detection_augment": (c_int, [P, P, P, _L, _I, _I, _I, _I, _I, _I, c_double, _I, P, P]),
    "sgb_pose_augment": (c_int, [P, P, P, _L, P, _L, _I, _I, _I, c_double, _I, P, P]),
    "sgb_imagenet_augment": (c_int, [P, P, P, _L, P, _L, _I, _I, _I, P, P, P, _I, c_float, c_float, P, P, P]),
    "sgb_cifar_augment": (c_int, [P, P, P, _L, _I, _I, P, P, P, P]),
    "sgb_detection_matching": (c_int, [POINTER(MatchDesc), P, P, P, P, P, P, P, P, P, P]),
    "sgb_detection_distance_matching": (c_int, [POINTER(MatchDesc), c_int32, P, P, P, P, P, P, P, P, P, P]),
    "sgb_pose_keypoint_matching": (c_int, [P] * 10 + [_I] * 6 + [P] * 7),
    "sgb_pose_tal_workspace_bytes": (c_int64, [POINTER(PoseLossDesc)]),
    "sgb_pose_tal_assign": (c_int, [POINTER(PoseLossDesc)] + [P] * 14 + [_L, P]),
    "sgb_pose_loss_fwd_bwd": (c_int, [POINTER(PoseLossDesc)] + [P] * 12 + [_F] + [P] * 5),
    "sgb_pose_loss_finalize": (c_int, [POINTER(PoseLossDesc), P, P, P]),
    "sgb_head_grad_scatter": (c_int, [P, _I, _I, _I, _I, _I, P, _I, P]),
    "sgb_sliding_window_gather": (c_int, [P, _I, _I, _I, _I, P, P, _I, _I, P, P]),
    "sgb_sliding_window_merge_workspace_bytes": (c_int64, [_I, P, _I, _I, _I]),
    "sgb_sliding_window_merge": (c_int, [P, P, P, P, P, _I, _I, _I, _I, c_double, P, P, P, _L, P]),
    "sgb_sliding_window_merge_launches": (c_int32, [_I, P, _I, _I]),
    "sgb_nms_workspace_bytes": (c_int64, [POINTER(NmsDesc)]),
    "sgb_batched_nms": (c_int, [POINTER(NmsDesc), P, P, P, P, P, P, _L, P]),
    "sgb_sgd_step": (c_int, [P, P, P, _L, P, P]),
    "sgb_adamw_step": (c_int, [P, P, P, P, _L, P, P]),
    "sgb_ema_update": (c_int, [P, P, _L, P, P]),
    "sgb_adam_step": (c_int, [P, P, P, P, _L, P, P]),
    "sgb_rmsprop_step": (c_int, [P, P, P, P, P, _L, P, P]),
    "sgb_rmsprop_tf_step": (c_int, [P, P, P, P, P, _L, P, P]),
    "sgb_lion_step": (c_int, [P, P, P, _L, P, P]),
    "sgb_lamb_grad_sqnorm": (c_int, [P, P, c_int32, P, P, P]),
    "sgb_lamb_step": (c_int, [P, P, P, P, P, _L, P, c_int32, P, P, P]),
    "sgb_clip_grad_norm": (c_int, [P, P, c_int32, P, c_int32, c_int32, _F, P, P, P]),
    "sgb_average_snapshots": (c_int, [P, c_int32, _L, P, P]),
}

_lib = None

# kernels launched by one call of each entry point (default 1); LAUNCHES[0] accumulates them (bench.py: gpu_launches)
LAUNCH_COUNT = {"sgb_tal_assign": 4, "sgb_lamb_step": 2, "sgb_clip_grad_norm": 2, "sgb_atss_assign": 3, "sgb_pose_tal_assign": 4, "sgb_sm100_launches": 0, "sgb_stem_recompute_launches": 0, "sgb_conv_halo_launches": 0, "sgb_conv_force_im2col": 0, "sgb_conv_wgrad_halo_launches": 0, "sgb_conv_wgrad_force_im2col": 0, "sgb_sliding_window_merge_workspace_bytes": 0, "sgb_sliding_window_merge_launches": 0, "sgb_last_error": 0, "sgb_version": 0, "sgb_check_device": 0}
LAUNCHES = [0]


def exported_names():
    return sorted(_SIGNATURES)


def load():
    """Loads libsgb200.so (raises SgbError if it has not been built)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise SgbError(f"{LIB_PATH} not found: run `python -c 'import __graft_entry__ as g; g.build()'` " "(there is no non-CUDA fallback for this package)")
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in _SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc, what=""):
    if rc != 0:
        msg = load().sgb_last_error()
        raise SgbError(f"{what} failed with code {rc}: {msg.decode() if msg else ''}")


def call(name, *args):
    lib = load()
    rc = getattr(lib, name)(*args)
    LAUNCHES[0] += LAUNCH_COUNT.get(name, 1)
    if rc != 0:
        msg = lib.sgb_last_error()
        raise SgbError(f"{name} failed with code {rc}: {msg.decode() if msg else ''}")
