"""ctypes binding of libswapnet_b200.so (the C ABI declared in include/swapnet_b200.h).

There is deliberately no fallback: if the shared library is missing or a call fails, the
product path raises.  (The CPU oracle under oracle/ is test infrastructure only.)
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libswapnet_b200.so")

SN_MAX_TAPS = 32
SN_MAX_SRC = 3
ACT_NONE, ACT_TANH, ACT_LRELU, ACT_RELU = 0, 1, 2, 3
LAYOUT_NCHW, LAYOUT_NHWC, LAYOUT_LABEL_U8, LAYOUT_MASK_I32 = 0, 1, 2, 3
FMT_BF16, FMT_F16 = 0, 1
AUG_NONE, AUG_HFLIP, AUG_VFLIP, AUG_AFFINE_NEAREST, AUG_PERSPECTIVE_BILINEAR = 0, 1, 2, 3, 4
AUG_MAX_OPS = 8


class SnTap(C.Structure):
    _fields_ = [("c_off", C.c_int), ("kb_off", C.c_int), ("dw", C.c_int), ("dh", C.c_int), ("hp", C.c_int)]


class SnTapGemmDesc(C.Structure):
    _fields_ = [
        ("a_hi", C.c_void_p), ("a_lo", C.c_void_p),
        ("a_n", C.c_int), ("a_h", C.c_int), ("a_w", C.c_int), ("a_c", C.c_int), ("a_pitch", C.c_int),
        ("a_parity", C.c_int), ("a_fmt", C.c_int), ("a_chunk", C.c_int),
        ("b_hi", C.c_void_p), ("b_lo", C.c_void_p),
        ("b_rows", C.c_int), ("b_k", C.c_longlong), ("b_fmt", C.c_int), ("b_scale", C.c_void_p),
        ("m_n", C.c_int), ("m_h", C.c_int), ("m_w", C.c_int),
        ("ntaps", C.c_int), ("k_per_tap", C.c_int),
        ("taps", SnTap * SN_MAX_TAPS),
        ("out", C.c_void_p),
        ("out_sn", C.c_longlong), ("out_sh", C.c_longlong), ("out_sw", C.c_longlong),
        ("out_mul_h", C.c_int), ("out_off_h", C.c_int), ("out_mul_w", C.c_int), ("out_off_w", C.c_int),
        ("n_valid", C.c_int), ("block_n", C.c_int),
        ("bias", C.c_void_p), ("act", C.c_int), ("nsplit", C.c_int), ("nphase", C.c_int),
        ("stack_slot", C.c_int), ("stack_c", C.c_int), ("stats", C.c_void_p),
    ]


class SnWgradDesc(C.Structure):
    _fields_ = [
        ("x_hi", C.c_void_p), ("x_lo", C.c_void_p),
        ("x_n", C.c_int), ("x_h", C.c_int), ("x_w", C.c_int), ("x_c", C.c_int), ("x_pitch", C.c_int),
        ("x_parity", C.c_int), ("x_fmt", C.c_int),
        ("y_hi", C.c_void_p), ("y_lo", C.c_void_p),
        ("y_n", C.c_int), ("y_h", C.c_int), ("y_w", C.c_int), ("y_c", C.c_int), ("y_pitch", C.c_int),
        ("y_parity", C.c_int), ("y_fmt", C.c_int),
        ("m_n", C.c_int), ("m_h", C.c_int), ("m_w", C.c_int),
        ("ntaps", C.c_int),
        ("xtaps", SnTap * SN_MAX_TAPS), ("ytaps", SnTap * SN_MAX_TAPS),
        ("tap_off", C.c_longlong * SN_MAX_TAPS),
        ("out", C.c_void_p), ("s_row", C.c_longlong), ("s_col", C.c_longlong),
        ("rows_valid", C.c_int), ("cols_valid", C.c_int),
        ("block_n", C.c_int), ("y_chunk", C.c_int),
        ("ngroups", C.c_int), ("group_start", C.c_int * SN_MAX_TAPS), ("group_size", C.c_int * SN_MAX_TAPS),
        ("ksplit", C.c_int), ("nsplit", C.c_int), ("deterministic", C.c_int),
    ]


class SnScaleItem(C.Structure):
    _fields_ = [("w", C.c_void_p), ("count", C.c_longlong), ("scale2", C.c_void_p)]


class SnPackItem(C.Structure):
    _fields_ = [("src", C.c_void_p), ("s_row", C.c_longlong), ("s_k", C.c_longlong),
                ("rows", C.c_int), ("taps", C.c_int), ("taps_pitch", C.c_int), ("k_real", C.c_int), ("k_pad", C.c_int),
                ("fmt", C.c_int), ("hi", C.c_void_p), ("lo", C.c_void_p), ("scale2", C.c_void_p),
                ("slot", C.c_int * 16), ("block_begin", C.c_int)]


class SnNormActDesc(C.Structure):
    _fields_ = [
        ("y", C.c_void_p), ("y_pitch", C.c_int),
        ("n", C.c_int), ("h", C.c_int), ("w", C.c_int), ("c", C.c_int),
        ("stats", C.c_void_p),
        ("act", C.c_int), ("slope", C.c_float),
        ("drop_p", C.c_float), ("drop_seed", C.c_ulonglong),
        ("drop_offset", C.c_ulonglong), ("drop_step_seed_dev", C.c_void_p), ("drop_stage_id", C.c_uint),
        ("residual", C.c_void_p), ("res_pitch", C.c_int),
        ("out_hi", C.c_void_p), ("out_lo", C.c_void_p), ("out_pitch", C.c_int), ("out_coff", C.c_int),
        ("out_fmt", C.c_int), ("out2_hi", C.c_void_p), ("out2_lo", C.c_void_p), ("out2_fmt", C.c_int),
        ("out_reflect_pad", C.c_int),
        ("out_f32", C.c_void_p), ("f32_pitch", C.c_int),
        ("gamma", C.c_void_p), ("beta", C.c_void_p),
    ]


class SnGradSrc(C.Structure):
    _fields_ = [("ptr", C.c_void_p), ("pitch", C.c_int), ("c_off", C.c_int), ("reflect_padded", C.c_int),
                ("up", C.c_int), ("act", C.c_int)]


class SnNormActBwdDesc(C.Structure):
    _fields_ = [
        ("src", SnGradSrc * SN_MAX_SRC), ("nsrc", C.c_int),
        ("y", C.c_void_p), ("y_pitch", C.c_int),
        ("n", C.c_int), ("h", C.c_int), ("w", C.c_int), ("c", C.c_int),
        ("stats", C.c_void_p),
        ("act", C.c_int), ("slope", C.c_float),
        ("drop_p", C.c_float), ("drop_seed", C.c_ulonglong),
        ("drop_offset", C.c_ulonglong), ("drop_step_seed_dev", C.c_void_p), ("drop_stage_id", C.c_uint),
        ("gstats", C.c_void_p),
        ("dy_hi", C.c_void_p), ("dy_lo", C.c_void_p), ("dy_pitch", C.c_int), ("dy_coff", C.c_int),
        ("dy_fmt", C.c_int), ("bias_grad", C.c_void_p),
        ("gamma", C.c_void_p), ("beta", C.c_void_p), ("bn_groups", C.c_int), ("bn_train", C.c_int),
        ("gamma_grad", C.c_void_p), ("beta_grad", C.c_void_p),
        ("det_slots", C.c_void_p), ("det_slots_cap", C.c_longlong),
        ("bn_phase", C.c_int), ("bn_gathered", C.c_void_p), ("bn_world", C.c_int), ("bn_rank", C.c_int),
    ]


class SnPixelDesc(C.Structure):
    _fields_ = [
        ("x_hi", C.c_void_p), ("x_lo", C.c_void_p), ("xb_hi", C.c_void_p), ("xb_lo", C.c_void_p),
        ("x_pitch", C.c_int), ("x_c", C.c_int), ("n", C.c_int), ("hw", C.c_int), ("cin", C.c_int),
        ("w1", C.c_void_p), ("b1", C.c_void_p), ("w2", C.c_void_p), ("b2", C.c_void_p), ("w3", C.c_void_p),
        ("b3", C.c_void_p), ("scale1", C.c_void_p), ("scale2", C.c_void_p),
        ("norm", C.c_int), ("nsplit", C.c_int), ("slope", C.c_float), ("eps", C.c_float),
        ("stats", C.c_void_p), ("gstats", C.c_void_p), ("pred", C.c_void_p), ("dpred", C.c_void_p),
        ("dw1", C.c_void_p), ("db1", C.c_void_p), ("dw2", C.c_void_p), ("db2", C.c_void_p), ("dw3", C.c_void_p),
        ("db3", C.c_void_p), ("dx", C.c_void_p), ("dx_pitch", C.c_int), ("debug", C.c_void_p),
        ("slots", C.c_void_p), ("slots_cap", C.c_longlong),
    ]


# name -> (restype, argtypes); every symbol declared in include/swapnet_b200.h
_VP, _I, _LL, _F, _ULL = C.c_void_p, C.c_int, C.c_longlong, C.c_float, C.c_ulonglong
SIGNATURES = {
    "sn_version": (C.c_char_p, []),
    "sn_last_error": (C.c_char_p, []),
    "sn_launch_count": (_LL, []),
    "sn_count_replayed": (None, [_LL]),
    "sn_tap_gemm_plan_create": (_I, [C.POINTER(SnTapGemmDesc), C.POINTER(_VP)]),
    "sn_wgrad_plan_create": (_I, [C.POINTER(SnWgradDesc), C.POINTER(_VP)]),
    "sn_plan_run": (_I, [_VP, _VP]),
    "sn_plan_destroy": (None, [_VP]),
    "sn_plan_has_stats": (_I, [_VP]),
    "sn_plan_geometry": (_I, [_VP, C.POINTER(C.c_int)]),
    "sn_plan_workspace_bytes": (_LL, [_VP]),
    "sn_wgrad_ksplit": (_I, [C.POINTER(SnWgradDesc), _I]),
    "sn_det_slots": (_LL, [_I, _I]),
    "sn_plane_sums_det": (_I, [_VP, _I, _I, _I, _I, _VP, _VP, _LL, _VP]),
    "sn_plane_stats_det": (_I, [_VP, _I, _I, _I, _I, _F, _VP, _VP, _LL, _VP]),
    "sn_bias_grad_det": (_I, [_VP, _VP, _I, _I, _I, _LL, _I, _VP, _VP, _VP, _LL, _VP]),
    "sn_ce_tanh_bwd_det": (_I, [_VP, _I, _VP, _I, C.POINTER(SnGradSrc), _I, _I, _I, _I, _I, _F, _VP, _VP, _VP, _I, _I,
                                _I, _VP, _LL, _VP]),
    "sn_gan_loss_fwd_bwd_det": (_I, [_I, _VP, _LL, _I, _F, _F, _VP, _F, _VP, _VP, _VP, _LL, _VP]),
    "sn_l1_loss_fwd_bwd_det": (_I, [_VP, _I, _VP, _I, _I, _I, _I, _F, _VP, _VP, _I, _VP, _LL, _VP]),
    "sn_to_one_wgrad_det": (_I, [_VP, _VP, _I, _I, _I, _I, _I, _I, _VP, _VP, _I, _I, _I, _I, _VP, _VP, _LL, _VP]),
    "sn_to_one_wgrad_det_slots": (_LL, [_I]),
    "sn_stats_finalize": (_I, [_VP, _I, _I, _F, _VP]),
    "sn_plane_sums": (_I, [_VP, _I, _I, _I, _I, _VP, _VP]),
    "sn_bn_finalize": (_I, [_VP, _I, _I, _I, _I, _F, _F, _VP, _VP, _VP, _VP]),
    "sn_bn_eval_stats": (_I, [_VP, _I, _I, _VP, _VP, _F, _VP]),
    "sn_bn_group_sums": (_I, [_VP, _I, _I, _I, _I, _VP, _VP]),
    "sn_bn_finalize_gathered": (_I, [_VP, _I, _I, _I, _VP, _I, _F, _F, _VP, _VP, _VP, _VP]),
    "sn_pack_planes": (_I, [_VP, _I, _I, _I, _I, _I, _I, _VP, _VP, _I, _I, _I, _VP]),
    "sn_pack_concat": (_I, [_I, _VP, _I, _I, _I, _VP, _I, _I, _I, _I, _I, _I, _I, _VP, _VP, _VP, _VP, _I, _I, _I, _I, _VP]),
    "sn_pack_head_weights": (_I, [_VP, _I, _I, _I, _I, _I, _I, _VP, _VP, _I, _VP, _VP]),
    "sn_weight_scale_multi": (_I, [_VP, _I, _VP, _VP]),
    "sn_pack_weights_multi": (_I, [_VP, _I, _I, _I, _VP]),
    "sn_pack_rows_per_block": (_I, []),
    "sn_pack_k_per_block": (_I, []),
    "sn_pack_head_stacked": (_I, [_VP, _I, _I, _I, _I, _VP, _VP, _I, _VP, _VP]),
    "sn_fold_head_wgrad": (_I, [_VP, _I, _I, _VP, _VP]),
    "sn_plane_stats": (_I, [_VP, _I, _I, _I, _I, _F, _VP, _VP]),
    "sn_norm_act_fwd": (_I, [C.POINTER(SnNormActDesc), _VP]),
    "sn_norm_act_bwd": (_I, [C.POINTER(SnNormActBwdDesc), _VP]),
    "sn_bias_grad": (_I, [_VP, _VP, _I, _I, _I, _LL, _I, _VP, _VP, _VP]),
    "sn_sum_grads": (_I, [C.POINTER(SnGradSrc), _I, _I, _I, _I, _I, _VP, _I, _VP]),
    "sn_tanh_bwd": (_I, [C.POINTER(SnGradSrc), _I, _VP, _I, _I, _I, _I, _I, _VP, _VP, _I, _I, _I, _VP]),
    "sn_upsample_planes": (_I, [_VP, _VP, _I, _I, _I, _I, _I, _I, _I, _VP, _VP, _I, _I, _VP]),
    "sn_adamw_step": (_I, [_VP, _VP, _VP, _VP, _LL, C.c_double, C.c_double, C.c_double, C.c_double, C.c_double, _I, _VP]),
    "sn_adamw_step_dev": (_I, [_VP, _VP, _VP, _VP, _LL, _VP, _VP]),
    "sn_adamw_hyper": (None, [C.c_double, C.c_double, C.c_double, C.c_double, C.c_double, _I, C.c_double,
                              C.POINTER(C.c_float)]),
    "sn_adabound_step": (_I, [_VP, _VP, _VP, _VP, _LL] + [C.c_double] * 8 + [_I, _VP]),
    "sn_adabound_step_dev": (_I, [_VP, _VP, _VP, _VP, _LL, _VP, _VP]),
    "sn_adabound_hyper": (None, [C.c_double] * 8 + [_I, C.c_double, C.POINTER(C.c_float)]),
    "sn_set_step_params": (_I, [_VP, C.POINTER(C.c_float), _I, _VP]),
    "sn_bce_logits_fwd_bwd_dev": (_I, [_VP, _LL, _I, _VP, _F, _VP, _VP, _VP]),
    "sn_dropout_mask": (_I, [_ULL, _F, _LL, _VP, _VP]),
    "sn_ce_loss_fwd_bwd": (_I, [_VP, _I, _VP, _I, _I, _I, _I, _I, _F, _VP, _VP, _I, _VP]),
    "sn_ce_tanh_bwd": (_I, [_VP, _I, _VP, _I, C.POINTER(SnGradSrc), _I, _I, _I, _I, _I, _F, _VP, _VP, _VP, _I, _I, _I, _VP]),
    "sn_bce_logits_fwd_bwd": (_I, [_VP, _LL, _I, _F, _F, _F, _VP, _VP, _VP]),
    "sn_gan_loss_fwd_bwd_dev": (_I, [_I, _VP, _LL, _I, _F, _F, _VP, _F, _VP, _VP, _VP]),
    "sn_l1_loss_fwd_bwd": (_I, [_VP, _I, _VP, _I, _I, _I, _I, _F, _VP, _VP, _I, _VP]),
    "sn_tap_sum_fwd": (_I, [_VP, _I, _I, _I, _I, _I, _I, _VP, _VP, _I, _VP]),
    "sn_to_one_fwd": (_I, [_VP, _VP, _I, _I, _LL, _I, _VP, _I, _VP, _I, _VP]),
    "sn_to_one_wgrad": (_I, [_VP, _VP, _I, _I, _I, _I, _I, _I, _VP, _VP, _I, _I, _I, _I, _VP, _VP]),
    "sn_to_one_dgrad": (_I, [_VP, _VP, _I, _I, _I, _I, _I, _I, _VP, _I, _I, _VP, _I, _VP]),
    "sn_affine_pack": (_I, [_VP, _I, _I, _I, _I, _I, _I, _F, _F, _VP, _VP, _I, _I, _I, _VP]),
    "sn_relu_pool_fwd": (_I, [_VP, _I, _I, _I, _I, _I, _VP, _VP, _I, _I, _I, _VP]),
    "sn_relu_pool_bwd": (_I, [_VP, _I, _VP, _I, _VP, _I, _I, _I, _I, _I, _VP, _VP, _I, _I, _I, _VP]),
    "sn_feat_loss_fwd_bwd": (_I, [_VP, _I, _VP, _I, _LL, _I, C.c_double, C.c_double, _VP, _VP, _I, _VP]),
    "sn_feat_loss_fwd_bwd_det": (_I, [_VP, _I, _VP, _I, _LL, _I, C.c_double, C.c_double, _VP, _VP, _I, _VP, _LL, _VP]),
    "sn_gram_rows": (_I, [_VP, _LL, _LL, _LL, _I, _VP, _LL, _LL, _LL, _I, _I, _LL, _VP, _VP]),
    "sn_gram_rows_det": (_I, [_VP, _LL, _LL, _LL, _I, _VP, _LL, _LL, _LL, _I, _I, _LL, _VP, _VP, _LL, _VP]),
    "sn_gram_rows_det_slots": (_LL, [_I, _I]),
    "sn_gram_rows_mse": (_I, [_VP, _VP, _I, _I, C.c_double, C.c_double, _VP, _VP, _VP]),
    "sn_gram_rows_bwd": (_I, [_VP, _I, _VP, _LL, _LL, _LL, _I, _I, _LL, _VP, _I, _I, _VP]),
    "sn_roi_align_pack_fwd": (_I, [_VP, _I, _I, _I, _I, _VP, _I, _I, _VP, _I, _VP, _VP, _I, _I, _I, _VP]),
    "sn_tap_gemm_simt": (_I, [C.POINTER(SnTapGemmDesc), _VP]),
    "sn_pixel_fwd_stats": (_I, [C.POINTER(SnPixelDesc), _VP]),
    "sn_pixel_fwd": (_I, [C.POINTER(SnPixelDesc), _VP]),
    "sn_pixel_bwd_reduce": (_I, [C.POINTER(SnPixelDesc), _VP]),
    "sn_pixel_bwd_apply": (_I, [C.POINTER(SnPixelDesc), _VP]),
    "sn_pixel_det_slots": (_LL, [_I, _I]),
    "sn_augment_channels": (_I, [_VP, _VP, _I, _I, _I, _I, _VP, _I, _I, _VP, _VP, _VP]),
}

_lib = None


class SwapnetB200Error(RuntimeError):
    pass


def load(build_if_missing: bool = False) -> C.CDLL:
    """Load the shared library (once) and attach prototypes.  Raises if unavailable."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        if build_if_missing:
            from . import build as _build

            _build.build(verbose=False)
        else:
            raise SwapnetB200Error(
                f"{LIB_PATH} is missing: build it with `python -m swapnet_b200.build` "
                "(there is no CPU / eager fallback for the hot path)"
            )
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the .so does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc: int) -> None:
    if rc != 0:
        msg = load().sn_last_error().decode("utf-8", "replace")
        raise SwapnetB200Error(f"libswapnet_b200 call failed ({rc}): {msg}")
