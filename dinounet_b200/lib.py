"""ctypes binding of the C-ABI in include/dinounet_b200.h (libdinounet_b200.so, built in-tree by csrc/build.py).

No torch types cross this boundary: callers pass raw device addresses (`tensor.data_ptr()`), sizes and a
`cudaStream_t`.  The library is REQUIRED: there is no Python/PyTorch fallback for any op — a missing or failing
extension raises (`NativeLibraryError`), it never silently degrades.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

F16, BF16 = 0, 1
ACT_NONE, ACT_GELU, ACT_RELU, ACT_LRELU, ACT_SWIGLU = 0, 1, 2, 3, 4
CONV_NONE, CONV3X3_S1, CONV3X3_S2 = 0, 1, 2

# DINOUNET_B200_LIB: load another build of the same C-ABI (A/B measurements of kernel variants; csrc/build.py)
_LIB_PATH = os.environ.get("DINOUNET_B200_LIB") or os.path.join(os.path.dirname(os.path.abspath(__file__)), "libdinounet_b200.so")


class NativeLibraryError(RuntimeError):
    pass


class Epilogue(C.Structure):
    _fields_ = [
        ("out", C.c_void_p), ("out_fp32", C.c_int32), ("ldc", C.c_int64), ("col_off", C.c_int32),
        ("rows_in", C.c_int32), ("rows_out", C.c_int32), ("row_off", C.c_int32),
        ("ps_cout", C.c_int32), ("ps_h", C.c_int32), ("ps_w", C.c_int32),
        ("bias", C.c_void_p), ("scale", C.c_void_p), ("shift", C.c_void_p),
        ("act1", C.c_int32), ("act2", C.c_int32), ("round16", C.c_int32),
        ("residual", C.c_void_p), ("ldres", C.c_int64), ("add16", C.c_void_p), ("ldadd", C.c_int64),
    ]


class GemmParams(C.Structure):
    _fields_ = [
        ("M", C.c_int32), ("N", C.c_int32), ("K", C.c_int32),
        ("A", C.c_void_p), ("lda", C.c_int64), ("Wp", C.c_void_p), ("ldw", C.c_int64),
        ("dtype", C.c_int32), ("conv", C.c_int32),
        ("B", C.c_int32), ("Hin", C.c_int32), ("Win", C.c_int32), ("C", C.c_int32),
        ("epi", Epilogue),
    ]


class QkvParams(C.Structure):
    _fields_ = [
        ("B", C.c_int32), ("ntok", C.c_int32), ("D", C.c_int32), ("heads", C.c_int32), ("prefix", C.c_int32),
        ("A", C.c_void_p), ("lda", C.c_int64), ("Wp", C.c_void_p), ("ldw", C.c_int64),
        ("bias", C.c_void_p), ("rope_sin", C.c_void_p), ("rope_cos", C.c_void_p),
        ("q", C.c_void_p), ("k", C.c_void_p), ("v", C.c_void_p), ("dtype", C.c_int32),
        ("v_transposed", C.c_int32), ("npad", C.c_int32), ("rope_w", C.c_int32),
    ]


class DsTargetsParams(C.Structure):
    """b2u_ds_targets_params (deep-supervision target downsampling)."""
    _fields_ = [
        ("src", C.c_void_p), ("dtype", C.c_int32), ("B", C.c_int32), ("C", C.c_int32), ("H", C.c_int32), ("W", C.c_int32),
        ("nscales", C.c_int32), ("fy", C.c_int32 * 4), ("fx", C.c_int32 * 4), ("dst", C.c_void_p * 4),
    ]


DS_MAX_SCALES, DS_INT16, DS_FP32 = 4, 0, 1


class F32GemmParams(C.Structure):
    """b2u_f32_gemm_params (fp32 parity tier)."""
    _fields_ = [
        ("M", C.c_int64), ("N", C.c_int32), ("K", C.c_int32),
        ("A", C.c_void_p), ("lda", C.c_int64),
        ("a_rows_in", C.c_int32), ("a_rows_out", C.c_int32), ("a_row_off", C.c_int32),
        ("W", C.c_void_p), ("ldw", C.c_int64),
        ("conv", C.c_int32), ("Hin", C.c_int32), ("Win", C.c_int32), ("C", C.c_int32), ("Cpad", C.c_int32),
        ("out", C.c_void_p), ("ldc", C.c_int64), ("col_off", C.c_int32),
        ("rows_in", C.c_int32), ("rows_out", C.c_int32), ("row_off", C.c_int32),
        ("ps_cout", C.c_int32), ("ps_h", C.c_int32), ("ps_w", C.c_int32),
        ("bias", C.c_void_p), ("scale", C.c_void_p), ("shift", C.c_void_p),
        ("act1", C.c_int32), ("act2", C.c_int32),
        ("residual", C.c_void_p), ("ldres", C.c_int64),
        ("a_trans", C.c_int32), ("w_mode", C.c_int32), ("w_cpad", C.c_int32), ("ksplit", C.c_int32), ("accumulate", C.c_int32),
    ]


i32, i64, f32, vp = C.c_int32, C.c_int64, C.c_float, C.c_void_p

# name -> argtypes (restype is int unless listed in _RESTYPES); mirrors include/dinounet_b200.h one to one
SIGNATURES = {
    "b2u_gemm": [C.POINTER(GemmParams), vp],
    "b2u_qkv_rope": [C.POINTER(QkvParams), vp],
    "b2u_attention_tc": [vp, vp, vp, vp, i32, i32, i32, i32, i32, f32, i32, vp],
    "b2u_attention_tc_hd": [vp, vp, vp, vp, i32, i32, i32, i32, i32, f32, i32, vp],
    "b2u_attention_rows": [vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, f32, i32, vp],
    "b2u_layernorm": [vp, vp, vp, vp, i32, i32, f32, i32, i32, i32, i32, i32, vp],
    "b2u_cast_rows": [vp, vp, i32, i32, i32, i32, i32, i32, vp],
    "b2u_copy_rows16": [vp, vp, i32, i32, i32, i32, i32, vp],
    "b2u_layernorm16": [vp, vp, vp, vp, i32, i32, f32, i32, i32, i32, i32, i32, vp],
    "b2u_patchify": [vp, vp, i32, i32, i32, vp],
    "b2u_write_prefix": [vp, vp, i32, i32, i32, i32, vp],
    "b2u_stem_conv0": [vp, vp, vp, vp, vp, i32, i32, i32, vp],
    "b2u_maxpool3x3s2": [vp, vp, i32, i32, i32, i32, i32, vp],
    "b2u_dwconv3x3": [vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, vp],
    "b2u_msda_forward": [vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, vp],
    "b2u_msda_forward_f32": [vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, vp],
    "b2u_sw_gather_tiles": [vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, vp],
    "b2u_sw_accumulate": [vp, vp, i32, i32, vp, vp, vp, i32, i32, i32, i32, i32, i32, vp],
    "b2u_sw_finalize": [vp, vp, i32, i64, vp, vp],
    "b2u_export_resample_f16": [vp, vp, i32, i32, i32, i32, i32, i32, vp],
    "b2u_export_segment": [vp, i32, i64, i32, vp, vp, i32, vp, vp],
    "b2u_export_segment_accumulate": [vp, i32, i64, i32, vp, i32, vp],
    "b2u_ensemble_accumulate": [vp, i32, vp, i64, i32, vp],
    "b2u_ensemble_segment": [vp, i32, i64, i32, i32, vp, vp, i32, vp],
    "b2u_pre_minmax_f32": [vp, i64, vp, vp, vp, vp],
    "b2u_pre_zscore": [vp, i64, i32, i32, i32, i64, i64, i64, vp, vp, vp],
    "b2u_pre_normalize": [vp, i64, i32, vp, f32, f32, f32, f32, vp],
    "b2u_pre_resample3_work_doubles": [i32, i32, i32, i32],
    "b2u_pre_resample3": [vp, i32, i32, i32, i64, i64, i64, i32, i32, i32, vp, vp, vp, vp],
    "b2u_pre_ensemble_f16": [vp, vp, i64, i32, vp],
    "b2u_pre_seg_check": [vp, i32, i64, vp, vp],
    "b2u_pre_resample_seg": [vp, i32, i32, i32, i32, i32, i32, vp, vp, vp],
    "b2u_pre_seg_count": [vp, i32, i64, vp, vp, i32, vp, vp],
    "b2u_pre_seg_compact_work_ints": [i64],
    "b2u_pre_seg_compact": [vp, i32, i64, vp, i32, vp, vp, vp],
    "b2u_pre_seg_gather": [vp, vp, i64, i32, i32, vp, vp],
    "b2u_fp_fg_compact": [vp, i32, i64, vp, vp, vp, vp],
    "b2u_fp_gather": [vp, i32, i64, vp, vp, i64, vp, i64, vp],
    "b2u_fp_select_work_bytes": [],
    "b2u_fp_select": [vp, i64, vp, i32, vp, vp, vp],
    "b2u_fp_moments_work_bytes": [i64, i32],
    "b2u_fp_moments": [vp, i64, i32, i32, vp, vp, vp],
    "b2u_vi_scan": [vp, i64, vp, i32, i64, i64, i64, vp, vp],
    "b2u_eval_masks": [vp, i32, vp, i32, i32, i32, i32, i32, C.POINTER(C.c_int64), i32, i32, i64, vp, vp, vp, vp],
    "b2u_eval_edt": [vp, i32, i32, i32, C.c_double, C.c_double, C.c_double, vp, vp, vp, vp],
    "b2u_eval_sum_f64": [vp, i64, vp, vp],
    "b2u_pp_largest_component": [vp, i32, i32, i32, i32, vp, i32, i64, vp, vp, vp],
    "b2u_aug_work_bytes": [i32, i32, i32, i32, i32, i32],
    "b2u_aug_apply": [vp, vp, i32, i32, i32, i32, i32, i32, vp, vp, C.c_uint64, vp, i32, vp, vp, vp, vp],
    "b2u_aug_noise_field": [C.c_uint64, i32, i32, i64, vp, vp],
    "b2u_dl_crop": [vp, vp, i32, i32, i32, i32, i32, vp, i32, vp, vp, vp],
    "b2u_ds_targets": [C.POINTER(DsTargetsParams), vp],
    "b2u_dice_ce_work_doubles": [i32, i32, i64, i32],
    "b2u_dice_ce_stats": [vp, vp, i32, i32, i32, vp, vp, vp, i32, i32, i64, vp],
    "b2u_dice_ce_finalize": [vp, vp, vp, vp, i32, i32, i64, i32, f32, f32, i32, i32, f32, vp],
    "b2u_dice_ce_backward": [vp, vp, i32, i32, i32, vp, vp, vp, i32, i32, i64, f32, f32, i32, i32, f32, vp, vp, vp],
    "b2u_dice_bce_work_doubles": [i32, i32, i64],
    "b2u_dice_bce_stats": [vp, vp, i32, i32, vp, vp, i32, i32, i64, vp],
    "b2u_dice_bce_finalize": [vp, vp, vp, vp, i32, i32, i64, f32, f32, i32, i32, f32, vp],
    "b2u_dice_bce_backward": [vp, vp, i32, i32, vp, vp, vp, i32, i32, i64, f32, f32, i32, f32, vp, vp, vp],
    "b2u_msda_backward_f32": [vp, vp, vp, vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, vp],
    "b2u_tail_fuse": [vp, i32, i64, vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, vp],
    "b2u_in_stats_work_floats": [i32, i32, i32],
    "b2u_in_stats": [vp, i64, vp, vp, i32, i32, i32, i32, vp],
    "b2u_in_apply": [vp, i64, vp, i64, vp, vp, vp, i32, i32, i32, f32, i32, vp],
    "b2u_film": [vp, vp, i64, i32, vp, i32, i32, i32, vp],
    "b2u_se_gate": [vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, vp],
    "b2u_se_apply": [vp, vp, i64, vp, vp, i32, i32, i32, i32, vp],
    "b2u_seg_head": [vp, vp, vp, vp, f32, vp, vp, vp, vp, i32, i32, i32, i32, i32, vp],
    "b2u_zero": [vp, i64, vp],
    "b2u_f32_gemm": [C.POINTER(F32GemmParams), vp],
    "b2u_tf32_gemm": [C.POINTER(F32GemmParams), vp],
    "b2u_f32_layernorm": [vp, vp, vp, vp, i64, i32, f32, i32, i32, i32, vp],
    "b2u_f32_patchify": [vp, vp, i32, i32, vp],
    "b2u_f32_nchw_to_nhwc": [vp, vp, i32, i32, i64, vp],
    "b2u_f32_seg_out": [vp, vp, vp, i32, i64, i32, vp],
    "b2u_f32_maxpool3x3s2": [vp, vp, i32, i32, i32, i32, vp],
    "b2u_f32_dwconv3x3": [vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, vp],
    "b2u_f32_attention": [vp, vp, vp, vp, i32, i32, i32, i32, i32, f32, vp],
    "b2u_f32_msda": [vp, vp, vp, i32, i32, i32, i32, i32, vp],
    "b2u_f32_instnorm": [vp, i64, vp, i64, vp, vp, vp, vp, i32, i64, i32, f32, i32, vp],
    "b2u_f32_se": [vp, vp, i64, vp, vp, vp, vp, vp, vp, i32, i64, i32, i32, vp],
    "b2u_f32_film": [vp, vp, vp, i64, i32, vp],
    "b2u_f32_tail": [vp, i64, i64, vp, vp, vp, vp, i32, i32, i32, i32, vp],
    "b2u_f32_add": [vp, vp, vp, i64, vp],
    "b2u_f32_act": [vp, vp, i64, i32, vp],
    "b2u_f32_act_bwd": [vp, vp, vp, i64, i32, vp],
    "b2u_f32_colsum": [vp, i64, i64, i32, vp, vp],
    "b2u_f32_layernorm_bwd": [vp, vp, vp, vp, vp, vp, i64, i32, f32, vp],
    "b2u_f32_instnorm_bwd": [vp, i64, vp, i64, vp, vp, vp, vp, vp, i64, vp, vp, i32, i64, i32, i32, vp],
    "b2u_f32_bn_act": [vp, vp, vp, vp, vp, vp, f32, i64, i32, i32, vp],
    "b2u_f32_bn_act_bwd": [vp, vp, vp, vp, vp, vp, f32, vp, vp, vp, i64, i32, i32, vp],
    "b2u_f32_dwconv_wgrad": [vp, vp, vp, vp, i32, i32, i32, i32, i32, vp],
    "b2u_f32_maxpool3x3s2_bwd": [vp, vp, vp, i32, i32, i32, i32, vp],
    "b2u_f32_film_bwd": [vp, vp, vp, vp, vp, i64, i32, vp],
    "b2u_f32_se_bwd": [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, i32, i64, i32, i32, vp],
    "b2u_f32_msda_prep": [vp, vp, vp, i32, i32, i32, i32, vp],
    "b2u_f32_msda_prep_bwd": [vp, vp, vp, vp, i32, i32, i32, i32, vp],
    "b2u_f32_unshuffle": [vp, i64, i32, vp, i32, i32, i32, i32, vp],
    "b2u_f32_conv3x3_dgrad": [vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, vp],
    "b2u_f32_conv3x3_wgrad": [vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, vp],
    "b2u_f32_sqsum": [vp, i64, vp, vp],
    "b2u_f32_sgd_nesterov": [vp, vp, vp, i64, f32, f32, f32, vp, f32, i32, vp],
    "b2u_f32_bn_work_doubles": [i64, i32],
    "b2u_f32_bn_stats": [vp, i64, i32, vp, vp, vp],
    "b2u_f32_bn_finalize": [vp, i32, vp, vp, vp, vp, vp, f32, vp],
    "b2u_f32_bn_train_bwd_reduce": [vp, vp, vp, vp, vp, vp, f32, i64, i32, i32, vp, vp, vp, vp, vp],
    "b2u_f32_bn_train_bwd_apply": [vp, vp, vp, vp, vp, vp, f32, vp, vp, i64, i32, i32, vp],
    "b2u_f32_droppath_add": [vp, vp, vp, vp, i64, i32, i64, vp],
    "b2u_rope_tables": [vp, vp, vp, vp, i32, i32, i32, i32, vp],
    "b2u_set_option": [i32, i32],
    "b2u_last_error": [],
    "b2u_version": [],
    "b2u_launch_count": [],
}
_RESTYPES = {"b2u_last_error": C.c_char_p, "b2u_launch_count": C.c_int64, "b2u_in_stats_work_floats": C.c_int64,
             "b2u_dice_ce_work_doubles": C.c_int64, "b2u_dice_bce_work_doubles": C.c_int64,
             "b2u_f32_bn_work_doubles": C.c_int64, "b2u_pre_resample3_work_doubles": C.c_int64,
             "b2u_aug_work_bytes": C.c_int64, "b2u_pre_seg_compact_work_ints": C.c_int64,
             "b2u_fp_select_work_bytes": C.c_int64, "b2u_fp_moments_work_bytes": C.c_int64}

_lib: Optional[C.CDLL] = None


def load() -> C.CDLL:
    """Load libdinounet_b200.so (raises NativeLibraryError if it was not built)."""
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            raise NativeLibraryError(
                f"{_LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(nvcc, sm_90a). dinounet_b200 has no CPU or PyTorch fallback.")
        try:
            lib = C.CDLL(_LIB_PATH)
        except OSError as e:  # pragma: no cover
            raise NativeLibraryError(f"cannot load {_LIB_PATH}: {e}") from e
        for name, argtypes in SIGNATURES.items():
            fn = getattr(lib, name)
            fn.argtypes = argtypes
            fn.restype = _RESTYPES.get(name, C.c_int)
        _lib = lib
    return _lib


def last_error() -> str:
    return load().b2u_last_error().decode()


def launch_count() -> int:
    return int(load().b2u_launch_count())


def check(rc: int, what: str = "native call"):
    if rc != 0:
        raise NativeLibraryError(f"{what} failed (rc={rc}): {last_error()}")
