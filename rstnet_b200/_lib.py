"""ctypes binding of librstnet_b200.so (the C ABI declared in include/rstnet_b200.h).

There is no CPU fallback: if the shared library is missing, or an entry point fails, this module
raises.  Build with ``python -m rstnet_b200.build`` (nvcc, sm_90a).
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "librstnet_b200.so")

ACT_NONE, ACT_ELU, ACT_GELU = 0, 1, 2

# every symbol include/rstnet_b200.h declares (tests assert the .so exports all of them)
SYMBOLS = [
    "rstnet_version", "rstnet_last_error", "rstnet_launch_count", "rstnet_device_error_flags",
    "rstnet_gemm_rows_f32", "rstnet_tc_gemm_create", "rstnet_tc_gemm_run", "rstnet_tc_gemm_destroy", "rstnet_tc_gemm_grid",
    "rstnet_tc_resblock_create", "rstnet_tc_resblock_run", "rstnet_tc_resblock_destroy", "rstnet_tf32_split_f32", "rstnet_conv1d_cin1_f32", "rstnet_conv1d_cout1_f32",
    "rstnet_convtr1d_depthwise_f32", "rstnet_rows_fill_f32", "rstnet_rows_copy_table_f32",
    "rstnet_counter_add", "rstnet_layer_norm_f32", "rstnet_rope_kv_append_f32",
    "rstnet_ring_attention_f32", "rstnet_rope_ring_attention_f32", "rstnet_rvq_encode_workspace", "rstnet_rvq_encode_f32",
    "rstnet_rvq_decode_gather_f32",
    "rstnet_skinny_gemm_workspace", "rstnet_skinny_gemm_create", "rstnet_skinny_gemm_create_fused", "rstnet_skinny_gemm_run", "rstnet_skinny_gemm_destroy",
    "rstnet_lm_embed_sum_bf16", "rstnet_lm_embed_rows_bf16", "rstnet_lm_rms_norm_bf16", "rstnet_lm_rope_kv_append_bf16",
    "rstnet_lm_rope_pair_kv_append_bf16",
    "rstnet_lm_ring_decode_attention_bf16", "rstnet_lm_silu_mul_bf16", "rstnet_lm_depth_attention_bf16", "rstnet_lm_sample_bf16",
    "rstnet_resample_f32", "rstnet_lm_delay_cache_in", "rstnet_lm_delay_cache_out",
    "rstnet_lm_rope_kv_append_rows_bf16", "rstnet_lm_ring_decode_attention_rows_bf16", "rstnet_lm_sample_rows_bf16",
    "rstnet_counter_add_rows", "rstnet_lm_cross_entropy_bf16",
]

RESAMPLE_MAX_TABLE_BYTES = 48 * 1024   # RSTNET_RESAMPLE_MAX_TABLE_BYTES


class GemmRowsArgs(C.Structure):
    _fields_ = [
        ("A", C.c_void_p), ("a_batch_stride", C.c_int64), ("a_row_stride", C.c_int64),
        ("Wt", C.c_void_p), ("bias", C.c_void_p), ("scale", C.c_void_p),
        ("R", C.c_void_p), ("r_batch_stride", C.c_int64), ("r_row_stride", C.c_int64),
        ("C", C.c_void_p), ("c_batch_stride", C.c_int64), ("c_row_stride", C.c_int64),
        ("batch", C.c_int32), ("rows", C.c_int32), ("N", C.c_int32), ("K", C.c_int32),
        ("pre_act", C.c_int32), ("post_act", C.c_int32), ("taps", C.c_int32), ("tap_stride", C.c_int64),
    ]


class TcGemmDesc(C.Structure):
    _fields_ = [
        ("A", C.c_void_p), ("a_i_stride", C.c_int64), ("a_o_stride", C.c_int64),
        ("a_c_extent", C.c_int32), ("a_i_extent", C.c_int32), ("a_o_extent", C.c_int32),
        ("taps", C.c_int32), ("tap_di", C.c_int32), ("tap_do", C.c_int32), ("o_mul", C.c_int32),
        ("W", C.c_void_p), ("W_lo", C.c_void_p), ("N", C.c_int32), ("Kc", C.c_int32), ("I_out", C.c_int32), ("O_out", C.c_int32),
        ("C", C.c_void_p), ("c_i_stride", C.c_int64), ("c_o_stride", C.c_int64), ("c_split_stride", C.c_int64),
        ("R", C.c_void_p), ("r_i_stride", C.c_int64), ("r_o_stride", C.c_int64), ("r_split_stride", C.c_int64),
        ("bias", C.c_void_p), ("scale", C.c_void_p),
        ("n_split", C.c_int32), ("pre_act", C.c_int32), ("post_act", C.c_int32), ("precision", C.c_int32),
        ("C2", C.c_void_p), ("act2", C.c_int32),
    ]


class TcResblockDesc(C.Structure):
    _fields_ = [
        ("Y", C.c_void_p), ("y_i_stride", C.c_int64), ("y_o_stride", C.c_int64),
        ("channels", C.c_int32), ("I_out", C.c_int32), ("O_out", C.c_int32), ("y_rows", C.c_int32),
        ("W1", C.c_void_p), ("W1_lo", C.c_void_p), ("b1", C.c_void_p),
        ("W2", C.c_void_p), ("W2_lo", C.c_void_p), ("b2", C.c_void_p),
        ("out", C.c_void_p), ("out_i_stride", C.c_int64), ("out_o_stride", C.c_int64),
    ]


class RowCopy(C.Structure):
    _fields_ = [("buf", C.c_void_p), ("batch_stride", C.c_int64), ("C", C.c_int32), ("src_row", C.c_int32),
                ("dst_row", C.c_int32), ("nrows", C.c_int32), ("cps", C.c_int32), ("reserved", C.c_int32)]


class RstnetError(RuntimeError):
    pass


_lib = None


def lib() -> C.CDLL:
    """Load the library once; fail loudly when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RstnetError(
            f"{LIB_PATH} not found: the CUDA extension is not built. Run `python -m rstnet_b200.build` "
            "(there is no CPU fallback).")
    # a library built from other sources than the ones next to it would be driven through mismatched structs:
    # compare the stamp the build wrote (git-ignored, like the .so) with the digest of the sources present
    from . import build as _build
    stamp = os.path.join(os.path.dirname(LIB_PATH), "build.sha256")
    if os.path.isdir(_build.CSRC) and (not os.path.exists(stamp) or open(stamp).read().strip() != _build._digest()):
        raise RstnetError(
            f"{LIB_PATH} is stale (built from different sources than rstnet_b200/csrc + include/). "
            "Run `python -m rstnet_b200.build`.")
    L = C.CDLL(LIB_PATH)
    vp, i32, i64, f32 = C.c_void_p, C.c_int32, C.c_int64, C.c_float
    L.rstnet_version.restype = C.c_int
    L.rstnet_last_error.restype = C.c_char_p
    L.rstnet_launch_count.restype = i64
    L.rstnet_gemm_rows_f32.argtypes = [C.POINTER(GemmRowsArgs), vp]
    L.rstnet_tc_gemm_create.argtypes = [C.POINTER(TcGemmDesc), C.POINTER(C.c_void_p)]
    L.rstnet_tc_gemm_run.argtypes = [vp, vp]
    L.rstnet_tc_gemm_destroy.argtypes = [vp]
    L.rstnet_tc_gemm_destroy.restype = None
    L.rstnet_tc_gemm_grid.argtypes = [vp, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32)]
    L.rstnet_tc_resblock_create.argtypes = [C.POINTER(TcResblockDesc), C.POINTER(C.c_void_p)]
    L.rstnet_tc_resblock_run.argtypes = [vp, vp]
    L.rstnet_tc_resblock_destroy.argtypes = [vp]
    L.rstnet_tc_resblock_destroy.restype = None
    L.rstnet_tf32_split_f32.argtypes = [vp, vp, vp, i64, vp]
    L.rstnet_conv1d_cin1_f32.argtypes = [vp, i64, i64, vp, vp, vp, vp, i64, i64, i32, i32, i32, i32, i32, i32, vp]
    L.rstnet_conv1d_cout1_f32.argtypes = [vp, i64, i64, vp, vp, vp, i64, i32, i32, i32, i32, vp]
    L.rstnet_convtr1d_depthwise_f32.argtypes = [vp, i64, i64, vp, vp, i64, i64, i32, i32, i32, i32, vp]
    L.rstnet_rows_fill_f32.argtypes = [vp, i64, i32, i32, i32, i32, i32, i32, vp, i32, i32, vp]
    L.rstnet_rows_copy_table_f32.argtypes = [vp, i32, i32, vp, vp]
    L.rstnet_counter_add.argtypes = [vp, i64, i32, vp, vp]
    L.rstnet_layer_norm_f32.argtypes = [vp, i64, vp, vp, vp, i32, i32, i32, f32, vp]
    L.rstnet_rope_kv_append_f32.argtypes = [vp, i64, i64, vp, vp, i32, vp, i32, i32, i32, i32, i32, vp]
    L.rstnet_ring_attention_f32.argtypes = [vp, i64, i64, vp, vp, i32, vp, i64, i64, i32, i32, i32, i32, i32, i32, i32, vp]
    L.rstnet_rope_ring_attention_f32.argtypes = [vp, i64, i64, vp, vp, i32, vp, vp, i64, i64, i32, i32, i32, i32, i32, i32, vp]
    L.rstnet_rvq_encode_workspace.argtypes = [i64, i32, i32, i32]
    L.rstnet_rvq_encode_workspace.restype = i64
    L.rstnet_rvq_encode_f32.argtypes = [vp, i64, vp, vp, vp, vp, vp, i64, i32, i32, i32, i32, i32, i32, vp]
    L.rstnet_rvq_decode_gather_f32.argtypes = [vp, vp, vp, i64, i32, i32, i32, i32, i32, i32, vp]
    L.rstnet_skinny_gemm_workspace.argtypes = [i32, i32, i32]
    L.rstnet_skinny_gemm_workspace.restype = i64
    L.rstnet_skinny_gemm_create.argtypes = [vp, vp, vp, vp, vp, i32, i32, i32, i32, C.POINTER(C.c_void_p)]
    L.rstnet_skinny_gemm_create_fused.argtypes = [vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, vp, vp, f32, i32, C.POINTER(C.c_void_p)]
    L.rstnet_skinny_gemm_run.argtypes = [vp, vp]
    L.rstnet_skinny_gemm_destroy.argtypes = [vp]
    L.rstnet_skinny_gemm_destroy.restype = None
    L.rstnet_lm_embed_sum_bf16.argtypes = [vp, i32, vp, i64, vp, i64, i32, i32, vp, i32, vp]
    L.rstnet_lm_embed_rows_bf16.argtypes = [vp, i32, vp, i64, i32, vp, i32, vp]
    L.rstnet_device_error_flags.argtypes = [i32]
    L.rstnet_device_error_flags.restype = C.c_uint32
    L.rstnet_lm_rms_norm_bf16.argtypes = [vp, vp, vp, i32, i32, f32, i32, vp]
    L.rstnet_lm_rope_kv_append_bf16.argtypes = [vp, vp, vp, i64, i32, vp, i32, vp, vp, i32, i32, i32, i32, i32, i32, vp]
    L.rstnet_lm_rope_pair_kv_append_bf16.argtypes = [vp, vp, i32, vp, vp, i32, i32, i32, i32, i32, vp, vp]
    L.rstnet_lm_ring_decode_attention_bf16.argtypes = [vp, vp, vp, i32, vp, i32, i32, i32, i32, i32, i32, i32, vp]
    L.rstnet_lm_silu_mul_bf16.argtypes = [vp, vp, i32, i32, vp]
    L.rstnet_lm_depth_attention_bf16.argtypes = [vp, vp, vp, i32, i32, i32, i32, i32, i32, vp]
    L.rstnet_lm_sample_bf16.argtypes = [vp, i32, i32, i32, i32, f32, C.c_uint32, vp, vp, i32, vp]
    L.rstnet_resample_f32.argtypes = [vp, i64, i64, i64, vp, vp, i32, i32, i32, i32, vp, i64, i64, i32, vp]
    L.rstnet_lm_delay_cache_in.argtypes = [vp, vp, vp, vp, vp, i32, vp, i32, i32, i32, i32, i32, i64, i64, vp]
    L.rstnet_lm_delay_cache_out.argtypes = [vp, vp, vp, vp, vp, i32, vp, i32, vp, i32, i32, i32, i32, i32, vp]
    L.rstnet_lm_rope_kv_append_rows_bf16.argtypes = [vp, vp, vp, i64, i32, vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, vp]
    L.rstnet_lm_ring_decode_attention_rows_bf16.argtypes = [vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, vp]
    L.rstnet_lm_sample_rows_bf16.argtypes = [vp, i32, i32, i32, vp, i32, i32, f32, C.c_uint32, vp, vp, vp, i32, vp]
    L.rstnet_counter_add_rows.argtypes = [vp, vp, i32, vp]
    L.rstnet_lm_cross_entropy_bf16.argtypes = [vp, i64, i32, i32, i32, vp, vp, vp, vp, i32, vp, vp, vp, vp]
    for name in SYMBOLS:
        fn = getattr(L, name)
        if fn.restype is C.c_int and name not in ("rstnet_version",):
            pass
    _lib = L
    return L


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = lib().rstnet_last_error()
        raise RstnetError(f"{what or 'rstnet call'} failed (rc={rc}): {msg.decode() if msg else '?'}")


def launch_count() -> int:
    return int(lib().rstnet_launch_count())
