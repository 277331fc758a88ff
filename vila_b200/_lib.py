"""ctypes binding of libvila_b200.so (the C-ABI declared in include/vila_b200.h).

There is no fallback: if the shared library is missing or a call fails, a RuntimeError is raised.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

_LIB_PATH = Path(__file__).resolve().parent / "libvila_b200.so"

c_void_p, c_int, c_i64, c_float = C.c_void_p, C.c_int, C.c_int64, C.c_float
c_i32_p = C.POINTER(C.c_int32)


class FmhaParams(C.Structure):
    _fields_ = [
        ("q", c_void_p), ("q_tok_stride", c_i64), ("q_head_stride", c_i64),
        ("k", c_void_p), ("v", c_void_p),
        ("kv_page_stride", c_i64), ("kv_tok_stride", c_i64), ("kv_head_stride", c_i64),
        ("kv_num_pages", c_i64),
        ("page_table", c_void_p), ("page_table_stride", C.c_int32),
        ("o", c_void_p), ("o_tok_stride", c_i64), ("o_head_stride", c_i64),
        ("B", C.c_int32), ("Sq", C.c_int32), ("Sk", C.c_int32), ("Hq", C.c_int32),
        ("Hkv", C.c_int32), ("D", C.c_int32), ("causal", C.c_int32),
        ("scale", c_float),
    ]


class GemvParams(C.Structure):
    _fields_ = [
        ("x", c_void_p), ("w", c_void_p), ("bias", c_void_p), ("norm_w", c_void_p),
        ("norm_eps", c_float), ("residual", c_void_p), ("y", c_void_p),
        ("N", C.c_int32), ("K", C.c_int32), ("flags", C.c_int32),
        ("argmax_key", c_void_p),
    ]


class GemvBatchParams(C.Structure):
    _fields_ = [
        ("x", c_void_p), ("ldx", c_i64), ("w", c_void_p), ("bias", c_void_p), ("residual", c_void_p),
        ("ld_res", c_i64), ("y", c_void_p), ("ldy", c_i64),
        ("M", C.c_int32), ("N", C.c_int32), ("K", C.c_int32), ("flags", C.c_int32),
    ]


class DecodeAttnParams(C.Structure):
    _fields_ = [
        ("qkv", c_void_p), ("position", c_void_p), ("k_pool", c_void_p), ("v_pool", c_void_p),
        ("page_table", c_void_p), ("out", c_void_p), ("ws", c_void_p), ("counters", c_void_p),
        ("inv_freq", c_void_p),
        ("Hq", C.c_int32), ("Hkv", C.c_int32), ("D", C.c_int32), ("num_splits", C.c_int32),
        ("scale", c_float),
    ]


class DecodeAttnSplitParams(C.Structure):
    _fields_ = [
        ("qkv", c_void_p), ("position", c_void_p), ("k_pool", c_void_p), ("v_pool", c_void_p),
        ("page_table", c_void_p), ("kv_num_pages", c_i64), ("out", c_void_p), ("o_partial", c_void_p),
        ("lse", c_void_p), ("counters", c_void_p), ("inv_freq", c_void_p),
        ("Hq", C.c_int32), ("Hkv", C.c_int32), ("D", C.c_int32), ("num_splits", C.c_int32),
        ("split_tokens", C.c_int32), ("scale", c_float),
    ]


class DecodeAttnFp8Params(C.Structure):
    _fields_ = [
        ("qkv", c_void_p), ("position", c_void_p), ("k_pool", c_void_p), ("v_pool", c_void_p),
        ("k_scale", c_void_p), ("v_scale", c_void_p), ("page_table", c_void_p), ("out", c_void_p),
        ("ws", c_void_p), ("counters", c_void_p), ("inv_freq", c_void_p),
        ("Hq", C.c_int32), ("Hkv", C.c_int32), ("D", C.c_int32), ("batch", C.c_int32), ("qkv_stride", C.c_int32),
        ("out_stride", C.c_int32), ("pt_stride", C.c_int32), ("num_splits", C.c_int32),
        ("split_tokens", C.c_int32), ("scale", c_float),
    ]


class SampleParams(C.Structure):
    _fields_ = [
        ("logits", c_void_p), ("ld", c_i64), ("inv_temperature", c_void_p), ("top_k", c_void_p),
        ("top_p", c_void_p), ("seed", c_void_p), ("step", c_void_p), ("position", c_void_p),
        ("tokens", c_void_p), ("n_kept", c_void_p), ("M", C.c_int32), ("V", C.c_int32),
    ]


# name -> argtypes; every function returns int (0 == ok) unless listed in _RESTYPES
SIGNATURES = {
    "vila_abi_version": [],
    "vila_device_info": [C.POINTER(c_int)] * 3,
    "vila_set_workspace": [c_void_p, C.c_uint64],
    "vila_linear": [c_void_p, c_i64, c_void_p, c_i64, c_void_p, c_void_p, c_i64, c_int, c_void_p,
                    c_i64, c_int, c_int, c_int, c_int, c_int, c_void_p],
    "vila_linear_cfg": [c_int, c_void_p, c_i64, c_void_p, c_i64, c_void_p, c_void_p, c_i64, c_int,
                        c_void_p, c_i64, c_int, c_int, c_int, c_int, c_int, c_void_p],
    "vila_layernorm": [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_float, c_void_p],
    "vila_rmsnorm": [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_float, c_void_p],
    "vila_fmha": [C.POINTER(FmhaParams), c_void_p],
    "vila_fmha_cfg": [c_int, C.POINTER(FmhaParams), c_void_p],
    "vila_patch_im2col": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p],
    "vila_resize_bicubic_tiles": [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p,
                                  c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_float, c_float, c_void_p],
    "vila_space_to_depth": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p],
    "vila_s2_merge": [c_void_p, c_void_p, c_int, c_int, c_int, C.POINTER(c_int), C.POINTER(c_int),
                      c_int, c_int, c_int, c_void_p],
    "vila_chessboard_merge": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p],
    "vila_tsp_pool": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p],
    "vila_embed_splice": [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p],
    "vila_rope_kv_append": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                            c_void_p, c_void_p, c_int, c_void_p],
    "vila_rope_kv_append_table": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                  c_int, c_void_p],
    "vila_linear_qkv_rope": [c_void_p, C.c_int64, c_void_p, C.c_int64, c_void_p, c_void_p, C.c_int64,
                             c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                             c_void_p, c_int, c_int, c_void_p],
    "vila_rope_table": [c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p],
    "vila_gemv": [C.POINTER(GemvParams), c_void_p],
    "vila_gemv_fp8": [C.POINTER(GemvParams), c_void_p, c_void_p],
    "vila_gemv_w4a16": [C.POINTER(GemvParams), c_void_p, c_void_p, c_void_p],
    "vila_gemv_batch_fp8": [C.POINTER(GemvBatchParams), c_void_p, c_void_p],
    "vila_gemv_batch_w4a16": [C.POINTER(GemvBatchParams), c_void_p, c_void_p, c_void_p],
    "vila_gemv_batch_partition": [c_int, c_int, c_int, c_i32_p],
    "vila_argmax_finalize": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                             c_int, c_void_p],
    "vila_decode_attention": [C.POINTER(DecodeAttnParams), c_void_p],
    "vila_decode_attention_batch": [C.POINTER(DecodeAttnParams), c_int, c_int, c_int, c_int, c_int, c_void_p],
    "vila_decode_attention_split": [C.POINTER(DecodeAttnSplitParams), c_void_p],
    "vila_decode_attention_split_batch": [C.POINTER(DecodeAttnSplitParams), c_int, c_int, c_int, c_int, c_void_p],
    "vila_kv_quantize_fp8": [c_void_p, c_i64, c_void_p, c_void_p, c_i64, c_void_p, c_int, c_int, c_int, c_int,
                             c_int, c_void_p],
    "vila_decode_attention_fp8_batch": [C.POINTER(DecodeAttnFp8Params), c_void_p],
    "vila_sample_batch": [C.POINTER(SampleParams), c_void_p],
}
_RESTYPES = {"vila_last_error": C.c_char_p}

_lib = None


def lib_path() -> Path:
    return _LIB_PATH


def load() -> C.CDLL:
    """Load the shared library (raises if it has not been built)."""
    global _lib
    if _lib is not None:
        return _lib
    if not _LIB_PATH.exists():
        raise RuntimeError(
            f"{_LIB_PATH} not found: build it with `python -m vila_b200.build` "
            "(vila_b200 has no CPU / PyTorch fallback path)")
    lib = C.CDLL(str(_LIB_PATH))
    lib.vila_last_error.restype = C.c_char_p
    lib.vila_last_error.argtypes = []
    for name, argtypes in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is missing
        fn.argtypes = argtypes
        fn.restype = c_int
    _lib = lib
    return lib


LAUNCHES = 0  # number of C-ABI compute calls issued from this process (bench.py reports it)


def check(rc: int, what: str) -> None:
    global LAUNCHES
    LAUNCHES += 1
    if rc != 0:
        msg = load().vila_last_error()
        raise RuntimeError(f"{what} failed (rc={rc}): {msg.decode() if msg else '?'}")
