"""ctypes binding of libeagle_b200.so (C ABI declared in include/eagle_b200.h).

There is no CPU path: importing this module on a box without the built library raises, and
engine creation on a machine without an H100 (sm_90) fails inside the library (eb200_create).
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libeagle_b200.so")

ABI_VERSION = 5
BF16, FP16 = 0, 1
DT_BF16, DT_FP16, DT_FP32, DT_INT64, DT_BOOL, DT_INT8, DT_UINT8, DT_FP8_E4M3 = 0, 1, 2, 3, 4, 5, 6, 7
FLAG_SIMT_GEMM, FLAG_NO_GRAPH, FLAG_NO_CHAIN, FLAG_TARGET_INT8 = 1, 2, 4, 8
FLAG_TARGET_NF4, FLAG_TARGET_FP4, FLAG_TARGET_FP8 = 16, 32, 64
EPI_STORE, EPI_RESIDUAL, EPI_SWIGLU = 0, 1, 2


class Config(C.Structure):
    _fields_ = [
        ("abi_version", C.c_int32), ("dtype", C.c_int32),
        ("vocab_size", C.c_int32), ("hidden_size", C.c_int32), ("intermediate_size", C.c_int32),
        ("num_layers", C.c_int32), ("num_heads", C.c_int32), ("num_kv_heads", C.c_int32),
        ("rms_norm_eps", C.c_float),
        ("eagle3", C.c_int32),
        ("head_hidden_size", C.c_int32), ("head_intermediate_size", C.c_int32), ("head_num_layers", C.c_int32),
        ("head_num_heads", C.c_int32), ("head_num_kv_heads", C.c_int32),
        ("draft_vocab_size", C.c_int32), ("head_fc_bias", C.c_int32), ("head_rms_norm_eps", C.c_float),
        ("total_token", C.c_int32), ("depth", C.c_int32), ("top_k", C.c_int32),
        ("max_length", C.c_int32), ("max_rope_positions", C.c_int32),
        ("tp_rank", C.c_int32), ("tp_size", C.c_int32), ("device", C.c_int32), ("flags", C.c_int32),
    ]


class GenParams(C.Structure):
    _fields_ = [
        ("temperature", C.c_float), ("top_p", C.c_float), ("top_k", C.c_int32),
        ("max_new_tokens", C.c_int32), ("max_length", C.c_int32),
        ("eos_token_id", C.c_int32), ("stop_token_id", C.c_int32), ("seed", C.c_uint64),
    ]


class Stats(C.Structure):
    _fields_ = [
        ("kernel_launches", C.c_uint64), ("cycles", C.c_uint64), ("tokens_committed", C.c_uint64),
        ("gemm_ms", C.c_double), ("gemm_bytes", C.c_double), ("gemm_launches", C.c_uint64),
        ("attn_ms", C.c_double), ("other_ms", C.c_double),
        ("verify_gemm_ms", C.c_double), ("verify_gemm_bytes", C.c_double),
        ("chain_ms", C.c_double), ("chain_bytes", C.c_double), ("chain_launches", C.c_uint64),
    ]


# name -> (restype, argtypes); mirrors include/eagle_b200.h one to one
_P = C.c_void_p
_I32 = C.c_int32
_I64 = C.c_int64
SIGNATURES = {
    "eb200_last_error": (C.c_char_p, []),
    "eb200_abi_version": (_I32, []),
    "eb200_create": (_I32, [C.POINTER(Config), C.POINTER(_P)]),
    "eb200_destroy": (None, [_P]),
    "eb200_load_tensor": (_I32, [_P, C.c_char_p, _P, C.POINTER(_I64), _I32, _I32]),
    "eb200_set_rope_table": (_I32, [_P, _I32, _P, _P, _I32]),
    "eb200_finalize": (_I32, [_P]),
    "eb200_tp_unique_id": (_I32, [_P]),
    "eb200_tp_shard": (_I32, [C.c_char_p, _I64, _I64, _I32, _I32, C.POINTER(_I64)]),
    "eb200_tp_init": (_I32, [_P, _P]),
    "eb200_tp_ipc_handle": (_I32, [_P, _P]),
    "eb200_tp_open_peers": (_I32, [_P, _P, _I32]),
    "eb200_generate": (_I32, [_P, _P, _I32, C.POINTER(GenParams), _P, _I32, C.POINTER(_I32), C.POINTER(_I32), C.POINTER(_I32)]),
    "eb200_naive_generate": (_I32, [_P, _P, _I32, C.POINTER(GenParams), _P, _I32, C.POINTER(_I32), C.POINTER(_I32), C.POINTER(_I32)]),
    "eb200_naive_begin": (_I32, [_P, _P, _I32, C.POINTER(GenParams), C.POINTER(_I64)]),
    "eb200_naive_step": (_I32, [_P, C.POINTER(_I64), C.POINTER(_I64)]),
    "eb200_time_target_forward": (_I32, [_P, _I32, _I32, C.POINTER(C.c_double)]),
    "eb200_set_total_token": (_I32, [_P, _I32]),
    "eb200_set_uniforms": (_I32, [_P, _P, _I32]),
    "eb200_set_static_tree": (_I32, [_P, _P, _P, _I32]),
    "eb200_static_tree_buffers": (_I32, [_P, _P, _I32, _I32, _P, _P, _P, _P, C.POINTER(_I32), C.POINTER(_I32), C.POINTER(_I32),
                                          _P, _P, _P, _P, C.POINTER(_I32)]),
    "eb200_prefill": (_I32, [_P, _P, _I32, C.POINTER(GenParams), C.POINTER(_I64)]),
    "eb200_step": (_I32, [_P, _P, C.POINTER(_I32), C.POINTER(_I64)]),
    "eb200_get_tree": (_I32, [_P, _P, _P, _P, _P, C.POINTER(_I32), C.POINTER(_I32)]),
    "eb200_get_verify": (_I32, [_P, _P, C.POINTER(_I32), C.POINTER(_I32), C.POINTER(_I32)]),
    "eb200_debug_read": (_I32, [_P, C.c_char_p, _P, _I64, C.POINTER(_I32), C.POINTER(_I32)]),
    "eb200_get_stream": (_P, [_P]),
    "eb200_set_profiling": (_I32, [_P, _I32]),
    "eb200_get_stats": (_I32, [_P, C.POINTER(Stats)]),
    "eb200_reset_stats": (_I32, [_P]),
    "eb200_k_gemm": (_I32, [_I32, _I32, _I32, _P, _P, _P, _P, _P, _P, _I32, _I32, _I32, _I32, _P]),
    "eb200_k_gemm_w8": (_I32, [_I32, _I32, _P, _P, _P, _P, _P, _P, _I32, _I32, _I32, _I32, _P]),
    "eb200_k_gemm_fp8": (_I32, [_I32, _I32, _P, _P, _P, _P, _P, _P, _I32, _I32, _I32, _I32, _P]),
    "eb200_k_gemm_w4": (_I32, [_I32, _I32, _I32, _P, _P, _P, _P, _P, _P, _I32, _I32, _I32, _I32, _P]),
    "eb200_k_chain_gemm": (_I32, [_I32, _I32, _P, _P, _P, _P, _P, _I32, _I32, _I32, _I32, _P]),
    "eb200_k_gemm_bench": (_I32, [_I32, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _I32, C.POINTER(C.c_double)]),
    "eb200_k_rmsnorm": (_I32, [_I32, _P, _P, _P, _I32, _I32, C.c_float, _P]),
    "eb200_k_prefetch": (_I32, [_I32, _I32, _I32, _P, _P, _P, _P, _I32, _I32, _I32, _I32, C.c_float, _P, _I32, _I32, _I32, _I32, _I32, _P]),
    "eb200_k_attention": (_I32, [_I32, _P, _P, _P, _P, _I32, _I32, _I32, _I64, _I32, _I32, _P, _P]),
    "eb200_k_attention_plan": (_I32, [_I32, _I32, _I32, _I32, _I32, C.POINTER(_I32), C.POINTER(_I32), C.POINTER(_I32),
                                      C.POINTER(_I64)]),
    "eb200_k_attention_ex": (_I32, [_I32, _P, _P, _P, _P, _I32, _I32, _I32, _I64, _I32, _P, _I32, _I32, _I32, _I32, _P, _I32,
                                    _I32, _P]),
    "eb200_k_qkv_rope": (_I32, [_I32, _I32, _P, _P, _P, _P, _P, _P, _P, _P, _I32, _I32, _I32, _I32, _I64, _I32, _I32, _P]),
    "eb200_k_argmax": (_I32, [_I32, _P, _I32, _I32, _P, _P]),
    "eb200_k_logsoftmax_topk": (_I32, [_I32, _P, _I32, _I32, _I32, _P, _P, _P]),
    "eb200_k_topk_raw": (_I32, [_I32, _P, _I32, _I32, _I32, _P, _P, _P]),
    "eb200_k_generate_candidates": (_I32, [_P, _I32, _I32, _P, _I32, _P, _I32, _I32, _P]),
    "eb200_k_tree_finalize": (_I32, [_I32, _P, _P, _P, _I32, _I32, _I32, _I32, _I32, _P, _P, _P, _P, C.POINTER(_I32), C.POINTER(_I32)]),
    "eb200_k_tree_grow": (_I32, [_I32, _P, _P, _P, _I32, _I32, _I32, _I32, _P, _P, _P, _P, _P, _P, _P, _P]),
    "eb200_k_sample_posterior": (_I32, [_I32, _P, _I32, _P, _P, _I32, _I32, _I32, C.c_float, C.c_float, _I32, _P, _I32,
                                         C.POINTER(_I32), C.POINTER(_I32), C.POINTER(_I32), C.POINTER(_I32)]),
    "eb200_k_greedy_accept": (_I32, [_P, _P, _P, _I32, _I32, _I32, C.POINTER(_I32), C.POINTER(_I32), C.POINTER(_I32)]),
    "eb200_k_sample_stats": (_I32, [_I32, _P, _I32, _I32, C.c_float, C.c_float, _I32, _P]),
    "eb200_k_sample_token": (_I32, [_I32, _P, _I32, C.c_float, C.c_float, _I32, C.c_float, C.POINTER(_I32)]),
}

_lib = None


class EngineError(RuntimeError):
    pass


def load():
    """Load the shared library (built by __graft_entry__.build() / eagle_b200/csrc/Makefile)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise EngineError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(eagle_b200 has no CPU or PyTorch fallback)")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the library does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    if lib.eb200_abi_version() != ABI_VERSION:
        raise EngineError("libeagle_b200.so ABI version mismatch")
    _lib = lib
    return lib


def check(rc: int):
    if rc != 0:
        raise EngineError(load().eb200_last_error().decode("utf-8", "replace"))
