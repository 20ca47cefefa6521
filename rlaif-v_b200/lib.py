"""ctypes binding of the C-ABI library ``librlaifv_b200.so`` (declared in include/rlaifv_b200.h).

There is no fallback: if the library is missing or a call fails, an exception is raised.  Torch is
used only for device memory and streams; every pointer handed to the library is a raw device
address (``tensor.data_ptr()``) and every launch goes on torch's current CUDA stream.
"""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "librlaifv_b200.so")

c_void_p = ctypes.c_void_p
c_int = ctypes.c_int
c_ll = ctypes.c_longlong
c_float = ctypes.c_float

# name -> argtypes (every function returns int: 0 ok, <0 error; message via rlaifv_last_error)
_SIGNATURES = {
    "rlaifv_gemm_bf16": [c_void_p, c_ll, c_int, c_void_p, c_ll, c_int, c_void_p, c_ll, c_int, c_int, c_int,
                         c_void_p, c_void_p, c_ll, c_int, c_int, c_int, c_void_p],
    "rlaifv_gemm_bf16_scaled": [c_void_p, c_ll, c_int, c_void_p, c_ll, c_int, c_void_p, c_ll, c_int, c_int, c_int,
                                c_void_p, c_void_p, c_ll, c_int, c_int, c_int, c_float, c_void_p],
    "rlaifv_gemm_bf16_dual": [c_void_p, c_ll, c_int, c_void_p, c_ll, c_int, c_void_p, c_ll, c_void_p, c_ll, c_int, c_int,
                              c_int, c_void_p, c_ll, c_int, c_int, c_int, c_void_p, c_void_p, c_ll, c_int, c_int,
                              c_void_p],
    "rlaifv_gemm_bf16_swiglu_bwd": [c_void_p, c_ll, c_void_p, c_ll, c_int, c_void_p, c_ll, c_void_p, c_ll, c_int, c_void_p,
                                    c_ll, c_void_p, c_ll, c_int, c_int, c_int, c_void_p],
    "rlaifv_attention_bwd_split": [c_void_p, c_ll, c_void_p, c_void_p, c_ll, c_void_p, c_ll, c_void_p, c_ll, c_void_p,
                                   c_void_p, c_ll, c_void_p, c_void_p, c_ll, c_void_p, c_int, c_int, c_int, c_int, c_int,
                                   c_int, c_int, c_float, c_void_p],
    "rlaifv_gemm_set_tuning": [c_int, c_int],
    "rlaifv_gemm_set_l2": [c_int],
    "rlaifv_gemm_max_active_clusters": [c_int, c_void_p],
    "rlaifv_gemm_set_split_k": [c_int, c_int],
    "rlaifv_rmsnorm_fwd": [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_float, c_void_p],
    "rlaifv_rmsnorm_bwd": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                           c_void_p, c_int, c_int, c_void_p],
    "rlaifv_layernorm_fwd": [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_float, c_void_p],
    "rlaifv_rope_fwd": [c_void_p, c_void_p, c_void_p, c_ll, c_int, c_int, c_int, c_ll, c_void_p],
    "rlaifv_rope_bwd": [c_void_p, c_void_p, c_void_p, c_void_p, c_ll, c_int, c_int, c_int, c_ll, c_void_p],
    "rlaifv_swiglu_fwd": [c_void_p, c_void_p, c_ll, c_int, c_void_p],
    "rlaifv_swiglu_bwd": [c_void_p, c_void_p, c_void_p, c_ll, c_int, c_void_p],
    "rlaifv_gelu_fwd": [c_void_p, c_void_p, c_ll, c_void_p],
    "rlaifv_gelu_bwd": [c_void_p, c_void_p, c_void_p, c_ll, c_void_p],
    "rlaifv_dropout_fwd": [c_void_p, c_void_p, c_ll, c_float, ctypes.c_ulonglong, c_void_p],
    "rlaifv_dropout_bwd_add": [c_void_p, c_void_p, c_ll, c_float, ctypes.c_ulonglong, c_void_p],
    "rlaifv_colsum": [c_void_p, c_ll, c_int, c_void_p, c_int, c_void_p, c_void_p],
    "rlaifv_clip_im2col": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p],
    "rlaifv_clip_embed": [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p],
    "rlaifv_clip_drop_cls": [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p],
    "rlaifv_splice_count": [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p],
    "rlaifv_splice_map": [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                          c_void_p, c_void_p, c_void_p],
    "rlaifv_splice_gather": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                             c_void_p],
    "rlaifv_splice_scatter": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                              c_void_p],
    "rlaifv_f32_to_bf16": [c_void_p, c_void_p, c_ll, c_int, c_void_p],
    "rlaifv_f32_to_bf16_2d": [c_void_p, c_ll, c_void_p, c_ll, c_ll, c_int, c_int, c_void_p],
    "rlaifv_splice_token_weight": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p],
    "rlaifv_supervised_rows": [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p],
    "rlaifv_rows_gather": [c_void_p, c_void_p, c_void_p, c_ll, c_int, c_void_p],
    "rlaifv_rows_scatter": [c_void_p, c_void_p, c_void_p, c_ll, c_int, c_void_p],
    "rlaifv_logp_fwd": [c_void_p, c_ll, c_void_p, c_void_p, c_ll, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                        c_void_p, c_void_p, c_void_p],
    "rlaifv_logp_bwd": [c_void_p, c_ll, c_void_p, c_void_p, c_ll, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                        c_int, c_int, c_void_p],
    "rlaifv_dpo_loss": [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_float, c_float, c_float, c_float,
                        c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p],
    "rlaifv_adamw_step": [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_ll, c_float, c_float,
                          c_float, c_float, c_float, c_int, c_float, c_void_p],
    "rlaifv_adamw_offload_bucket": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_ll, c_ll, c_void_p, c_int, c_ll,
                                    c_float, c_float, c_float, c_float, c_float, c_int, c_void_p, c_void_p, c_void_p],
    "rlaifv_adamw_offload_release": [c_void_p],
    "rlaifv_adamw8bit_step": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_ll, c_ll, c_void_p,
                              c_void_p, c_float, c_float, c_float, c_float, c_float, c_int, c_void_p],
    "rlaifv_adamw8bit_offload_bucket": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_ll, c_ll,
                                        c_void_p, c_void_p, c_void_p, c_int, c_ll, c_float, c_float, c_float, c_float,
                                        c_float, c_int, c_void_p, c_void_p, c_void_p],
    "rlaifv_attention_fwd_gqa": [c_void_p, c_void_p, c_void_p, c_ll, c_void_p, c_ll, c_void_p, c_int, c_int,
                                 c_int, c_int, c_int, c_int, c_float, c_void_p],
    "rlaifv_attention_bwd_gqa": [c_void_p, c_void_p, c_void_p, c_ll, c_void_p, c_ll, c_void_p, c_ll, c_void_p,
                                 c_void_p, c_void_p, c_void_p, c_ll, c_void_p, c_int, c_int, c_int, c_int, c_int,
                                 c_float, c_void_p],
    "rlaifv_rope_fwd_gqa": [c_void_p, c_void_p, c_void_p, c_ll, c_int, c_int, c_int, c_int, c_ll, c_void_p],
    "rlaifv_rope_bwd_gqa": [c_void_p, c_void_p, c_void_p, c_void_p, c_ll, c_int, c_int, c_int, c_int, c_ll, c_void_p],
    "rlaifv_attention_fwd": [c_void_p, c_void_p, c_void_p, c_ll, c_void_p, c_ll, c_void_p, c_int, c_int,
                             c_int, c_int, c_int, c_float, c_void_p],
    "rlaifv_attention_bwd": [c_void_p, c_void_p, c_void_p, c_ll, c_void_p, c_ll, c_void_p, c_ll, c_void_p,
                             c_void_p, c_void_p, c_void_p, c_ll, c_void_p, c_int, c_int, c_int, c_int,
                             c_float, c_void_p],
    "rlaifv_cross_attention_fwd": [c_void_p, c_ll, c_void_p, c_void_p, c_ll, c_void_p, c_ll, c_void_p, c_int, c_int,
                                   c_int, c_int, c_int, c_int, c_float, c_void_p],
    "rlaifv_cross_attention_bwd": [c_void_p, c_ll, c_void_p, c_void_p, c_ll, c_void_p, c_ll, c_void_p, c_ll, c_void_p,
                                   c_void_p, c_void_p, c_void_p, c_ll, c_void_p, c_int, c_int, c_int, c_int, c_int,
                                   c_int, c_float, c_void_p],
    "rlaifv_layernorm_bwd": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int,
                             c_int, c_float, c_void_p],
    "rlaifv_add_rows_bcast": [c_void_p, c_void_p, c_void_p, c_ll, c_int, c_int, c_void_p],
    "rlaifv_logp_weighted_reduce": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p],
    "rlaifv_splice_map_inplace": [c_void_p, c_void_p, c_int, c_int, c_int, c_ll, c_ll, c_ll, c_void_p, c_void_p,
                                  c_void_p],
    "rlaifv_attention_varlen_fwd": [c_void_p, c_void_p, c_void_p, c_ll, c_void_p, c_ll, c_void_p, c_void_p, c_int,
                                    c_int, c_ll, c_int, c_int, c_int, c_float, c_void_p],
    "rlaifv_attention_varlen_bwd": [c_void_p, c_void_p, c_void_p, c_ll, c_void_p, c_ll, c_void_p, c_ll, c_void_p,
                                    c_void_p, c_ll, c_void_p, c_void_p, c_ll, c_void_p, c_void_p, c_int, c_int, c_ll,
                                    c_int, c_int, c_int, c_float, c_void_p],
    "rlaifv_attention_varlen_prefix_fwd": [c_void_p, c_void_p, c_void_p, c_ll, c_void_p, c_ll, c_void_p, c_void_p,
                                           c_void_p, c_void_p, c_int, c_int, c_ll, c_int, c_int, c_int, c_float,
                                           c_void_p],
    "rlaifv_attention_varlen_prefix_bwd": [c_void_p, c_void_p, c_void_p, c_ll, c_void_p, c_ll, c_void_p, c_ll,
                                           c_void_p, c_void_p, c_ll, c_void_p, c_void_p, c_ll, c_void_p, c_void_p,
                                           c_void_p, c_void_p, c_int, c_int, c_ll, c_int, c_int, c_int, c_float,
                                           c_void_p],
    "rlaifv_rope_pos_fwd": [c_void_p, c_void_p, c_void_p, c_void_p, c_ll, c_int, c_int, c_int, c_ll, c_void_p],
    "rlaifv_rope_pos_bwd": [c_void_p, c_void_p, c_void_p, c_void_p, c_ll, c_int, c_int, c_int, c_ll, c_void_p],
    "rlaifv_dropout_rows_fwd": [c_void_p, c_void_p, c_void_p, c_ll, c_int, c_float, ctypes.c_ulonglong, c_void_p],
    "rlaifv_dropout_rows_bwd_add": [c_void_p, c_void_p, c_void_p, c_ll, c_int, c_float, ctypes.c_ulonglong, c_void_p],
    "rlaifv_quant_fp8_rows": [c_void_p, c_ll, c_void_p, c_ll, c_void_p, c_ll, c_int, c_int, c_void_p],
    "rlaifv_quant_fp8_blocks": [c_void_p, c_ll, c_void_p, c_ll, c_void_p, c_ll, c_void_p, c_ll, c_int, c_int, c_void_p],
    "rlaifv_gemm_fp8": [c_void_p, c_ll, c_void_p, c_ll, c_void_p, c_ll, c_void_p, c_int, c_void_p, c_ll, c_void_p, c_ll,
                        c_int, c_int, c_int, c_void_p, c_ll, c_int, c_int, c_int, c_void_p, c_ll, c_void_p, c_ll,
                        c_void_p],
}
_INT_RETURNING_PLAIN = {"rlaifv_rmsnorm_bwd_partials": []}

_lib = None


class B200Error(RuntimeError):
    pass


def exported_symbols():
    """Every symbol the header declares (used by the CPU-side load/export test)."""
    return sorted(list(_SIGNATURES) + list(_INT_RETURNING_PLAIN) + ["rlaifv_last_error"])


def load():
    """Load the shared library (building is a separate, explicit step: __graft_entry__.build())."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise B200Error(
            "CUDA extension %s is missing: run `python rlaif-v_b200/build.py` "
            "(there is no CPU or eager fallback)" % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    missing = []
    for name, argtypes in _SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError:
            missing.append(name)
            continue
        fn.argtypes = argtypes
        fn.restype = c_int
    if missing:
        raise B200Error("library %s lacks symbols %s (stale build?)" % (LIB_PATH, missing))
    for name, argtypes in _INT_RETURNING_PLAIN.items():
        fn = getattr(lib, name)
        fn.argtypes = argtypes
        fn.restype = c_int
    lib.rlaifv_last_error.restype = ctypes.c_char_p
    lib.rlaifv_last_error.argtypes = []
    _lib = lib
    return lib


def last_error():
    return load().rlaifv_last_error().decode("utf-8", "replace")


_launches = 0


def launch_count():
    """Number of C-ABI kernel-launching calls made so far (each launches >= 1 CUDA kernel)."""
    return _launches


def call(name, *args):
    global _launches
    lib = load()
    _launches += 1
    rc = getattr(lib, name)(*args)
    if rc != 0:
        raise B200Error("%s failed (rc=%d): %s" % (name, rc, last_error()))


_bound_stream = None


def bind_stream(stream=None):
    """Pin the stream all following launches go to (saves the ~13 us torch.cuda.current_stream() lookup
    per launch). Call with None to return to per-call lookup. The engine binds at the start of a step."""
    global _bound_stream
    _bound_stream = None if stream is None else c_void_p(stream.cuda_stream)


_override_stream = None


class use_stream:
    """Context manager: launches inside go to `stream` (side streams for overlapped optimizer work)."""

    def __init__(self, stream):
        self.stream = stream

    def __enter__(self):
        global _override_stream
        self._prev = _override_stream
        _override_stream = c_void_p(self.stream.cuda_stream)

    def __exit__(self, *exc):
        global _override_stream
        _override_stream = self._prev


def stream_ptr():
    if _override_stream is not None:
        return _override_stream
    if _bound_stream is not None:
        return _bound_stream
    return c_void_p(torch.cuda.current_stream().cuda_stream)


def ptr(t):
    """Raw device pointer of a tensor (or NULL for None)."""
    if t is None:
        return c_void_p(0)
    return c_void_p(t.data_ptr())
