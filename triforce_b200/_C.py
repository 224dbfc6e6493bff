"""ctypes binding of libtriforce_b200.so (the C ABI in include/triforce_b200.h).

There is NO fallback: if the library is missing or a kernel call fails, this raises.  PyTorch is used only for device
memory and streams — every wrapper passes raw pointers + the current CUDA stream.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import c_char_p, c_float, c_int, c_int64, c_longlong, c_size_t, c_void_p
from typing import Optional

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libtriforce_b200.so")

_lib: Optional[ctypes.CDLL] = None

# name -> (restype, argtypes); mirrors include/triforce_b200.h one to one
_SIGNATURES = {
    "tf_version": (c_int, []),
    "tf_last_error": (c_char_p, []),
    "tf_set_pdl": (c_int, [c_int]),
    "tf_sm_count": (c_int, []),
    "tf_kv_tensormap_encode": (c_int, [c_void_p, c_void_p, c_int, c_longlong, c_int, c_int, c_longlong, c_longlong, c_int]),
    "tf_kv_tensormap_encode_e4m3": (c_int, [c_void_p, c_void_p, c_int, c_longlong, c_int, c_int, c_longlong, c_longlong, c_int]),
    "tf_kv_quantize_e4m3": (c_int, [c_void_p, c_longlong, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_longlong, c_void_p]),
    "tf_rope_append_e4m3": (c_int, [c_void_p, c_void_p, c_void_p, c_longlong, c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p,
                                    c_int, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                    c_longlong, c_void_p]),
    "tf_verify_attn_e4m3": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_longlong, c_int, c_int, c_void_p, c_int, c_int,
                                    c_int, c_int, c_int, c_float, c_void_p, c_void_p, c_size_t, c_void_p]),
    "tf_retrieval_build_e4m3": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_longlong, c_longlong, c_void_p, c_int, c_int, c_int,
                                        c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_longlong, c_longlong, c_void_p, c_void_p,
                                        c_void_p, c_size_t, c_void_p]),
    "tf_tail_update_e4m3": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_longlong, c_longlong, c_void_p, c_void_p, c_longlong,
                                    c_longlong, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int, c_void_p]),
    "tf_retrieval_build_workspace_bytes": (c_size_t, [c_int] * 6),
    "tf_retrieval_build": (c_int, [c_void_p, c_void_p, c_longlong, c_longlong, c_void_p, c_int, c_int, c_int, c_int, c_int,
                                   c_int, c_void_p, c_void_p, c_longlong, c_longlong, c_void_p, c_void_p, c_void_p,
                                   c_size_t, c_void_p]),
    "tf_retrieval_build_gqa": (c_int, [c_void_p, c_void_p, c_longlong, c_longlong, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int,
                                       c_int, c_void_p, c_void_p, c_longlong, c_longlong, c_void_p, c_void_p, c_void_p,
                                       c_size_t, c_void_p]),
    "tf_rope_append_gqa": (c_int, [c_void_p, c_void_p, c_void_p, c_longlong, c_void_p, c_void_p, c_int, c_void_p, c_int,
                                   c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                                   c_void_p, c_longlong, c_longlong, c_void_p]),
    "tf_verify_attn_gqa_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int]),
    "tf_verify_attn_gqa": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int,
                                   c_float, c_void_p, c_void_p, c_size_t, c_int, c_int, c_void_p]),
    "tf_verify_attn_tree_gqa": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int,
                                        c_float, c_void_p, c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
    "tf_tree_attn_tc_gqa": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p, c_int,
                                    c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
    "tf_rope_append": (c_int, [c_void_p, c_void_p, c_void_p, c_longlong, c_void_p, c_void_p, c_int, c_void_p, c_int,
                               c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                               c_longlong, c_longlong, c_void_p]),
    "tf_verify_attn_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "tf_verify_attn": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_int, c_int, c_int, c_int, c_float,
                               c_void_p, c_void_p, c_size_t, c_int, c_int, c_void_p]),
    "tf_verify_attn_prefetch": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_int, c_int, c_int, c_int, c_float,
                                        c_void_p, c_void_p, c_size_t, c_int, c_int, c_void_p, c_size_t, c_void_p]),
    "tf_verify_attn_calibrate": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p,
                                         c_void_p, c_size_t, c_int, c_void_p, c_void_p]),
    "tf_verify_attn_tree": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_int, c_int, c_int, c_int, c_float,
                                    c_void_p, c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
    "tf_tree_attn_tc_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "tf_tree_attn_tc": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p, c_int, c_int, c_void_p,
                                c_void_p, c_size_t, c_void_p, c_void_p]),
    "tf_kv_compact": (c_int, [c_void_p, c_void_p, c_longlong, c_longlong, c_int, c_int, c_int, c_void_p, c_int, c_int, c_void_p]),
    "tf_draft_attn": (c_int, [c_void_p, c_void_p, c_void_p, c_longlong, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                              c_float, c_void_p, c_void_p]),
    "tf_tail_update": (c_int, [c_void_p, c_void_p, c_longlong, c_longlong, c_void_p, c_void_p, c_longlong, c_longlong,
                               c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int, c_void_p]),
    "tf_window_slide": (c_int, [c_void_p, c_void_p, c_longlong, c_longlong, c_int, c_int, c_int, c_int, c_int, c_int,
                                c_void_p]),
    "tf_add_rmsnorm": (c_int, [c_void_p, c_void_p, c_void_p, c_float, c_void_p, c_int, c_int, c_void_p]),
    "tf_silu_mul": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "tf_skinny_gemm_workspace_bytes": (c_size_t, [c_int]),
    "tf_skinny_gemm": (c_int, [c_void_p, c_longlong, c_void_p, c_longlong, c_int, c_int, c_int, c_void_p, c_longlong, c_void_p,
                               c_size_t, c_void_p]),
    "tf_weight_tensormap_encode": (c_int, [c_void_p, c_void_p, c_int, c_int, c_longlong, c_int]),
    "tf_stream_linear_workspace_bytes": (c_size_t, []),
    "tf_stream_linear": (c_int, [c_void_p, c_longlong, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_longlong, c_void_p, c_size_t,
                                 c_void_p]),
    "tf_weight_quantize_e4m3": (c_int, [c_void_p, c_longlong, c_int, c_int, c_void_p, c_longlong, c_void_p, c_void_p, c_void_p]),
    "tf_weight_dequantize_e4m3": (c_int, [c_void_p, c_longlong, c_void_p, c_int, c_int, c_void_p, c_longlong, c_void_p]),
    "tf_weight_tensormap_encode_e4m3": (c_int, [c_void_p, c_void_p, c_int, c_int, c_longlong]),
    "tf_stream_linear_e4m3": (c_int, [c_void_p, c_longlong, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_longlong, c_void_p,
                                      c_size_t, c_void_p]),
    "tf_stream_linear_allreduce_buffer_bytes": (c_size_t, []),
    "tf_stream_linear_allreduce": (c_int, [c_void_p, c_longlong, c_void_p, c_int, c_int, c_int, c_void_p, c_longlong, c_void_p, c_size_t,
                                           c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "tf_skinny_gemm_allreduce_buffer_bytes": (c_size_t, []),
    "tf_skinny_gemm_allreduce": (c_int, [c_void_p, c_longlong, c_void_p, c_longlong, c_int, c_int, c_int, c_void_p, c_longlong,
                                         c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "tf_allreduce_buffer_bytes": (c_size_t, [c_size_t]),
    "tf_stream_linear_ll_push": (c_int, [c_void_p, c_longlong, c_void_p, c_int, c_int, c_int, c_void_p, c_size_t, c_void_p, c_void_p, c_int, c_int,
                                         c_size_t, c_void_p, c_void_p]),
    "tf_add_rmsnorm_ll": (c_int, [c_void_p, c_void_p, c_int, c_size_t, c_void_p, c_void_p, c_float, c_void_p, c_int, c_int, c_void_p]),
    "tf_allreduce_ll_buffer_bytes": (c_size_t, [c_size_t]),
    "tf_allreduce_ll": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_longlong, c_size_t, c_void_p, c_void_p]),
    "tf_allreduce_oneshot": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_longlong, c_size_t, c_void_p, c_void_p]),
    "tf_philox_fill": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p]),
    "tf_loop_begin": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "tf_loop_draft_sample": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "tf_loop_middle_accept": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "tf_loop_prepare_full": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p]),
    "tf_loop_verify": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int64, c_void_p, c_void_p, c_void_p,
                               c_void_p, c_int, c_void_p, c_void_p]),
    "tf_window_slide_dev": (c_int, [c_void_p, c_void_p, c_longlong, c_longlong, c_int, c_int, c_int, c_int, c_void_p, c_int, c_int,
                                    c_void_p]),
    "tf_loop_graph_build": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p]),
    "tf_loop_graph_launch": (c_int, [c_void_p, c_void_p]),
    "tf_loop_graph_destroy": (c_int, [c_void_p]),
    "tf_norm_logits_workspace_bytes": (c_size_t, [c_int, c_int]),
    "tf_norm_logits": (c_int, [c_void_p, c_longlong, c_int, c_int, c_float, c_float, c_void_p, c_void_p, c_size_t, c_void_p]),
    "tf_sample_argmax": (c_int, [c_void_p, c_longlong, c_void_p, c_longlong, c_int, c_int, c_void_p, c_void_p]),
    "tf_residual_probs": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    "tf_tree_accept_walk": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_int, c_int, c_void_p,
                                    c_void_p, c_void_p, c_void_p]),
    "tf_middle_accept": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p,
                                 c_void_p, c_void_p]),
    "tf_verify_accept": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_int64, c_int64, c_void_p,
                                 c_void_p, c_void_p]),
    "tf_verify_resample": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p,
                                   c_void_p]),
}

EXPORTED_SYMBOLS = tuple(_SIGNATURES)
DEFAULT_PDL_MASK = 1 | 2 | 4 | 8 | 16 | 32 | 128 | 256


class TriForceNativeError(RuntimeError):
    pass


def lib() -> ctypes.CDLL:
    """Load the shared library (built in-tree by `python -m triforce_b200.build` / `__graft_entry__.build()`)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise TriForceNativeError(
            f"{LIB_PATH} is missing: the CUDA extension has not been built (run `python -m triforce_b200.build`). "
            "There is no CPU or PyTorch fallback for the TriForce hot path.")
    L = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in _SIGNATURES.items():
        fn = getattr(L, name)  # AttributeError if the header and the library drifted apart
        fn.restype = res
        fn.argtypes = args
    _lib = L
    # programmatic dependent launch mask of the decode-path kernels (tf_set_pdl): on by default for every kernel of the chain
    # (1 add_rmsnorm, 2 silu_mul, 4 rope_append, 8 draft_attn, 16 verify_attn on short stores, 32 skinny_gemm, 128 stream_linear, 256 the one-shot peer all-reduce);
    L.tf_set_pdl(int(os.environ.get("TRIFORCE_PDL", str(DEFAULT_PDL_MASK))))
    return L


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = lib().tf_last_error()
        raise TriForceNativeError(f"{what} failed (code {rc}): {msg.decode() if msg else '?'}")


def stream_ptr() -> int:
    return torch.cuda.current_stream().cuda_stream


def ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def require_cuda(*tensors: torch.Tensor) -> None:
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise TriForceNativeError("triforce_b200 kernels need CUDA tensors; there is no CPU path")
