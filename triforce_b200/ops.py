"""Tensor-level wrappers over the C ABI (one function per entry point of include/triforce_b200.h).

Each wrapper validates what only the host can know (dtype, contiguity, device), then hands raw pointers and the current
stream to the library.  Nothing here computes anything with torch.
"""
from __future__ import annotations

import ctypes
from typing import Optional

import torch

from . import _C
from ._C import check, lib, ptr, require_cuda, stream_ptr

class _LaunchCounter:
    """Number of THIS library's kernels enqueued (bench.py reports it as `gpu_launches`).  Graph replays add the count
    recorded at capture time (see engine._capture)."""
    n = 0


COUNTER = _LaunchCounter()

VERIFY_MAX_ROWS = 32
VERIFY_BOX_KEYS = 64
SAMPLING_MAX_VOCAB = 32768


def _f16c(t: torch.Tensor, name: str):
    if t.dtype != torch.float16:
        raise TypeError(f"{name} must be float16, got {t.dtype}")


class KVTensorMaps:
    """Host-side TMA descriptors for one head-major KV store [L,H,cap,d] (K and V)."""

    def __init__(self, key_store: torch.Tensor, value_store: torch.Tensor):
        require_cuda(key_store, value_store)
        L, H, cap, d = key_store.shape
        assert key_store.is_contiguous() and value_store.is_contiguous()
        self.k = (ctypes.c_uint8 * 128)()
        self.v = (ctypes.c_uint8 * 128)()
        for buf, t in ((self.k, key_store), (self.v, value_store)):
            check(lib().tf_kv_tensormap_encode(ctypes.addressof(buf), t.data_ptr(), d, cap, H, L, t.stride(1), t.stride(0),
                                               VERIFY_BOX_KEYS), "tf_kv_tensormap_encode")
        self.k_ptr = ctypes.addressof(self.k)
        self.v_ptr = ctypes.addressof(self.v)
        self.shape = (L, H, cap, d)


class E4m3Store:
    """One E4M3 full-KV store (the format of include/triforce_b200.h): codes uint8 [L,Hkv,cap,d] and exponents int8 [L,Hkv,cap],
    for K and for V, plus the TMA descriptors of the codes.  cap must be a multiple of VERIFY_BOX_KEYS."""

    def __init__(self, k_codes: torch.Tensor, v_codes: torch.Tensor, k_exp: torch.Tensor, v_exp: torch.Tensor):
        require_cuda(k_codes, v_codes, k_exp, v_exp)
        L, H, cap, d = k_codes.shape
        for t in (k_codes, v_codes):
            assert t.dtype == torch.uint8 and t.is_contiguous() and t.shape == (L, H, cap, d)
        for t in (k_exp, v_exp):
            assert t.dtype == torch.int8 and t.is_contiguous() and t.shape == (L, H, cap)
        if cap % VERIFY_BOX_KEYS:
            raise ValueError(f"an e4m3 store needs a capacity that is a multiple of {VERIFY_BOX_KEYS}, got {cap}")
        self.k_codes, self.v_codes, self.k_exp, self.v_exp = k_codes, v_codes, k_exp, v_exp
        self.k = (ctypes.c_uint8 * 128)()
        self.v = (ctypes.c_uint8 * 128)()
        for buf, t in ((self.k, k_codes), (self.v, v_codes)):
            check(lib().tf_kv_tensormap_encode_e4m3(ctypes.addressof(buf), t.data_ptr(), d, cap, H, L, t.stride(1), t.stride(0),
                                                    VERIFY_BOX_KEYS), "tf_kv_tensormap_encode_e4m3")
        self.k_ptr = ctypes.addressof(self.k)
        self.v_ptr = ctypes.addressof(self.v)
        self.shape = (L, H, cap, d)

    @staticmethod
    def empty(L: int, H: int, cap: int, d: int, device) -> "E4m3Store":
        return E4m3Store(torch.zeros((L, H, cap, d), dtype=torch.uint8, device=device),
                         torch.zeros((L, H, cap, d), dtype=torch.uint8, device=device),
                         torch.zeros((L, H, cap), dtype=torch.int8, device=device),
                         torch.zeros((L, H, cap), dtype=torch.int8, device=device))


def kv_quantize_e4m3(src_layer: torch.Tensor, codes_layer: torch.Tensor, exp_layer: torch.Tensor, slot0: int, n: int):
    """fp16 rows [slot0, slot0+n) of src_layer [Hkv, >=cap, d] -> the same slots of one layer of K or V codes [Hkv, cap, d]
    and exponents [Hkv, cap] (tf_kv_quantize_e4m3)."""
    require_cuda(src_layer, codes_layer, exp_layer)
    _f16c(src_layer, "src_layer")
    H, cap, d = codes_layer.shape
    assert codes_layer.dtype == torch.uint8 and codes_layer.is_contiguous()
    assert exp_layer.dtype == torch.int8 and exp_layer.is_contiguous() and exp_layer.shape == (H, cap)
    assert src_layer.shape[0] == H and src_layer.shape[2] == d and src_layer.stride(2) == 1 and src_layer.stride(1) == d
    check(lib().tf_kv_quantize_e4m3(src_layer.data_ptr(), src_layer.stride(0), slot0, n, H, d, codes_layer.data_ptr(),
                                    exp_layer.data_ptr(), cap, stream_ptr()), "tf_kv_quantize_e4m3")
    COUNTER.n += 1


def rope_append_e4m3(qkv: torch.Tensor, Hq: int, Hkv: int, d: int, cos, sin, q_out, store: E4m3Store, layer: int, *,
                     pos_ids=None, pos0: int = 0, pos0_dev=None, slot0: int = 0, slot0_dev=None):
    """rope_append_gqa with the appended K/V rows quantized into `layer` of the e4m3 store (tf_rope_append_e4m3)."""
    require_cuda(qkv, cos, sin, q_out)
    _f16c(qkv, "qkv")
    R = qkv.shape[0]
    L, H, cap, _ = store.shape
    assert H == Hkv and qkv.stride(1) == 1 and qkv.shape[1] == (Hq + 2 * Hkv) * d
    assert q_out.is_contiguous() and q_out.shape == (R, Hq, d)
    base = qkv.data_ptr()
    es = qkv.element_size()
    if pos_ids is not None:
        assert pos_ids.dtype == torch.int32 and pos_ids.numel() >= R
    check(lib().tf_rope_append_e4m3(base, base + Hq * d * es, base + (Hq + Hkv) * d * es, qkv.stride(0), cos.data_ptr(),
                                    sin.data_ptr(), cos.shape[0], ptr(pos_ids), pos0, ptr(pos0_dev), slot0, ptr(slot0_dev), R, Hq,
                                    Hkv, d, q_out.data_ptr(), store.k_codes[layer].data_ptr(), store.v_codes[layer].data_ptr(),
                                    store.k_exp[layer].data_ptr(), store.v_exp[layer].data_ptr(), cap, stream_ptr()),
          "tf_rope_append_e4m3")
    COUNTER.n += 1


def verify_attn_e4m3(q, store: E4m3Store, layer: int, kv_len: int, R: int, Hq: int, Hkv: int, d: int, scale: float, out,
                     workspace, kv_len_dev=None, kv_len_max: Optional[int] = None):
    """verify_attn_gqa (causal, Hq == Hkv is MHA) over the e4m3 store (tf_verify_attn_e4m3); workspace from
    verify_attn_gqa_workspace.  Rows are cut into bottom-right aligned blocks of gqa_row_block(Hq, Hkv) token rows."""
    require_cuda(q, out, workspace)
    _f16c(q, "q")
    assert q.is_contiguous() and out.is_contiguous() and q.shape[-3:] == (R, Hq, d) and out.shape == q.shape
    L, H, cap, _ = store.shape
    assert H == Hkv, (store.shape, Hkv)
    if kv_len_max is None:
        kv_len_max = cap if kv_len_dev is not None else kv_len
    step = gqa_row_block(Hq, Hkv)
    if step < 1:
        raise ValueError(f"{Hq // Hkv} query heads per KV head exceed the {VERIFY_MAX_ROWS} rows of a verify-attention CTA")
    for r0 in range(0, R, step):
        r1 = min(R, r0 + step)
        check(lib().tf_verify_attn_e4m3(q[r0:r1].data_ptr(), store.k_ptr, store.v_ptr, store.k_exp.data_ptr(), store.v_exp.data_ptr(),
                                        cap, layer, kv_len - (R - r1), ptr(kv_len_dev), min(kv_len_max, cap), r1 - r0, Hq, Hkv, d,
                                        scale, out[r0:r1].data_ptr(), workspace.data_ptr(), workspace.numel(), stream_ptr()),
              "tf_verify_attn_e4m3")
        COUNTER.n += 1


def retrieval_build_e4m3(store: E4m3Store, q, retr_key_store, retr_value_store, prefill: int, chunk: int, budget: int,
                         layer0: int = 0, n_layers: Optional[int] = None, out_idx=None, out_scores=None):
    """retrieval_build / retrieval_build_gqa ("group_sum" when Hq > Hkv) over the e4m3 store (tf_retrieval_build_e4m3):
    q [n_layers,Hq,d]; the gather writes D into the fp16 retrieval store."""
    require_cuda(q, retr_key_store, retr_value_store)
    L, Hkv, cap, d = store.shape
    n = q.shape[0] if n_layers is None else n_layers
    Hq = q.shape[1]
    _f16c(q, "q")
    assert q.is_contiguous() and q.shape == (n, Hq, d), (q.shape, (n, Hq, d))
    ws_bytes = lib().tf_retrieval_build_workspace_bytes(n, Hkv, d, prefill, chunk, budget)
    ws = torch.empty(max(ws_bytes, 16), dtype=torch.uint8, device=q.device)
    if out_idx is not None:
        assert out_idx.dtype == torch.int32 and out_idx.is_contiguous() and out_idx.shape == (n, Hkv, budget // chunk)
    if out_scores is not None:
        assert out_scores.dtype == torch.float16 and out_scores.is_contiguous() and out_scores.shape == (n, Hkv, prefill // chunk)
    kc = store.k_codes
    check(lib().tf_retrieval_build_e4m3(kc[layer0].data_ptr(), store.v_codes[layer0].data_ptr(), store.k_exp[layer0].data_ptr(),
                                        store.v_exp[layer0].data_ptr(), kc.stride(0), kc.stride(1), q.data_ptr(), n, Hq, Hkv, d,
                                        prefill, chunk, budget, retr_key_store[layer0].data_ptr(), retr_value_store[layer0].data_ptr(),
                                        retr_key_store.stride(0), retr_key_store.stride(1), ptr(out_idx), ptr(out_scores),
                                        ws.data_ptr(), ws.numel(), stream_ptr()), "tf_retrieval_build_e4m3")
    COUNTER.n += 3


def tail_update_e4m3(store: E4m3Store, retr_key_store, retr_value_store, prefill: int, budget: int, seq_len: int,
                     seq_len_dev=None, max_new: int = 0, layer0: int = 0, n_layers: Optional[int] = None):
    """tail_update from the e4m3 store into the fp16 retrieval store (tf_tail_update_e4m3), layers [layer0, layer0+n): writes D."""
    L, H, cap, d = store.shape
    n = L - layer0 if n_layers is None else n_layers
    kc = store.k_codes
    check(lib().tf_tail_update_e4m3(kc[layer0].data_ptr(), store.v_codes[layer0].data_ptr(), store.k_exp[layer0].data_ptr(),
                                    store.v_exp[layer0].data_ptr(), kc.stride(0), kc.stride(1), retr_key_store[layer0].data_ptr(),
                                    retr_value_store[layer0].data_ptr(), retr_key_store.stride(0), retr_key_store.stride(1), n, H, d,
                                    prefill, budget, seq_len, ptr(seq_len_dev), max_new, stream_ptr()), "tf_tail_update_e4m3")
    COUNTER.n += 1


def retrieval_build(key_store, value_store, q, retr_key_store, retr_value_store, prefill: int, chunk: int, budget: int,
                    layer0: int = 0, n_layers: Optional[int] = None, out_idx=None, out_scores=None):
    """key_store/value_store [L,H,cap,d]; q [n_layers,H,d]; retr_* [L,H,rcap,d].  Builds layers [layer0, layer0+n)."""
    require_cuda(key_store, value_store, q, retr_key_store, retr_value_store)
    L, H, cap, d = key_store.shape
    n = q.shape[0] if n_layers is None else n_layers
    _f16c(q, "q")
    assert q.is_contiguous() and q.shape == (n, H, d), (q.shape, (n, H, d))
    ws_bytes = lib().tf_retrieval_build_workspace_bytes(n, H, d, prefill, chunk, budget)
    ws = torch.empty(max(ws_bytes, 16), dtype=torch.uint8, device=q.device)
    if out_idx is not None:
        assert out_idx.dtype == torch.int32 and out_idx.is_contiguous() and out_idx.shape == (n, H, budget // chunk)
    if out_scores is not None:
        assert out_scores.dtype == torch.float16 and out_scores.is_contiguous() and out_scores.shape == (n, H, prefill // chunk)
    check(lib().tf_retrieval_build(key_store[layer0].data_ptr(), value_store[layer0].data_ptr(), key_store.stride(0),
                                   key_store.stride(1), q.data_ptr(), n, H, d, prefill, chunk, budget,
                                   retr_key_store[layer0].data_ptr(), retr_value_store[layer0].data_ptr(),
                                   retr_key_store.stride(0), retr_key_store.stride(1), ptr(out_idx), ptr(out_scores),
                                   ws.data_ptr(), ws.numel(), stream_ptr()), "tf_retrieval_build")
    COUNTER.n += 3


def retrieval_build_gqa(key_store, value_store, q, retr_key_store, retr_value_store, prefill: int, chunk: int, budget: int,
                        layer0: int = 0, n_layers: Optional[int] = None, out_idx=None, out_scores=None):
    """retrieval_build for a grouped-query target under the "group_sum" rule (tf_retrieval_build_gqa): stores [L,Hkv,cap,d];
    q [n_layers,Hq,d]; out_idx [n,Hkv,budget/chunk]; out_scores [n,Hkv,prefill/chunk]."""
    require_cuda(key_store, value_store, q, retr_key_store, retr_value_store)
    L, Hkv, cap, d = key_store.shape
    n = q.shape[0] if n_layers is None else n_layers
    Hq = q.shape[1]
    _f16c(q, "q")
    assert q.is_contiguous() and q.shape == (n, Hq, d), (q.shape, (n, Hq, d))
    ws_bytes = lib().tf_retrieval_build_workspace_bytes(n, Hkv, d, prefill, chunk, budget)
    ws = torch.empty(max(ws_bytes, 16), dtype=torch.uint8, device=q.device)
    if out_idx is not None:
        assert out_idx.dtype == torch.int32 and out_idx.is_contiguous() and out_idx.shape == (n, Hkv, budget // chunk)
    if out_scores is not None:
        assert out_scores.dtype == torch.float16 and out_scores.is_contiguous() and out_scores.shape == (n, Hkv, prefill // chunk)
    check(lib().tf_retrieval_build_gqa(key_store[layer0].data_ptr(), value_store[layer0].data_ptr(), key_store.stride(0),
                                       key_store.stride(1), q.data_ptr(), n, Hq, Hkv, d, prefill, chunk, budget,
                                       retr_key_store[layer0].data_ptr(), retr_value_store[layer0].data_ptr(),
                                       retr_key_store.stride(0), retr_key_store.stride(1), ptr(out_idx), ptr(out_scores),
                                       ws.data_ptr(), ws.numel(), stream_ptr()), "tf_retrieval_build_gqa")
    COUNTER.n += 3


def rope_append(qkv: torch.Tensor, H: int, d: int, cos, sin, q_out, key_layer, value_layer, *, pos_ids=None, pos0: int = 0,
                pos0_dev=None, slot0: int = 0, slot0_dev=None, rotate_q=True, rotate_k=True):
    """qkv [R, 3*H*d] (q|k|v); key_layer/value_layer [H,cap,d] of one layer; q_out [R,H,d]."""
    require_cuda(qkv, cos, sin, q_out, key_layer, value_layer)
    _f16c(qkv, "qkv")
    R = qkv.shape[0]
    assert qkv.stride(1) == 1 and qkv.shape[1] == 3 * H * d
    assert q_out.is_contiguous() and key_layer.stride(2) == 1 and key_layer.stride(1) == d
    base = qkv.data_ptr()
    es = qkv.element_size()
    if pos_ids is not None:
        assert pos_ids.dtype == torch.int32 and pos_ids.numel() >= R
    check(lib().tf_rope_append(base, base + H * d * es, base + 2 * H * d * es, qkv.stride(0), cos.data_ptr(), sin.data_ptr(),
                               cos.shape[0], ptr(pos_ids), pos0, ptr(pos0_dev), slot0, ptr(slot0_dev), R, H, d,
                               int(rotate_q), int(rotate_k), q_out.data_ptr(), key_layer.data_ptr(), value_layer.data_ptr(),
                               key_layer.stride(0), key_layer.shape[1], stream_ptr()), "tf_rope_append")
    COUNTER.n += 1


def rope_append_gqa(qkv: torch.Tensor, Hq: int, Hkv: int, d: int, cos, sin, q_out, key_layer, value_layer, *, pos_ids=None,
                    pos0: int = 0, pos0_dev=None, slot0: int = 0, slot0_dev=None):
    """qkv [R, (Hq + 2 Hkv) d] (q|k|v); key_layer/value_layer [Hkv,cap,d] of one layer; q_out [R,Hq,d] (tf_rope_append_gqa)."""
    require_cuda(qkv, cos, sin, q_out, key_layer, value_layer)
    _f16c(qkv, "qkv")
    R = qkv.shape[0]
    assert qkv.stride(1) == 1 and qkv.shape[1] == (Hq + 2 * Hkv) * d
    assert q_out.is_contiguous() and q_out.shape == (R, Hq, d) and key_layer.stride(2) == 1 and key_layer.stride(1) == d
    assert key_layer.shape[0] == Hkv
    base = qkv.data_ptr()
    es = qkv.element_size()
    if pos_ids is not None:
        assert pos_ids.dtype == torch.int32 and pos_ids.numel() >= R
    check(lib().tf_rope_append_gqa(base, base + Hq * d * es, base + (Hq + Hkv) * d * es, qkv.stride(0), cos.data_ptr(),
                                   sin.data_ptr(), cos.shape[0], ptr(pos_ids), pos0, ptr(pos0_dev), slot0, ptr(slot0_dev), R, Hq,
                                   Hkv, d, 1, 1, q_out.data_ptr(), key_layer.data_ptr(), value_layer.data_ptr(),
                                   key_layer.stride(0), key_layer.shape[1], stream_ptr()), "tf_rope_append_gqa")
    COUNTER.n += 1


def verify_attn_workspace(R: int, H: int, d: int, device) -> torch.Tensor:
    n = lib().tf_verify_attn_workspace_bytes(R, H, d)
    return torch.zeros(n, dtype=torch.uint8, device=device)  # the per-head arrival counters must start at zero


def verify_attn(q, maps: KVTensorMaps, layer: int, kv_len: int, R: int, H: int, d: int, scale: float, out, workspace,
                kv_len_dev=None, kv_len_max: Optional[int] = None, variant: int = 0, clean_keys: int = 0,
                next_weights: Optional[torch.Tensor] = None):
    """`next_weights`: the weight matrix the next kernel streams (o_proj); behind a short store the kernel prefetches it into L2
    (tf_verify_attn_prefetch).  Must be one dense allocation (the whole storage range [data_ptr, +nbytes) is prefetched)."""
    require_cuda(q, out, workspace)
    _f16c(q, "q")
    assert q.is_contiguous() and out.is_contiguous() and q.shape[-3:] == (R, H, d)
    cap = maps.shape[2]
    if kv_len_max is None:
        kv_len_max = cap if kv_len_dev is not None else kv_len
    if next_weights is not None and next_weights.is_contiguous():
        check(lib().tf_verify_attn_prefetch(q.data_ptr(), maps.k_ptr, maps.v_ptr, layer, kv_len, ptr(kv_len_dev), min(kv_len_max, cap), R, H,
                                            d, scale, out.data_ptr(), workspace.data_ptr(), workspace.numel(), variant, clean_keys,
                                            next_weights.data_ptr(), next_weights.numel() * next_weights.element_size(), stream_ptr()),
              "tf_verify_attn_prefetch")
        COUNTER.n += 1
        return
    check(lib().tf_verify_attn(q.data_ptr(), maps.k_ptr, maps.v_ptr, layer, kv_len, ptr(kv_len_dev), min(kv_len_max, cap), R, H,
                               d, scale, out.data_ptr(), workspace.data_ptr(), workspace.numel(), variant, clean_keys, stream_ptr()),
          "tf_verify_attn")
    COUNTER.n += 1


def verify_attn_calibrate(q, maps: KVTensorMaps, layer: int, kv_len: int, R: int, H: int, d: int, scale: float, out, workspace,
                          rounds: int = 4) -> dict:
    """Init-time load balancing of `verify_attn` (tf_verify_attn_calibrate): measures per-CTA streaming time on this KV
    store and installs a split table in `workspace`.  Synchronises the stream.  Returns the before/after report."""
    import ctypes

    require_cuda(q, out, workspace)
    _f16c(q, "q")
    assert q.is_contiguous() and out.is_contiguous() and q.shape[-3:] == (R, H, d)
    rep = (ctypes.c_double * 4)()
    check(lib().tf_verify_attn_calibrate(q.data_ptr(), maps.k_ptr, maps.v_ptr, layer, min(kv_len, maps.shape[2]), R, H, d, scale,
                                         out.data_ptr(), workspace.data_ptr(), workspace.numel(), rounds,
                                         ctypes.addressof(rep), stream_ptr()), "tf_verify_attn_calibrate")
    COUNTER.n += 3 * (rounds + 1) if rounds > 0 else 0
    return {"spread_before": rep[0], "spread_after": rep[1], "median_ns_before": rep[2], "median_ns_after": rep[3]}


def verify_attn_tree(q, maps: KVTensorMaps, layer: int, kv_len: int, R: int, H: int, d: int, scale: float, tree_mask: torch.Tensor,
                     tree_cols: int, out, workspace, kv_len_dev=None, kv_len_max: Optional[int] = None):
    """Tree-masked variant: `tree_mask` uint32/int32 [R, tree_cols/32] (bit set = visible) for the LAST tree_cols keys."""
    require_cuda(q, out, workspace, tree_mask)
    _f16c(q, "q")
    assert q.is_contiguous() and out.is_contiguous() and q.shape[-3:] == (R, H, d)
    assert tree_mask.is_contiguous() and tree_mask.element_size() == 4 and tree_mask.numel() >= R * (tree_cols // 32)
    cap = maps.shape[2]
    if kv_len_max is None:
        kv_len_max = cap if kv_len_dev is not None else kv_len
    check(lib().tf_verify_attn_tree(q.data_ptr(), maps.k_ptr, maps.v_ptr, layer, kv_len, ptr(kv_len_dev), min(kv_len_max, cap), R, H, d,
                                    scale, tree_mask.data_ptr(), tree_cols, out.data_ptr(), workspace.data_ptr(), workspace.numel(),
                                    stream_ptr()), "tf_verify_attn_tree")
    COUNTER.n += 1


def verify_attn_gqa_workspace(Hq: int, Hkv: int, d: int, device) -> torch.Tensor:
    n = lib().tf_verify_attn_gqa_workspace_bytes(VERIFY_MAX_ROWS, Hq, Hkv, d)
    if n == 0:
        raise ValueError(f"no verify-attention workspace for Hq={Hq}, Hkv={Hkv}, d={d}")
    return torch.zeros(n, dtype=torch.uint8, device=device)  # the per-KV-head arrival counters must start at zero


def gqa_row_block(Hq: int, Hkv: int) -> int:
    """Token rows per tf_verify_attn_gqa launch: a CTA holds the rows of a whole query-head group, at most VERIFY_MAX_ROWS."""
    return VERIFY_MAX_ROWS // (Hq // Hkv)


def verify_attn_gqa(q, maps: KVTensorMaps, layer: int, kv_len: int, R: int, Hq: int, Hkv: int, d: int, scale: float, out,
                    workspace, kv_len_dev=None, kv_len_max: Optional[int] = None, clean_keys: int = 0, tree_mask=None,
                    tree_cols: int = 0):
    """Verify attention of R token rows of Hq query heads over the Hkv-head store `maps` (tf_verify_attn_gqa, or
    tf_verify_attn_tree_gqa with `tree_mask` [R, tree_cols/32] over token rows).  The rows are cut into blocks of
    gqa_row_block(Hq, Hkv) token rows; block [r0, r1) sees kv_len - (R - r1) keys, which keeps it bottom-right aligned in
    causal mode.  Tree blocks keep kv_len (the tree columns are the last keys) and take their own rows of the mask."""
    require_cuda(q, out, workspace)
    _f16c(q, "q")
    assert q.is_contiguous() and out.is_contiguous() and q.shape[-3:] == (R, Hq, d) and out.shape == q.shape
    assert maps.shape[1] == Hkv, (maps.shape, Hkv)
    cap = maps.shape[2]
    if kv_len_max is None:
        kv_len_max = cap if kv_len_dev is not None else kv_len
    if tree_mask is not None:
        assert tree_mask.is_contiguous() and tree_mask.element_size() == 4 and tree_mask.shape == (R, tree_cols // 32)
    step = gqa_row_block(Hq, Hkv)
    if step < 1:
        raise ValueError(f"{Hq // Hkv} query heads per KV head exceed the {VERIFY_MAX_ROWS} rows of a verify-attention CTA")
    for r0 in range(0, R, step):
        r1 = min(R, r0 + step)
        shift = R - r1  # rows after this block: their keys are not visible to it
        if tree_mask is None:
            check(lib().tf_verify_attn_gqa(q[r0:r1].data_ptr(), maps.k_ptr, maps.v_ptr, layer, kv_len - shift, ptr(kv_len_dev),
                                           min(kv_len_max, cap), r1 - r0, Hq, Hkv, d, scale, out[r0:r1].data_ptr(),
                                           workspace.data_ptr(), workspace.numel(), 0, clean_keys, stream_ptr()),
                  "tf_verify_attn_gqa")
        else:
            check(lib().tf_verify_attn_tree_gqa(q[r0:r1].data_ptr(), maps.k_ptr, maps.v_ptr, layer, kv_len, ptr(kv_len_dev),
                                                min(kv_len_max, cap), r1 - r0, Hq, Hkv, d, scale, tree_mask[r0:r1].data_ptr(),
                                                tree_cols, out[r0:r1].data_ptr(), workspace.data_ptr(), workspace.numel(),
                                                stream_ptr()),
                  "tf_verify_attn_tree_gqa")
        COUNTER.n += 1


def tree_attn_tc_workspace(R: int, H: int, kv_len_max: int, device) -> torch.Tensor:
    return torch.empty(lib().tf_tree_attn_tc_workspace_bytes(R, H, kv_len_max), dtype=torch.uint8, device=device)


def tree_attn_tc(q, maps: KVTensorMaps, layer: int, kv_len: int, R: int, H: int, d: int, scale: float, tree_mask: Optional[torch.Tensor],
                 tree_cols: int, out, workspace, debug_scores: Optional[torch.Tensor] = None, causal: bool = False):
    """wgmma tensor-core attention (tf_tree_attn_tc), d = 128: tree-verify (`tree_mask` as in verify_attn_tree), plain, or — with
    causal=True — the bottom-right causal attention of R new rows over kv_len keys (prefill chunks)."""
    require_cuda(q, out, workspace)
    _f16c(q, "q")
    assert q.is_contiguous() and out.is_contiguous() and q.shape[-3:] == (R, H, d)
    if tree_cols:
        assert tree_mask is not None and tree_mask.is_contiguous() and tree_mask.element_size() == 4 and tree_mask.numel() >= R * (tree_cols // 32)
    if debug_scores is not None:
        assert debug_scores.dtype == torch.float32 and debug_scores.is_contiguous() and debug_scores.numel() >= 128 * 128
    check(lib().tf_tree_attn_tc(q.data_ptr(), maps.k_ptr, maps.v_ptr, layer, kv_len, R, H, d, scale, ptr(tree_mask) if tree_cols else None,
                                tree_cols, 1 if causal else 0, out.data_ptr(), workspace.data_ptr(), workspace.numel(), ptr(debug_scores),
                                stream_ptr()),
          "tf_tree_attn_tc")
    COUNTER.n += 2


def tree_attn_tc_gqa(q, maps: KVTensorMaps, layer: int, kv_len: int, R: int, Hq: int, Hkv: int, d: int, scale: float,
                     tree_mask: Optional[torch.Tensor], tree_cols: int, out, workspace, causal: bool = False):
    """tree_attn_tc for Hq query heads over the Hkv-head store `maps` (tf_tree_attn_tc_gqa); workspace from
    tree_attn_tc_workspace(R, Hq, kv_len_max)."""
    require_cuda(q, out, workspace)
    _f16c(q, "q")
    assert q.is_contiguous() and out.is_contiguous() and q.shape[-3:] == (R, Hq, d) and maps.shape[1] == Hkv
    if tree_cols:
        assert tree_mask is not None and tree_mask.is_contiguous() and tree_mask.element_size() == 4 and tree_mask.numel() >= R * (tree_cols // 32)
    check(lib().tf_tree_attn_tc_gqa(q.data_ptr(), maps.k_ptr, maps.v_ptr, layer, kv_len, R, Hq, Hkv, d, scale,
                                    ptr(tree_mask) if tree_cols else None, tree_cols, 1 if causal else 0, out.data_ptr(),
                                    workspace.data_ptr(), workspace.numel(), stream_ptr()), "tf_tree_attn_tc_gqa")
    COUNTER.n += 2


def kv_compact(key_store, value_store, src_idx: torch.Tensor, dst_start: int):
    """gather_kv_incremental: rows src_idx (absolute slots, int32 device tensor) -> dst_start.. in every (layer, head)."""
    L, H, cap, d = key_store.shape
    assert src_idx.dtype == torch.int32 and src_idx.is_cuda
    check(lib().tf_kv_compact(key_store.data_ptr(), value_store.data_ptr(), key_store.stride(0), key_store.stride(1), L, H, d,
                              src_idx.data_ptr(), src_idx.numel(), dst_start, stream_ptr()), "tf_kv_compact")
    COUNTER.n += 1


def draft_attn(q, key_layer, value_layer, cos, sin, kv_len: int, scale: float, out):
    require_cuda(q, key_layer, value_layer, cos, sin, out)
    R, H, d = q.shape
    assert q.is_contiguous() and out.is_contiguous() and key_layer.stride(1) == d
    check(lib().tf_draft_attn(q.data_ptr(), key_layer.data_ptr(), value_layer.data_ptr(), key_layer.stride(0), cos.data_ptr(),
                              sin.data_ptr(), kv_len, R, H, d, scale, out.data_ptr(), stream_ptr()), "tf_draft_attn")
    COUNTER.n += 1


def tail_update(key_store, value_store, retr_key_store, retr_value_store, prefill: int, budget: int, seq_len: int,
                seq_len_dev=None, max_new: int = 0):
    L, H, cap, d = key_store.shape
    check(lib().tf_tail_update(key_store.data_ptr(), value_store.data_ptr(), key_store.stride(0), key_store.stride(1),
                               retr_key_store.data_ptr(), retr_value_store.data_ptr(), retr_key_store.stride(0),
                               retr_key_store.stride(1), L, H, d, prefill, budget, seq_len, ptr(seq_len_dev), max_new,
                               stream_ptr()), "tf_tail_update")
    COUNTER.n += 1


def window_slide(key_store, value_store, src_start: int, dst_start: int, n_rows: int):
    L, H, cap, d = key_store.shape
    assert src_start + n_rows <= cap and dst_start + n_rows <= cap
    check(lib().tf_window_slide(key_store.data_ptr(), value_store.data_ptr(), key_store.stride(0), key_store.stride(1), L, H, d,
                                src_start, dst_start, n_rows, stream_ptr()), "tf_window_slide")
    COUNTER.n += 1


def add_rmsnorm(h, delta, weight, eps: float, out):
    require_cuda(h, weight, out)
    rows, hidden = h.shape
    assert h.is_contiguous() and out.is_contiguous() and (delta is None or delta.is_contiguous())
    check(lib().tf_add_rmsnorm(h.data_ptr(), ptr(delta), weight.data_ptr(), eps, out.data_ptr(), rows, hidden, stream_ptr()),
          "tf_add_rmsnorm")
    COUNTER.n += 1


def silu_mul(gate_up, out):
    rows, two_i = gate_up.shape
    assert gate_up.is_contiguous() and out.is_contiguous()
    check(lib().tf_silu_mul(gate_up.data_ptr(), out.data_ptr(), rows, two_i // 2, stream_ptr()), "tf_silu_mul")
    COUNTER.n += 1


def skinny_gemm(x: torch.Tensor, W: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """y = x @ W.T for x [M<=16, K], W [N, K] (fp16, K % 32 == 0)."""
    require_cuda(x, W)
    _f16c(x, "x")
    _f16c(W, "W")
    M, K = x.shape
    N = W.shape[0]
    assert W.shape[1] == K and x.stride(1) == 1 and W.stride(1) == 1
    if out is None:
        out = torch.empty((M, N), dtype=torch.float16, device=x.device)
    check(lib().tf_skinny_gemm(x.data_ptr(), x.stride(0), W.data_ptr(), W.stride(0), M, N, K, out.data_ptr(), out.stride(0),
                               None, 0, stream_ptr()), "tf_skinny_gemm")
    COUNTER.n += 1
    return out


class WeightMap:
    """TMA descriptor of one weight matrix W [N, K] for `stream_linear` (tf_weight_tensormap_encode); keeps W alive.
    silu=True describes the [gate; up] stack of an MLP (8-row boxes, so that a tile pairs gate rows with their up rows)."""

    def __init__(self, W: torch.Tensor, silu: bool = False):
        require_cuda(W)
        _f16c(W, "W")
        assert W.dim() == 2 and W.stride(1) == 1
        self.W, self.silu = W, silu
        self.N, self.K = int(W.shape[0]), int(W.shape[1])
        self.buf = (ctypes.c_uint8 * 128)()
        check(lib().tf_weight_tensormap_encode(ctypes.addressof(self.buf), W.data_ptr(), self.N, self.K, W.stride(0), 8 if silu else 16),
              "tf_weight_tensormap_encode")
        self.ptr = ctypes.addressof(self.buf)

    @staticmethod
    def supported(W: torch.Tensor, rows: int = 8) -> bool:
        """K a multiple of 64 (the TMA view is [rows][K/64][64]); up to STREAM_MAX_ROWS token rows."""
        return W.is_cuda and W.dtype == torch.float16 and int(W.shape[1]) % 64 == 0 and rows <= STREAM_MAX_ROWS


class E4m3WeightMap:
    """One projection matrix stored in E4M3 (the format of include/triforce_b200.h): codes uint8 [N, K], exponents int8 [N] and
    the TMA descriptor of the codes for `stream_linear` (tf_weight_tensormap_encode_e4m3).  The matrix it stands for is
    D = code * 2^e, exact in fp16 (`weight_dequantize_e4m3`).  silu=True: the [gate; up] stack of an MLP."""

    def __init__(self, codes: torch.Tensor, exps: torch.Tensor, silu: bool = False):
        require_cuda(codes, exps)
        assert codes.dtype == torch.uint8 and codes.dim() == 2 and codes.is_contiguous()
        assert exps.dtype == torch.int8 and exps.is_contiguous() and exps.shape == (codes.shape[0],)
        self.codes, self.exps, self.silu = codes, exps, silu
        self.N, self.K = int(codes.shape[0]), int(codes.shape[1])
        self.buf = (ctypes.c_uint8 * 128)()
        check(lib().tf_weight_tensormap_encode_e4m3(ctypes.addressof(self.buf), codes.data_ptr(), self.N, self.K, codes.stride(0)),
              "tf_weight_tensormap_encode_e4m3")
        self.ptr = ctypes.addressof(self.buf)

    @staticmethod
    def quantize(W: torch.Tensor, silu: bool = False) -> "E4m3WeightMap":
        codes, exps = weight_quantize_e4m3(W)
        return E4m3WeightMap(codes, exps, silu=silu)

    def nbytes(self) -> int:
        return self.codes.numel() + self.exps.numel()


WEIGHT_E4M3_MAX = 61440.0  # 240 * 2^8: above it D = code * 2^e can round past the fp16 maximum


def weight_quantize_e4m3(W: torch.Tensor, codes: Optional[torch.Tensor] = None, exps: Optional[torch.Tensor] = None):
    """fp16 W [N, K] (K % 64 == 0) -> (codes uint8 [N, K], exponents int8 [N]) (tf_weight_quantize_e4m3).  Raises ValueError
    when a row is not finite or has max|w| > WEIGHT_E4M3_MAX (synchronises the stream to read the count)."""
    require_cuda(W)
    _f16c(W, "W")
    assert W.dim() == 2 and W.stride(1) == 1
    N, K = int(W.shape[0]), int(W.shape[1])
    if K % 64:
        raise ValueError(f"E4M3 weights need K a multiple of 64, got K={K}")
    if codes is None:
        codes = torch.empty((N, K), dtype=torch.uint8, device=W.device)
    if exps is None:
        exps = torch.empty(N, dtype=torch.int8, device=W.device)
    assert codes.dtype == torch.uint8 and codes.shape == (N, K) and codes.stride(1) == 1
    assert exps.dtype == torch.int8 and exps.shape == (N,) and exps.is_contiguous()
    refused = torch.zeros(1, dtype=torch.int32, device=W.device)
    check(lib().tf_weight_quantize_e4m3(W.data_ptr(), W.stride(0), N, K, codes.data_ptr(), codes.stride(0), exps.data_ptr(),
                                        refused.data_ptr(), stream_ptr()), "tf_weight_quantize_e4m3")
    COUNTER.n += 1
    bad = int(refused.item())
    if bad:
        raise ValueError(f"{bad} of {N} weight rows cannot be stored in E4M3: not finite, or max|w| > {WEIGHT_E4M3_MAX:g}")
    return codes, exps


def weight_dequantize_e4m3(codes: torch.Tensor, exps: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """D = code * 2^e as fp16 [N, K] (tf_weight_dequantize_e4m3); `out` may be a wider-strided view."""
    require_cuda(codes, exps)
    N, K = int(codes.shape[0]), int(codes.shape[1])
    assert codes.dtype == torch.uint8 and codes.stride(1) == 1 and exps.dtype == torch.int8 and exps.shape == (N,)
    if out is None:
        out = torch.empty((N, K), dtype=torch.float16, device=codes.device)
    _f16c(out, "out")
    assert out.shape == (N, K) and out.stride(1) == 1
    check(lib().tf_weight_dequantize_e4m3(codes.data_ptr(), codes.stride(0), exps.data_ptr(), N, K, out.data_ptr(), out.stride(0),
                                          stream_ptr()), "tf_weight_dequantize_e4m3")
    COUNTER.n += 1
    return out


STREAM_MAX_ROWS = 24
_LINEAR_WS = {}


def stream_linear_workspace(device) -> torch.Tensor:
    """Zero-filled hand-over buffer of `stream_linear` (one per device and stream; the kernel leaves it zero)."""
    key = (torch.device(device).index, stream_ptr())
    ws = _LINEAR_WS.get(key)
    if ws is None:
        ws = _LINEAR_WS[key] = torch.zeros(lib().tf_stream_linear_workspace_bytes(), dtype=torch.uint8, device=device)
    return ws


def stream_linear(x: torch.Tensor, W, *, silu: bool = False, out_fp32: bool = False, out: Optional[torch.Tensor] = None,
                  workspace: Optional[torch.Tensor] = None) -> torch.Tensor:
    """y = epilogue(x @ W.T) in one weight-streaming kernel (tf_stream_linear), x [M<=24, K], W a WeightMap (or a tensor,
    encoded on the fly).  silu: W = [gate; up] and y[M, N/2] = SiLU(gate) * up.  out_fp32: y = float(fp16(x @ W.T)).
    W an E4m3WeightMap: tf_stream_linear_e4m3, bit-identical to the fp16 kernel on D."""
    e4m3 = isinstance(W, E4m3WeightMap)
    if not e4m3 and not isinstance(W, WeightMap):
        W = WeightMap(W, silu=silu)
    assert W.silu == silu, "the WeightMap was encoded for the other epilogue"
    assert not (silu and out_fp32)
    require_cuda(x)
    _f16c(x, "x")
    M, K = x.shape
    N = W.N
    assert W.K == K and x.stride(1) == 1
    if out is None:
        out = torch.empty((M, N // 2 if silu else N), dtype=torch.float32 if out_fp32 else torch.float16, device=x.device)
    if workspace is None:
        workspace = stream_linear_workspace(x.device)
    epilogue = 1 if silu else (2 if out_fp32 else 0)
    if e4m3:
        check(lib().tf_stream_linear_e4m3(x.data_ptr(), x.stride(0), W.ptr, W.exps.data_ptr(), M, N, K, epilogue, out.data_ptr(),
                                          out.stride(0), workspace.data_ptr(), workspace.numel(), stream_ptr()), "tf_stream_linear_e4m3")
    else:
        check(lib().tf_stream_linear(x.data_ptr(), x.stride(0), W.ptr, M, N, K, epilogue, out.data_ptr(), out.stride(0),
                                     workspace.data_ptr(), workspace.numel(), stream_ptr()), "tf_stream_linear")
    COUNTER.n += 1
    return out


def norm_logits(logits: torch.Tensor, temperature: float, top_p: float, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    require_cuda(logits)
    assert logits.dim() == 2 and logits.dtype == torch.float32 and logits.stride(1) == 1
    rows, V = logits.shape
    if out is None:
        out = torch.empty((rows, V), dtype=torch.float32, device=logits.device)
    check(lib().tf_norm_logits(logits.data_ptr(), logits.stride(0), rows, V, temperature, top_p, out.data_ptr(), None, 0,
                               stream_ptr()), "tf_norm_logits")
    return out


def sample_argmax(probs: torch.Tensor, expo: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    require_cuda(probs, expo)
    p2 = probs.reshape(-1, probs.shape[-1])
    e2 = expo.reshape(-1, expo.shape[-1])
    assert p2.dtype == torch.float32 and e2.dtype == torch.float32 and p2.stride(1) == 1 and e2.stride(1) == 1
    rows, V = p2.shape
    if out is None:
        out = torch.empty(rows, dtype=torch.int64, device=probs.device)
    check(lib().tf_sample_argmax(p2.data_ptr(), p2.stride(0), e2.data_ptr(), e2.stride(0) if e2.shape[0] > 1 else 0, rows, V,
                                 out.data_ptr(), stream_ptr()), "tf_sample_argmax")
    COUNTER.n += 1
    return out


def residual_probs(p: torch.Tensor, q: torch.Tensor) -> torch.Tensor:
    out = torch.empty_like(p)
    check(lib().tf_residual_probs(p.data_ptr(), q.data_ptr(), p.shape[-1], out.data_ptr(), stream_ptr()), "tf_residual_probs")
    COUNTER.n += 1
    return out


def tree_accept_walk(target_probs, draft_logits, verify_tokens, succ_off, succ, uniforms, temperature: float, out, residual, scratch,
                     max_accept: int = 24):
    V = target_probs.shape[-1]
    assert target_probs.is_contiguous() and draft_logits.is_contiguous() and out.dtype == torch.int32 and out.numel() >= 32
    check(lib().tf_tree_accept_walk(target_probs.data_ptr(), draft_logits.data_ptr(), verify_tokens.data_ptr(), succ_off.data_ptr(),
                                    succ.data_ptr(), uniforms.data_ptr(), temperature, V, max_accept, out.data_ptr(), residual.data_ptr(),
                                    scratch.data_ptr(), stream_ptr()), "tf_tree_accept_walk")
    COUNTER.n += 1


def middle_accept(draft_probs, verify_probs, verify_tokens, uniform, expo, gamma: int, state, out_ids, spec_probs):
    V = draft_probs.shape[-1]
    check(lib().tf_middle_accept(draft_probs.data_ptr(), verify_probs.data_ptr(), verify_tokens.data_ptr(), uniform.data_ptr(),
                                 expo.data_ptr(), gamma, V, state.data_ptr(), out_ids.data_ptr(), spec_probs.data_ptr(),
                                 stream_ptr()), "tf_middle_accept")
    COUNTER.n += 1


def verify_accept(p_rows, q_rows, gen, g2: int, uniforms, strict_less: bool, eos_token: int, first_token: int, res, pass_tokens):
    V = p_rows.shape[-1]
    check(lib().tf_verify_accept(p_rows.data_ptr(), q_rows.data_ptr(), gen.data_ptr(), g2, uniforms.data_ptr(), V,
                                 int(strict_less), eos_token, first_token, res.data_ptr(), pass_tokens.data_ptr(), stream_ptr()),
          "tf_verify_accept")
    COUNTER.n += 1


def verify_resample(p_rows, q_rows, gen, g2: int, expo, res, out_token, pass_tokens):
    V = p_rows.shape[-1]
    check(lib().tf_verify_resample(p_rows.data_ptr(), q_rows.data_ptr(), gen.data_ptr(), g2, expo.data_ptr(), V, res.data_ptr(),
                                   out_token.data_ptr(), pass_tokens.data_ptr(), stream_ptr()), "tf_verify_resample")
    COUNTER.n += 1



# ---- whole-loop graph (tf_loop_*): device-side Middle_Spec / accept walk, Philox noise --------------------------------------------
def philox_fill(state: torch.Tensor, kind: int, out: torch.Tensor) -> torch.Tensor:
    """One draw of the device Philox stream (`state` int64[2] = {seed, next draw}) into `out` (fp32): kind 0 uniform, 1 exponential."""
    assert state.dtype == torch.int64 and state.numel() == 2 and out.dtype == torch.float32 and out.is_contiguous()
    check(lib().tf_philox_fill(state.data_ptr(), kind, out.data_ptr(), out.numel(), stream_ptr()), "tf_philox_fill")
    COUNTER.n += 1
    return out


def loop_begin(state, verify_tokens, first_token, gamma: int, seq_len_dev, position_ids):
    check(lib().tf_loop_begin(state.data_ptr(), verify_tokens.data_ptr(), first_token.data_ptr(), gamma, seq_len_dev.data_ptr(),
                              position_ids.data_ptr(), stream_ptr()), "tf_loop_begin")
    COUNTER.n += 1


def loop_draft_sample(draft_probs, state, rng, verify_tokens):
    assert draft_probs.is_contiguous() and draft_probs.dtype == torch.float32
    check(lib().tf_loop_draft_sample(draft_probs.data_ptr(), draft_probs.shape[-1], state.data_ptr(), rng.data_ptr(), verify_tokens.data_ptr(),
                                     stream_ptr()), "tf_loop_draft_sample")
    COUNTER.n += 1


def loop_middle_accept(draft_probs, verify_probs, verify_tokens, rng, gamma: int, state, out_ids, spec_probs):
    assert draft_probs.is_contiguous() and verify_probs.is_contiguous() and spec_probs.is_contiguous()
    check(lib().tf_loop_middle_accept(draft_probs.data_ptr(), verify_probs.data_ptr(), verify_tokens.data_ptr(), rng.data_ptr(), gamma,
                                      draft_probs.shape[-1], state.data_ptr(), out_ids.data_ptr(), spec_probs.data_ptr(), stream_ptr()),
          "tf_loop_middle_accept")
    COUNTER.n += 1


def loop_prepare_full(state, out_ids, first_token, full_ids):
    check(lib().tf_loop_prepare_full(state.data_ptr(), out_ids.data_ptr(), first_token.data_ptr(), full_ids.data_ptr(), full_ids.numel(),
                                     stream_ptr()), "tf_loop_prepare_full")
    COUNTER.n += 1


def loop_verify(p_rows, q_rows, out_ids, state, rng, strict_less: bool, eos: int, first_token, res, tokens, pass_tokens, seq_len_dev):
    assert p_rows.is_contiguous() and q_rows.is_contiguous() and res.dtype == torch.int32 and res.numel() >= 16
    check(lib().tf_loop_verify(p_rows.data_ptr(), q_rows.data_ptr(), out_ids.data_ptr(), state.data_ptr(), rng.data_ptr(), p_rows.shape[-1],
                               int(strict_less), eos, first_token.data_ptr(), res.data_ptr(), tokens.data_ptr(), pass_tokens.data_ptr(),
                               pass_tokens.numel(), seq_len_dev.data_ptr(), stream_ptr()), "tf_loop_verify")
    COUNTER.n += 1


def window_slide_dev(key_store, value_store, src_base: int, shift_dev, dst_start: int, n_rows: int):
    L, H, cap, d = key_store.shape
    check(lib().tf_window_slide_dev(key_store.data_ptr(), value_store.data_ptr(), key_store.stride(0), key_store.stride(1), L, H, d, src_base,
                                    shift_dev.data_ptr(), dst_start, n_rows, stream_ptr()), "tf_window_slide_dev")
    COUNTER.n += 1
