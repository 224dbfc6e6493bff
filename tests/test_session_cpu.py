"""CPU-side checks of follow-up turns: the argument checks of tf_tree_attn_tc_causal_e4m3 (no launch), the retrieval boundary
arithmetic and its refusals, RetrievalCache's shapes without max_context, and the refusals of LlamaModel.extend and Session
that run before anything touches a device."""
import ctypes
from types import SimpleNamespace

import pytest
import torch

from triforce_b200 import _C
from triforce_b200.cache import RetrievalCache
from triforce_b200.llama import LlamaModel
from triforce_b200.session import Session


def _buf():
    buf = (ctypes.c_uint8 * 512)()
    p = ctypes.addressof(buf)
    return buf, p, (p + 15) & ~15


def test_causal_e4m3_checks_its_arguments():
    lib = _C.lib()
    _keep, p, a = _buf()
    f = lib.tf_tree_attn_tc_causal_e4m3
    # (q, kmap, vmap, k_exp, v_exp, cap, layer, kv_len, R, Hq, Hkv, d, scale, out, ws, ws_bytes, stream)
    R, H, S, cap = 300, 32, 125228, 125248
    ws = lib.tf_tree_attn_tc_workspace_bytes(R, H, S)
    assert f(a, p, p, None, a, cap, 0, S, R, H, H, 128, 0.1, p, a, ws, None) == -1
    assert b"NULL exponent" in lib.tf_last_error()
    assert f(a, p, p, a, a, cap, 0, S, R, H, H, 64, 0.1, p, a, ws, None) == -2                  # head_dim 64
    assert f(a, p, p, a, a, cap, 0, S, R, H, H, 128, 0.1, p, a, ws - 1, None) == -1             # workspace 1 B short
    assert b"workspace" in lib.tf_last_error()
    assert f(a, p, p, a + 1, a, cap, 0, S, R, H, H, 128, 0.1, p, a, ws, None) == -1             # misaligned exponents
    assert b"16-byte aligned" in lib.tf_last_error()
    assert f(a, p, p, a, a, 125250, 0, S, R, H, H, 128, 0.1, p, a, ws, None) == -1             # cap % 64
    assert b"cap" in lib.tf_last_error()
    assert f(a, p, p, a, a, 125184, 0, S, R, H, H, 128, 0.1, p, a, ws, None) == -1             # kv_len > cap
    assert b"exceeds cap" in lib.tf_last_error()
    assert f(a, p, p, a, a, cap, 0, S, R, 32, 6, 128, 0.1, p, a, ws, None) == -1                # Hq % Hkv
    assert b"multiple of Hkv" in lib.tf_last_error()
    assert f(a, p, p, a, a, cap, 0, 299, R, H, H, 128, 0.1, p, a, ws, None) == -1               # kv_len < R
    assert b"causal" in lib.tf_last_error()
    assert f(a, p, p, a, a, cap, 0, S, 0, H, H, 128, 0.1, p, a, ws, None) == -1                 # no rows
    # R = 1 and R = 300 (not a multiple of 128), MHA and GQA pass every check up to the next one (a misaligned q), before any launch
    for rows, hkv in ((1, 32), (300, 32), (300, 8)):
        w = lib.tf_tree_attn_tc_workspace_bytes(rows, H, S)
        assert f(a + 2, p, p, a, a, cap, 0, S, rows, H, hkv, 128, 0.1, p, a, w, None) == -1
        assert b"q must be 16-byte aligned" in lib.tf_last_error()


def _model_stub(L=2, H=4, hidden=512):
    cfg = SimpleNamespace(num_hidden_layers=L, num_key_value_heads=H, hidden_size=hidden, num_attention_heads=H)
    return SimpleNamespace(config=cfg, device=torch.device("cpu"))


def test_retrieval_cache_without_max_context_keeps_its_shapes():
    gc = RetrievalCache(_model_stub(), max_budget=4096, prefill=124928, chunk_size=8, gamma=6)
    assert gc.max_context == 124928
    assert gc.chunk_scores.shape == (2, 4, 15616) and gc.chunk_scores.is_contiguous()
    assert gc.topk_idx.shape == (2, 4, 512) and gc.key_store.shape == (2, 4, 4103, 128)
    big = RetrievalCache(_model_stub(), max_budget=4096, prefill=124928, chunk_size=8, gamma=6, max_context=131072)
    assert big.chunk_scores.shape == (2, 4, 15616) and big.chunks == 15616
    with pytest.raises(ValueError, match="below prefill"):
        RetrievalCache(_model_stub(), max_budget=64, prefill=1024, max_context=512)


def test_boundary_arithmetic_and_refusals():
    gc = RetrievalCache(_model_stub(), max_budget=4096, prefill=124928, chunk_size=8, gamma=6, max_context=131072)
    assert gc.boundary(124928) == 124928
    assert gc.boundary(124928 + 7) == 124928
    assert gc.boundary(124928 + 300) == 125224
    assert gc.boundary(4096) == 4096 and gc.boundary(4103) == 4096
    with pytest.raises(ValueError, match="fewer than the retrieval budget"):
        gc.boundary(4095)
    with pytest.raises(ValueError, match="beyond max_context"):
        gc.boundary(131080)
    assert gc.boundary(131079) == 131072
    # reset returns to the constructed boundary
    gc.prefill, gc.chunks = 125224, 125224 // 8
    assert gc.chunk_scores.shape == (2, 4, 15653)
    gc.reset()
    assert (gc.prefill, gc.chunks) == (124928, 15616)


def test_extend_refuses_an_append_past_the_capacity():
    model = object.__new__(LlamaModel)
    kv = SimpleNamespace(seq_len=1000, slots=1024, kv_dtype="fp16")
    with pytest.raises(ValueError, match="exceeds the 1024 slots"):
        model.extend(torch.zeros(25, dtype=torch.long), kv)
    with pytest.raises(ValueError, match="at least one id"):
        model.extend(torch.zeros(0, dtype=torch.long), kv)


def _session(seq_len=5000, slots=8192, budget=4096):
    kv = SimpleNamespace(seq_len=seq_len, slots=slots)
    gc = RetrievalCache(_model_stub(), max_budget=budget, prefill=4096, chunk_size=8, gamma=6, max_context=slots)
    ge = SimpleNamespace(engine=SimpleNamespace(kv_cache=kv, graph_cache=gc))
    return Session(ge, gamma=6)


def test_session_refuses_calls_out_of_order():
    s = _session()
    with pytest.raises(RuntimeError, match="append before prefill"):
        s.append([1, 2, 3])
    with pytest.raises(RuntimeError, match="generate before prefill"):
        s.generate(16)
    with pytest.raises(RuntimeError, match="truncate before prefill"):
        s.truncate(10)
    s.ids = list(range(5000))  # as after a prefill whose turn was generated
    with pytest.raises(RuntimeError, match="call append"):
        s.generate(16)


def test_session_refuses_out_of_range_appends_and_truncations():
    s = _session()
    s.ids = list(range(5000))
    with pytest.raises(ValueError, match="exceeds the 8192 slots"):
        s.append(list(range(3193)))
    with pytest.raises(ValueError, match="at least one id"):
        s.append([])
    for n in (0, 5001, -3):
        with pytest.raises(ValueError, match="committed length is 5000"):
            s.truncate(n)
    s = _session(seq_len=4000)
    s.ids = list(range(4000))
    with pytest.raises(ValueError, match="fewer than the retrieval budget"):
        s.append(list(range(95)))  # 4095 tokens: a boundary of 4088 < 4096
    assert s.ids == list(range(4000)) and s.pending is None  # nothing changed
