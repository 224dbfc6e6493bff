"""CPU-side checks of the C-ABI boundary: the library loads, exports every symbol the header declares, and its argument
validation fails loudly with reference-style messages — no compute calls (there is no GPU in this tier)."""
import ctypes
import os
import re

import pytest

from triforce_b200 import _C

REPO = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))


def _header_symbols():
    src = open(os.path.join(REPO, "include", "triforce_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(tf_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_header_symbol():
    lib = _C.lib()
    names = _header_symbols()
    assert len(names) >= 20
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/triforce_b200.h but not exported"
    assert set(names) == set(_C.EXPORTED_SYMBOLS), set(names) ^ set(_C.EXPORTED_SYMBOLS)


def test_version_and_error_string():
    lib = _C.lib()
    assert lib.tf_version() >= 100
    rc = lib.tf_retrieval_build(None, None, 0, 0, None, 1, 1, 128, 64, 8, 8, None, None, 0, 0, None, None, None, 0, None)
    assert rc == -1
    assert b"NULL" in lib.tf_last_error()


def test_reference_assert_messages_are_kept():
    """RetrievalCache.__init__ asserts (cache.py:126-127) surface from the C ABI with the same wording."""
    lib = _C.lib()
    buf = (ctypes.c_uint8 * 64)()
    p = ctypes.addressof(buf)
    rc = lib.tf_retrieval_build(p, p, 8, 8, p, 1, 1, 128, 100, 8, 64, p, p, 8, 8, None, None, p, 64, None)
    assert rc == -1 and b"prefill should be multiple of chunk_size" in lib.tf_last_error()
    rc = lib.tf_retrieval_build(p, p, 8, 8, p, 1, 1, 128, 64, 8, 12, p, p, 8, 8, None, None, p, 64, None)
    assert rc == -1 and b"max_budget should be multiple of chunk_size" in lib.tf_last_error()
    rc = lib.tf_retrieval_build(p, p, 8, 8, p, 1, 1, 128, 64, 8, 128, p, p, 8, 8, None, None, p, 64, None)
    assert rc == -1 and b"out of range" in lib.tf_last_error()  # torch.topk's error in the reference


def test_unsupported_shapes_are_rejected():
    lib = _C.lib()
    buf = (ctypes.c_uint8 * 256)()
    p = ctypes.addressof(buf)
    assert lib.tf_verify_attn(p, p, p, 0, 64, None, 64, 33, 1, 128, 0.1, p, p, 1 << 30, 0, 0, None) == -1  # R > 32
    assert lib.tf_verify_attn(p, p, p, 0, 64, None, 64, 4, 1, 96, 0.1, p, p, 1 << 30, 0, 0, None) == -2   # head_dim 96
    assert lib.tf_norm_logits(p, 70000, 1, 70000, 1.0, 0.9, p, None, 0, None) == -2                    # vocab too large
    assert lib.tf_verify_attn_workspace_bytes(8, 32, 128) > 0
    # tf_tree_attn_tc(q, kmap, vmap, layer, kv_len, R, H, d, scale, tree_mask, tree_cols, causal, out, ws, ws_bytes, dbg, stream)
    a = (p + 15) & ~15  # 16-byte aligned workspace
    R, H, S = 512, 32, 4096
    ws = lib.tf_tree_attn_tc_workspace_bytes(R, H, S)
    assert ws > 0
    assert lib.tf_tree_attn_tc(p, p, p, 0, S, R, H, 64, 0.1, p, 512, 0, p, a, ws, None, None) == -2   # head_dim 64
    assert lib.tf_tree_attn_tc(p, p, p, 0, S, R, H, 128, 0.1, p, 512, 1, p, a, ws, None, None) == -1  # causal with a tree
    assert b"causal" in lib.tf_last_error()
    assert lib.tf_tree_attn_tc(p, p, p, 0, S, R, H, 128, 0.1, p, 500, 0, p, a, ws, None, None) == -1  # tree_cols % 32
    assert b"multiple of 32" in lib.tf_last_error()
    assert lib.tf_tree_attn_tc(p, p, p, 0, S, R, H, 128, 0.1, p, 512, 0, p, a, ws - 1, None, None) == -1  # workspace 1 B short
    assert b"workspace" in lib.tf_last_error()
    # the exact workspace size passes that check: the call stops at the next one (a misaligned q), before any launch
    assert lib.tf_tree_attn_tc(a + 2, p, p, 0, S, R, H, 128, 0.1, p, 512, 0, p, a, ws, None, None) == -1
    assert b"q must be 16-byte aligned" in lib.tf_last_error()


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    monkeypatch.setattr(_C, "_lib", None)
    monkeypatch.setattr(_C, "LIB_PATH", str(tmp_path / "nope.so"))
    with pytest.raises(_C.TriForceNativeError, match="no CPU or PyTorch fallback"):
        _C.lib()
