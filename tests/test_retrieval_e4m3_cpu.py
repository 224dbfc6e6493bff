"""E4M3 retrieval cache without a GPU: argument checks of the three new entry points of the C ABI, the refusals, the bytes a
retrieval forward reads, and the --retrieval_dtype switch of test/on_chip.py and test/offloading_TP.py."""
from __future__ import annotations

import ctypes
from types import SimpleNamespace

import pytest

from triforce_b200 import _C


def test_retrieval_e4m3_entry_points_check_their_arguments():
    lib = _C.lib()
    buf = (ctypes.c_uint8 * 512)()
    p = ctypes.addressof(buf)
    a = (p + 15) & ~15
    big = 1 << 30
    # tf_retrieval_build_to_e4m3(K, V, Ke, Ve, ls, hs, q, n_layers, Hq, Hkv, d, prefill, chunk, budget, rK, rV, rKe, rVe, rls, rhs,
    #                            idx, scores, ws, ws_bytes, stream)
    build = lib.tf_retrieval_build_to_e4m3
    assert build(a, a, None, a, 8192, 8192, a, 1, 8, 8, 128, 64, 8, 8, a, a, a, a, 8192, 128, None, None, a, 64, None) == -1
    assert b"exponent" in lib.tf_last_error()  # one source exponent pointer without the other
    assert build(a, a, None, None, 8192, 8192, a, 1, 8, 8, 128, 64, 8, 8, a, a, None, a, 8192, 128, None, None, a, 64, None) == -1
    assert build(a, a, None, None, 8192, 8192, a, 1, 30, 8, 128, 64, 8, 8, a, a, a, a, 8192, 128, None, None, a, 64, None) == -1
    assert b"multiple" in lib.tf_last_error()
    assert build(a, a, None, None, 8192, 8192, a, 1, 8, 8, 128, 64, 8, 8, a, a, a, a, 8200, 128, None, None, a, 64, None) == -1
    assert b"strides" in lib.tf_last_error()
    assert build(a, a, None, None, 8192, 8192, a, 1, 8, 8, 256, 64, 8, 8, a, a, a, a, 8192, 256, None, None, a, 64, None) == -2
    assert build(a, a, None, None, 8192, 8192, a, 1, 8, 8, 128, 64, 8, 16, a, a, a, a, 8192, 128, None, None, a, 0, None) == -1
    # tf_tail_update_to_e4m3(K, V, Ke, Ve, ls, hs, rK, rV, rKe, rVe, rls, rhs, L, H, d, prefill, budget, seq_len, seq_len_dev,
    #                        max_new, stream)
    tail = lib.tf_tail_update_to_e4m3
    assert tail(a, a, None, None, 8192, 8192, a, a, None, a, 8192, 128, 1, 1, 128, 0, 8, 4, None, 0, None) == -1
    assert b"NULL" in lib.tf_last_error()
    assert tail(a, a, a, None, 8192, 8192, a, a, a, a, 8192, 128, 1, 1, 128, 0, 8, 4, None, 0, None) == -1
    assert tail(a, a, None, None, 8192, 8192, a, a, a, a, 8192, 128, 1, 1, 96, 0, 8, 4, None, 0, None) == -2
    assert tail(a, a, None, None, 8192, 8200, a, a, a, a, 8192, 128, 1, 1, 128, 0, 8, 4, None, 0, None) == -1  # stride % d
    assert tail(a, a, None, None, 8192, 8192, a, a, a, a, 8192, 128, 1, 1, 128, 0, 8, 12, None, 0, None) == -1  # > budget
    assert b"budget" in lib.tf_last_error()
    assert tail(a, a, None, None, 8192, 8192, a, a, a, a, 8192, 128, 1, 1, 128, 0, 8, 0, a, 9, None) == -1   # max_new > budget
    assert tail(a, a, None, None, 8192, 8192, a, a, a, a, 8192, 128, 1, 1, 128, 16, 8, 4, None, 0, None) == 0  # nothing new
    # tf_verify_attn_e4m3_clean(q, kmap, vmap, kexp, vexp, cap, layer, kv_len, kv_len_dev, kv_len_max, R, Hq, Hkv, d, scale, out,
    #                           ws, ws_bytes, clean_keys, stream)
    ver = lib.tf_verify_attn_e4m3_clean
    assert ver(a, p, p, a, a, 128, 0, 64, None, 64, 8, 32, 8, 128, 0.1, a, a, big, -1, None) == -1
    assert b"clean_keys" in lib.tf_last_error()
    assert ver(a, p, p, a, a, 128, 0, 64, None, 64, 8, 32, 8, 128, 0.1, a, a, big, 192, None) == -1
    assert ver(a, p, p, None, a, 128, 0, 64, None, 64, 8, 32, 8, 128, 0.1, a, a, big, 64, None) == -1
    assert b"NULL" in lib.tf_last_error()
    assert ver(a, p, p, a, a, 100, 0, 64, None, 64, 8, 32, 8, 128, 0.1, a, a, big, 64, None) == -1  # cap % 64
    assert ver(a, p, p, a, a, 128, 0, 64, None, 64, 8, 30, 8, 128, 0.1, a, a, big, 64, None) == -1  # Hq % Hkv
    assert ver(a, p, p, a, a, 128, 0, 64, None, 64, 8, 32, 8, 96, 0.1, a, a, big, 64, None) == -2


def test_paths_without_an_e4m3_retrieval_cache_refuse_it():
    from triforce_b200.cache import RetrievalCache, RetrievalCacheSeqouia
    from triforce_b200.tp import DistributedLlama

    with pytest.raises(NotImplementedError, match="Sequoia tree path"):
        RetrievalCacheSeqouia(SimpleNamespace(), kv_dtype="e4m3")
    with pytest.raises(ValueError, match="kv_dtype"):
        RetrievalCache(SimpleNamespace(), kv_dtype="fp8")
    with pytest.raises(ValueError, match="retrieval_dtype"):
        DistributedLlama("llama-7B-128K", retrieval_dtype="int8")
    # the TP refusals of the full store and the weights stay as they are
    with pytest.raises(NotImplementedError, match="tensor parallel"):
        DistributedLlama("llama-7B-128K", kv_dtype="e4m3", retrieval_dtype="e4m3")
    with pytest.raises(NotImplementedError, match="tensor parallel"):
        DistributedLlama("llama-7B-128K", weight_dtype="e4m3", retrieval_dtype="e4m3")
    assert DistributedLlama("llama-7B-128K", retrieval_dtype="e4m3").retrieval_dtype == "e4m3"
    cache = object.__new__(RetrievalCache)
    cache.e4m3 = object()
    with pytest.raises(NotImplementedError, match="rope_append_e4m3"):
        cache.update(None, None, 0)


def _read_bytes(layers, heads, slots, d, dtype):
    """K and V bytes one retrieval forward reads: every slot of every layer, plus one exponent byte per E4M3 row."""
    per_row = 2 * d if dtype == "fp16" else d + 1
    return 2 * layers * heads * slots * per_row


def test_retrieval_forward_bytes_from_shapes():
    import torch

    from triforce_b200 import ops

    # cfg2: 7B (32 layers, 32 heads, d = 128), budget 4096, gamma 6: 4103 slots, rounded to 4160 in the E4M3 cache's capacity
    slots, gamma = 4096 + 6 + 1, 6
    cap = -(-slots // ops.VERIFY_BOX_KEYS) * ops.VERIFY_BOX_KEYS
    assert cap == 4160
    fp16 = _read_bytes(32, 32, slots, 128, "fp16")
    e4m3 = _read_bytes(32, 32, slots, 128, "e4m3")
    assert round(fp16 / 1e9, 2) == 2.15 and round(e4m3 / 1e9, 2) == 1.08
    assert 2 * e4m3 == fp16 + 2 * 2 * 32 * 32 * slots  # codes are half the fp16 bytes; exponents add one byte per row
    # cfg4: budget 12288, gamma 16
    assert round(_read_bytes(32, 32, 12288 + 17, 128, "fp16") / 1e9, 2) == 6.45
    # the cache's allocation from shapes, on the meta device
    codes = torch.empty((32, 32, cap, 128), dtype=torch.uint8, device="meta")
    ex = torch.empty((32, 32, cap), dtype=torch.int8, device="meta")
    assert 2 * (codes.numel() + ex.numel()) == _read_bytes(32, 32, cap, 128, "e4m3")
    assert gamma + 1 + 4096 == slots


@pytest.mark.parametrize("entry", ["on_chip", "offloading_TP"])
def test_entry_points_take_the_retrieval_dtype_switch(entry):
    from triforce_b200.cli import build_parser

    assert build_parser(entry).parse_args([]).retrieval_dtype == "fp16"
    assert build_parser(entry).parse_args(["--retrieval_dtype", "e4m3"]).retrieval_dtype == "e4m3"
    with pytest.raises(SystemExit):
        build_parser(entry).parse_args(["--retrieval_dtype", "int8"])


def test_the_sequoia_entry_point_has_no_retrieval_dtype_switch():
    from triforce_b200.cli import build_parser

    assert not hasattr(build_parser("offloading_seqouia").parse_args([]), "retrieval_dtype")
    with pytest.raises(SystemExit):
        build_parser("offloading_seqouia").parse_args(["--retrieval_dtype", "e4m3"])
