"""E4M3 full-KV store without a GPU: the quantization rule of tests/kv_e4m3_oracle.py and the argument checks of the six
e4m3 entry points of the C ABI."""
from __future__ import annotations

import ctypes

import pytest
import torch

import kv_e4m3_oracle as eo
from triforce_b200 import _C


def _row(vals, d=128):
    x = torch.zeros(d, dtype=torch.float16)
    x[: len(vals)] = torch.tensor(vals, dtype=torch.float16)
    return x


@pytest.mark.parametrize("e", [-20, -9, 0, 1, 5, 7])
def test_amax_on_the_boundary_and_one_ulp_above(e):
    at = _row([448.0 * 2.0 ** e, -1.0 * 2.0 ** e])
    assert float(at.abs().max()) == 448.0 * 2.0 ** e  # exactly representable in fp16
    assert int(eo.row_exponent(at)) == e
    above = at.clone()
    above[0] = torch.tensor(448.0 * 2.0 ** e, dtype=torch.float16).view(torch.int16).add(1).view(torch.float16)  # one fp16 ulp up
    assert float(above[0]) > 448.0 * 2.0 ** e
    assert int(eo.row_exponent(above)) == e + 1
    codes, ex = eo.quantize(at)
    assert codes[0].item() == 0x7E  # 448 = the largest finite e4m3 code
    assert torch.equal(eo.dequantize(codes, ex), at)


def test_all_zero_row():
    codes, e = eo.quantize(torch.zeros(3, 64, dtype=torch.float16))
    assert torch.equal(e, torch.zeros(3, dtype=torch.int8))
    assert torch.equal(codes, torch.zeros(3, 64, dtype=torch.uint8))
    assert torch.equal(eo.roundtrip(torch.zeros(64, dtype=torch.float16)), torch.zeros(64, dtype=torch.float16))


def test_fp16_extremes():
    x = _row([65504.0, -65504.0, 1.0])
    codes, e = eo.quantize(x)
    assert int(e) == 8
    # 65504 / 256 = 255.875 rounds to the code 256, and 256 * 2^8 = 65536 is past fp16: D overflows like the fp16 cast
    assert float(eo.dequantize(codes, e)[0]) == float("inf")
    assert float(eo.dequantize(codes, e)[1]) == float("-inf")
    # fp16 subnormals: max 3 * 2^-24 = 1.5 * 2^-23 needs e = -31 (448 * 2^-32 < 1.5 * 2^-23 <= 448 * 2^-31); a row of
    # subnormals is stored without loss, and the smallest subnormal alone gives the bottom of the range
    tiny = _row([2.0 ** -24, -3 * 2.0 ** -24, 2.0 ** -23])
    codes, e = eo.quantize(tiny)
    assert int(e) == -31
    assert torch.equal(eo.dequantize(codes, e), tiny)
    assert int(eo.row_exponent(_row([2.0 ** -24]))) == -32


def test_exponent_range_on_random_rows():
    g = torch.Generator().manual_seed(0)
    scales = torch.exp2(torch.randint(-30, 16, (512, 1), generator=g).double())
    x = (torch.randn(512, 128, generator=g, dtype=torch.float64) * scales).clamp(-65504, 65504).half()
    x = x[x.abs().amax(-1) > 0]  # rows flushed to zero by the fp16 cast have e = 0
    e = eo.row_exponent(x).double()
    amax = x.double().abs().amax(-1)
    assert bool(((amax <= 448 * torch.exp2(e)) & (amax > 448 * torch.exp2(e - 1))).all())
    assert int(e.min()) >= -32 and int(e.max()) <= 8


def test_rounding_ties_go_to_even():
    # at e = 0 the e4m3 step in [1, 2) is 1/8 and in [256, 448] it is 32: midpoints go to the even code
    x = _row([448.0, 1.0625, 1.1875, 272.0, 304.0, -1.0625, 2.0 ** -10 * 1.5])
    codes, e = eo.quantize(x)
    assert int(e) == 0
    d = eo.dequantize(codes, e)
    assert d[1].item() == 1.0 and d[2].item() == 1.25 and d[3].item() == 256.0 and d[4].item() == 320.0
    assert d[5].item() == -1.0
    # e4m3 subnormals are multiples of 2^-9: 1.5 * 2^-10 = 0.75 * 2^-9 rounds to 2^-9
    assert d[6].item() == 2.0 ** -9


def test_store_bytes_from_shapes():
    # cfg2: 32 layers x 32 heads x 124 944 (rounded to 125 056 slots) x 128; codes are half the fp16 bytes and the
    # exponents add one byte per row
    L, H, cap, d = 32, 32, 125056, 128
    codes = torch.empty((L, H, cap, d), dtype=torch.uint8, device="meta")
    ex = torch.empty((L, H, cap), dtype=torch.int8, device="meta")
    fp16 = L * H * cap * d * 2
    e4m3 = codes.numel() * codes.element_size() + ex.numel() * ex.element_size()
    assert 2 * e4m3 == fp16 + 2 * L * H * cap
    assert codes.view(torch.float8_e4m3fn).shape == codes.shape


def test_e4m3_entry_points_check_their_arguments():
    lib = _C.lib()
    buf = (ctypes.c_uint8 * 512)()
    p = ctypes.addressof(buf)
    a = (p + 15) & ~15
    big = 1 << 30
    ws = lib.tf_verify_attn_gqa_workspace_bytes(8, 32, 8, 128)
    # tf_kv_tensormap_encode_e4m3(out, base, d, cap, heads, layers, head_stride, layer_stride, box)
    assert lib.tf_kv_tensormap_encode_e4m3(p, None, 128, 64, 1, 1, 8192, 8192, 64) == -1
    assert lib.tf_kv_tensormap_encode_e4m3(p, a, 96, 64, 1, 1, 6144, 6144, 64) == -1
    assert lib.tf_kv_tensormap_encode_e4m3(p, a, 128, 64, 1, 1, 8200, 8200, 64) == -1  # 8-byte strides
    # tf_kv_quantize_e4m3(src, src_head_stride, slot0, n, Hkv, d, codes, exps, cap, stream)
    assert lib.tf_kv_quantize_e4m3(None, 8192, 0, 1, 1, 128, a, a, 64, None) == -1
    assert lib.tf_kv_quantize_e4m3(a, 6144, 0, 1, 1, 96, a, a, 64, None) == -2
    assert lib.tf_kv_quantize_e4m3(a, 8192, 60, 8, 1, 128, a, a, 64, None) == -1  # past cap
    # tf_rope_append_e4m3(q, k, v, stride, cos, sin, max_pos, pos_ids, pos0, pos0_dev, slot0, slot0_dev, R, Hq, Hkv, d, q_out,
    #                     Kc, Vc, Ke, Ve, cap, stream)
    assert lib.tf_rope_append_e4m3(p, p, p, 8, p, p, 4, None, 0, None, 0, None, 1, 8, 8, 128, p, p, p, None, p, 128, None) == -1
    assert lib.tf_rope_append_e4m3(p, p, p, 8, p, p, 4, None, 0, None, 0, None, 1, 30, 8, 128, p, p, p, p, p, 128, None) == -1
    assert b"multiple" in lib.tf_last_error()
    assert lib.tf_rope_append_e4m3(p, p, p, 8, p, p, 4, None, 0, None, 0, None, 1, 32, 8, 96, p, p, p, p, p, 128, None) == -2
    # tf_verify_attn_e4m3(q, kmap, vmap, kexp, vexp, cap, layer, kv_len, kv_len_dev, kv_len_max, R, Hq, Hkv, d, scale, out, ws,
    #                     ws_bytes, stream)
    assert lib.tf_verify_attn_e4m3(p, p, p, None, a, 128, 0, 64, None, 64, 8, 32, 8, 128, 0.1, p, a, big, None) == -1
    assert b"NULL" in lib.tf_last_error()
    assert lib.tf_verify_attn_e4m3(a, p, p, a, a, 100, 0, 64, None, 64, 8, 32, 8, 128, 0.1, a, a, big, None) == -1  # cap % 64
    assert lib.tf_verify_attn_e4m3(a, p, p, a, a, 128, 0, 192, None, 192, 8, 32, 8, 128, 0.1, a, a, big, None) == -1  # > cap
    assert lib.tf_verify_attn_e4m3(a, p, p, a, a, 128, 0, 64, None, 64, 4, 30, 8, 128, 0.1, a, a, big, None) == -1  # Hq % Hkv
    assert b"multiple" in lib.tf_last_error()
    assert lib.tf_verify_attn_e4m3(a, p, p, a, a, 128, 0, 64, None, 64, 9, 32, 8, 128, 0.1, a, a, big, None) == -1  # R·G = 36
    assert b"packed rows" in lib.tf_last_error()
    assert lib.tf_verify_attn_e4m3(a, p, p, a, a, 128, 0, 64, None, 64, 8, 32, 8, 128, 0.1, a, a, ws - 1, None) == -1
    assert b"workspace" in lib.tf_last_error()
    assert lib.tf_verify_attn_e4m3(a, p, p, a, a, 128, 0, 64, None, 64, 8, 32, 8, 96, 0.1, a, a, big, None) == -2
    # tf_retrieval_build_e4m3(K, V, Ke, Ve, ls, hs, q, n_layers, Hq, Hkv, d, prefill, chunk, budget, rK, rV, rls, rhs, idx, scores,
    #                         ws, ws_bytes, stream)
    assert lib.tf_retrieval_build_e4m3(a, a, None, a, 8192, 8192, a, 1, 8, 8, 128, 64, 8, 8, a, a, 8, 8, None, None, a, 64, None) == -1
    assert lib.tf_retrieval_build_e4m3(a, a, a, a, 8192, 8192, a, 1, 30, 8, 128, 64, 8, 8, a, a, 8, 8, None, None, a, 64, None) == -1
    assert lib.tf_retrieval_build_e4m3(a, a, a, a, 8192, 8192, a, 1, 32, 8, 96, 64, 8, 8, a, a, 8, 8, None, None, a, 64, None) == -1
    assert lib.tf_retrieval_build_e4m3(a, a, a, a, 8192, 8192, a, 1, 32, 8, 256, 64, 8, 8, a, a, 8, 8, None, None, a, 64, None) == -2
    # tf_tail_update_e4m3(K, V, Ke, Ve, ls, hs, rK, rV, rls, rhs, L, H, d, prefill, budget, seq_len, seq_len_dev, max_new, stream)
    assert lib.tf_tail_update_e4m3(a, a, None, a, 8192, 8192, a, a, 8, 8, 1, 1, 128, 0, 8, 4, None, 0, None) == -1
    assert lib.tf_tail_update_e4m3(a, a, a, a, 8200, 8192, a, a, 8, 8, 1, 1, 128, 0, 8, 4, None, 0, None) == -1  # stride % d
    assert lib.tf_tail_update_e4m3(a, a, a, a, 8192, 8192, a, a, 8, 8, 1, 1, 128, 0, 8, 12, None, 0, None) == -1  # > budget


# ---------------------------------------------------------------------------------------------------------------------
# refusals and the switch (no device needed: every check runs before anything is allocated)
# ---------------------------------------------------------------------------------------------------------------------
def test_paths_that_keep_an_fp16_store_refuse_e4m3():
    from types import SimpleNamespace

    from triforce_b200.cache import FlashSimpleCache, RetrievalCacheSeqouia
    from triforce_b200.tp import DistributedLlama

    kv = SimpleNamespace(kv_dtype="e4m3")
    with pytest.raises(ValueError, match="kv_dtype"):
        FlashSimpleCache(SimpleNamespace(), 64, kv_dtype="bf16")
    with pytest.raises(NotImplementedError, match="Sequoia"):
        object.__new__(RetrievalCacheSeqouia).init_graph_cache(kv, None, 0)
    with pytest.raises(NotImplementedError, match="tensor parallel"):
        DistributedLlama("llama-7B-128K", kv_dtype="e4m3")
    cache = object.__new__(FlashSimpleCache)
    cache.kv_dtype = "e4m3"
    with pytest.raises(NotImplementedError, match="update"):
        cache.update(None, None, 0)


def test_on_chip_takes_the_kv_dtype_switch():
    from triforce_b200.cli import build_parser

    assert build_parser("on_chip").parse_args([]).kv_dtype == "fp16"
    assert build_parser("on_chip").parse_args(["--kv_dtype", "e4m3"]).kv_dtype == "e4m3"
    with pytest.raises(SystemExit):
        build_parser("on_chip").parse_args(["--kv_dtype", "int8"])
