"""Kernels of the E4M3 retrieval cache on the GPU.

* Build (tf_retrieval_build_to_e4m3): indices and scores bit-identical to the build into an fp16 cache from the same store;
  the cache holds the oracle's quantization of the rows that build gathered (fp16 store) or the store's own codes and
  exponents (E4M3 store), and nothing past the budget.
* Tail copy (tf_tail_update_to_e4m3), host and device length: the same, for rows [prefill, seq_len).
* Retrieval verify (tf_verify_attn_e4m3_clean) chained after tf_rope_append_e4m3 in a captured graph, with the early ring fill
  of the clean budget under PDL: bit-identical to the launch without PDL, and within the fp64-over-D tolerance of
  tests/test_kv_e4m3_gpu.py."""
from __future__ import annotations

import os

import pytest
import torch

import kv_e4m3_oracle as eo
from attn_needles import report_time_and_memory  # noqa: F401  (autouse fixture: wall time and peak memory per test)
from oracle import triforce_oracle as orc
from test_kv_e4m3_gpu import _check_verify, _dequant, _rows_with_spread_exponents, _store_from, _verify_inputs
from triforce_b200 import _C, ops

pytestmark = pytest.mark.gpu
DEV = "cuda"
CHUNK = 8


def _cache(L, H, budget, gamma, d):
    cap = -(-(budget + gamma + 1) // ops.VERIFY_BOX_KEYS) * ops.VERIFY_BOX_KEYS
    return ops.E4m3Store.empty(L, H, cap, d, DEV)


def _gathered_rows(idx):
    """[L, H, budget] source slots of the selected chunks."""
    return (idx.long()[..., None] * CHUNK + torch.arange(CHUNK, device=DEV)).flatten(-2)


def _take(t, rows):
    """t [L, H, slots, ...] at rows [L, H, n] -> [L, H, n, ...]."""
    ix = rows.view(rows.shape + (1,) * (t.dim() - 3)).expand(rows.shape + t.shape[3:])
    return torch.gather(t, 2, ix)


@pytest.mark.parametrize("src,Hq,Hkv,L,prefill,budget", [
    ("fp16", 32, 32, 2, 124928, 4096),     # 7B, production prefill
    ("fp16", 32, 32, 2, 124928, 12288),
    ("fp16", 32, 8, 2, 124928, 4096),      # GQA under group_sum
    ("e4m3", 32, 32, 2, 124928, 4096),
    ("e4m3", 32, 8, 2, 124928, 12288),
    ("fp16", 32, 32, 32, 16384, 4096),     # all 32 layers in one launch sequence
    ("e4m3", 32, 8, 32, 16384, 4096),
    ("fp16", 12, 12, 2, 2048, 256),        # d = 64, parity size
    ("e4m3", 12, 12, 2, 2048, 256),
])
def test_build_into_e4m3_cache(src, Hq, Hkv, L, prefill, budget):
    d = 64 if Hq == 12 else 128
    slots = prefill + 64
    K = _rows_with_spread_exponents((L, Hkv, slots, d), 1, -6, 2)
    V = _rows_with_spread_exponents((L, Hkv, slots, d), 2, -6, 4)
    if src == "e4m3":
        store = _store_from(K, V)
        del K, V
    g = torch.Generator(device=DEV).manual_seed(L * Hkv + budget)
    q = torch.randn((L, Hq, d), generator=g, device=DEV).half()
    n_sel = budget // CHUNK
    idx16 = torch.empty((L, Hkv, n_sel), dtype=torch.int32, device=DEV)
    sc16 = torch.empty((L, Hkv, prefill // CHUNK), dtype=torch.float16, device=DEV)
    rK = torch.zeros((L, Hkv, budget, d), dtype=torch.float16, device=DEV)
    rV = torch.zeros_like(rK)
    if src == "e4m3":
        ops.retrieval_build_e4m3(store, q, rK, rV, prefill, CHUNK, budget, out_idx=idx16, out_scores=sc16)
    elif Hq == Hkv:
        ops.retrieval_build(K, V, q, rK, rV, prefill, CHUNK, budget, out_idx=idx16, out_scores=sc16)
    else:
        ops.retrieval_build_gqa(K, V, q, rK, rV, prefill, CHUNK, budget, out_idx=idx16, out_scores=sc16)
    cache = _cache(L, Hkv, budget, 6, d)
    for t in (cache.k_codes, cache.v_codes):
        t.fill_(0xAA)
    idx8 = torch.empty_like(idx16)
    sc8 = torch.empty_like(sc16)
    ops.retrieval_build_to_e4m3(store if src == "e4m3" else (K, V), q, cache, prefill, CHUNK, budget, out_idx=idx8, out_scores=sc8)
    torch.cuda.synchronize()
    assert torch.equal(idx8, idx16) and torch.equal(sc8.view(torch.int16), sc16.view(torch.int16))
    if src == "e4m3":  # the store's own codes and exponents of the selected rows
        rows = _gathered_rows(idx16)
        for codes, ex, sc_, se in ((cache.k_codes, cache.k_exp, store.k_codes, store.k_exp),
                                   (cache.v_codes, cache.v_exp, store.v_codes, store.v_exp)):
            assert torch.equal(codes[:, :, :budget], _take(sc_, rows)) and torch.equal(ex[:, :, :budget], _take(se, rows))
        assert torch.equal(_dequant(cache.k_codes[:, :, :budget], cache.k_exp[:, :, :budget]), rK)  # = D of the fp16-cache build
    else:  # the quantization of the rows the fp16-cache build gathered: the oracle's on the host for the first, middle and last
        # layer, tf_kv_quantize_e4m3's (which test_kv_e4m3_gpu.py pins to the oracle) for every layer
        for codes, ex, ref in ((cache.k_codes, cache.k_exp, rK), (cache.v_codes, cache.v_exp, rV)):
            for l in sorted({0, L // 2, L - 1}):
                want_c, want_e = eo.quantize(ref[l].cpu())
                assert torch.equal(codes[l, :, :budget].cpu(), want_c) and torch.equal(ex[l, :, :budget].cpu(), want_e)
            wc, we = torch.empty_like(codes[0, :, :budget]), torch.empty_like(ex[0, :, :budget])
            for l in range(L):
                ops.kv_quantize_e4m3(ref[l], wc, we, 0, budget)
                assert torch.equal(codes[l, :, :budget], wc) and torch.equal(ex[l, :, :budget], we)
    assert bool((cache.k_codes[:, :, budget:] == 0xAA).all()) and bool((cache.v_codes[:, :, budget:] == 0xAA).all())


@pytest.mark.parametrize("src", ["fp16", "e4m3"])
@pytest.mark.parametrize("device_len", [False, True])
@pytest.mark.parametrize("d", [64, 128])
def test_tail_update_into_e4m3_cache(src, device_len, d):
    L, H, slots, prefill, budget, n = 2, 4, 512, 320, 64, 25
    K = _rows_with_spread_exponents((L, H, slots, d), 1, -30, 8)
    V = _rows_with_spread_exponents((L, H, slots, d), 2, -30, 8)
    source = _store_from(K, V) if src == "e4m3" else (K, V)
    cache = _cache(L, H, budget, 4, d)
    if device_len:
        ops.tail_update_to_e4m3(source, cache, prefill, budget, 300, seq_len_dev=torch.tensor([45], dtype=torch.int32, device=DEV),
                                max_new=40)
    else:
        ops.tail_update_to_e4m3(source, cache, prefill, budget, prefill + n)
    torch.cuda.synchronize()
    for codes, ex, (sc_, se, ref) in ((cache.k_codes, cache.k_exp, (source.k_codes, source.k_exp, K) if src == "e4m3" else (None, None, K)),
                                      (cache.v_codes, cache.v_exp, (source.v_codes, source.v_exp, V) if src == "e4m3" else (None, None, V))):
        if src == "e4m3":
            want_c, want_e = sc_[:, :, prefill:prefill + n], se[:, :, prefill:prefill + n]
        else:
            want_c, want_e = (t.to(DEV) for t in eo.quantize(ref[:, :, prefill:prefill + n].cpu()))
        assert torch.equal(codes[:, :, budget - n:budget], want_c) and torch.equal(ex[:, :, budget - n:budget], want_e)
        assert int(codes[:, :, :budget - n].count_nonzero()) == 0 and int(codes[:, :, budget:].count_nonzero()) == 0
    # one layer of a rebuild's per-layer copy
    one = _cache(L, H, budget, 4, d)
    ops.tail_update_to_e4m3(source, one, prefill, budget, prefill + n, layer0=1, n_layers=1)
    torch.cuda.synchronize()
    assert torch.equal(one.k_codes[1], cache.k_codes[1]) and torch.equal(one.v_exp[1], cache.v_exp[1])
    assert int(one.k_codes[0].count_nonzero()) == 0


@pytest.mark.parametrize("Hq,Hkv", [(32, 32), (32, 8)])
@pytest.mark.parametrize("gamma", [4, 6, 16])
def test_pdl_retrieval_verify_after_rope_append(Hq, Hkv, gamma):
    """rope_append_e4m3 writes the gamma+1 rows at slot `budget`; the verify over budget + gamma + 1 keys fills its ring from
    the clean budget before it waits.  RoPE with cos = 1, sin = 0 keeps q and the appended rows as given, so the needles of
    _verify_inputs (q aligned with chosen keys, the fresh rows included) stay in place and the controls can reject mutants."""
    d, budget, R = 128, 4096, gamma + 1
    kv_len = budget + R
    cap = -(-kv_len // 64) * 64
    q, st = _verify_inputs(Hq, Hkv, d, R, kv_len, cap, seed=gamma * 3 + Hkv)
    KD, VD = _dequant(st.k_codes[0], st.k_exp[0]), _dequant(st.v_codes[0], st.v_exp[0])
    qkv = torch.cat([q.reshape(R, -1), KD[:, budget:kv_len].transpose(0, 1).reshape(R, -1),
                     VD[:, budget:kv_len].transpose(0, 1).reshape(R, -1)], dim=1).contiguous()
    for t in (st.k_codes, st.v_codes, st.k_exp, st.v_exp):
        t[0, :, budget:kv_len] = 0  # the append must write them
    pos = torch.arange(10, 10 + R, dtype=torch.int32, device=DEV)
    cos = torch.ones((64, d), dtype=torch.float16, device=DEV)
    sin = torch.zeros((64, d), dtype=torch.float16, device=DEV)
    ws = ops.verify_attn_gqa_workspace(Hq, Hkv, d, DEV)
    scale = orc.softmax_scale_fp16(d)
    qo = torch.empty_like(q)
    out = torch.empty_like(q)

    def chain(clean):
        ops.rope_append_e4m3(qkv, Hq, Hkv, d, cos, sin, qo, st, 0, pos_ids=pos, slot0=budget)
        ops.verify_attn_e4m3(qo, st, 0, kv_len, R, Hq, Hkv, d, scale, out, ws, clean_keys=clean)

    lib = _C.lib()
    mask = int(os.environ.get("TRIFORCE_PDL", str(_C.DEFAULT_PDL_MASK)))
    try:
        lib.tf_set_pdl(mask & ~16)  # the verify launched without PDL, no early fill
        chain(0)
        torch.cuda.synchronize()
        ref = out.clone()
        lib.tf_set_pdl(mask)
        assert torch.equal(qo, q)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            chain(budget)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=s):
                chain(budget)
        torch.cuda.current_stream().wait_stream(s)
        for _ in range(3):
            out.zero_()
            g.replay()
            torch.cuda.synchronize()
            assert torch.equal(out, ref)
        chain(budget)  # eager, PDL with the early fill
        torch.cuda.synchronize()
        assert torch.equal(out, ref)
    finally:
        lib.tf_set_pdl(mask)
    print(f"worst excess {_check_verify(q, st, out, kv_len, R, Hq, Hkv):.3f}")
