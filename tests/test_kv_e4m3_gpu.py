"""Kernels of the E4M3 full-KV store on the GPU: the quantizer and the RoPE append bit for bit against tests/kv_e4m3_oracle.py,
the tail copy and the retrieval build bit for bit against their fp16 kernels on the dequantized store D, and the verify
attention against an fp64 reference over D with the needle method of tests/attn_needles.py."""
from __future__ import annotations

import pytest
import torch

import kv_e4m3_oracle as eo
from attn_needles import Needles, base_logit, excess, assert_rejected, reference, visibility, report_time_and_memory  # noqa: F401
from oracle import triforce_oracle as orc
from triforce_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _rows_with_spread_exponents(shape, seed, lo=-12, hi=6):
    """fp16 rows whose scales are random powers of two, so neighbouring rows have very different exponents."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(shape, generator=g, device=DEV, dtype=torch.float32)
    s = torch.randint(lo, hi + 1, shape[:-1] + (1,), generator=g, device=DEV).float()
    return (x * torch.exp2(s)).half()


def _dequant(codes, e):
    """D on the device (the oracle's dequantize without the trip to the host)."""
    return (codes.view(torch.float8_e4m3fn).double() * torch.exp2(e.double()).unsqueeze(-1)).half()


def _store_from(K: torch.Tensor, V: torch.Tensor) -> ops.E4m3Store:
    L, H, cap, d = K.shape
    st = ops.E4m3Store.empty(L, H, cap, d, DEV)
    for l in range(L):
        ops.kv_quantize_e4m3(K[l], st.k_codes[l], st.k_exp[l], 0, cap)
        ops.kv_quantize_e4m3(V[l], st.v_codes[l], st.v_exp[l], 0, cap)
    return st


# ---------------------------------------------------------------------------------------------------------------------
# quantizer and RoPE append: bit-exact
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", [64, 128])
def test_quantize_matches_the_oracle(d):
    H, cap = 4, 1024
    x = _rows_with_spread_exponents((H, cap, d), seed=d, lo=-40, hi=14).clamp(-65504, 65504)
    x[:, 5] = 0                       # all-zero row
    x[:, 6, 0] = 65504                # the top of the range
    x[:, 7] = (x[:, 7] * 0).add_(2.0 ** -24)  # subnormals only
    codes = torch.full((H, cap, d), 0xAA, dtype=torch.uint8, device=DEV)
    ex = torch.full((H, cap), 99, dtype=torch.int8, device=DEV)
    ops.kv_quantize_e4m3(x, codes, ex, 3, 1000)
    want_c, want_e = eo.quantize(x[:, 3:1003].cpu())
    assert torch.equal(codes[:, 3:1003].cpu(), want_c) and torch.equal(ex[:, 3:1003].cpu(), want_e)
    assert bool((codes[:, :3] == 0xAA).all()) and bool((ex[:, 1003:] == 99).all())  # nothing outside the rows
    assert torch.equal(_dequant(codes[:, 3:1003], ex[:, 3:1003]).cpu(), eo.dequantize(want_c, want_e))


@pytest.mark.parametrize("Hq,Hkv,d", [(8, 8, 128), (32, 8, 128), (8, 2, 64)])
@pytest.mark.parametrize("path", ["pos0", "pos_ids", "dev"])
def test_rope_append_matches_the_oracle(Hq, Hkv, d, path):
    R, cap, max_pos = 7, 256, 512
    g = torch.Generator(device=DEV).manual_seed(Hq * 100 + d)
    qkv = (torch.randn((R, (Hq + 2 * Hkv) * d), generator=g, device=DEV) * 3).half()
    cos, sin = (torch.randn((max_pos, d), generator=g, device=DEV).half() for _ in range(2))
    kw = {}
    if path == "pos0":
        kw = dict(pos0=40, slot0=100)
    elif path == "pos_ids":
        kw = dict(pos_ids=torch.tensor([5, 9, 2, 300, 7, 8, 1], dtype=torch.int32, device=DEV), slot0=100)
    else:
        kw = dict(pos0=30, pos0_dev=torch.tensor([10], dtype=torch.int32, device=DEV), slot0=60,
                  slot0_dev=torch.tensor([40], dtype=torch.int32, device=DEV))
    Kf = torch.zeros((Hkv, cap, d), dtype=torch.float16, device=DEV)
    Vf = torch.zeros_like(Kf)
    q16 = torch.empty((R, Hq, d), dtype=torch.float16, device=DEV)
    ops.rope_append_gqa(qkv, Hq, Hkv, d, cos, sin, q16, Kf, Vf, **kw)
    st = ops.E4m3Store.empty(2, Hkv, cap, d, DEV)
    q8 = torch.empty_like(q16)
    ops.rope_append_e4m3(qkv, Hq, Hkv, d, cos, sin, q8, st, 1, **kw)
    torch.cuda.synchronize()
    assert torch.equal(q8, q16)
    for codes, ex, ref in ((st.k_codes, st.k_exp, Kf), (st.v_codes, st.v_exp, Vf)):
        want_c, want_e = eo.quantize(ref[:, 100:107].cpu())
        assert torch.equal(codes[1, :, 100:107].cpu(), want_c) and torch.equal(ex[1, :, 100:107].cpu(), want_e)
        assert int(codes[0].count_nonzero()) == 0 and int(codes[1].count_nonzero()) == int(codes[1, :, 100:107].count_nonzero())


# ---------------------------------------------------------------------------------------------------------------------
# tail copy and retrieval build: bit-identical to the fp16 kernels on D
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("device_len", [False, True])
def test_tail_update_writes_D(device_len):
    L, H, cap, d, prefill, budget = 2, 4, 512, 128, 320, 64
    st = _store_from(_rows_with_spread_exponents((L, H, cap, d), 1, -30, 8), _rows_with_spread_exponents((L, H, cap, d), 2, -30, 8))
    rK = torch.zeros((L, H, budget, d), dtype=torch.float16, device=DEV)
    rV = torch.zeros_like(rK)
    if device_len:
        ops.tail_update_e4m3(st, rK, rV, prefill, budget, 300, seq_len_dev=torch.tensor([45], dtype=torch.int32, device=DEV), max_new=40)
    else:
        ops.tail_update_e4m3(st, rK, rV, prefill, budget, 345)
    n = 25
    assert torch.equal(rK[:, :, budget - n:], _dequant(st.k_codes[:, :, prefill:prefill + n], st.k_exp[:, :, prefill:prefill + n]))
    assert torch.equal(rV[:, :, budget - n:], _dequant(st.v_codes[:, :, prefill:prefill + n], st.v_exp[:, :, prefill:prefill + n]))
    assert int(rK[:, :, :budget - n].count_nonzero()) == 0


@pytest.mark.parametrize("Hq,Hkv", [(32, 32), (32, 8)])
def test_retrieval_build_is_the_fp16_build_on_D(Hq, Hkv):
    d, prefill, chunk, budget = 128, 124928, 8, 4096
    cap = prefill + 64
    g = torch.Generator(device=DEV).manual_seed(Hkv)
    K = _rows_with_spread_exponents((1, Hkv, cap, d), 3, -6, 2)
    V = _rows_with_spread_exponents((1, Hkv, cap, d), 4, -6, 2)
    st = _store_from(K, V)
    del K, V
    KD, VD = _dequant(st.k_codes, st.k_exp), _dequant(st.v_codes, st.v_exp)
    q = torch.randn((1, Hq, d), generator=g, device=DEV).half()
    outs = []
    for e4m3 in (True, False):
        rK = torch.zeros((1, Hkv, budget, d), dtype=torch.float16, device=DEV)
        rV = torch.zeros_like(rK)
        idx = torch.empty((1, Hkv, budget // chunk), dtype=torch.int32, device=DEV)
        sc = torch.empty((1, Hkv, prefill // chunk), dtype=torch.float16, device=DEV)
        if e4m3:
            ops.retrieval_build_e4m3(st, q, rK, rV, prefill, chunk, budget, out_idx=idx, out_scores=sc)
        else:
            ops.retrieval_build_gqa(KD, VD, q, rK, rV, prefill, chunk, budget, out_idx=idx, out_scores=sc)
        outs.append((idx, sc, rK, rV))
    for a, b in zip(*outs):
        assert torch.equal(a.view(torch.int16) if a.dtype == torch.float16 else a,
                           b.view(torch.int16) if b.dtype == torch.float16 else b)


# ---------------------------------------------------------------------------------------------------------------------
# verify attention against fp64 over D
# ---------------------------------------------------------------------------------------------------------------------
def _verify_inputs(Hq, Hkv, d, R, kv_len, cap, seed):
    G = Hq // Hkv
    nd = Needles(Hkv, seed, d)
    K = nd.store(1, cap)
    V = nd.store(1, cap)
    gs = torch.Generator(device=DEV).manual_seed(seed + 1)
    # background rows at random power-of-two scales (K only downwards, so needles keep their share of the softmax)
    K *= torch.exp2(torch.randint(-6, 1, (1, Hkv, cap, 1), generator=gs, device=DEV).half())
    V *= torch.exp2(torch.randint(-6, 4, (1, Hkv, cap, 1), generator=gs, device=DEV).half())
    L0 = base_logit(kv_len)
    fresh = list(range(kv_len - R, kv_len))
    spots = sorted(set(torch.randint(0, kv_len - R, (24,), generator=gs, device=DEV).tolist()) | {0, 63, 64, kv_len // 2})
    nd.plant(K, V, 0, fresh, [L0 - 0.5] * R)
    for i, k in enumerate(spots):  # needles of very different V scales
        nd.plant(K, V, 0, [k], [L0 - 1.0 + 0.1 * (i % 5)], v_amp=4.0 * 2.0 ** (i % 9 - 6))
    nd.plant(K, V, 0, [kv_len // 2], [L0 - 0.5])  # full-size needle in a middle tile: the dropped-partial control sees it
    if kv_len < cap:  # a stale needle right behind the last key
        nd.plant(K, V, 0, [kv_len], [L0 + 6.0], v_amp=16.0)
    q = nd.queries(R * G).view(R, G, Hkv, d).permute(0, 2, 1, 3).reshape(R, Hq, d).contiguous()
    return q, _store_from(K, V)


def _check_verify(q, st, out, kv_len, R, Hq, Hkv, controls=True):
    G = Hq // Hkv
    KD, VD = _dequant(st.k_codes[0], st.k_exp[0]), _dequant(st.v_codes[0], st.v_exp[0])
    n = min(kv_len + 1, KD.shape[1])
    vis = visibility(R, n, kv_len, causal=True)
    worst = 0.0
    for h in range(Hq):
        want = reference(q[:, h], KD[h // G], VD[h // G], vis)
        worst = max(worst, excess(out[:, h], want))
    assert worst <= 1.0, f"verify e4m3: excess {worst:.3g}"
    if controls:
        h = 0
        want = reference(q[:, h], KD[0], VD[0], vis)
        ones = torch.zeros_like(st.k_exp[0, 0])
        mutants = [
            ("K exponents ignored", reference(q[:, h], _dequant(st.k_codes[0, 0], ones), VD[0], vis)),
            ("V exponents ignored", reference(q[:, h], KD[0], _dequant(st.v_codes[0, 0], ones), vis)),
            ("previous key's K exponent", reference(q[:, h], _dequant(st.k_codes[0, 0], st.k_exp[0, 0].roll(1)), VD[0], vis)),
            ("previous key's V exponent", reference(q[:, h], KD[0], _dequant(st.v_codes[0, 0], st.v_exp[0, 0].roll(1)), vis)),
            ("diagonal shifted", reference(q[:, h], KD[0], VD[0], visibility(R, n, kv_len - 1, causal=True))),
        ]
        lost = visibility(R, n, kv_len, causal=True)
        t0 = (kv_len // 2) // 64 * 64
        lost[:, t0:t0 + 64] = False  # the 64-key tile of the middle needle: a lost (CTA, head) partial drops at least this
        mutants.append(("dropped partial", reference(q[:, h], KD[0], VD[0], lost)))
        if n > kv_len:
            mutants.append(("kv_len + 1 keys", reference(q[:, h], KD[0], VD[0], visibility(R, n, kv_len + 1, causal=True))))
        assert_rejected(mutants, want, "verify e4m3")
    return worst


@pytest.mark.parametrize("Hq,Hkv,d,R,kv_len,cap,dev_len", [
    (32, 32, 128, 8, 124944, 125056, True),   # cfg2 verify through kv_len_dev
    (32, 8, 128, 1, 124944, 125056, False),
    (32, 8, 128, 7, 124944, 125056, False),
    (32, 8, 128, 8, 124944, 125056, True),
    (12, 12, 64, 5, 20000, 20032, False),     # d = 64
    (8, 8, 128, 8, 259, 131072, False),       # a short store in a long capacity
    (8, 8, 128, 20, 4103, 4160, False),       # R > 16: the two-row-block instance
])
def test_verify_attn_e4m3(Hq, Hkv, d, R, kv_len, cap, dev_len):
    q, st = _verify_inputs(Hq, Hkv, d, R, kv_len, cap, seed=R * 7 + d)
    ws = ops.verify_attn_gqa_workspace(Hq, Hkv, d, DEV)
    scale = orc.softmax_scale_fp16(d)
    outs = []
    for _ in range(2):
        out = torch.empty_like(q)
        if dev_len:
            ops.verify_attn_e4m3(q, st, 0, kv_len - 1000, R, Hq, Hkv, d, scale, out, ws,
                                 kv_len_dev=torch.tensor([1000], dtype=torch.int32, device=DEV), kv_len_max=cap)
        else:
            ops.verify_attn_e4m3(q, st, 0, kv_len, R, Hq, Hkv, d, scale, out, ws)
        outs.append(out)
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1])
    print(f"worst excess {_check_verify(q, st, outs[0], kv_len, R, Hq, Hkv):.3f}")


def test_verify_attn_e4m3_graph_follows_the_device_length():
    Hq, Hkv, d, R, cap = 32, 8, 128, 8, 8192
    q, st = _verify_inputs(Hq, Hkv, d, R, 6000, cap, seed=5)
    ws = ops.verify_attn_gqa_workspace(Hq, Hkv, d, DEV)
    scale = orc.softmax_scale_fp16(d)
    n_dev = torch.tensor([0], dtype=torch.int32, device=DEV)
    out = torch.empty_like(q)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.verify_attn_e4m3(q, st, 0, 0, R, Hq, Hkv, d, scale, out, ws, kv_len_dev=n_dev, kv_len_max=cap)  # warm-up
        n_dev.fill_(6000)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            ops.verify_attn_e4m3(q, st, 0, 0, R, Hq, Hkv, d, scale, out, ws, kv_len_dev=n_dev, kv_len_max=cap)
    torch.cuda.current_stream().wait_stream(s)
    for kv_len in (5990, 6000, 6055, 6100, 5000):  # grows across a 64-key tile, then shrinks
        n_dev.fill_(kv_len)
        g.replay()
        eager = torch.empty_like(q)  # same kv_len_max, hence the same grid and summation order as the graph
        ops.verify_attn_e4m3(q, st, 0, 0, R, Hq, Hkv, d, scale, eager, ws, kv_len_dev=n_dev, kv_len_max=cap)
        torch.cuda.synchronize()
        assert torch.equal(out, eager)
        _check_verify(q, st, out, kv_len, R, Hq, Hkv, controls=False)


def test_decode_chain_eager_and_graph_agree():
    """tf_rope_append_e4m3 -> tf_verify_attn_e4m3 under the default PDL mask, eagerly and as a captured graph."""
    Hq, Hkv, d, R, cap, pos = 32, 8, 128, 6, 4160, 4000
    q0, st = _verify_inputs(Hq, Hkv, d, R, pos, cap, seed=11)
    g = torch.Generator(device=DEV).manual_seed(3)
    qkv = torch.randn((R, (Hq + 2 * Hkv) * d), generator=g, device=DEV).half()
    cos, sin = (torch.randn((cap, d), generator=g, device=DEV).half() for _ in range(2))
    ws = ops.verify_attn_gqa_workspace(Hq, Hkv, d, DEV)
    scale = orc.softmax_scale_fp16(d)
    seq = torch.tensor([pos], dtype=torch.int32, device=DEV)
    qo = torch.empty((R, Hq, d), dtype=torch.float16, device=DEV)
    out = torch.empty_like(qo)

    def chain():
        ops.rope_append_e4m3(qkv, Hq, Hkv, d, cos, sin, qo, st, 0, pos0_dev=seq, slot0_dev=seq)
        ops.verify_attn_e4m3(qo, st, 0, R, R, Hq, Hkv, d, scale, out, ws, kv_len_dev=seq, kv_len_max=cap)

    chain()
    torch.cuda.synchronize()
    eager = out.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, stream=s):
            chain()
    torch.cuda.current_stream().wait_stream(s)
    out.zero_()
    gr.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)
