"""Grouped-query attention on the GPU: tf_verify_attn_gqa (and its tree form), tf_tree_attn_tc_gqa, tf_rope_append_gqa,
tf_retrieval_build_gqa, and a GQA target through the model forward.

Attention outputs are compared with an fp64 reference built with `repeat_kv` (query head h reads KV head h // G), with
the tolerance and the needle inputs of attn_needles.  The query heads of one group share their KV head's needle
direction but weigh it differently (scale 1 + g/(2G) for member g), so members have distinct outputs.  Each comparison
must reject three mutated references: KV head h % Hkv instead of h // G, the causal diagonal taken from the packed row
r·G + g instead of the token row r, and a member's output computed from its neighbour's query.

On one H100 80GB HBM3 at a 700 W power limit the file runs in about 15 s; the largest test peaks at 2.2 GiB of device
memory (the 512-row tree at cfg2 depth), the model test at 0.9 GiB."""
import numpy as np
import pytest
import torch

import gqa_oracle
from attn_needles import (DEV, Q_ALONG, Needles, assert_rejected, base_logit, excess, plant_stale, reference,
                          report_time_and_memory, visibility)  # noqa: F401  (report_time_and_memory: autouse fixture)
from test_verify_attn_production_gpu import Plan, partial_m, sm_count, workspace_layout
from oracle import triforce_oracle as orc
from triforce_b200 import ops

pytestmark = pytest.mark.gpu
D = 128


def group_queries(nd: Needles, R: int, G: int) -> torch.Tensor:
    """q [R, Hkv·G, d]: member g of KV head k is (1 + g / 2G)·Q_ALONG·u_k plus noise orthogonal to u_k."""
    Hkv = nd.H
    u = nd.u.repeat_interleave(G, 0)  # [Hq, d]
    s = (1.0 + torch.arange(G, device=DEV, dtype=torch.float64) / (2 * G)).repeat(Hkv)[:, None]
    n = torch.randn((R, Hkv * G, nd.d), generator=nd.g, device=DEV, dtype=torch.float64)
    n -= (n * u).sum(-1, keepdim=True) * u
    return (Q_ALONG * s * u + n).half().contiguous()


def plant(nd: Needles, K, V, kv_len: int, R: int, cap: int, plan: Plan = None):
    """Stale rows past kv_len; per KV head, needles at the first and last key of its partials (when a plan is given),
    at a few spread keys, and a record needle e^3 above them; needles at the R fresh keys."""
    L0 = base_logit(kv_len)
    plant_stale(nd, K, V, 0, kv_len, cap)
    body = kv_len - R
    for h in range(nd.H):
        keys = {body * f // 8 for f in range(8)}
        if plan is not None:
            keys |= {k for _, lo, hi in plan.partials(h) for k in (lo, hi - 1) if k < body}
        record = body // 2 + 1
        keys.discard(record)
        keys = sorted(keys) + [record]
        nd.plant(K, V, 0, keys, [L0] * (len(keys) - 1) + [L0 + 3.0], head=h)
    nd.plant(K, V, 0, range(body, kv_len), [L0] * R)


def check_heads(out, q, K, V, vis, G: int, what: str, causal_rows: bool = True):
    """Every query head against its KV head's fp64 reference; the three mutants on the first and last group."""
    R, Hq, d = q.shape
    Hkv = Hq // G
    worst, weakest = 0.0, float("inf")
    for h in range(Hq):
        kvh, g = h // G, h % G
        want = reference(q[:, h], K[0, kvh], V[0, kvh], vis)
        e = excess(out[:, h], want)
        assert e <= 1.0, f"{what}: query head {h} (KV head {kvh}) exceeds the tolerance ({e:.3g})"
        worst = max(worst, e)
        if kvh not in (0, Hkv - 1):
            continue
        mutants = []
        if h % Hkv != kvh:
            mutants.append(("KV head h % Hkv", reference(q[:, h], K[0, h % Hkv], V[0, h % Hkv], vis)))
        if G > 1:
            mutants.append(("neighbour's query", reference(q[:, kvh * G + (g + 1) % G], K[0, kvh], V[0, kvh], vis)))
        if causal_rows and G > 1 and g > 0 and R > 1:
            n = vis.shape[1]
            i = torch.arange(R, device=DEV)[:, None] * G + g
            j = torch.arange(n, device=DEV)[None, :]
            kv_len = int(vis[-1].sum())  # the last token row sees every key below kv_len
            vm = (j <= kv_len - R + i) & (j < kv_len)
            if not torch.equal(vm, vis):
                mutants.append(("diagonal of the packed row", reference(q[:, h], K[0, kvh], V[0, kvh], vm)))
        if mutants:
            weakest = min(weakest, assert_rejected(mutants, want, f"{what}, head {h}"))
    print(f"{what}: worst error/tolerance {worst:.3f}, weakest negative control {weakest:.1f}")


# ---------------------------------------------------------------------------------------------------------------------
# tf_verify_attn_gqa
# ---------------------------------------------------------------------------------------------------------------------
HEADS = [(32, 8), (8, 1), (64, 8), (8, 4)]


@pytest.mark.parametrize("kv_len", [259, 4103, 124944])
@pytest.mark.parametrize("R", [1, 7, 8])
@pytest.mark.parametrize("Hq,Hkv", HEADS, ids=[f"{a}q{b}kv" for a, b in HEADS])
def test_verify_attn_gqa(Hq, Hkv, R, kv_len):
    G = Hq // Hkv
    cap = max(2048, kv_len + 64) if kv_len < 100000 else 131072
    sms = sm_count()
    nd = Needles(Hkv, seed=1000 + Hq + R + kv_len, d=D)
    K, V = nd.store(1, cap), nd.store(1, cap)
    block = ops.gqa_row_block(Hq, Hkv)
    single = R <= block
    plan = Plan(R * G, Hkv, D, kv_len, kv_len, sms) if single else None
    plant(nd, K, V, kv_len, R, cap, plan)
    q = group_queries(nd, R, G)
    maps = ops.KVTensorMaps(K, V)
    ws = ops.verify_attn_gqa_workspace(Hq, Hkv, D, DEV)
    lay = workspace_layout(Hkv, D, sms)
    assert ws.numel() == lay["bytes"], "the GQA workspace is the MHA workspace of Hkv heads"
    out = torch.empty_like(q)
    if single:  # the slots of exactly the (CTA, KV head) segments of the plan are written: each KV head streamed once
        partial_m(ws, lay).fill_(float("nan"))
    ops.verify_attn_gqa(q, maps, 0, kv_len, R, Hq, Hkv, D, nd.scale, out, ws)
    torch.cuda.synchronize()
    if single:
        want = torch.zeros((lay["slots"], 32), dtype=torch.bool, device=DEV)
        for b, h, _, _ in plan.segments:
            want[b + h, :R * G] = True
        bad = torch.nonzero((~partial_m(ws, lay).isnan()) != want)[:, 0].unique().tolist()
        assert not bad, f"partial slots {bad[:8]} written unlike the plan ({plan.summary()})"
    assert not ws[:4 * Hkv].view(torch.int32).any(), "an arrival counter was left non-zero"
    again = torch.empty_like(q)
    ops.verify_attn_gqa(q, maps, 0, kv_len, R, Hq, Hkv, D, nd.scale, again, ws)
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.int16), again.view(torch.int16)), "two launches differ"
    vis = visibility(R, kv_len, kv_len, causal=True)
    check_heads(out, q, K, V, vis, G, f"Hq {Hq} / Hkv {Hkv}, R {R}, kv_len {kv_len}"
                                      f"{', ' + plan.summary() if plan else f', blocks of {block} rows'}")


@pytest.mark.parametrize("R", [1, 8, 16])
def test_verify_attn_gqa_at_g1_gives_the_mha_bits(R):
    H, kv_len, cap = 8, 9000, 16384
    nd = Needles(H, seed=7, d=D)
    K, V = nd.store(1, cap), nd.store(1, cap)
    plant(nd, K, V, kv_len, R, cap)
    q = group_queries(nd, R, 1)
    maps = ops.KVTensorMaps(K, V)
    a, b = torch.empty_like(q), torch.empty_like(q)
    ops.verify_attn(q, maps, 0, kv_len, R, H, D, nd.scale, a, ops.verify_attn_workspace(32, H, D, DEV))
    ops.verify_attn_gqa(q, maps, 0, kv_len, R, H, H, D, nd.scale, b, ops.verify_attn_gqa_workspace(H, H, D, DEV))
    torch.cuda.synchronize()
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))


def test_verify_attn_gqa_device_length_in_a_graph():
    """kv_len from device memory inside a captured graph, replayed as the length grows and crosses a tile."""
    Hq, Hkv, R, cap = 32, 8, 7, 131072
    nd = Needles(Hkv, seed=11, d=D)
    K, V = nd.store(1, cap), nd.store(1, cap)
    q = group_queries(nd, R, Hq // Hkv)
    maps = ops.KVTensorMaps(K, V)
    ws = ops.verify_attn_gqa_workspace(Hq, Hkv, D, DEV)
    out = torch.empty_like(q)
    dev_len = torch.zeros(1, dtype=torch.int32, device=DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        dev_len.fill_(R + 1)
        ops.verify_attn_gqa(q, maps, 0, 0, R, Hq, Hkv, D, nd.scale, out, ws, kv_len_dev=dev_len)  # warm-up
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            ops.verify_attn_gqa(q, maps, 0, 0, R, Hq, Hkv, D, nd.scale, out, ws, kv_len_dev=dev_len)
    torch.cuda.current_stream().wait_stream(s)
    for kv_len in (120001, 120064, 120065, 124944):
        K.copy_(nd.store(1, cap))  # in place (the graph holds the store's tensor maps): no needles of the previous length
        V.copy_(nd.store(1, cap))
        plant(nd, K, V, kv_len, R, cap)
        dev_len.fill_(kv_len)
        g.replay()
        eager = torch.empty_like(q)
        ops.verify_attn_gqa(q, maps, 0, kv_len, R, Hq, Hkv, D, nd.scale, eager, ws, kv_len_max=cap)
        torch.cuda.synchronize()
        assert torch.equal(out.view(torch.int16), eager.view(torch.int16)), f"graph replay at {kv_len} differs from eager"
        check_heads(out, q, K, V, visibility(R, kv_len, kv_len, causal=True), Hq // Hkv, f"graph replay at kv_len {kv_len}")


@pytest.mark.parametrize("Hq,Hkv", [(32, 8), (64, 8)])
def test_verify_attn_tree_gqa(Hq, Hkv):
    """A 32-row tree mask over the last 32 keys, cut into blocks of 32 / G token rows."""
    G, T, kv_len, cap = Hq // Hkv, 32, 4103 + 32, 8192
    nd = Needles(Hkv, seed=13 + Hq, d=D)
    K, V = nd.store(1, cap), nd.store(1, cap)
    plant(nd, K, V, kv_len, T, cap)
    q = group_queries(nd, T, G)
    gen = torch.Generator().manual_seed(5)
    tree = torch.rand((T, T), generator=gen) < 0.4
    tree = (tree.tril(-1) | torch.eye(T, dtype=torch.bool)).to(DEV)
    bits = torch.from_numpy(orc.pack_tree_mask(tree.cpu().numpy()).view(np.int32)).to(DEV)
    bits = bits.view(T, T // 32).contiguous()
    out = torch.empty_like(q)
    ops.verify_attn_gqa(q, ops.KVTensorMaps(K, V), 0, kv_len, T, Hq, Hkv, D, nd.scale, out,
                        ops.verify_attn_gqa_workspace(Hq, Hkv, D, DEV), tree_mask=bits, tree_cols=T)
    torch.cuda.synchronize()
    vis = visibility(T, kv_len, kv_len, tree=tree)
    check_heads(out, q, K, V, vis, G, f"tree Hq {Hq} / Hkv {Hkv}", causal_rows=False)
    # the tree row of a packed row is its token row: a mask read at the packed row is rejected
    h = G - 1
    want = reference(q[:, h], K[0, 0], V[0, 0], vis)
    rows = torch.clamp(torch.arange(T, device=DEV) * G + h, max=T - 1)
    assert_rejected([("tree row of the packed row", reference(q[:, h], K[0, 0], V[0, 0],
                                                              visibility(T, kv_len, kv_len, tree=tree[rows])))], want, "tree")


# ---------------------------------------------------------------------------------------------------------------------
# tf_tree_attn_tc_gqa
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kv_len", [4096, 124928])
def test_tree_attn_tc_gqa_causal_chunk(kv_len):
    Hq, Hkv, R = 32, 8, 128
    G, cap = Hq // Hkv, kv_len + 256
    nd = Needles(Hkv, seed=17, d=D)
    K, V = nd.store(1, cap), nd.store(1, cap)
    plant(nd, K, V, kv_len, R, cap)
    q = group_queries(nd, R, G)
    out = torch.empty_like(q)
    ops.tree_attn_tc_gqa(q, ops.KVTensorMaps(K, V), 0, kv_len, R, Hq, Hkv, D, nd.scale, None, 0, out,
                         ops.tree_attn_tc_workspace(R, Hq, kv_len, DEV), causal=True)
    torch.cuda.synchronize()
    check_heads(out, q, K, V, visibility(R, kv_len, kv_len, causal=True), G, f"tc causal 128 rows over {kv_len}",
                causal_rows=False)


def test_tree_attn_tc_gqa_512_tree_at_cfg2_depth():
    Hq, Hkv, T = 32, 8, 512
    G, kv_len = Hq // Hkv, 124941 + 512
    cap = kv_len + 128
    nd = Needles(Hkv, seed=19, d=D)
    K, V = nd.store(1, cap), nd.store(1, cap)
    plant(nd, K, V, kv_len, T, cap)
    q = group_queries(nd, T, G)
    gen = torch.Generator().manual_seed(9)
    parent = [max(0, i - 1 - int(torch.randint(0, 4, (1,), generator=gen))) for i in range(T)]
    tree = torch.zeros((T, T), dtype=torch.bool)
    for i in range(T):
        tree[i, i] = True
        if i:
            tree[i] |= tree[parent[i]]
    tree = tree.to(DEV)
    bits = torch.from_numpy(orc.pack_tree_mask(tree.cpu().numpy()).view(np.int32)).to(DEV)
    out = torch.empty_like(q)
    ops.tree_attn_tc_gqa(q, ops.KVTensorMaps(K, V), 0, kv_len, T, Hq, Hkv, D, nd.scale, bits.view(T, T // 32).contiguous(), T, out,
                         ops.tree_attn_tc_workspace(T, Hq, kv_len, DEV))
    torch.cuda.synchronize()
    check_heads(out, q, K, V, visibility(T, kv_len, kv_len, tree=tree), G, "tc 512-row tree", causal_rows=False)


# ---------------------------------------------------------------------------------------------------------------------
# tf_rope_append_gqa
# ---------------------------------------------------------------------------------------------------------------------
def _rope_ref(x, cos, sin):
    """fp16 at the reference's rounding points: fp16(fp16(x·cos) + fp16(rotate_half(x)·sin)), on the GPU in fp16."""
    h = x.shape[-1] // 2
    rot = torch.cat([-x[..., h:], x[..., :h]], -1)
    return (x * cos) + (rot * sin)


@pytest.mark.parametrize("Hq,Hkv", [(32, 8), (8, 8)])
def test_rope_append_gqa(Hq, Hkv):
    from triforce_b200.config import named_config
    from triforce_b200.rope import tables_for
    cos, sin = (t.to(DEV) for t in tables_for(named_config("llama-7B-128K")))
    R, cap, slot0 = 7, 256, 100
    gen = torch.Generator(device=DEV).manual_seed(3)
    qkv = torch.randn((R, (Hq + 2 * Hkv) * D), generator=gen, device=DEV).half()
    pos = torch.tensor([5000, 17, 124000, 3, 99999, 1, 64000], dtype=torch.int32, device=DEV)
    K = torch.zeros((Hkv, cap, D), dtype=torch.float16, device=DEV)
    V = torch.zeros_like(K)
    q_out = torch.empty((R, Hq, D), dtype=torch.float16, device=DEV)
    ops.rope_append_gqa(qkv, Hq, Hkv, D, cos, sin, q_out, K, V, pos_ids=pos, slot0=slot0)
    torch.cuda.synchronize()
    c, s = cos[pos.long()][:, None], sin[pos.long()][:, None]
    q = qkv[:, :Hq * D].view(R, Hq, D)
    k = qkv[:, Hq * D:(Hq + Hkv) * D].view(R, Hkv, D)
    v = qkv[:, (Hq + Hkv) * D:].view(R, Hkv, D)
    assert torch.equal(q_out.view(torch.int16), _rope_ref(q, c, s).view(torch.int16))
    assert torch.equal(K[:, slot0:slot0 + R].view(torch.int16), _rope_ref(k, c, s).transpose(0, 1).view(torch.int16))
    assert torch.equal(V[:, slot0:slot0 + R], v.transpose(0, 1))
    assert not K[:, :slot0].any() and not K[:, slot0 + R:].any()
    if Hq == Hkv:  # the MHA entry point gives the same bits
        K2, V2, q2 = torch.zeros_like(K), torch.zeros_like(V), torch.empty_like(q_out)
        ops.rope_append(qkv, Hq, D, cos, sin, q2, K2, V2, pos_ids=pos, slot0=slot0)
        torch.cuda.synchronize()
        assert torch.equal(q2, q_out) and torch.equal(K2, K) and torch.equal(V2, V)


# ---------------------------------------------------------------------------------------------------------------------
# tf_retrieval_build_gqa
# ---------------------------------------------------------------------------------------------------------------------
def test_retrieval_build_gqa_matches_the_group_rule():
    Hq, Hkv, P, chunk, budget, cap = 32, 8, 124928, 8, 4096, 124928 + 64
    gen = torch.Generator(device=DEV).manual_seed(23)
    K = torch.randn((1, Hkv, cap, D), generator=gen, device=DEV).half()
    V = torch.randn((1, Hkv, cap, D), generator=gen, device=DEV).half()
    q = torch.randn((1, Hq, D), generator=gen, device=DEV).half()
    rK = torch.zeros((1, Hkv, budget + 8, D), dtype=torch.float16, device=DEV)
    rV = torch.zeros_like(rK)
    idx = torch.empty((1, Hkv, budget // chunk), dtype=torch.int32, device=DEV)
    sc = torch.empty((1, Hkv, P // chunk), dtype=torch.float16, device=DEV)
    ops.retrieval_build_gqa(K, V, q, rK, rV, P, chunk, budget, out_idx=idx, out_scores=sc)
    torch.cuda.synchronize()
    Kn = K[0].permute(1, 0, 2).cpu().numpy()
    Vn = V[0].permute(1, 0, 2).cpu().numpy()
    wK, wV, widx, wsc = gqa_oracle.retrieval_build_group_sum(Kn, Vn, q[0].cpu().numpy(), P, chunk, budget)
    assert np.array_equal(sc[0].cpu().numpy().view(np.uint16), wsc.view(np.uint16))
    assert np.array_equal(idx[0].cpu().numpy(), widx)
    assert np.array_equal(rK[0, :, :budget].permute(1, 0, 2).cpu().numpy(), wK)
    assert np.array_equal(rV[0, :, :budget].permute(1, 0, 2).cpu().numpy(), wV)
    # the rule is not the per-head MHA selection of any single query head
    assert not np.array_equal(widx, orc.topk_chunks(orc.chunk_scores(q[0, ::4].cpu().numpy(),
                                                                     orc.chunk_mean_keys(Kn, P, chunk)), budget // chunk))
    # G = 1: the bits of tf_retrieval_build
    a_idx, b_idx = torch.empty_like(idx), torch.empty_like(idx)
    a_sc, b_sc = torch.empty_like(sc), torch.empty_like(sc)
    ops.retrieval_build(K, V, q[:, :Hkv].contiguous(), rK, rV, P, chunk, budget, out_idx=a_idx, out_scores=a_sc)
    ops.retrieval_build_gqa(K, V, q[:, :Hkv].contiguous(), rK, rV, P, chunk, budget, out_idx=b_idx, out_scores=b_sc)
    torch.cuda.synchronize()
    assert torch.equal(a_idx, b_idx) and torch.equal(a_sc.view(torch.int16), b_sc.view(torch.int16))


# ---------------------------------------------------------------------------------------------------------------------
# model level: a GQA target and its repeat_kv twin
# ---------------------------------------------------------------------------------------------------------------------
def test_gqa_model_matches_its_repeat_kv_twin():
    """A two-layer d = 128 GQA target (8 query / 2 KV heads) and the MHA model whose k_proj / v_proj repeat each KV head
    for its group compute the same attention.  Prefill (wgmma chunks), a full-KV verify and decode (verify attention) must
    agree; the KV store of the GQA model must equal every G-th head of the twin's, and the retrieval selection must be the
    top-k of the chunk scores it reports.  (test_gqa_model_gpu.py checks those scores against an fp64 group_sum reference.)"""
    from triforce_b200.cache import FlashSimpleCache, RetrievalCache
    from triforce_b200.config import LlamaShape
    from triforce_b200.llama import LlamaModel
    from triforce_b200.synth import numpy_state_dict

    Hq, Hkv, hid = 8, 2, 1024
    G = Hq // Hkv
    kw = dict(hidden_size=hid, intermediate_size=2048, num_hidden_layers=2, num_attention_heads=Hq, vocab_size=32000,
              max_position_embeddings=8192, rms_norm_eps=1e-5)
    gcfg = LlamaShape(num_key_value_heads=Hkv, gqa_retrieval="group_sum", **kw)
    mcfg = LlamaShape(**kw)
    sd = numpy_state_dict(gcfg, seed=31, lm_head_std=0.05)
    twin = dict(sd)
    for l in range(2):
        for n in ("k_proj", "v_proj"):
            w = sd[f"model.layers.{l}.self_attn.{n}.weight"]
            twin[f"model.layers.{l}.self_attn.{n}.weight"] = w.view(Hkv, D, hid).repeat_interleave(G, 0).reshape(Hq * D, hid)
    gm, mm = LlamaModel(gcfg, sd, device=DEV), LlamaModel(mcfg, twin, device=DEV)
    assert gm.gqa and gm.local_num_kv_heads == Hkv and gm.layers[0].wqkv.shape[0] == (Hq + 2 * Hkv) * D
    P, cap = 2048, 4096
    gen = torch.Generator().manual_seed(4)
    ids = torch.randint(0, 32000, (1, P + 16), generator=gen).to(DEV)
    gk, mk = FlashSimpleCache(gm, cap), FlashSimpleCache(mm, cap)
    rc = RetrievalCache(gm, max_budget=256, prefill=P, chunk_size=8, gamma=6)
    assert rc.topk_idx.shape == (2, Hkv, 32)
    for c in range(0, P - 1, 128):  # prefill chunks, then the last prompt token builds the retrieval cache
        gm.forward_target(ids[:, c:min(c + 128, P - 1)], gk)
        mm.forward_target(ids[:, c:min(c + 128, P - 1)], mk)
    gl = gm.forward_target(ids[:, P - 1:P], gk, graph_cache=rc)
    ml = mm.forward_target(ids[:, P - 1:P], mk)
    torch.cuda.synchronize()
    # the two models' q|k|v GEMMs have different widths (cuBLAS may pick other algorithms): equal up to fp16 rounding
    assert (gk.key_store[:, :, :P].float() - mk.key_store[:, ::G, :P].float()).abs().max() < 2e-2
    worst = 0.0
    for a, b in [(gl, ml)] + [(gm.forward_target(ids[:, P + i:P + i + n], gk), mm.forward_target(ids[:, P + i:P + i + n], mk))
                              for i, n in ((0, 7), (7, 1), (8, 8))]:
        torch.cuda.synchronize()
        err = (a - b).abs().max().item() / b.abs().max().item()
        worst = max(worst, err)
        assert err < 2e-2, f"GQA logits differ from the repeat_kv twin by {err:.3g} of the logit scale"
    print(f"GQA vs repeat_kv twin: worst logit difference {worst:.2e} of the logit scale")
    # the last prompt token built the retrieval cache per (layer, KV head): its selection is the top-k of its own scores
    sc = rc.chunk_scores.cpu().numpy()
    for l in range(2):
        idx = orc.topk_chunks(sc[l], 32)
        assert np.array_equal(idx, rc.topk_idx[l].cpu().numpy())
