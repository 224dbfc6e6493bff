"""A grouped-query target through the engine: a two-layer `llama-7B-gqa8-128K`-wide model (32 query / 8 KV heads,
head_dim 128, YaRN factor 32) run by GraphInferenceEngine with its graphs captured, compared with an fp64 evaluation on
the GPU, as test_model_production_gpu.py does for the MHA widths.

The sequence: a 16 383-token prefill in 128-row chunks (causal tf_tree_attn_tc_gqa), the last prompt token (full-KV
attention, then the retrieval build under the "group_sum" rule), a retrieval verify through the captured graph and
eagerly (tf_verify_attn_gqa with clean_keys), a full-KV verify of gamma + 2 rows and a decode step through the seq_len_dev
graphs, then tail_update on the 8-head store and a second retrieval verify.

The reference is that file's Reference with `repeat_kv`: k_proj / v_proj have Hkv heads, the K / V store holds Hkv heads,
and query head h attends to KV head h // G.  Chunk scores are checked against fp16(q̄ · k̄) with q̄ the fp64 sum of the
group's reference queries (the group_sum rule).  The error budget, the tolerances and the KV-store bounds are those of
test_model_production_gpu.py (written above its checks); this model has the same widths and rounding points.  Each check
must also reject negative controls built from the reference alone, among them query head h reading KV head h % Hkv.

On one H100 80GB HBM3 at a 700 W power limit the test took 2.2 s with a peak of 6.1 GiB of device memory.  Maximum logit
excess 0.19-0.30, chunk scores 0.79, layer-1 K / V at most 8.5 ulps (bound 16); the weakest negative control is 6.7 (the
retrieval verify without the tail update), the KV-head mutant 180-195."""
import dataclasses
import types

import pytest
import torch

from test_model_production_gpu import (DEV, F16, LAYERS, LM_HEAD_STD, PEAKED, ROWS, TIED, Reference, attention_ref,
                                       build_engine, check_kv_store, check_logits, check_selection, linear, random_ids,
                                       rmsnorm, rope, _report_time_and_memory)  # noqa: F401  (autouse fixture)
from triforce_b200.config import named_config
from triforce_b200.synth import cuda_state_dict

pytestmark = pytest.mark.gpu


def gqa_model(seed: int):
    """Two layers of llama-7B-gqa8-128K, shaped like production_model: RMSNorm weights 1 + 0.1 N(0, 1); in the first half
    of the KV heads k_proj equals the q_proj of the group's first query head (scaled by TIED), the other q / k heads are
    scaled by PEAKED."""
    cfg = dataclasses.replace(named_config("llama-7B-gqa8-128K"), num_hidden_layers=LAYERS)
    sd = cuda_state_dict(cfg, seed=seed, lm_head_std=LM_HEAD_STD)
    g = torch.Generator(device=DEV).manual_seed(seed + 1000)
    for w in sd.values():
        if w.dim() == 1:
            w.copy_(1 + 0.1 * torch.randn(w.shape, generator=g, device=DEV))
    H, Hkv, d = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim
    G = H // Hkv
    for l in range(LAYERS):
        q = sd[f"model.layers.{l}.self_attn.q_proj.weight"].view(H, d, -1)
        k = sd[f"model.layers.{l}.self_attn.k_proj.weight"].view(Hkv, d, -1)
        q[:H // 2].mul_(TIED)
        k[:Hkv // 2].copy_(q[0:H // 2:G])
        q[H // 2:].mul_(PEAKED)
        k[Hkv // 2:].mul_(PEAKED)
    return cfg, sd


class GQAReference(Reference):
    """Reference with Hkv-head K / V; attention reads KV head kv_map[h] for query head h (h // G, or a mutant map)."""

    def __init__(self, cfg, sd, slots):
        super().__init__(cfg, sd, slots)
        self.Hkv = cfg.num_key_value_heads
        self.G = self.H // self.Hkv
        self.K = [torch.zeros((self.Hkv, slots, self.d), dtype=F16, device=DEV) for _ in range(LAYERS)]
        self.V = [torch.zeros_like(k) for k in self.K]
        self.kv_map = torch.arange(self.H, device=DEV) // self.G

    def store_view(self):
        """What check_kv_store / check_selection need, over the Hkv store heads."""
        return types.SimpleNamespace(H=self.Hkv, d=self.d, K=self.K, V=self.V)

    def attend_store(self, q, K, V, limit, kv_map=None):
        m = self.kv_map if kv_map is None else kv_map
        return attention_ref(q, K[m], V[m], limit, self.scale)

    def qkv(self, x, W, pos):
        n = x.shape[0]
        q = rope(linear(x, W["q"]).view(n, self.H, self.d), self.cos, self.sin, pos)
        k = rope(linear(x, W["k"]).view(n, self.Hkv, self.d), self.cos, self.sin, pos)
        return q, k, linear(x, W["v"]).view(n, self.Hkv, self.d)

    def prefill(self, ids):
        N = ids.numel()
        pos = torch.arange(N, device=DEV)
        h = self.sd["model.embed_tokens.weight"][ids]
        q0 = torch.empty((N, self.H, self.d), dtype=F16, device=DEV)
        W = self.w64(0, ("q", "k", "v"))
        for r0 in range(0, N, ROWS):
            r1 = min(N, r0 + ROWS)
            q0[r0:r1], k, v = self.qkv(rmsnorm(h[r0:r1], self.ln(0, 1), self.eps), W, pos[r0:r1])
            self.K[0][:, r0:r1], self.V[0][:, r0:r1] = k.transpose(0, 1), v.transpose(0, 1)
        del W
        a0 = self.attend_store(q0, self.K[0], self.V[0], pos)
        W = self.w64(0, ("o", "gate", "up", "down"))
        for r0 in range(0, N, ROWS):
            r1 = min(N, r0 + ROWS)
            h[r0:r1] = self.post_attention(0, h[r0:r1], a0[r0:r1], W)
        del W, a0
        W = self.w64(1, ("q", "k", "v"))
        for r0 in range(0, N, ROWS):
            r1 = min(N, r0 + ROWS)
            _, k, v = self.qkv(rmsnorm(h[r0:r1], self.ln(1, 1), self.eps), W, pos[r0:r1])
            self.K[1][:, r0:r1], self.V[1][:, r0:r1] = k.transpose(0, 1), v.transpose(0, 1)

    def full_kv(self, slot0, limit, kv_of_layer=lambda l: l, kv_map=None):
        def attend(l, q, k, v):
            n = q.shape[0]
            self.K[l][:, slot0:slot0 + n], self.V[l][:, slot0:slot0 + n] = k.transpose(0, 1), v.transpose(0, 1)
            src = kv_of_layer(l)
            return self.attend_store(q, self.K[src], self.V[src], limit, kv_map)
        return attend

    def retrieval(self, K, V, B, kv_map=None):
        """attend() of a retrieval verify over the reference's retrieval store (K / V: per layer [Hkv, B + gamma + 1, d])."""
        def attend(l, q, k, v):
            n = q.shape[0]
            K[l][:, B:B + n], V[l][:, B:B + n] = k.transpose(0, 1), v.transpose(0, 1)
            return self.attend_store(q, K[l], V[l], B + torch.arange(n, device=DEV), kv_map)
        return attend

    def retrieval_store(self, idx, B, c, gamma):
        rows = (idx.long()[:, :, :, None] * c + torch.arange(c, device=DEV)).reshape(LAYERS, self.Hkv, B)
        K, V = [], []
        for l in range(LAYERS):
            k = torch.zeros((self.Hkv, B + gamma + 1, self.d), dtype=F16, device=DEV)
            v = torch.zeros_like(k)
            k[:, :B] = torch.gather(self.K[l], 1, rows[l][:, :, None].expand(-1, -1, self.d))
            v[:, :B] = torch.gather(self.V[l], 1, rows[l][:, :, None].expand(-1, -1, self.d))
            K.append(k)
            V.append(v)
        return K, V


@torch.inference_mode()
def test_gqa_7b_width_prefill_retrieval_full_verify_decode_and_tail_update():
    P, B, c, gamma = 16384, 4096, 8, 6
    cfg, sd = gqa_model(seed=41)
    ge = build_engine(cfg, sd, P, P + 64, B, c, gamma)
    kv, gc = ge.engine.kv_cache, ge.engine.graph_cache
    target = ge.engine.model
    assert target.gqa and target.local_num_kv_heads == 8 and kv.key_store.shape[1] == 8 and gc.topk_idx.shape[1] == 8
    ref = GQAReference(cfg, sd, P + 64)
    store = ref.store_view()
    wrong_kv = torch.arange(ref.H, device=DEV) % ref.Hkv  # the mutant head map: h % Hkv instead of h // G
    ids = random_ids(P + 32, seed=42)
    prompt, extra = ids[:P], ids[P:]

    # 1. prefill of P - 1 tokens in 128-row chunks
    ge.inference(prompt[None, :-1])
    torch.cuda.synchronize()
    assert kv.seq_len == P - 1
    ref.prefill(prompt[:-1])
    check_kv_store(kv, store, P - 1)

    # 2. the last prompt token, then the retrieval build: chunk scores against fp16(q̄·k̄) of the reference's queries
    logits = ge.inference(prompt[None, -1:])
    q_bar = [None] * LAYERS

    def last_attend(l, q, k, v):
        q_bar[l] = q[0].double().view(ref.Hkv, ref.G, ref.d).sum(1)  # the group_sum query of each KV head
        return ref.full_kv(P - 1, torch.tensor([P - 1], device=DEV))(l, q, k, v)

    want = ref.forward(prompt[-1:], torch.tensor([P - 1], device=DEV), last_attend)
    check_logits("last prompt token", logits, want)
    assert kv.seq_len == P
    check_selection(gc, kv, store, q_bar, P)
    rK, rV = ref.retrieval_store(gc.topk_idx, B, c, gamma)

    # 3. retrieval verify of gamma + 1 rows (7 x 4 = 28 packed rows per CTA): captured graph, then eagerly
    vt = extra[:gamma + 1]
    vpos = torch.arange(P, P + gamma + 1, device=DEV)
    got_graph = ge.graph_verify(vt[None], vpos[None])
    got_eager = ge.engine.model_verify(vt[None], vpos[None])
    assert torch.equal(got_graph, got_eager), "retrieval verify: graph replay and eager forward differ"
    copy = lambda: ([k.clone() for k in rK], [v.clone() for v in rV])
    mutants = [
        ("RoPE positions + 1", ref.forward(vt, vpos + 1, ref.retrieval(*copy(), B))),
        ("query head h reads KV head h % Hkv", ref.forward(vt, vpos, ref.retrieval(*copy(), B, kv_map=wrong_kv))),
        ("gate and up swapped", ref.forward(vt, vpos, ref.retrieval(*copy(), B), swap_gate_up=True)),
    ]
    want = ref.forward(vt, vpos, ref.retrieval(rK, rV, B))
    check_logits("retrieval verify", got_graph, want, mutants)

    # 4. full-KV verify of gamma + 2 rows (8 x 4 = 32 packed rows) through the seq_len_dev graph, then one decode step
    ft = extra[gamma + 1:2 * gamma + 3]
    fpos = torch.arange(P, P + gamma + 2, device=DEV)
    snap = [k.clone() for k in ref.K], [v.clone() for v in ref.V]

    def restore():
        for l in range(LAYERS):
            ref.K[l].copy_(snap[0][l])
            ref.V[l].copy_(snap[1][l])

    mutants = []
    for name, kw, lim in (("layer 1 attends to layer 0's K/V", dict(kv_of_layer=lambda l: 0), fpos),
                          ("kv_len short by the row count", {}, fpos - (gamma + 2)),
                          ("query head h reads KV head h % Hkv", dict(kv_map=wrong_kv), fpos)):
        restore()
        mutants.append((name, ref.forward(ft, fpos, ref.full_kv(P, lim, **kw))))
    restore()
    got = ge.inference(ft[None])
    assert kv.seq_len == P + gamma + 2
    want = ref.forward(ft, fpos, ref.full_kv(P, fpos))
    check_logits("full-KV verify", got, want, mutants)

    dt = extra[2 * gamma + 3:2 * gamma + 4]
    p1 = P + gamma + 2
    got = ge.decode_step(dt)
    assert kv.seq_len == p1 + 1
    dpos = torch.tensor([p1], device=DEV)
    mutants = [("decode at kv_len - 1", ref.forward(dt, dpos, ref.full_kv(p1, dpos - 1)))]
    want = ref.forward(dt, dpos, ref.full_kv(p1, dpos))
    check_logits("decode step", got, want, mutants)

    # 5. tail update on the 8-head stores, then a retrieval verify that attends to the committed tokens
    ge.update_graph_cache()
    n_new = kv.seq_len - P
    stale = [k.clone() for k in rK], [v.clone() for v in rV]
    for l in range(LAYERS):
        rK[l][:, B - n_new:B], rV[l][:, B - n_new:B] = ref.K[l][:, P:P + n_new], ref.V[l][:, P:P + n_new]
        assert torch.equal(gc.key_store[l, :, B - n_new:B], kv.key_store[l, :, P:P + n_new])
        assert torch.equal(gc.value_store[l, :, B - n_new:B], kv.value_store[l, :, P:P + n_new])
    ut = torch.cat([ft, dt])[:gamma + 1]
    upos = torch.arange(kv.seq_len, kv.seq_len + gamma + 1, device=DEV)
    got = ge.graph_verify(ut[None], upos[None])
    mutants = [("retrieval verify without the tail update", ref.forward(ut, upos, ref.retrieval(*stale, B)))]
    want = ref.forward(ut, upos, ref.retrieval(rK, rV, B))
    check_logits("retrieval verify after the tail update", got, want, mutants)
