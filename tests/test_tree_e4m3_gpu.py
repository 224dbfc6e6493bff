"""The Sequoia tree path over an E4M3 full-KV store and E4M3 weights, on the GPU.

* tf_tree_attn_tc_e4m3 is bit-identical to tf_tree_attn_tc over the dequantized store D (MHA 40 and 32 heads, GQA 32/8; R = 128
  and 512; a short store whose last tile is partial, 49 664 and 130 560 keys; the real 512-node mask and random masks; rows at
  exponents -32 and 8 and zero rows), and close to fp64 attention over D.
* tf_kv_compact_e4m3 equals torch indexing on codes and exponents, bit for bit, for overlapping ranges in every layer and head.
* Greedy SpecTree runs at 13B width (and a grouped-query 7B shape) emit the greedy autoregressive sequence of the same engine,
  the T = 0 walk equals its CPU restatement, and after each compaction the store and the retrieval tail hold the accepted rows.
* At T = 0.6 an E4M3-weight SpecTree and one whose fp16 weights are D agree bit for bit for 4 rounds."""
from __future__ import annotations

import dataclasses

import pytest
import torch

from attn_needles import report_time_and_memory  # noqa: F401  (autouse fixture: wall time and peak memory per test)
from test_greedy_gpu import NEAR_TIE, NEAR_TIE_E4M3_STORE, _one_hot_rows, compare_to_greedy, cpu_greedy_walk
from test_weights_e4m3_model_gpu import d_state_dict
from triforce_b200 import ops
from triforce_b200.config import named_config
from triforce_b200.rng import CounterNoise
from triforce_b200.spectree import SpecTree, load_grow_map, pack_mask_bits
from triforce_b200.synth import agreement_state_dicts, numpy_prompt
from triforce_b200.tp import SingleGpuLlama

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _dequant(codes, e):
    """D = fp16_rn(code * 2^e), rounded once (the oracle's rule, on the device)."""
    return (codes.view(torch.float8_e4m3fn).double() * torch.exp2(e.double()).unsqueeze(-1)).half()


def _random_store(H, cap, d, seed):
    """One layer of random codes (no NaN codes) at exponents in [-12, 4], with rows at -32 and at 8 (codes below 0x78 there, so D
    stays finite) and all-zero rows.  Returns the E4m3Store and its D (K, V)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    stores = []
    for _ in range(2):
        c = torch.randint(0, 256, (1, H, cap, d), generator=g, device=DEV, dtype=torch.uint8)
        c = torch.where((c & 0x7F) == 0x7F, c ^ 1, c)
        e = torch.randint(-12, 5, (1, H, cap), generator=g, device=DEV, dtype=torch.int8)
        e[..., 5::97] = -32
        e[..., 11::131] = 8
        big = (c[..., 11::131, :] & 0x7F).clamp(max=0x77)
        c[..., 11::131, :] = (c[..., 11::131, :] & 0x80) | big
        c[..., 17::113, :] = 0
        stores.append((c.contiguous(), e.contiguous()))
    (kc, ke), (vc, ve) = stores
    return ops.E4m3Store(kc, vc, ke, ve), _dequant(kc, ke), _dequant(vc, ve)


def _mask(R, kind, seed):
    if kind == "tree":
        return pack_mask_bits(load_grow_map("512")["mask"][:R, :R]).to(DEV)
    g = torch.Generator().manual_seed(seed)
    m = (torch.rand(R, R, generator=g) < 0.3).to(torch.int64)
    m.fill_diagonal_(1)
    return pack_mask_bits(m).to(DEV)


def _both(Hq, Hkv, R, kv_len, kind, seed):
    d = 128
    cap = (kv_len + 63) // 64 * 64 + 64
    st, KD, VD = _random_store(Hkv, cap, d, seed)
    g = torch.Generator(device=DEV).manual_seed(seed + 1)
    q = (torch.randn((R, Hq, d), generator=g, device=DEV) * 0.05).half()
    mask = _mask(R, kind, seed)
    scale = d ** -0.5
    ws = ops.tree_attn_tc_workspace(R, Hq, kv_len, DEV)
    got, want = torch.empty_like(q), torch.empty_like(q)
    ops.tree_attn_tc_e4m3(q, st, 0, kv_len, R, Hq, Hkv, d, scale, mask, R, got, ws)
    maps = ops.KVTensorMaps(KD, VD)
    if Hq == Hkv:
        ops.tree_attn_tc(q, maps, 0, kv_len, R, Hq, d, scale, mask, R, want, ws)
    else:
        ops.tree_attn_tc_gqa(q, maps, 0, kv_len, R, Hq, Hkv, d, scale, mask, R, want, ws)
    torch.cuda.synchronize()
    return q, KD, VD, mask, got, want


CASES = [  # (Hq, Hkv, R, kv_len, mask)
    (40, 40, 512, 1000, "tree"),
    (32, 32, 128, 777, "random"),
    (32, 8, 512, 1000, "random"),
    (40, 40, 512, 49664, "tree"),
    (32, 8, 128, 49664, "random"),
    (32, 32, 512, 130560, "tree"),
    (40, 40, 512, 130560, "random"),
]


@pytest.mark.parametrize("Hq,Hkv,R,kv_len,kind", CASES, ids=[f"{a}-{b}-R{r}-S{s}-{k}" for a, b, r, s, k in CASES])
def test_tree_attn_tc_e4m3_is_the_fp16_kernel_on_d(Hq, Hkv, R, kv_len, kind):
    *_, got, want = _both(Hq, Hkv, R, kv_len, kind, seed=kv_len + R + Hkv)
    assert torch.isfinite(want).all()
    assert torch.equal(got, want), (got.float() - want.float()).abs().max().item()


def test_tree_attn_tc_e4m3_against_fp64_on_d():
    Hq, Hkv, R, kv_len = 8, 2, 128, 900
    q, KD, VD, mask, got, _ = _both(Hq, Hkv, R, kv_len, "tree", seed=4)
    grp = Hq // Hkv
    K = KD[0, :, :kv_len].double().repeat_interleave(grp, 0)  # [Hq, S, d]
    V = VD[0, :, :kv_len].double().repeat_interleave(grp, 0)
    s = torch.einsum("rhd,hsd->hrs", q.double(), K) * (128 ** -0.5)
    words = mask.view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    bits = ((words.unsqueeze(-1) >> torch.arange(32, device=DEV)) & 1).reshape(R, -1)[:, :R].bool()
    vis = torch.cat([torch.ones(R, kv_len - R, dtype=torch.bool, device=DEV), bits], dim=1)
    s = s.masked_fill(~vis, float("-inf"))
    ref = torch.einsum("hrs,hsd->rhd", torch.softmax(s, dim=-1), V)
    # fp16 P and output rounding, relative to the largest |V| a row can mix (the exponent-8 rows dominate where visible)
    vmax = V.abs().amax(dim=(1, 2)).view(1, Hq, 1)
    err = ((got.double() - ref).abs() / vmax).max().item()
    assert err < 2e-3, err


@pytest.mark.parametrize("n", [1, 2, 5, 9, 17])
def test_kv_compact_e4m3_is_torch_indexing(n):
    L, H, cap, d = 3, 8, 512, 128
    g = torch.Generator(device=DEV).manual_seed(n)
    st = ops.E4m3Store(*(torch.randint(0, 256, (L, H, cap, d), generator=g, device=DEV, dtype=torch.uint8) for _ in range(2)),
                       *(torch.randint(-32, 9, (L, H, cap), generator=g, device=DEV, dtype=torch.int8) for _ in range(2)))
    for offset in (100, 301):
        # accepted nodes lie at offset + i, i ascending from 0: the first ones are their own destination, later ones overlap it
        idx = torch.sort(torch.randperm(40, generator=torch.Generator().manual_seed(n + offset))[:n]).values
        idx[0] = 0
        src = (idx + offset).to(torch.int32).to(DEV)
        before = [t.clone() for t in (st.k_codes, st.v_codes, st.k_exp, st.v_exp)]
        ops.kv_compact_e4m3(st, src, offset)
        for b, a in zip(before, (st.k_codes, st.v_codes, st.k_exp, st.v_exp)):
            want = b.clone()
            want[:, :, offset:offset + n] = b[:, :, src.long()]
            assert torch.equal(a, want)


# ---------------------------------------------------------------------------------------------------------------------
# the tree path end to end
# ---------------------------------------------------------------------------------------------------------------------
def _tree_engine(name, kv, weights, P, B, gen_len, temperature, alpha=0.001):
    cfg = dataclasses.replace(named_config(name), num_hidden_layers=2)
    tsd, _ = agreement_state_dicts(cfg, named_config("llama-68M"), alpha, alpha, seed=0, device=DEV)
    gm = load_grow_map("512")
    llm = SingleGpuLlama(name, local_rank=0, world_size=1, prefill=P, gen_len=gen_len, retrieval_budget=B, retrieval_chunk_size=8,
                         gamma=6, temperature=temperature, config=cfg, tree_size=gm["size"], kv_dtype=kv, weight_dtype=weights)
    return llm, tsd, gm, cfg


class _CompactionCheck:
    """Wraps gather_kv_incremental over an E4M3 store: the store rows [offset, offset + accepted) must hold exactly the accepted nodes' codes and
    exponents afterwards, and the retrieval tail their D."""

    def __init__(self, llm):
        self.llm, self.kv = llm, llm.kv_cache
        self.orig = self.kv.gather_kv_incremental
        self.kv.gather_kv_incremental = self
        self.checked = 0

    def __call__(self, indices, offset):
        st = self.kv.e4m3
        rows = [st.k_codes, st.v_codes, st.k_exp, st.v_exp]
        src = torch.tensor([offset + int(i) for i in indices], device=DEV)
        want = [t[:, :, src].clone() for t in rows]
        self.orig(indices, offset)
        for t, w in zip(rows, want):
            assert torch.equal(t[:, :, offset:offset + len(indices)], w)
        self.pending = (offset + len(indices))
        self.checked += 1

    def check_tail(self):
        rc, st = self.llm.retrieval_cache, self.kv.e4m3
        n = self.pending - rc.prefill
        KD = _dequant(st.k_codes[:, :, rc.prefill:self.pending], st.k_exp[:, :, rc.prefill:self.pending])
        VD = _dequant(st.v_codes[:, :, rc.prefill:self.pending], st.v_exp[:, :, rc.prefill:self.pending])
        assert torch.equal(rc.key_store[:, :, rc.max_budget - n:rc.max_budget], KD)
        assert torch.equal(rc.value_store[:, :, rc.max_budget - n:rc.max_budget], VD)


GREEDY = [  # (target shape, full-KV store, weights)
    ("llama-13B-128K", "e4m3", "fp16"),
    ("llama-13B-128K", "fp16", "e4m3"),
    ("llama-13B-128K", "e4m3", "e4m3"),
    ("llama-7B-gqa8-128K", "e4m3", "fp16"),
]


@pytest.mark.parametrize("name,kv,weights", GREEDY, ids=[f"{a}-kv_{b}-w_{c}" for a, b, c in GREEDY])
@torch.inference_mode()
def test_greedy_spectree_over_e4m3_formats_is_greedy_ar(name, kv, weights):
    P, B, rounds = 16384, 4096, 16
    llm, tsd, gm, cfg = _tree_engine(name, kv, weights, P, B, rounds * 24 + 64, 0.0)
    llm.init_parameters(state_dict=tsd, cuda_graphs=False)
    del tsd
    ids = numpy_prompt(P, seed=9)[0].to(DEV)
    n_ar = rounds * 17 + 8
    llm.reset()
    row = llm.prefill(ids.unsqueeze(0))[:, -1, :].float()
    ar, ar_rows = [], []
    for i in range(n_ar + 1):
        ar_rows.append(row[0].clone())
        ar.append(int(torch.argmax(row[0])))
        if i < n_ar:
            row = llm.inference(torch.tensor([[ar[-1]]], device=DEV))[:, -1, :].float()
    ar_rows = torch.stack(ar_rows)

    st = SpecTree(engine=llm, temperature=0.0, top_p=0.9, max_length=P + 512, grow_map=gm, vocab_size=cfg.vocab_size)
    chk = _CompactionCheck(llm) if kv == "e4m3" else None
    nt = st.prefill(prefix=ids)
    emitted = [int(nt.reshape(-1)[0])]
    counts = []
    for r in range(rounds):
        st.construct_grow_map(next_token=nt)
        tokens = st.verify_tokens.clone()
        nt, acc, toks = st.verify()
        assert nt is not None, "an EOS was accepted"
        probs = st.target_logits.cpu()
        assert torch.equal(probs, _one_hot_rows(probs))
        walk, code, terminal, nxt = cpu_greedy_walk(probs, tokens.cpu(), gm["Successors"])
        toks = [int(t) for t in toks.tolist()]
        assert not terminal and st._walk_out[2].item() == 0
        assert acc == len(walk) + 1 and toks[1:-1] == tokens[walk].tolist() and toks[-1] == nxt, (r, walk, toks)
        if chk is not None:
            chk.check_tail()
        emitted.extend(toks[1:])
        counts.append(acc)
        nt = nt.unsqueeze(0)
    assert chk is None or chk.checked == rounds
    print(f"Sequoia {name} kv={kv} weights={weights}, greedy: tokens per round {counts}")
    compare_to_greedy(emitted, ar, ar_rows, rounds + 1, f"SpecTree 512 nodes, {name}, kv={kv}, weights={weights}",
                      near_tie=NEAR_TIE_E4M3_STORE if kv == "e4m3" else NEAR_TIE)
    assert sum(counts) / len(counts) > 1.0


@pytest.mark.parametrize("kv", ["fp16", "e4m3"])
@torch.inference_mode()
def test_e4m3_weight_spectree_is_the_fp16_spectree_on_d(kv):
    P, B, rounds = 8192, 4096, 4
    out = []
    for weights in ("e4m3", "fp16"):
        llm, tsd, gm, cfg = _tree_engine("llama-13B-128K", kv, weights, P, B, rounds * 24 + 64, 0.6, alpha=0.01)
        llm.init_parameters(state_dict=tsd if weights == "e4m3" else d_state_dict(cfg, tsd), cuda_graphs=False)
        del tsd
        st = SpecTree(engine=llm, temperature=0.6, top_p=0.9, max_length=P + 512, grow_map=gm, vocab_size=cfg.vocab_size,
                      noise=CounterNoise(7, device=DEV))
        nt = st.prefill(prefix=numpy_prompt(P, seed=11)[0].to(DEV))
        trace = [nt.cpu()]
        for _ in range(rounds):
            st.construct_grow_map(next_token=nt)
            draft = st.draft_logits.cpu()
            tokens = st.verify_tokens.cpu()
            nt, acc, toks = st.verify()
            trace += [draft, tokens, st.target_logits.cpu(), acc, torch.as_tensor(toks).cpu(), llm.kv_cache.seq_len]
            if nt is None:
                break
            nt = nt.unsqueeze(0)
        out.append(trace)
        del st, llm
        torch.cuda.empty_cache()
    a, b = out
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert (torch.equal(x, y) if isinstance(x, torch.Tensor) else x == y), f"entry {i} of the trace differs"
