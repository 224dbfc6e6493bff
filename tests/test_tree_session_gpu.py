"""Follow-up turns on the Sequoia tree path (session.TreeSession), on the GPU.

* Wiring: the first turn emits the tokens, per-round counts and store length of SpecTree.prefill plus rounds driven by hand on
  the same Philox stream (the session draws no race at the prompt, so its stream starts one draw later).
* append: the store rows and the last-row logits are bit-identical to the same forwards run on the model directly (the prompt
  phase, then LlamaModel.extend); after the re-selection, topk_idx equals a fresh build at the new boundary with the same
  queries and the budget tail holds the store's rows [B, len).  13B width and a grouped-query 7B, 2 layers, fp16 store.
* T = 0: turn 2 (after append) is the engine's greedy continuation of the transcript, for fp16, an E4M3 store, E4M3 store and
  weights, and GQA over an E4M3 store; at T = 0.6, truncate + the same append + the same seed repeat turn 2, another seed
  does not.
* T > 0 on the stub engine of test_tree_lossless_gpu.py, driven as the session drives it (session.tree_round: fp32 Philox race
  redrawn every round): the first token of round 1 and of round 2 follow the root's target row (chi-square)."""
from __future__ import annotations

import dataclasses

import numpy as np
import pytest
import torch

from attn_needles import report_time_and_memory  # noqa: F401  (autouse fixture: wall time and peak memory per test)
from chi2_util import chi2, chi2_threshold
from test_greedy_gpu import NEAR_TIE, NEAR_TIE_E4M3_STORE, compare_to_greedy
from test_tree_lossless_gpu import _assert_follows, _t
from tree_lossless_util import SMALL_TREE, StubEngine, grow_map_of, softmax64, synthetic_logits
from triforce_b200 import ops
from triforce_b200.cache import FlashSimpleCache, RetrievalCacheSeqouia
from triforce_b200.config import named_config
from triforce_b200.device_loop import PhiloxNoise
from triforce_b200.session import TreeSession, tree_round
from triforce_b200.spectree import SpecTree, load_grow_map
from triforce_b200.synth import agreement_state_dicts, numpy_prompt
from triforce_b200.tp import SingleGpuLlama

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _engine(name, kv, weights, P, B, temperature, extra=1024, gen_len=256, alpha=0.001):
    """test_tree_e4m3_gpu._tree_engine's 2-layer engine, with room for `extra` appended tokens."""
    cfg = dataclasses.replace(named_config(name), num_hidden_layers=2)
    tsd, _ = agreement_state_dicts(cfg, named_config("llama-68M"), alpha, alpha, seed=0, device=DEV)
    gm = load_grow_map("512")
    llm = SingleGpuLlama(name, local_rank=0, world_size=1, prefill=P, gen_len=gen_len, retrieval_budget=B, retrieval_chunk_size=8,
                         gamma=6, temperature=temperature, config=cfg, tree_size=gm["size"], kv_dtype=kv, weight_dtype=weights,
                         max_context=P + extra)
    llm.init_parameters(state_dict=tsd, cuda_graphs=False)
    del tsd
    assert llm.kv_cache.max_budget == P + extra + gen_len + 32 + gm["size"] and llm.retrieval_cache.max_context == P + extra
    return llm, gm, cfg


@torch.inference_mode()
def test_first_turn_is_spectree_driven_by_hand():
    P, B, seed = 8192, 4096, 3
    llm, gm, cfg = _engine("llama-13B-128K", "fp16", "fp16", P, B, 0.6)
    ids = numpy_prompt(P, seed=11)[0].to(DEV)
    s = TreeSession(llm)
    s.prefill(ids)
    # SpecTree.prefill draws the race (draw 0) before the first token (draw 1); the session draws no race at the prompt
    toks = s.generate(100, temperature=0.6, top_p=0.9, noise=PhiloxNoise(DEV, state=torch.tensor([seed, 1], device=DEV)))
    turn, length = s.last_turn, s.length
    assert turn.rounds >= 4, turn
    st = SpecTree(llm, temperature=0.6, top_p=0.9, grow_map=gm, vocab_size=cfg.vocab_size, noise=PhiloxNoise(DEV, 99),
                  race_dtype=torch.float32)
    st.noise = PhiloxNoise(DEV, seed)
    nt = st.prefill(prefix=ids)
    emitted, counts = [int(nt.reshape(-1)[0])], []
    for _ in range(turn.rounds):
        st.noise.tree_uniform_into(st.rand)
        st.construct_grow_map(next_token=nt)
        nt, acc, t = st.verify()
        assert nt is not None
        emitted += [int(x) for x in t[1:].tolist()]
        counts.append(acc)
        nt = nt.unsqueeze(0)
    print(f"\n[tree session] turn 1 by hand: {turn.rounds} rounds, tokens per round {counts}")
    assert emitted == toks and counts == turn.accepted and llm.kv_cache.seq_len == length == P + len(toks) - 1


CONFIGS = ["llama-13B-128K", "llama-7B-gqa8-128K"]


@pytest.mark.parametrize("name", CONFIGS)
@torch.inference_mode()
def test_append_state_is_the_models_own_forwards(name):
    P, B, Q = 16384, 4096, 300
    llm, gm, cfg = _engine(name, "fp16", "fp16", P, B, 0.0)
    ids = numpy_prompt(P + Q, seed=5)[0].to(DEV)
    s = TreeSession(llm)
    s.prefill(ids[:P])
    s.append(ids[P:])
    n = s.length
    assert n == P + Q and s.ids == ids.tolist()
    # the same forwards on the model: the prompt phase (all ids but the last, then the last one), then extend
    m, kv = llm.model, llm.kv_cache
    ref = FlashSimpleCache(m, kv.max_budget)
    m.prefill(ids[:P - 1], ref)
    m.forward_target(ids[P - 1:P], ref)
    q = torch.empty((cfg.num_hidden_layers, cfg.num_attention_heads, cfg.head_dim), dtype=torch.float16, device=DEV)
    want = m.extend(ids[P:], ref, queries=q)
    assert torch.equal(s._logits, want)
    assert torch.equal(kv.key_store[:, :, :n], ref.key_store[:, :, :n]) and torch.equal(kv.value_store[:, :, :n], ref.value_store[:, :, :n])
    # the re-selection: a fresh build at the new boundary with the same queries, and the tail
    rc = llm.retrieval_cache
    Bn = n // 8 * 8
    assert rc.prefill == Bn
    fresh = RetrievalCacheSeqouia(m, max_budget=B, prefill=Bn, chunk_size=8, tree_size=gm["size"], max_context=Bn)
    fresh.build_all_layers(ref, q)
    assert torch.equal(rc.topk_idx, fresh.topk_idx)
    t = n - Bn
    assert t > 0
    assert torch.equal(rc.key_store[:, :, B - t:B], kv.key_store[:, :, Bn:n])
    assert torch.equal(rc.value_store[:, :, B - t:B], kv.value_store[:, :, Bn:n])
    assert torch.equal(rc.key_store[:, :, :B - t], fresh.key_store[:, :, :B - t])


LOSSLESS = [("llama-13B-128K", "fp16", "fp16"), ("llama-13B-128K", "e4m3", "fp16"), ("llama-13B-128K", "e4m3", "e4m3"),
            ("llama-7B-gqa8-128K", "e4m3", "fp16")]


@pytest.mark.parametrize("name,kv,weights", LOSSLESS, ids=[f"{a}-kv_{b}-w_{c}" for a, b, c in LOSSLESS])
@torch.inference_mode()
def test_second_turn_at_temperature_zero_is_greedy_ar(name, kv, weights):
    P, B, Q, gen = 16384, 4096, 200, 64
    llm, gm, cfg = _engine(name, kv, weights, P, B, 0.0)
    ids = numpy_prompt(P + Q, seed=7)[0].to(DEV)
    s = TreeSession(llm)
    s.prefill(ids[:P])
    s.generate(24, temperature=0.0)
    s.append(ids[P:])
    L2 = s.length
    first_row = s._logits[0, -1].float().clone()
    tri = s.generate(gen, temperature=0.0)
    turn = s.last_turn
    # the engine alone from the same state: one-row forwards after the appended rows
    s.truncate(L2)
    rows, ar = [first_row], [int(torch.argmax(first_row))]
    for _ in range(len(tri) + 8):
        row = llm.inference(torch.tensor([[ar[-1]]], device=DEV))[0, -1].float()
        rows.append(row)
        ar.append(int(torch.argmax(row)))
    what = f"TreeSession {name} kv={kv} weights={weights}, turn 2"
    print(f"\n[{what}] {turn.rounds} rounds, tokens per round {turn.accepted}, stop {turn.stop}")
    compare_to_greedy(tri, ar, torch.stack(rows), 16, what, near_tie=NEAR_TIE_E4M3_STORE if kv == "e4m3" else NEAR_TIE)
    assert turn.tokens_per_round > 1.0


@torch.inference_mode()
def test_truncate_and_the_same_turn_again_repeat_it():
    P, B, Q = 8192, 4096, 150
    llm, gm, cfg = _engine("llama-13B-128K", "fp16", "fp16", P, B, 0.6)
    ids = numpy_prompt(P + Q, seed=13)[0].to(DEV)
    s = TreeSession(llm)
    s.prefill(ids[:P])
    s.generate(16, seed=1)
    n0 = s.length
    turns = []
    for seed in (7, 7, 8):
        s.truncate(n0)
        s.append(ids[P:])
        toks = s.generate(24, seed=seed)
        turns.append((toks, s.last_turn.accepted, s.length, llm.retrieval_cache.prefill))
    assert turns[0] == turns[1]
    assert turns[0][0] != turns[2][0]
    print(f"\n[tree session] rollback: {len(turns[0][0])} tokens in {len(turns[0][1])} rounds, identical twice; seed 8 differs")


# ---------------------------------------------------------------------------------------------------------------------
# T > 0 through the session's round driver, on the stub engine
# ---------------------------------------------------------------------------------------------------------------------
def _stub_tree(gm, V, T, top_p, seed):
    draft, target = synthetic_logits(gm["size"], V, seed)
    st = SpecTree(StubEngine(_t(draft), _t(target)), temperature=T, top_p=top_p, grow_map=gm, vocab_size=V,
                  noise=PhiloxNoise(DEV, 0), race_dtype=torch.float32)
    return st, draft, target


def _two_rounds(st, nt):
    out = []
    for _ in range(2):
        nxt, acc, toks = tree_round(st, nt)
        assert nxt is not None
        out.append(toks[1])
        nt = nxt.reshape(1, 1)
    return out


@torch.inference_mode()
def test_session_rounds_are_lossless_at_temperature():
    gm = grow_map_of(SMALL_TREE)
    V, T, top_p, N = 1000, 0.6, 0.9, 16_000
    st, draft, target = _stub_tree(gm, V, T, top_p, seed=25)
    st.noise = PhiloxNoise(DEV, 41)
    p = ops.norm_logits(_t(target), T, top_p).cpu().numpy()[0].astype(np.float64)
    q = softmax64(draft[0], T)
    nt = torch.ones((1, 1), dtype=torch.long, device=DEV)
    firsts = torch.stack([torch.stack(_two_rounds(st, nt)) for _ in range(N)]).cpu().numpy()  # [N, 2]
    for r in range(2):
        counts = np.bincount(firsts[:, r], minlength=V)
        _assert_follows(f"TreeSession rounds, fp32 Philox race, round {r + 1} first token, 4/3/4 tree V {V} T {T} top_p {top_p}",
                        firsts[:, r], p, V, [("q_root", counts, q)])
    # the rounds are not copies of each other: a fresh race each round
    assert (firsts[:, 0] != firsts[:, 1]).mean() > 0.05
    # the same seed gives the same rounds, another seed other ones
    runs = []
    for seed in (5, 5, 6):
        st.noise = PhiloxNoise(DEV, seed)
        runs.append([int(x) for _ in range(8) for x in _two_rounds(st, nt)])
    assert runs[0] == runs[1] and runs[0] != runs[2]
    stat, df = chi2(np.bincount(firsts[:, 1], minlength=V), p)
    assert stat < chi2_threshold(df)
