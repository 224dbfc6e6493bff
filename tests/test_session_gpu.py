"""Follow-up turns over a prefilled context, on the GPU.

* tf_tree_attn_tc_causal_e4m3 is bit-identical to the fp16 wgmma kernel in causal mode over the dequantized store D (MHA 32 heads
  and GQA 32/8; prefixes of 49 152 and 124 928 keys; R = 1, 65, 128, 300; rows at exponents -32 and 8).
* LlamaModel.extend: prefill(A) then extend(B) equals prefill(A + B) bit for bit over fp16 (MHA and GQA); over an E4M3 store
  with E4M3 weights it stays within the fp64-reference logit tolerance of test_model_production_gpu.py.
* RetrievalCache.reselect selects what the CPU oracle selects over the new boundary's chunks with the new query (fp16 store;
  E4M3 store into an E4M3 retrieval cache, the oracle over D), and the budget tail holds the store's rows [B, len).
* Session: turn 2 at T = 0 is the target's greedy continuation of the same state (fp16, E4M3 store + weights + retrieval, GQA);
  truncate + the same append + the same seed repeats a turn exactly; the whole-loop graph equals the step-wise loop over two
  turns; the first turn replays tests/golden/e2e_tiny.json event for event."""
from __future__ import annotations

import dataclasses
import json
import os

import numpy as np
import pytest
import torch

import kv_e4m3_oracle as eo
from attn_needles import report_time_and_memory  # noqa: F401  (autouse fixture: wall time and peak memory per test)
from e2e_util import TokenizerStub, matching_prefix
from oracle import triforce_oracle as orc
from test_greedy_gpu import NEAR_TIE, NEAR_TIE_E4M3_STORE, compare_to_greedy
from test_model_production_gpu import Reference, attention_ref, check_logits, production_model
from test_tree_e4m3_gpu import _random_store
from test_weights_e4m3_model_gpu import d_state_dict
from triforce_b200 import ops
from triforce_b200.cache import FlashSimpleCache, RetrievalCache, StreamingLLMEvictionCache
from triforce_b200.config import named_config
from triforce_b200.engine import GraphInferenceEngine
from triforce_b200.llama import LlamaModel
from triforce_b200.rng import CounterNoise
from triforce_b200.sampling import norm_logits
from triforce_b200.session import Session
from triforce_b200.synth import agreement_state_dicts, cuda_state_dict, numpy_prompt, numpy_state_dict

pytestmark = pytest.mark.gpu
DEV = "cuda"
TOK = TokenizerStub()


# ---------------------------------------------------------------------------------------------------------------------
# the kernel
# ---------------------------------------------------------------------------------------------------------------------
_STORES = {}


def _store(Hkv, cap):
    if (Hkv, cap) not in _STORES:
        _STORES.clear()
        _STORES[(Hkv, cap)] = _random_store(Hkv, cap, 128, seed=Hkv + cap)
    return _STORES[(Hkv, cap)]


KERNEL_CASES = [(hq, hkv, prefix, R) for hq, hkv in ((32, 32), (32, 8)) for prefix in (49152, 124928) for R in (1, 65, 128, 300)]


@pytest.mark.parametrize("Hq,Hkv,prefix,R", KERNEL_CASES, ids=[f"{a}-{b}-P{p}-R{r}" for a, b, p, r in KERNEL_CASES])
def test_causal_e4m3_is_the_fp16_causal_kernel_on_d(Hq, Hkv, prefix, R):
    d, kv_len = 128, prefix + R
    cap = 124928 + 320
    st, KD, VD = _store(Hkv, cap)
    g = torch.Generator(device=DEV).manual_seed(prefix + R + Hkv)
    q = (torch.randn((R, Hq, d), generator=g, device=DEV) * 0.05).half()
    scale = d ** -0.5
    ws = ops.tree_attn_tc_workspace(R, Hq, kv_len, DEV)
    got, want = torch.empty_like(q), torch.empty_like(q)
    ops.tree_attn_tc_causal_e4m3(q, st, 0, kv_len, R, Hq, Hkv, d, scale, got, ws)
    maps = ops.KVTensorMaps(KD, VD)
    if Hq == Hkv:
        ops.tree_attn_tc(q, maps, 0, kv_len, R, Hq, d, scale, None, 0, want, ws, causal=True)
    else:
        ops.tree_attn_tc_gqa(q, maps, 0, kv_len, R, Hq, Hkv, d, scale, None, 0, want, ws, causal=True)
    torch.cuda.synchronize()
    assert torch.isfinite(want).all()
    assert torch.equal(got, want), (got.float() - want.float()).abs().max().item()
    # the rows near the exponent -32 / 8 keys did see them: the store holds both kinds below kv_len
    assert (st.k_exp[0, :, :kv_len] == 8).any() and (st.k_exp[0, :, :kv_len] == -32).any()


# ---------------------------------------------------------------------------------------------------------------------
# LlamaModel.extend
# ---------------------------------------------------------------------------------------------------------------------
def _two_layer(name, seed=11):
    if name == "llama-7B-128K":
        return production_model(name, seed=seed)
    cfg = dataclasses.replace(named_config(name), num_hidden_layers=2)
    return cfg, cuda_state_dict(cfg, seed=seed, lm_head_std=0.01)


@pytest.mark.parametrize("name", ["llama-7B-128K", "llama-7B-gqa8-128K"])
@torch.inference_mode()
def test_extend_after_prefill_is_the_longer_prefill_fp16(name):
    cfg, sd = _two_layer(name)
    A, Bn = 8192, 300  # the 300 rows: pieces of 128, 128 (wgmma causal) and 44 (wgmma causal, > 32 rows)
    model = LlamaModel(cfg, sd, device=DEV)
    ids = numpy_prompt(A + Bn + 17, seed=4).cuda()[0]
    one, two = FlashSimpleCache(model, A + Bn + 64), FlashSimpleCache(model, A + Bn + 64)
    want = model.prefill(ids[:A + Bn], one)
    model.prefill(ids[:A], two)
    got = model.extend(ids[A:A + Bn], two)
    assert one.seq_len == two.seq_len == A + Bn
    assert got.shape == (1, 1, cfg.vocab_size)
    assert torch.equal(got, want[:, -1:]), (got - want[:, -1:]).abs().max().item()
    assert torch.equal(one.key_store, two.key_store) and torch.equal(one.value_store, two.value_store)
    # and a short append (17 rows: the verify attention) is forward_target's
    q = torch.empty((2, cfg.num_attention_heads, cfg.head_dim), dtype=torch.float16, device=DEV)
    got = model.extend(ids[A + Bn:], two, queries=q)
    want = model.forward_target(ids[A + Bn:], one)[:, -1:]
    assert torch.equal(got, want) and torch.equal(one.key_store, two.key_store)
    assert q.abs().sum() > 0


@torch.inference_mode()
def test_extend_over_e4m3_store_and_weights_against_fp64():
    cfg, sd = production_model("llama-7B-128K", seed=11)
    sdD = d_state_dict(cfg, sd)
    A, Bn = 16001, 300
    slots = A + Bn + 64
    model = LlamaModel(cfg, sd, device=DEV, weight_dtype="e4m3")
    kv = FlashSimpleCache(model, slots, kv_dtype="e4m3")
    ids = numpy_prompt(A + Bn, seed=6).cuda()[0]
    model.prefill(ids[:A], kv)
    got = model.extend(ids[A:], kv)
    assert kv.seq_len == A + Bn
    # the reference: weights D, the engine's prefix rows as D, the new rows' K / V rounded through the E4M3 format
    ref = Reference(cfg, sdD, slots)
    for l in range(2):
        ref.K[l][:, :A] = eo.dequantize(kv.e4m3.k_codes[l, :, :A], kv.e4m3.k_exp[l, :, :A]).to(DEV)
        ref.V[l][:, :A] = eo.dequantize(kv.e4m3.v_codes[l, :, :A], kv.e4m3.v_exp[l, :, :A]).to(DEV)
    pos = torch.arange(A, A + Bn, device=DEV)

    def attend(limit):
        def f(l, q, k, v):
            ref.K[l][:, A:A + Bn] = eo.roundtrip(k).to(DEV).transpose(0, 1)
            ref.V[l][:, A:A + Bn] = eo.roundtrip(v).to(DEV).transpose(0, 1)
            return attention_ref(q, ref.K[l], ref.V[l], limit, ref.scale)
        return f

    mutants = [("RoPE positions from 0", ref.forward(ids[A:], pos - A, attend(pos))[-1:])]
    want = ref.forward(ids[A:], pos, attend(pos))[-1:]
    check_logits("extend over an E4M3 store and E4M3 weights", got[0], want, mutants)


# ---------------------------------------------------------------------------------------------------------------------
# RetrievalCache.reselect
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", ["fp16", "e4m3"])
@torch.inference_mode()
def test_reselect_is_the_oracle_selection_at_the_new_boundary(fmt):
    cfg, sd = _two_layer("llama-7B-128K")
    P, budget, c, extra = 8192, 4096, 8, 1031
    model = LlamaModel(cfg, sd, device=DEV)
    kv = FlashSimpleCache(model, P + extra + 64, kv_dtype=fmt)
    gc = RetrievalCache(model, max_budget=budget, prefill=P, chunk_size=c, gamma=6, kv_dtype=fmt, max_context=P + extra + 64)
    ids = numpy_prompt(P + extra, seed=9).cuda()[0]
    model.prefill(ids[:P - 1], kv)
    model.forward_target(ids[P - 1:P], kv, gc)
    q = torch.empty((2, cfg.num_attention_heads, cfg.head_dim), dtype=torch.float16, device=DEV)
    model.extend(ids[P:], kv, queries=q)
    n = kv.seq_len
    B = gc.reselect(kv, q)
    assert B == n // c * c and gc.prefill == B and gc.chunk_scores.shape == (2, cfg.num_key_value_heads, B // c)
    for l in range(2):
        if fmt == "e4m3":
            K = eo.dequantize(kv.e4m3.k_codes[l, :, :n], kv.e4m3.k_exp[l, :, :n])
            V = eo.dequantize(kv.e4m3.v_codes[l, :, :n], kv.e4m3.v_exp[l, :, :n])
        else:
            K, V = kv.key_store[l, :, :n].cpu(), kv.value_store[l, :, :n].cpu()
        Kn, Vn = K.permute(1, 0, 2).numpy(), V.permute(1, 0, 2).numpy()
        _, _, idx, scores = orc.retrieval_build(Kn, Vn, q[l].cpu().numpy(), B, c, budget)
        assert np.array_equal(gc.topk_idx[l].cpu().numpy(), idx), f"layer {l}: selection differs from the oracle"
        assert np.array_equal(gc.chunk_scores[l].cpu().numpy(), scores), f"layer {l}: chunk scores differ from the oracle"
        # the budget tail holds the rows past the boundary (D of them, in the E4M3 cache's format)
        t = n - B
        assert t > 0
        if fmt == "e4m3":
            got_k = eo.dequantize(gc.e4m3.k_codes[l, :, budget - t:budget], gc.e4m3.k_exp[l, :, budget - t:budget])
        else:
            got_k = gc.key_store[l, :, budget - t:budget].cpu()
        assert torch.equal(got_k, K[:, B:n])


# ---------------------------------------------------------------------------------------------------------------------
# Session
# ---------------------------------------------------------------------------------------------------------------------
def _engine(target, draft, P, slots, budget=4096, gamma=6, kv="fp16", retrieval="fp16", temperature=0.0, chunk=8):
    cache = FlashSimpleCache(target, slots, kv_dtype=kv)
    graph_cache = RetrievalCache(target, max_budget=budget, prefill=P, gamma=gamma, chunk_size=chunk, kv_dtype=retrieval,
                                 max_context=slots // chunk * chunk)
    draft_cache = StreamingLLMEvictionCache(draft, start_size=16, recent_size=256 - 16 - gamma, gamma=gamma)
    ge = GraphInferenceEngine(target, cache, graph_cache, draft, draft_cache)
    ge.initialize_cuda_graph(gamma, probs=True, temperature=temperature, top_p=0.9)
    return ge


LOSSLESS = [("llama-7B-128K", "fp16", "fp16", "fp16"), ("llama-7B-128K", "e4m3", "e4m3", "e4m3"),
            ("llama-7B-gqa8-128K", "fp16", "fp16", "fp16")]


@pytest.mark.parametrize("name,kv,weights,retrieval", LOSSLESS, ids=[f"{a}-kv_{b}-w_{c}-r_{d}" for a, b, c, d in LOSSLESS])
@torch.inference_mode()
def test_second_turn_at_temperature_zero_is_the_targets_greedy_continuation(name, kv, weights, retrieval):
    P, Q, gen, gamma = 16384, 200, 48, 6
    cfg_t = dataclasses.replace(named_config(name), num_hidden_layers=2)
    cfg_d = named_config("llama-68M")
    tsd, dsd = agreement_state_dicts(cfg_t, cfg_d, 0.01, 0.01, seed=0, device=DEV)
    target = LlamaModel(cfg_t, tsd, device=DEV, weight_dtype=weights)
    draft = LlamaModel(cfg_d, dsd, device=DEV, is_draft=True)
    del tsd, dsd
    ge = _engine(target, draft, P, P + Q + 4 * gen + 64, kv=kv, retrieval=retrieval, gamma=gamma)
    ids = numpy_prompt(P + Q, seed=5).cuda()[0]
    s = Session(ge, gamma=gamma, tokenizer=TOK)
    s.prefill(ids[:P])
    s.generate(gen, temperature=0.0)
    s.append(ids[P:])
    L2 = s.length
    first_row = s._logits[0, -1].float().clone()
    tri = s.generate(gen, temperature=0.0)
    run = s.last_run
    tps = (len(tri) - 1) / len(run.acc_rate_middle_list)
    # the target alone from the same state: one-row decode steps after the appended rows
    s.truncate(L2)
    expo = torch.ones(cfg_t.vocab_size, device=DEV)
    rows, ar = [first_row], [int(torch.argmax(first_row))]
    for _ in range(gen + 8):
        row = ge.decode_step(torch.tensor([[ar[-1]]], device=DEV))[0, -1].float()
        rows.append(row)
        ar.append(int(ops.sample_argmax(norm_logits(row[None], temperature=0.0, top_k=-1, top_p=0.9), expo)))
    what = f"{name} kv={kv} weights={weights} retrieval={retrieval}, turn 2"
    print(f"{what}: {tps:.2f} tokens per step, accepted {run.accepted_count} of {run.draft_count}")
    compare_to_greedy(tri, ar, torch.stack(rows), 32, what, near_tie=NEAR_TIE_E4M3_STORE if kv == "e4m3" else NEAR_TIE)
    if kv == "fp16" and weights == "fp16":
        assert tps > 1.0 and run.accepted_count > 0


TINY = dict(target="tiny-yarn-target", draft="llama-68M", target_seed=1, draft_seed=2, prompt_seed=3, prefill=512, budget=64,
            chunk=8, gamma=4)


def _tiny_engine(temperature=0.6):
    ts, ds = named_config(TINY["target"]), named_config(TINY["draft"])
    target = LlamaModel(ts, numpy_state_dict(ts, TINY["target_seed"]), device=DEV)
    draft = LlamaModel(ds, numpy_state_dict(ds, TINY["draft_seed"]), device=DEV, is_draft=True)
    return _engine(target, draft, TINY["prefill"], TINY["prefill"] + 1024, budget=TINY["budget"], gamma=TINY["gamma"],
                   temperature=temperature)


@torch.inference_mode()
def test_truncate_and_the_same_turn_again_repeat_it():
    ge = _tiny_engine()
    ids = numpy_prompt(TINY["prefill"] + 300, seed=3).cuda()[0]
    s = Session(ge, gamma=TINY["gamma"], tokenizer=TOK)
    s.prefill(ids[:TINY["prefill"]])
    s.generate(24, seed=1)
    n0 = s.length
    turns = []
    for _ in range(2):
        s.truncate(n0)
        s.append(ids[TINY["prefill"]:])
        toks = s.generate(40, seed=7)
        r = s.last_run
        turns.append((toks, r.accepted_count, r.draft_count, r.resample_count, s.length))
    assert turns[0] == turns[1]
    assert turns[0][1] > 0
    print(f"rollback: {len(turns[0][0])} tokens, accepted {turns[0][1]} of {turns[0][2]}, identical twice")


@torch.inference_mode()
def test_device_loop_equals_step_wise_loop_over_two_turns():
    ids = numpy_prompt(TINY["prefill"] + 200, seed=3).cuda()[0]
    out = []
    for device_loop in (False, True):
        ge = _tiny_engine()
        s = Session(ge, gamma=TINY["gamma"], tokenizer=TOK, pad_full_verify=True)
        s.prefill(ids[:TINY["prefill"]])
        t1 = s.generate(20, seed=5, device_loop=device_loop)
        s.append(ids[TINY["prefill"]:])
        t2 = s.generate(30, seed=6, device_loop=device_loop)
        out.append((t1, t2, s.length, list(s.ids)))
        del s, ge
    assert out[0] == out[1]
    print(f"two turns: {len(out[0][0])} + {len(out[0][1])} tokens, identical on both loops")


@torch.inference_mode()
def test_first_turn_replays_the_reference_trace(golden_dir):
    from e2e_util import build_engine
    rec = json.load(open(os.path.join(golden_dir, "e2e_tiny.json")))
    case = rec["case"]
    ge = build_engine(case, graphs=True)
    ids = numpy_prompt(case["prefill"], seed=case["prompt_seed"]).cuda()
    trace = []
    s = Session(ge, gamma=case["gamma"], tokenizer=TOK, trace=trace)
    s.prefill(ids)
    s.generate(case["gen_len"], temperature=case["temperature"], top_p=case["top_p"], noise=CounterNoise(case["noise_seed"]))
    want = rec["calls"][0]["trace"]
    same = matching_prefix(trace, want)
    assert same == len(want) == len(trace), f"leaves the reference after {same} of {len(want)} events"
    assert abs(s.last_run.acceptance_rate - rec["calls"][0]["acceptance_rate"]) < 1e-9
    assert s.length == case["prefill"] + len(s.last_run.generated) - 1
