"""The E4M3 retrieval cache in the engine.

* The target does not read the retrieval cache outside the retrieval verify: two-layer 7B-wide targets (cfg2, and
  llama-7B-gqa8-128K) on a 16K-token prompt give bit-identical prefill, full-verify and decode logits with an fp16 and with an
  E4M3 retrieval cache, on fp16 and E4M3 stores and weights.  The E4M3 cache holds the quantized selection (fp16 store) or the
  store's own codes (E4M3 store).  Retrieval-verify logits are finite; their difference from the fp16 cache is printed.
* The whole-loop device graph equals the step-wise loop on the same Philox stream, on the tiny and gamma = 16 golden cases and
  on the TP engine at world 1 (and 2 where two GPUs exist).
* Losslessness: the first token the whole-loop graph emits, over many runs from one committed state with fresh noise, is
  distributed as the target's p (chi-square with tokens binned by p, as in test_sampling_loop_gpu.py)."""
import dataclasses
import json
import os

import numpy as np
import pytest
import torch

import kv_e4m3_oracle as eo
from attn_needles import report_time_and_memory  # noqa: F401  (autouse fixture: wall time and peak memory per test)
from e2e_util import TokenizerStub
from test_model_production_gpu import production_model
from chi2_util import chi2, chi2_threshold
from test_tp_gpu import _run
from triforce_b200.cache import FlashSimpleCache, RetrievalCache, StreamingLLMEvictionCache
from triforce_b200.config import named_config
from triforce_b200.decoding import TriForceRun
from triforce_b200.device_loop import DeviceLoop, DeviceLoopRun, PhiloxNoise
from triforce_b200.engine import GraphInferenceEngine
from triforce_b200.llama import LlamaModel
from triforce_b200.sampling import norm_logits
from triforce_b200.synth import cuda_state_dict, numpy_prompt, numpy_state_dict

pytestmark = pytest.mark.gpu
DEV = "cuda"
REPO = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
P, B, CHUNK, GAMMA = 16384, 4096, 8, 6


def dequant(codes, e):
    return (codes.view(torch.float8_e4m3fn).double() * torch.exp2(e.double()).unsqueeze(-1)).half()


def engine(cfg, sd, kv_dtype, weight_dtype, retrieval_dtype):
    target = LlamaModel(cfg, sd, device=DEV, weight_dtype=weight_dtype)
    ds = named_config("llama-68M")
    draft = LlamaModel(ds, numpy_state_dict(ds, 3), device=DEV, is_draft=True)
    cache = FlashSimpleCache(target, P + 64, kv_dtype=kv_dtype)
    graph_cache = RetrievalCache(target, max_budget=B, prefill=P, gamma=GAMMA, chunk_size=CHUNK, kv_dtype=retrieval_dtype)
    draft_cache = StreamingLLMEvictionCache(draft, start_size=16, recent_size=256 - 16 - GAMMA, gamma=GAMMA)
    ge = GraphInferenceEngine(target, cache, graph_cache, draft, draft_cache)
    ge.initialize_cuda_graph(GAMMA, probs=False)
    return ge


@pytest.mark.parametrize("name,kv,weights", [
    ("llama-7B-128K", "fp16", "fp16"),
    ("llama-7B-128K", "e4m3", "fp16"),
    ("llama-7B-128K", "fp16", "e4m3"),
    ("llama-7B-gqa8-128K", "fp16", "fp16"),
    ("llama-7B-gqa8-128K", "e4m3", "e4m3"),
])
def test_target_logits_do_not_depend_on_the_retrieval_cache(name, kv, weights):
    if name == "llama-7B-128K":
        cfg, sd = production_model(name, seed=11)
    else:
        cfg = dataclasses.replace(named_config(name), num_hidden_layers=2)
        sd = cuda_state_dict(cfg, seed=11, lm_head_std=0.01)
    ids = numpy_prompt(P + 16, seed=5).cuda()
    g16, g8 = engine(cfg, sd, kv, weights, "fp16"), engine(cfg, sd, kv, weights, "e4m3")
    kv16, kv8 = g16.engine.kv_cache, g8.engine.kv_cache
    gc16, gc8 = g16.engine.graph_cache, g8.engine.graph_cache
    assert gc8.kv_dtype == "e4m3" and gc8.slots % 64 == 0 and gc8.slots >= gc8.real_budget

    assert torch.equal(g16.engine.model_run(ids[:, :P - 1]), g8.engine.model_run(ids[:, :P - 1]))
    # the last prompt token builds the retrieval caches: same logits, same selection
    assert torch.equal(g16.engine.model_run(ids[:, P - 1:P]), g8.engine.model_run(ids[:, P - 1:P]))
    assert torch.equal(gc16.topk_idx, gc8.topk_idx) and torch.equal(gc16.chunk_scores.view(torch.int16), gc8.chunk_scores.view(torch.int16))
    for l in range(cfg.num_hidden_layers):
        if kv == "fp16":  # the oracle's quantization of the rows the fp16 cache holds
            for rows, codes, ex in ((gc16.key_store, gc8.e4m3.k_codes, gc8.e4m3.k_exp), (gc16.value_store, gc8.e4m3.v_codes, gc8.e4m3.v_exp)):
                want_c, want_e = eo.quantize(rows[l, :, :B].cpu())
                assert torch.equal(codes[l, :, :B].cpu(), want_c) and torch.equal(ex[l, :, :B].cpu(), want_e)
        else:  # the store's codes: D equals what the fp16 cache received
            assert torch.equal(dequant(gc8.e4m3.k_codes[l, :, :B], gc8.e4m3.k_exp[l, :, :B]), gc16.key_store[l, :, :B])
            assert torch.equal(dequant(gc8.e4m3.v_codes[l, :, :B], gc8.e4m3.v_exp[l, :, :B]), gc16.value_store[l, :, :B])

    pos = torch.arange(P, P + GAMMA + 1, device=DEV).unsqueeze(0)
    r16, r8 = g16.graph_verify(ids[:, :GAMMA + 1], pos), g8.graph_verify(ids[:, :GAMMA + 1], pos)
    assert bool(torch.isfinite(r8).all())
    rms = r16.double().pow(2).mean().sqrt().item()
    print(f"{name} kv={kv} weights={weights}: retrieval verify, fp16 vs e4m3 cache: max |dlogit| / logit RMS "
          f"{(r8.double() - r16.double()).abs().max().item() / rms:.4f}, top-1 agree on "
          f"{int((r8.argmax(-1) == r16.argmax(-1)).sum())} of {GAMMA + 1} rows")
    assert torch.equal(g16.inference(ids[:, P:P + GAMMA + 1]), g8.inference(ids[:, P:P + GAMMA + 1]))
    assert torch.equal(g16.decode_step(ids[:, P + GAMMA + 1:P + GAMMA + 2]), g8.decode_step(ids[:, P + GAMMA + 1:P + GAMMA + 2]))
    assert kv8.seq_len == kv16.seq_len == P + GAMMA + 2

    # the tail copy: the E4M3 cache holds the quantized (fp16 store) or copied (E4M3 store) rows the fp16 cache holds as fp16
    g16.update_graph_cache()
    g8.update_graph_cache()
    n = kv8.seq_len - P
    torch.cuda.synchronize()
    if kv == "fp16":
        want_c, want_e = eo.quantize(gc16.key_store[:, :, B - n:B].cpu())
        assert torch.equal(gc8.e4m3.k_codes[:, :, B - n:B].cpu(), want_c) and torch.equal(gc8.e4m3.k_exp[:, :, B - n:B].cpu(), want_e)
    else:
        assert torch.equal(gc8.e4m3.v_codes[:, :, B - n:B], kv8.e4m3.v_codes[:, :, P:P + n])
        assert torch.equal(gc8.e4m3.k_exp[:, :, B - n:B], kv8.e4m3.k_exp[:, :, P:P + n])


# ---------------------------------------------------------------------------------------------------------------------
# the whole-loop graph
# ---------------------------------------------------------------------------------------------------------------------
def _case(name):
    return json.load(open(os.path.join(REPO, "tests", "golden", f"e2e_{name}.json")))["case"]


def build_engine(case, retrieval_dtype="e4m3"):
    """tests/e2e_util.build_engine with the retrieval cache's format as a parameter."""
    ts, ds = named_config(case["target"]), named_config(case["draft"])
    target = LlamaModel(ts, numpy_state_dict(ts, case["target_seed"]), device=DEV)
    draft = LlamaModel(ds, numpy_state_dict(ds, case["draft_seed"]), device=DEV, is_draft=True)
    Pc, Bc, c, g = case["prefill"], case["budget"], case["chunk"], case["gamma"]
    cache = FlashSimpleCache(target, Pc + case.get("gen_len", 16) + 32)
    graph_cache = RetrievalCache(target, max_budget=Bc, prefill=Pc, gamma=g, chunk_size=c, kv_dtype=retrieval_dtype)
    draft_cache = StreamingLLMEvictionCache(draft, start_size=16, recent_size=256 - 16 - g, gamma=g)
    ge = GraphInferenceEngine(target, cache, graph_cache, draft, draft_cache)
    ge.initialize_cuda_graph(g, probs=True, temperature=case["temperature"], top_p=case["top_p"])
    return ge


def _steps(loop, gen):
    steps = []
    while loop.n < gen:
        before = len(loop.generated)
        loop.step()
        steps.append(loop.generated[before:])
    return steps


@pytest.mark.parametrize("name,seed", [("tiny", 3), ("g16", 7)])
def test_device_loop_matches_the_step_wise_loop(name, seed):
    case = _case(name)
    ids = numpy_prompt(case["prefill"], seed=case["prompt_seed"]).cuda()
    gen = min(case["gen_len"], 32)
    tok = TokenizerStub()
    kw = dict(gamma=case["gamma"], top_p=case["top_p"], temperature=case["temperature"])
    ge = build_engine(case)
    host = TriForceRun(tok, ge, noise=PhiloxNoise(torch.device("cuda"), seed), pad_full_verify=True, **kw)
    host.prefill(ids)
    host_steps = _steps(host, gen)
    host_tokens, host_len = list(host.generated), ge.engine.kv_cache.seq_len
    counts = host.accepted_count, host.draft_count, host.inner_iterations
    del host
    ge = build_engine(case)  # a fresh engine: both loops see a first prompt
    dev = DeviceLoopRun(tok, ge, seed=seed, **kw)
    dev.prefill(ids)
    dev_steps = _steps(dev, gen)
    assert dev.generated == host_tokens, (dev_steps[:6], host_steps[:6])
    assert dev_steps == host_steps
    assert ge.engine.kv_cache.seq_len == host_len
    assert (dev.accepted_count, dev.draft_count, dev.inner_iterations) == counts
    assert ge.engine.graph_cache.kv_dtype == "e4m3" and counts[1] > 0
    print(f"{name}, seed {seed}: {len(host_tokens)} tokens, accepted {counts[0]} of {counts[1]}, {counts[2]} inner iterations: identical")


@pytest.mark.parametrize("world", [1, 2])
def test_device_loop_on_the_tp_engine(world):
    if world > torch.cuda.device_count():
        pytest.skip(f"needs {world} GPUs")
    got = _run(world, "tiny", extra=("--device_loop", 3, "--retrieval_dtype", "e4m3"))
    assert got["identical"], (got["host"]["steps"][:6], got["device"]["steps"][:6])
    assert len(got["device"]["tokens"]) >= 16


def test_first_emitted_token_is_distributed_as_the_target():
    """Many whole-loop launches from one committed state (prompt + first token), each on a fresh Philox stream: the first token
    of every launch must follow the target's p at that position, whatever the E4M3 retrieval level proposed."""
    case = _case("tiny")
    ge = build_engine(case)
    eng = ge.engine
    kv, gc, dc = eng.kv_cache, eng.graph_cache, eng.draft_cache
    ids = numpy_prompt(case["prefill"], seed=case["prompt_seed"]).cuda()
    run = DeviceLoopRun(TokenizerStub(), ge, gamma=case["gamma"], top_p=case["top_p"], temperature=case["temperature"], seed=1)
    t0 = run.prefill(ids)
    loop: DeviceLoop = run.loop
    P0 = kv.seq_len
    with torch.inference_mode():
        logits = eng.model.forward_target(torch.tensor([[t0]], device=DEV), kv, None, None)
        p = norm_logits(logits[0], temperature=case["temperature"], top_k=-1, top_p=case["top_p"])[0].double().cpu().numpy()
        p_t1 = norm_logits(logits[0], temperature=1.0, top_k=-1, top_p=case["top_p"])[0].double().cpu().numpy()  # the power control
    state = [dc.key_store, dc.value_store, gc.e4m3.k_codes, gc.e4m3.v_codes, gc.e4m3.k_exp, gc.e4m3.v_exp]
    saved = [t.clone() for t in state]
    V = p.size
    counts = np.zeros(V, dtype=np.int64)
    N = 20000
    for trial in range(N):
        for t, s in zip(state, saved):
            t.copy_(s)
        kv.seq_len, kv._dev_mirror = P0, -1
        kv.sync_seq_len_to_device()
        loop.rng.copy_(torch.tensor([1000 + trial, 0], dtype=torch.int64))
        loop.set_first_token(t0)
        loop.launch()
        r, toks = loop.read()
        counts[toks[0]] += 1
    assert counts[p == 0].sum() == 0, np.flatnonzero((p == 0) & (counts > 0))[:10]
    stat, df = chi2(counts, p)
    stat_c, df_c = chi2(counts, p_t1)
    print(f"\n[lossless, e4m3 retrieval cache] {N} launches: chi2 vs p {stat:.1f} (df {df}, 1e-6 threshold {chi2_threshold(df):.1f}); "
          f"vs p at temperature 1 {stat_c:.1f} (df {df_c}, threshold {chi2_threshold(df_c):.1f})")
    assert stat < chi2_threshold(df)
    assert stat_c > chi2_threshold(df_c)
