"""Model-level runs with E4M3 projection weights.  An E4M3-weight target is compared with an fp16 target built from the state
dict of D = code * 2^e: since tf_stream_linear_e4m3 is bit-identical to tf_stream_linear on D and the > 24-row GEMMs run on D,
every logit, every KV row and every sampled token must agree bit for bit.

* Two-layer 7B-wide targets (cfg2's production inputs, and llama-7B-gqa8-128K), each on an fp16 and on an E4M3 full-KV store,
  with an 8K prompt through GraphInferenceEngine: the prefill (layer-major for E4M3 weights; chunk-major for the fp16 target
  on an fp16 store), the stores after it, the last prompt token with the retrieval build, a retrieval verify, a full-KV verify
  and a decode step through the graphs.
* The whole-loop device graph on the tiny and gamma = 16 parity models emits the same tokens, splits and counts.
* The E4M3-weight target holds no fp16 projection weights, and its weights take about half the memory."""
import dataclasses
import json
import os

import pytest
import torch

from attn_needles import report_time_and_memory  # noqa: F401  (autouse fixture: wall time and peak memory per test)
from e2e_util import TokenizerStub
from test_model_production_gpu import production_model
from triforce_b200 import ops
from triforce_b200.cache import FlashSimpleCache, RetrievalCache, StreamingLLMEvictionCache
from triforce_b200.config import LlamaShape, named_config
from triforce_b200.device_loop import DeviceLoopRun
from triforce_b200.engine import GraphInferenceEngine
from triforce_b200.llama import LlamaModel
from triforce_b200.synth import cuda_state_dict, numpy_prompt, numpy_state_dict

pytestmark = pytest.mark.gpu
DEV = "cuda"
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P, B, CHUNK, GAMMA = 8192, 4096, 8, 6
SLOTS = P + 64
PROJ = ("self_attn.q_proj", "self_attn.k_proj", "self_attn.v_proj", "self_attn.o_proj", "mlp.gate_proj", "mlp.up_proj", "mlp.down_proj")


def proj_keys(cfg):
    return [f"model.layers.{l}.{p}.weight" for l in range(cfg.num_hidden_layers) for p in PROJ] + ["lm_head.weight"]


def d_state_dict(cfg, sd):
    """The state dict whose projection weights are D of the E4M3 format (the rule is per row, so quantizing q, k, v apart or
    fused gives the same D)."""
    out = dict(sd)
    for k in proj_keys(cfg):
        w = sd[k].to(device=DEV, dtype=torch.float16).contiguous()
        codes, e = ops.weight_quantize_e4m3(w)
        out[k] = ops.weight_dequantize_e4m3(codes, e).to(sd[k].device)
    return out


def make_engine(target, kv_dtype, draft_seed=3, gamma=GAMMA, prefill=P, budget=B, slots=SLOTS, chunk=CHUNK, probs=False,
                temperature=0.6, top_p=0.9, draft_budget=256):
    ds = named_config("llama-68M")
    draft = LlamaModel(ds, numpy_state_dict(ds, draft_seed), device=DEV, is_draft=True)
    cache = FlashSimpleCache(target, slots, kv_dtype=kv_dtype)
    graph_cache = RetrievalCache(target, max_budget=budget, prefill=prefill, gamma=gamma, chunk_size=chunk)
    draft_cache = StreamingLLMEvictionCache(draft, start_size=16, recent_size=draft_budget - 16 - gamma, gamma=gamma)
    ge = GraphInferenceEngine(target, cache, graph_cache, draft, draft_cache)
    ge.initialize_cuda_graph(gamma, probs=probs, temperature=temperature, top_p=top_p)
    return ge


def check_no_fp16_projections(model):
    assert model.weight_dtype == "e4m3" and model.lm_head is None and isinstance(model.m_lm_head, ops.E4m3WeightMap)
    for w in model.layers:
        assert w.wqkv is None and w.wo is None and w.wgu is None and w.wd is None
        for m in (w.m_qkv, w.m_o, w.m_gu, w.m_d):
            assert isinstance(m, ops.E4m3WeightMap) and m.codes.dtype == torch.uint8


def model_pair(name):
    if name == "llama-7B-128K":
        cfg, sd = production_model(name, seed=11)
    else:
        cfg = dataclasses.replace(named_config(name), num_hidden_layers=2)
        sd = cuda_state_dict(cfg, seed=11, lm_head_std=0.01)
    sd = {k: v.cpu() for k, v in sd.items()}  # host copies: each model's device memory is its own
    sdD = d_state_dict(cfg, sd)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    m16 = LlamaModel(cfg, sdD, device=DEV)
    torch.cuda.synchronize()
    bytes16 = torch.cuda.memory_allocated() - base
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    m8 = LlamaModel(cfg, sd, device=DEV, weight_dtype="e4m3")
    torch.cuda.synchronize()
    bytes8 = torch.cuda.memory_allocated() - base
    check_no_fp16_projections(m8)
    fp16_proj = sum(sd[k].numel() * 2 for k in proj_keys(cfg))
    e4m3_proj = sum(sd[k].numel() + sd[k].shape[0] for k in proj_keys(cfg))
    saved = bytes16 - bytes8
    print(f"{name}: model bytes fp16 {bytes16 / 2**30:.3f} GiB, e4m3 {bytes8 / 2**30:.3f} GiB, saved {saved / 2**30:.3f} GiB "
          f"(projection bytes {fp16_proj / 2**30:.3f} -> {e4m3_proj / 2**30:.3f} GiB)")
    assert abs(saved - (fp16_proj - e4m3_proj)) < 0.02 * fp16_proj
    return cfg, m16, m8


def assert_bits(a, b, what):
    assert torch.equal(a, b), f"{what}: max |diff| {(a.double() - b.double()).abs().max().item()}"


@pytest.mark.parametrize("kv_dtype", ["fp16", "e4m3"])
@pytest.mark.parametrize("name", ["llama-7B-128K", "llama-7B-gqa8-128K"])
@torch.inference_mode()
def test_e4m3_weights_against_fp16_on_d(name, kv_dtype):
    cfg, m16, m8 = model_pair(name)
    ids = numpy_prompt(P + 16, seed=5).cuda()
    g16, g8 = make_engine(m16, kv_dtype), make_engine(m8, kv_dtype)
    kv16, kv8 = g16.engine.kv_cache, g8.engine.kv_cache

    # prefill: layer-major on the E4M3-weight side (one dequantization per layer), the fp16 engine's own path on the other
    l16 = g16.engine.model_run(ids[:, :P - 1])
    l8 = g8.engine.model_run(ids[:, :P - 1])
    assert kv8.seq_len == kv16.seq_len == P - 1
    assert_bits(l16, l8, "prefill logits")
    if kv_dtype == "fp16":
        assert torch.equal(kv16.key_store, kv8.key_store) and torch.equal(kv16.value_store, kv8.value_store)
    else:
        for a, b in ((kv16.e4m3.k_codes, kv8.e4m3.k_codes), (kv16.e4m3.v_codes, kv8.e4m3.v_codes),
                     (kv16.e4m3.k_exp, kv8.e4m3.k_exp), (kv16.e4m3.v_exp, kv8.e4m3.v_exp)):
            assert torch.equal(a, b)

    # the last prompt token with the retrieval build
    last = ids[:, P - 1:P]
    assert_bits(g16.engine.model_run(last), g8.engine.model_run(last), "retrieval-build step logits")
    gc16, gc8 = g16.engine.graph_cache, g8.engine.graph_cache
    assert torch.equal(gc16.key_store, gc8.key_store) and torch.equal(gc16.value_store, gc8.value_store)

    # retrieval verify, full-KV verify and decode step through the graphs
    pos = torch.arange(P, P + GAMMA + 1, device=DEV).unsqueeze(0)
    assert_bits(g16.graph_verify(ids[:, :GAMMA + 1], pos), g8.graph_verify(ids[:, :GAMMA + 1], pos), "retrieval verify")
    assert_bits(g16.inference(ids[:, P:P + GAMMA + 1]), g8.inference(ids[:, P:P + GAMMA + 1]), "full-KV verify")
    tok = ids[:, P + GAMMA + 1:P + GAMMA + 2]
    assert_bits(g16.decode_step(tok), g8.decode_step(tok), "decode step")
    assert kv8.seq_len == kv16.seq_len == P + GAMMA + 2
    # an eager forward of more than 24 rows runs cuBLAS on the one-layer D scratch
    rows = ids[:, P + 8:P + 48]
    assert_bits(g16.engine.model(input_ids=rows, kv_cache=kv16, graph_cache=None).logits,
                g8.engine.model(input_ids=rows, kv_cache=kv8, graph_cache=None).logits, "40-row full-KV forward")


def _case(name):
    return json.load(open(os.path.join(REPO, "tests", "golden", f"e2e_{name}.json")))["case"]


@pytest.mark.parametrize("name,seed", [("tiny", 3), ("g16", 7)])
@torch.inference_mode()
def test_device_loop_with_e4m3_weights_matches_fp16_on_d(name, seed):
    case = _case(name)
    ts = named_config(case["target"])
    sd = numpy_state_dict(ts, case["target_seed"])
    sdD = d_state_dict(ts, sd)
    ids = numpy_prompt(case["prefill"], seed=case["prompt_seed"]).cuda()
    gen = min(case["gen_len"], 32)
    P_, g = case["prefill"], case["gamma"]
    results = []
    for target in (LlamaModel(ts, sdD, device=DEV), LlamaModel(ts, sd, device=DEV, weight_dtype="e4m3")):
        ge = make_engine(target, "fp16", draft_seed=case["draft_seed"], gamma=g, prefill=P_, budget=case["budget"],
                         slots=P_ + case.get("gen_len", 16) + 32, chunk=case["chunk"], probs=True, temperature=case["temperature"],
                         top_p=case["top_p"])
        dev = DeviceLoopRun(TokenizerStub(), ge, gamma=g, top_p=case["top_p"], temperature=case["temperature"], seed=seed)
        dev.prefill(ids)
        steps = []
        while dev.n < gen:
            before = len(dev.generated)
            dev.step()
            steps.append(dev.generated[before:])
        results.append((list(dev.generated), steps, ge.engine.kv_cache.seq_len, dev.accepted_count, dev.draft_count,
                        dev.inner_iterations))
        del dev, ge
    assert results[0] == results[1], (results[0][1][:6], results[1][1][:6])
    print(f"{name}, seed {seed}: {len(results[0][0])} tokens in {len(results[0][1])} outer steps, accepted {results[0][3]} of "
          f"{results[0][4]}: identical")


def test_projection_k_not_a_multiple_of_64_is_refused():
    ts = LlamaShape(hidden_size=256, intermediate_size=1000, num_hidden_layers=1, num_attention_heads=4, num_key_value_heads=4,
                    vocab_size=512, max_position_embeddings=2048, rms_norm_eps=1e-6, name="k1000")
    sd = numpy_state_dict(ts, 1)
    with pytest.raises(ValueError, match="multiple of 64"):
        LlamaModel(ts, sd, device=DEV, weight_dtype="e4m3")
    w = torch.ones((16, 96), dtype=torch.float16, device=DEV)
    with pytest.raises(ValueError, match="multiple of 64"):
        ops.weight_quantize_e4m3(w)
