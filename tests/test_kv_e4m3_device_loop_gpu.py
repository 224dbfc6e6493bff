"""The whole-loop graph on E4M3 full-KV stores: the device loop (one CUDA-graph launch per outer step) and the step-wise loop
on the same device Philox stream must emit the same tokens, the same tokens per step, the same final sequence length and the
same accepted / drafted / inner-iteration counts, as test_device_loop_gpu.py / test_gqa_device_loop_gpu.py require of fp16
stores.  Targets: a tiny MHA target with d = 64 (the 68M-shaped YaRN target: its prompt attention takes the library path on
the fp16 scratch layer) and the G = 4 GQA target of test_gqa_device_loop_gpu.py."""
import pytest
import torch

from attn_needles import report_time_and_memory  # noqa: F401  (autouse fixture: wall time and peak memory per test)
from e2e_util import TokenizerStub
from triforce_b200.cache import FlashSimpleCache, RetrievalCache, StreamingLLMEvictionCache
from triforce_b200.config import LlamaShape, named_config
from triforce_b200.decoding import TriForceRun
from triforce_b200.device_loop import DeviceLoopRun, PhiloxNoise
from triforce_b200.engine import GraphInferenceEngine
from triforce_b200.llama import LlamaModel
from triforce_b200.synth import numpy_prompt, numpy_state_dict

pytestmark = pytest.mark.gpu
CASE = dict(prefill=512, budget=64, chunk=8, gamma=4, gen=32, temperature=0.6, top_p=0.9)


def e4m3_engine(kind: str):
    if kind == "mha64":
        ts = LlamaShape(hidden_size=768, intermediate_size=3072, num_hidden_layers=2, num_attention_heads=12, num_key_value_heads=12,
                        vocab_size=32000, max_position_embeddings=4096, rms_norm_eps=1e-6,
                        rope_scaling={"type": "yarn", "factor": 2.0, "original_max_position_embeddings": 2048}, name="mha-d64")
    else:
        ts = LlamaShape(hidden_size=1024, intermediate_size=2048, num_hidden_layers=2, num_attention_heads=8, num_key_value_heads=2,
                        vocab_size=32000, max_position_embeddings=4096, rms_norm_eps=1e-6,
                        rope_scaling={"type": "yarn", "factor": 2.0, "original_max_position_embeddings": 2048},
                        gqa_retrieval="group_sum", name="gqa-8q2kv")
    ds = named_config("llama-68M")
    target = LlamaModel(ts, numpy_state_dict(ts, 5, lm_head_std=0.05), device="cuda")
    draft = LlamaModel(ds, numpy_state_dict(ds, 6), device="cuda", is_draft=True)
    P, B, c, g = CASE["prefill"], CASE["budget"], CASE["chunk"], CASE["gamma"]
    cache = FlashSimpleCache(target, P + CASE["gen"] + 32, kv_dtype="e4m3")
    graph_cache = RetrievalCache(target, max_budget=B, prefill=P, gamma=g, chunk_size=c)
    draft_cache = StreamingLLMEvictionCache(draft, start_size=16, recent_size=256 - 16 - g, gamma=g)
    ge = GraphInferenceEngine(target, cache, graph_cache, draft, draft_cache)
    ge.initialize_cuda_graph(g, probs=True, temperature=CASE["temperature"], top_p=CASE["top_p"])
    return ge


def run_loop(loop, gen):
    steps = []
    while loop.n < gen:
        before = len(loop.generated)
        loop.step()
        steps.append(loop.generated[before:])
    return steps


@pytest.mark.parametrize("kind,seed", [("mha64", 3), ("gqa4", 9)])
def test_e4m3_device_loop_matches_the_step_wise_loop(kind, seed):
    ids = numpy_prompt(CASE["prefill"], seed=seed).cuda()
    tok = TokenizerStub()
    kw = dict(gamma=CASE["gamma"], top_p=CASE["top_p"], temperature=CASE["temperature"])
    ge = e4m3_engine(kind)
    host = TriForceRun(tok, ge, noise=PhiloxNoise(torch.device("cuda"), seed), pad_full_verify=True, **kw)
    host.prefill(ids)
    host_steps = run_loop(host, CASE["gen"])
    host_tokens, host_len = list(host.generated), ge.engine.kv_cache.seq_len
    counts = host.accepted_count, host.draft_count, host.inner_iterations
    del host
    ge = e4m3_engine(kind)  # a fresh engine: both loops see a first prompt
    dev = DeviceLoopRun(tok, ge, seed=seed, **kw)
    dev.prefill(ids)
    dev_steps = run_loop(dev, CASE["gen"])
    assert dev.generated == host_tokens, (dev_steps[:6], host_steps[:6])
    assert dev_steps == host_steps
    assert ge.engine.kv_cache.seq_len == host_len
    assert (dev.accepted_count, dev.draft_count, dev.inner_iterations) == counts
    assert len(host_tokens) >= CASE["gen"] and counts[1] > 0
    assert ge.engine.kv_cache.kv_dtype == "e4m3"
    print(f"{kind}, seed {seed}: {len(host_tokens)} tokens in {len(dev_steps)} outer steps, accepted {counts[0]} of {counts[1]}, "
          f"{counts[2]} inner iterations: identical")
