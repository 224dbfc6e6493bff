"""Model-level runs on an E4M3 full-KV store: two-layer 7B-wide targets (cfg2, and llama-7B-gqa8-128K with 8 KV heads) run a
16K-token prompt through GraphInferenceEngine, once on an fp16 and once on an E4M3 store.

* The layer-major E4M3 prefill runs every op of the fp16 chunk-major prefill with the same shapes, so its logits must be
  bit-identical to the fp16 engine's, and its store must equal the oracle's quantization of the fp16 store bit for bit.
* Every later step reads E4M3 and runs through the engine: the last prompt token with the retrieval build (the retrieval
  store must hold D of the selected chunks, bit for bit), a retrieval verify, a full-KV verify and a decode step through the
  seq_len_dev graphs, and tail_update (which must write exactly D).  Their attention is checked against fp64 over D by
  tests/test_kv_e4m3_gpu.py.
* The fp16-vs-E4M3 logit difference is printed, not asserted: with random weights it is a weak quality signal."""
import dataclasses

import pytest
import torch

import kv_e4m3_oracle as eo
from attn_needles import report_time_and_memory  # noqa: F401  (autouse fixture: wall time and peak memory per test)
from test_model_production_gpu import production_model
from triforce_b200.cache import FlashSimpleCache, RetrievalCache, StreamingLLMEvictionCache
from triforce_b200.config import named_config
from triforce_b200.engine import GraphInferenceEngine
from triforce_b200.llama import LlamaModel
from triforce_b200.synth import cuda_state_dict, numpy_prompt, numpy_state_dict

pytestmark = pytest.mark.gpu
DEV = "cuda"
P, B, CHUNK, GAMMA = 16384, 4096, 8, 6
SLOTS = P + 64


def engine(cfg, sd, kv_dtype):
    target = LlamaModel(cfg, sd, device=DEV)
    ds = named_config("llama-68M")
    draft = LlamaModel(ds, numpy_state_dict(ds, 3), device=DEV, is_draft=True)
    cache = FlashSimpleCache(target, SLOTS, kv_dtype=kv_dtype)
    graph_cache = RetrievalCache(target, max_budget=B, prefill=P, gamma=GAMMA, chunk_size=CHUNK)
    draft_cache = StreamingLLMEvictionCache(draft, start_size=16, recent_size=256 - 16 - GAMMA, gamma=GAMMA)
    ge = GraphInferenceEngine(target, cache, graph_cache, draft, draft_cache)
    ge.initialize_cuda_graph(GAMMA, probs=False)
    return ge


def dequant(codes, e):
    return (codes.view(torch.float8_e4m3fn).double() * torch.exp2(e.double()).unsqueeze(-1)).half()


@pytest.mark.parametrize("name", ["llama-7B-128K", "llama-7B-gqa8-128K"])
def test_e4m3_engine_against_fp16(name):
    if name == "llama-7B-128K":
        cfg, sd = production_model(name, seed=11)
    else:  # the production inputs tie k_proj to q_proj per head, which needs as many KV heads as query heads
        cfg = dataclasses.replace(named_config(name), num_hidden_layers=2)
        sd = cuda_state_dict(cfg, seed=11, lm_head_std=0.01)
    ids = numpy_prompt(P + 16, seed=5).cuda()
    g16, g8 = engine(cfg, sd, "fp16"), engine(cfg, sd, "e4m3")
    kv16, kv8 = g16.engine.kv_cache, g8.engine.kv_cache
    assert kv8.slots == kv16.slots == SLOTS

    # prefill: bit-identical logits, store = oracle(fp16 store)
    l16 = g16.engine.model_run(ids[:, :P - 1])
    l8 = g8.engine.model_run(ids[:, :P - 1])
    assert kv8.seq_len == kv16.seq_len == P - 1
    assert torch.equal(l16, l8)
    for l in range(cfg.num_hidden_layers):
        for store, codes, ex in ((kv16.key_store, kv8.e4m3.k_codes, kv8.e4m3.k_exp), (kv16.value_store, kv8.e4m3.v_codes, kv8.e4m3.v_exp)):
            want_c, want_e = eo.quantize(store[l, :, :P - 1].cpu())
            assert torch.equal(codes[l, :, :P - 1].cpu(), want_c) and torch.equal(ex[l, :, :P - 1].cpu(), want_e)

    # the last prompt token with the retrieval build: the fp16 engine's logits against the e4m3 engine's (printed only), and
    # the retrieval store must hold D of the chunks the build selected
    last = ids[:, P - 1:P]
    ref16 = g16.engine.model_run(last)[0, -1]
    got = g8.engine.model_run(last)[0, -1]
    assert kv8.seq_len == P and bool(torch.isfinite(got).all())
    rms = ref16.double().pow(2).mean().sqrt().item()
    print(f"{name}: fp16 vs e4m3 store, last prompt token: max |dlogit| / logit RMS "
          f"{(got.double() - ref16.double()).abs().max().item() / rms:.4f}, top-1 agree {bool(got.argmax() == ref16.argmax())}")
    gc8 = g8.engine.graph_cache
    Hkv = kv8.num_heads
    for l in range(cfg.num_hidden_layers):
        idx = gc8.topk_idx[l].long()  # [Hkv, select_sets]
        assert bool((idx[:, 0] == 0).all())
        rows = (idx[:, :, None] * CHUNK + torch.arange(CHUNK, device=DEV)).reshape(Hkv, -1)
        h = torch.arange(Hkv, device=DEV)[:, None]
        assert torch.equal(gc8.key_store[l, :, :B], dequant(kv8.e4m3.k_codes[l][h, rows], kv8.e4m3.k_exp[l][h, rows]))
        assert torch.equal(gc8.value_store[l, :, :B], dequant(kv8.e4m3.v_codes[l][h, rows], kv8.e4m3.v_exp[l][h, rows]))

    # retrieval verify, full-KV verify and decode step through the graphs (seq_len_dev for the full KV)
    pos = torch.arange(P, P + GAMMA + 1, device=DEV).unsqueeze(0)
    assert bool(torch.isfinite(g8.graph_verify(ids[:, :GAMMA + 1], pos)).all())
    assert bool(torch.isfinite(g8.inference(ids[:, P:P + GAMMA + 1])).all())
    assert kv8.seq_len == P + GAMMA + 1
    assert bool(torch.isfinite(g8.decode_step(ids[:, P + GAMMA + 1:P + GAMMA + 2])).all())
    assert kv8.seq_len == P + GAMMA + 2

    # tail_update writes exactly D of the e4m3 store
    g8.update_graph_cache()
    n = kv8.seq_len - P
    torch.cuda.synchronize()
    assert torch.equal(gc8.key_store[:, :, B - n:B], dequant(kv8.e4m3.k_codes[:, :, P:P + n], kv8.e4m3.k_exp[:, :, P:P + n]))
    assert torch.equal(gc8.value_store[:, :, B - n:B], dequant(kv8.e4m3.v_codes[:, :, P:P + n], kv8.e4m3.v_exp[:, :, P:P + n]))
