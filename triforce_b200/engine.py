"""CUDA-graph runtime of the hierarchy — the reference's `utils/graph_infer.py` (InferenceEngine :14-72,
capture helpers :74-127, GraphInferenceEngine :129-194) rebuilt around device-side sequence lengths.

What is captured (one shared memory pool, like graph_infer.py:138):
  * gamma+3 draft graphs (gamma_offset = 0..gamma+2 → 1..gamma+3 rows), each ending in the fused top-p kernel,
  * one retrieval-verify graph (gamma+1 rows over the retrieval cache),
  * NEW vs the reference, which runs these eagerly because `kv_cache.seq_len` is a Python int (decoding.py:31,85):
    full-KV graphs for 1..gamma+2 rows.  The attention / RoPE-append kernels read the committed length from
    `kv_cache.seq_len_dev`, so the 320-launch full verify and the autoregressive step replay as one graph each.
Chunked prefill stays eager (graph_infer.py:30-37: 128-token chunks for the target, 64 for the draft).
"""
from __future__ import annotations

import gc
import math
from typing import Dict, Optional

import torch

from . import ops
from .cache import FlashSimpleCache, RetrievalCache, StreamingLLMEvictionCache
from .llama import LlamaModel
from .sampling import norm_logits


class InferenceEngine:
    """Eager runtime over the three caches (graph_infer.py:14-72).  It owns no tensors of its own: `model` / `draft` are
    `LlamaModel`s whose every non-GEMM op is a kernel of libtriforce_b200.so, `cache` is the full head-major KV store,
    `graph_cache` the retrieval cache (budget + gamma + 1 slots) and `draft_cache` the StreamingLLM window.  The three
    `*_run` / `*_verify` methods keep the reference's argument meaning so that `decoding.py`'s loops, the golden-trace
    tests and user scripts can call either implementation."""

    def __init__(self, model: LlamaModel, cache: FlashSimpleCache, graph_cache: RetrievalCache, draft: LlamaModel,
                 draft_cache: StreamingLLMEvictionCache) -> None:
        self.model = model
        self.kv_cache = cache
        self.graph_cache = graph_cache
        self.draft = draft
        self.draft_cache = draft_cache
        self.target_prefill_chunk = 128  # graph_infer.py:30
        # balance the verify-attention split on this GPU before anything is captured (no reference counterpart)
        self.attn_balance = model.calibrate_attention(cache) if hasattr(model, "calibrate_attention") else None
        self.draft_prefill_chunk = 64    # graph_infer.py:45-47

    @torch.inference_mode()
    def model_run(self, input_ids: torch.LongTensor):
        """Target forward over the FULL cache.  More than 64 ids = prompt: appended in `target_prefill_chunk`-token pieces
        (the reference's chunking, kept because it fixes the fp16 summation order the golden logits were produced with);
        the last call with exactly one id also builds the retrieval cache inside `LlamaModel.forward_target`
        (modeling_llama.py:230-238).  Up to 64 ids = a verify / decode step over the full KV (`tf_verify_attn`)."""
        if input_ids.shape[-1] > 64 and (getattr(self.kv_cache, "kv_dtype", "fp16") == "e4m3"
                                         or getattr(self.model, "weight_dtype", "fp16") == "e4m3"):
            # layer-major prefill: on an E4M3 store the prompt's attention runs on an fp16 scratch layer, then the layer is
            # quantized; E4M3 weights are dequantized once per layer instead of once per chunk
            logits = self.model.prefill_e4m3(input_ids, self.kv_cache, chunk=self.target_prefill_chunk)
        elif input_ids.shape[-1] > 64:  # prefill
            c = self.target_prefill_chunk
            for i in range(math.ceil(input_ids.shape[1] / c)):
                logits = self.model(input_ids=input_ids[:, i * c:(i + 1) * c], kv_cache=self.kv_cache, graph_cache=None).logits
        else:  # verification
            logits = self.model(input_ids=input_ids, kv_cache=self.kv_cache, graph_cache=self.graph_cache).logits
        return logits

    @torch.inference_mode()
    def draft_run(self, input_ids: torch.LongTensor, gamma_offset: int = 0, probs=False, temperature=0.6, top_p=0.9):
        """Draft (Llama-68M) forward on its StreamingLLM window.  Prompt: chunks with an eviction before each one, so the
        window holds 16 sinks + the most recent keys (cache.py:252-261).  Decode: `gamma_offset` + 1 rows are written at the
        speculation slots behind the window (`spec_update`, cache.py:237-245) and attended with RoPE applied at the SLOT
        index while the keys are staged (`tf_draft_attn`).  `probs=True` returns the last row after the fused
        temperature / top-p / softmax kernel — what the draft graphs capture."""
        if input_ids.shape[-1] > 64:  # prefill
            c = self.draft_prefill_chunk
            for i in range(math.ceil(input_ids.shape[1] / c)):
                self.draft_cache.evict_prefill(c)
                logits = self.draft(input_ids=input_ids[:, i * c:(i + 1) * c], kv_cache=self.draft_cache, graph_cache=None).logits
        else:  # decoding
            logits = self.draft(input_ids=input_ids, kv_cache=self.draft_cache, graph_cache=self.draft_cache,
                                gamma_offset=gamma_offset).logits
        if probs:
            return norm_logits(logits[0], temperature=temperature, top_k=-1, top_p=top_p)[-1]
        return logits

    @torch.inference_mode()
    def model_verify(self, input_ids: torch.LongTensor, position_ids: Optional[torch.LongTensor] = None, probs=False,
                     temperature=0.6, top_p=0.9):
        """Retrieval-cache verify: exactly gamma + 1 rows, their K/V written to the slots behind the budget
        (cache.py:184-189) and attended over budget + gamma + 1 keys; `position_ids` carry the true positions for RoPE."""
        logits = self.model(input_ids=input_ids, kv_cache=self.kv_cache, graph_cache=self.graph_cache,
                            position_ids=position_ids, spec=True).logits
        if probs:
            return norm_logits(logits[0], temperature=temperature, top_k=-1, top_p=top_p)
        return logits

    def clear_kv(self):
        """Reset the three caches with the reference's semantics — including the two quirks the golden traces depend on:
        the draft window keeps `seq_len` (zero sinks from the second prompt on) and the retrieval cache keeps
        `init_graph` (later prompts rebuild through `update_graph_cache_retrieval`)."""
        self.kv_cache.reset()
        self.graph_cache.reset()
        self.draft_cache.reset()


def _capture(fn, n_warmups: int, mempool):
    """Warm `fn` up on a side stream, then capture one call into a CUDA graph of the shared pool.  Also records how many
    kernels of this library one replay launches (`bench.py` reports them as `gpu_launches`)."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(n_warmups):
            out = fn()
        s.synchronize()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    before = ops.COUNTER.n
    with torch.cuda.graph(graph, pool=mempool):
        out = fn()
    graph.tf_kernels = ops.COUNTER.n - before  # this library's kernels inside one replay
    return graph, out


def draft_run_capture_graph(engine: InferenceEngine, gamma_offset: int = 0, mempool=None, n_warmups: int = 3, probs=False,
                            temperature=0.6, top_p=0.9):
    device = engine.draft.device
    static_input_ids = torch.full((1, gamma_offset + 1), 0, dtype=torch.long, device=device)
    graph, static_out = _capture(lambda: engine.draft_run(input_ids=static_input_ids, gamma_offset=gamma_offset, probs=probs,
                                                          temperature=temperature, top_p=top_p), n_warmups, mempool)

    def run(input_ids):
        static_input_ids.copy_(input_ids)
        graph.replay()
        ops.COUNTER.n += graph.tf_kernels
        return static_out.clone()

    return run


def model_verify_capture_graph(engine: InferenceEngine, mempool=None, n_warmups: int = 3, gamma: int = 6, probs=False,
                               temperature=0.6, top_p=0.9):
    device = engine.model.device
    static_input_ids = torch.full((1, gamma + 1), 0, dtype=torch.long, device=device)
    static_position_ids = torch.arange(gamma + 1, device=device).unsqueeze(0)
    graph, static_out = _capture(lambda: engine.model_verify(input_ids=static_input_ids, position_ids=static_position_ids,
                                                             probs=probs, temperature=temperature, top_p=top_p),
                                 n_warmups, mempool)

    def run(input_ids, position_ids):
        static_input_ids.copy_(input_ids)
        static_position_ids.copy_(position_ids)
        graph.replay()
        ops.COUNTER.n += graph.tf_kernels
        return static_out.clone()

    return run


def full_kv_capture_graph(engine: InferenceEngine, rows: int, mempool=None, n_warmups: int = 2):
    """Full-KV forward of `rows` new tokens with the committed length read from the device (not in the reference)."""
    device = engine.model.device
    kv = engine.kv_cache
    static_input_ids = torch.full((1, rows), 0, dtype=torch.long, device=device)

    def fn():
        return engine.model.forward_target(static_input_ids, kv, None, None, spec=False, use_device_len=True)

    kv.sync_seq_len_to_device()
    graph, static_out = _capture(fn, n_warmups, mempool)  # use_device_len leaves the Python int untouched

    def run(input_ids):
        static_input_ids.copy_(input_ids)
        kv.sync_seq_len_to_device()
        graph.replay()
        ops.COUNTER.n += graph.tf_kernels
        kv.advance_on_device(rows)
        return static_out.clone()

    return run


class GraphInferenceEngine:
    def __init__(self, model, cache, graph_cache, draft, draft_cache) -> None:
        self.engine = InferenceEngine(model, cache, graph_cache, draft, draft_cache)
        self.callables: Dict[int, callable] = {}
        self.callable_model_verify = None
        self.full_kv_callables: Dict[int, callable] = {}
        self.mempool = None
        self.gamma = None
        self.temperature, self.top_p = 0.6, 0.9
        self.capture_full_kv_graphs = True

    @torch.inference_mode()
    def initialize_cuda_graph(self, gamma=6, probs=False, temperature=0.6, top_p=0.9):
        gc.collect()
        self.gamma, self.temperature, self.top_p = gamma, temperature, top_p
        self.mempool = torch.cuda.graphs.graph_pool_handle()
        for gamma_offset in range(gamma + 3):
            self.callables[gamma_offset] = draft_run_capture_graph(engine=self.engine, gamma_offset=gamma_offset, mempool=self.mempool,
                                                                   n_warmups=3, probs=probs, temperature=temperature, top_p=top_p)
        self.callable_model_verify = model_verify_capture_graph(engine=self.engine, mempool=self.mempool, n_warmups=3, gamma=gamma,
                                                                probs=probs, temperature=temperature, top_p=top_p)
        if self.capture_full_kv_graphs:
            for rows in range(1, gamma + 3):
                self.full_kv_callables[rows] = full_kv_capture_graph(self.engine, rows, mempool=self.mempool)
        self.engine.clear_kv()

    def clear_kv(self):
        self.engine.clear_kv()

    @torch.inference_mode()
    def graph_draft_inference(self, input_ids: torch.LongTensor, gamma_offset: int = 0):
        if gamma_offset in self.callables:
            return self.callables[gamma_offset](input_ids)
        return self.engine.draft_run(input_ids=input_ids, gamma_offset=gamma_offset, probs=True, temperature=self.temperature,
                                     top_p=self.top_p)

    @torch.inference_mode()
    def graph_draft_prefill(self, input_ids: torch.LongTensor):
        return self.engine.draft_run(input_ids=input_ids)

    @torch.inference_mode()
    def inference(self, input_ids: torch.LongTensor):
        n = input_ids.shape[-1]
        if 1 < n and n in self.full_kv_callables:  # gamma2+1 rows over the full KV: one graph replay
            return self.full_kv_callables[n](input_ids)
        return self.engine.model_run(input_ids=input_ids)

    @torch.inference_mode()
    def decode_step(self, next_token: torch.LongTensor):
        """One autoregressive step over the full KV (decoding.py:31 runs this eagerly with graph_cache=None)."""
        if 1 in self.full_kv_callables:
            return self.full_kv_callables[1](next_token.reshape(1, 1))
        return self.engine.model(input_ids=next_token.reshape(1, 1), kv_cache=self.engine.kv_cache, graph_cache=None).logits

    @torch.inference_mode()
    def graph_verify(self, input_ids: torch.LongTensor, position_ids: torch.LongTensor):
        if self.callable_model_verify is not None:
            return self.callable_model_verify(input_ids, position_ids)
        return self.engine.model_verify(input_ids=input_ids, position_ids=position_ids, probs=True,
                                        temperature=self.temperature, top_p=self.top_p)

    def update_graph_cache(self):
        self.engine.graph_cache.update_graph_cache(kv_cache=self.engine.kv_cache)
