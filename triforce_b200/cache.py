"""KV caches of the TriForce hierarchy — same classes, constructor arguments, attributes and method names as the
reference's `models/cache.py` (FlashSimpleCache :20-61, RetrievalCache :117-198, StreamingLLMEvictionCache :200-265),
re-laid-out for the GPU kernels.

Physical layout is HEAD-MAJOR `[L, H, slots, d]` fp16: one (layer, head) stream is contiguous, so the verify kernel's
TMA boxes are dense 128-byte rows and an 8-token retrieval chunk is one contiguous 2 KB block.  `.key_cache` /
`.value_cache` expose the reference's `[L, 1, slots, H, d]` shape as permuted VIEWS of that storage, so reference-style
slicing (`cache.key_cache[layer][:, a:b] = …`) keeps working.

`seq_len` stays a Python int that callers mutate (decoding.py:124 rolls back by decrementing it); the engine mirrors
it into a device int before replaying captured graphs.
"""
from __future__ import annotations

from typing import Optional

import torch

from . import ops


def _model_geometry(model):
    cfg = model.config
    heads = getattr(model, "local_num_kv_heads", None) or cfg.num_key_value_heads
    head_dim = cfg.hidden_size // cfg.num_attention_heads
    return cfg.num_hidden_layers, heads, head_dim


class Cache:
    def update(self, key_states, value_states, layer_idx):
        raise NotImplementedError("Make sure to implement `update` in a subclass.")


class _HeadMajorStore(Cache):
    def _alloc(self, L, H, slots, d, device, kv_dtype: str = "fp16"):
        """K and V stores [L, H, slots, d].  kv_dtype="e4m3": the E4M3 format of include/triforce_b200.h, with one power-of-two
        exponent per (layer, head, slot) row; `e4m3` holds codes and exponents, `key_store` / `value_store` are the uint8 codes
        and the slot count is rounded up to a multiple of 64."""
        self.e4m3: Optional[ops.E4m3Store] = None
        if kv_dtype == "e4m3":
            slots = -(-slots // ops.VERIFY_BOX_KEYS) * ops.VERIFY_BOX_KEYS
            self.e4m3 = ops.E4m3Store.empty(L, H, slots, d, device)
            self.key_store, self.value_store = self.e4m3.k_codes, self.e4m3.v_codes
        else:
            self.key_store = torch.zeros((L, H, slots, d), dtype=torch.float16, device=device)
            self.value_store = torch.zeros((L, H, slots, d), dtype=torch.float16, device=device)
        self.layers, self.num_heads, self.head_dim, self.slots = L, H, d, slots
        self._maps = self.e4m3  # an fp16 store builds its KVTensorMaps on first use

    def reset(self):
        self.key_store.zero_()
        self.value_store.zero_()
        if self.e4m3 is not None:
            self.e4m3.k_exp.zero_()
            self.e4m3.v_exp.zero_()

    @property
    def tensor_maps(self) -> ops.KVTensorMaps:
        if self._maps is None:
            self._maps = ops.KVTensorMaps(self.key_store, self.value_store)
        return self._maps

    # reference-shaped views [L, 1, slots, H, d]
    @property
    def key_cache(self) -> torch.Tensor:
        return self.key_store.permute(0, 2, 1, 3).unsqueeze(1)

    @property
    def value_cache(self) -> torch.Tensor:
        return self.value_store.permute(0, 2, 1, 3).unsqueeze(1)


KV_DTYPES = ("fp16", "e4m3")


def kv_dtype_of(cache) -> str:
    return getattr(cache, "kv_dtype", "fp16")


def _full_store_of(kv_cache):
    """The full-KV store as the E4M3 retrieval-cache entries take it: an E4m3Store, or the fp16 (key_store, value_store) pair."""
    return kv_cache.e4m3 if kv_dtype_of(kv_cache) == "e4m3" else (kv_cache.key_store, kv_cache.value_store)


def require_fp16_store(cache, what: str) -> None:
    if kv_dtype_of(cache) != "fp16":
        raise NotImplementedError(f"{what} needs an fp16 full-KV store; this one is {kv_dtype_of(cache)}")


class FlashSimpleCache(_HeadMajorStore):
    """Full KV of the target (reference cache.py:20-61).

    kv_dtype="e4m3" stores the full KV in FP8 E4M3 (see _HeadMajorStore._alloc).  Every kernel reading it computes what its
    fp16 counterpart computes on the dequantized rows, so the target's numerics change with the store."""

    def __init__(self, model, max_budget=1024, kv_dtype: str = "fp16") -> None:
        if kv_dtype not in KV_DTYPES:
            raise ValueError(f"kv_dtype must be one of {KV_DTYPES}, got {kv_dtype!r}")
        self.kv_dtype = kv_dtype
        self.seq_len = 0
        self.max_budget = max_budget
        L, H, d = _model_geometry(model)
        self.hidden_size = model.config.hidden_size
        self._alloc(L, H, max_budget, d, model.device, kv_dtype)
        self.seq_len_dev = torch.zeros(1, dtype=torch.int32, device=model.device)
        self._dev_mirror = 0  # value `seq_len_dev` holds once everything enqueued so far has run
        self.scores = []

    def print_status(self):
        print("[Full Cache] Cached:", self.seq_len, "| Budget:", self.max_budget)

    def reset(self):
        self.seq_len = 0
        super().reset()

    def gather_kv_incremental(self, indices, offset: int):
        """DistributedSimpleCache.gather_kv_incremental (reference cache.py:333-343): after a tree verify the KV rows of the
        accepted nodes (`offset + i` for i in `indices`) are packed to `offset ..` in every layer; `seq_len` follows.  An E4M3
        store moves the accepted nodes' codes and exponents bit for bit (tf_kv_compact_e4m3)."""
        idx = torch.tensor([int(i) + offset for i in indices], dtype=torch.int32, device=self.key_store.device)
        if self.e4m3 is not None:
            ops.kv_compact_e4m3(self.e4m3, idx, offset)
        else:
            ops.kv_compact(self.key_store, self.value_store, idx, offset)
        self.seq_len = offset + len(indices)

    def sync_seq_len_to_device(self):
        """Mirror the Python `seq_len` into `seq_len_dev` on the current stream (graphs read kv_len from there).
        Stream-ordered (`fill_` carries the value as a kernel argument), so the host may run ahead of the GPU."""
        if self._dev_mirror != self.seq_len:
            self.seq_len_dev.fill_(self.seq_len)
            self._dev_mirror = self.seq_len

    def advance_on_device(self, rows: int):
        """After a captured full-KV forward of `rows` tokens: bump both the int and its device mirror."""
        self.seq_len_dev.add_(rows)
        self.seq_len += rows
        self._dev_mirror += rows

    def update(self, key_states, value_states, layer_idx):
        """Reference-compatible append (cache.py:46-61): key_states [1, n, H, d].  The engine's own forward appends
        through the fused RoPE kernel instead; this exists for API parity."""
        require_fp16_store(self, "FlashSimpleCache.update")
        n = key_states.shape[-3]
        self.key_cache[layer_idx][:, self.seq_len:self.seq_len + n] = key_states
        self.value_cache[layer_idx][:, self.seq_len:self.seq_len + n] = value_states
        key = self.key_cache[layer_idx][:, :self.seq_len + n]
        value = self.value_cache[layer_idx][:, :self.seq_len + n]
        if layer_idx == self.layers - 1:
            self.seq_len += n
        return key, value


class RetrievalCache(_HeadMajorStore):
    """Retrieval ("graph") cache (reference cache.py:117-198): `max_budget` slots filled with the top-k chunks of the
    full KV, followed by gamma+1 slots for the tokens being verified.

    kv_dtype="e4m3" stores it in the E4M3 format of the full-KV store (see _HeadMajorStore._alloc).  The build and tail copy
    quantize the rows of an fp16 full store, or copy the codes of an E4M3 one.  The retrieval level only proposes tokens, so
    this changes acceptance but not the target: TriForce stays lossless with respect to the full model.  Like the reference,
    `reset` does not clear `init_graph`."""

    def __init__(self, model, max_budget=1024, prefill=1024, chunk_size=8, gamma=6, kv_dtype: str = "fp16",
                 max_context: Optional[int] = None) -> None:
        """`max_context` (default `prefill`): the longest context `reselect` may select from; it sizes `chunk_scores`."""
        if kv_dtype not in KV_DTYPES:
            raise ValueError(f"kv_dtype must be one of {KV_DTYPES}, got {kv_dtype!r}")
        self.kv_dtype = kv_dtype
        self.chunk_size = chunk_size
        self.prefill = prefill
        self.chunks = prefill // self.chunk_size
        self.select_sets = max_budget // self.chunk_size
        self.gamma = gamma
        self.max_budget = max_budget
        self.max_context = prefill if max_context is None else max_context
        assert prefill % self.chunk_size == 0, f"prefill should be multiple of chunk_size, got {prefill} % {self.chunk_size}"
        assert max_budget % self.chunk_size == 0, f"max_budget should be multiple of chunk_size, got {max_budget} % {self.chunk_size}"
        if self.max_context < prefill:
            raise ValueError(f"max_context ({self.max_context}) is below prefill ({prefill})")
        self.real_budget = max_budget + gamma + 1
        L, H, d = _model_geometry(model)
        self.hidden_size = model.config.hidden_size
        self._alloc(L, H, self.real_budget, d, model.device, kv_dtype)
        self.init_graph = False
        # last build's selection, kept for inspection / parity tests: int32 [L, H, select_sets], fp16 [L, H, chunks]
        self.topk_idx = torch.zeros((L, H, self.select_sets), dtype=torch.int32, device=model.device)
        self._scores = torch.zeros(L * H * (self.max_context // chunk_size), dtype=torch.float16, device=model.device)
        self._prefill0 = prefill

    def reset(self):
        """Clears the stores and returns to the constructed `prefill` boundary (a new prompt builds there, whatever a
        re-selection moved it to)."""
        super().reset()
        self.prefill, self.chunks = self._prefill0, self._prefill0 // self.chunk_size

    @property
    def chunk_scores(self) -> torch.Tensor:
        """fp16 [L, H, chunks]: the scores of the last build, contiguous whatever the current boundary."""
        return self._scores[:self.layers * self.num_heads * self.chunks].view(self.layers, self.num_heads, self.chunks)

    def boundary(self, seq_len: int) -> int:
        """The selection boundary `reselect` takes at a context of seq_len tokens: the last whole chunk, which must leave at
        least the budget to select from and fit `max_context`."""
        B = seq_len // self.chunk_size * self.chunk_size
        if B < self.max_budget:
            raise ValueError(f"a context of {seq_len} tokens has {B} tokens of whole chunks, fewer than the retrieval budget "
                             f"{self.max_budget}")
        if B > self.max_context:
            raise ValueError(f"a context of {seq_len} tokens selects from {B} tokens, beyond max_context {self.max_context} of "
                             f"the retrieval cache")
        return B

    def reselect(self, kv_cache: FlashSimpleCache, queries: torch.Tensor) -> int:
        """Re-select the budget for a new question over the full KV's seq_len tokens: score the chunks below the boundary B
        (`boundary`) with `queries` [L, Hq, d], the post-RoPE queries of the context's last token, gather the top-k, and copy
        rows [B, seq_len) to the budget tail.  `prefill` becomes B, so later tail copies start there.  Returns B."""
        B = self.boundary(kv_cache.seq_len)
        self.prefill, self.chunks = B, B // self.chunk_size
        self.build_all_layers(kv_cache, queries)
        self._tail_copy(kv_cache, kv_cache.seq_len)
        return B

    def print_status(self):
        print("[Retrieval Cache] Budget:", self.max_budget, " | PreFill:", self.prefill, " | Chunk Size:", self.chunk_size,
              " | Chunks:", self.chunks, " | Select Sets:", self.select_sets)

    def init_graph_cache(self, kv_cache: FlashSimpleCache, query_states: torch.Tensor, layer_idx: int):
        """Per-layer build (cache.py:146-178).  query_states: [1, 1, H, d] post-RoPE query of the last prompt token."""
        assert 1 == query_states.shape[1], "query_states should be 1 for init"
        q = query_states.reshape(1, -1, self.head_dim).contiguous()
        self._build(kv_cache, q, layer_idx, 1)
        if layer_idx == self.layers - 1:
            self.init_graph = True

    def _build(self, kv_cache: FlashSimpleCache, q: torch.Tensor, layer0: int, n: int):
        out = dict(layer0=layer0, n_layers=n, out_idx=self.topk_idx[layer0:layer0 + n], out_scores=self.chunk_scores[layer0:layer0 + n])
        if self.e4m3 is not None:  # into the E4M3 cache, from either store (MHA, or GQA under the "group_sum" rule)
            ops.retrieval_build_to_e4m3(_full_store_of(kv_cache), q, self.e4m3, self.prefill, self.chunk_size, self.max_budget, **out)
            return
        if kv_dtype_of(kv_cache) == "e4m3":  # MHA, or GQA under the "group_sum" rule, over the E4M3 store
            ops.retrieval_build_e4m3(kv_cache.e4m3, q, self.key_store, self.value_store, self.prefill, self.chunk_size,
                                     self.max_budget, **out)
            return
        build = ops.retrieval_build if q.shape[1] == self.num_heads else ops.retrieval_build_gqa  # GQA: the "group_sum" rule
        build(kv_cache.key_store, kv_cache.value_store, q, self.key_store, self.value_store, self.prefill, self.chunk_size,
              self.max_budget, **out)

    def build_all_layers(self, kv_cache: FlashSimpleCache, queries: torch.Tensor):
        """All layers in ONE launch sequence (3 kernels instead of 3*L): `queries` [L, H, d].  The selection of layer l
        only needs that layer's query and full K, both final once the last prompt token has gone through layer l.
        A grouped-query target passes its Hq query heads and is scored by the "group_sum" rule (tf_retrieval_build_gqa)."""
        self._build(kv_cache, queries.contiguous(), 0, self.layers)
        self.init_graph = True

    def update_graph_cache(self, kv_cache: Optional[FlashSimpleCache] = None, use_device_len: bool = False, max_new: int = 0):
        """cache.py:180-182: KV of every committed generated token overwrites the budget tail, all layers."""
        if use_device_len:
            self._tail_copy(kv_cache, 0, seq_len_dev=kv_cache.seq_len_dev, max_new=max_new)
        else:
            self._tail_copy(kv_cache, kv_cache.seq_len)

    def _tail_copy(self, kv_cache, seq_len: int, **kw):
        """Full-KV rows [prefill, seq_len) to the budget tail in one launch: into an E4M3 cache (quantized, or the E4M3 store's
        codes), from an E4M3 store into an fp16 cache (its dequantized rows), or fp16 to fp16.  `kw`: the device length
        (seq_len_dev, max_new), or for the E4M3 entries a layer range (layer0, n_layers)."""
        if self.e4m3 is not None:
            ops.tail_update_to_e4m3(_full_store_of(kv_cache), self.e4m3, self.prefill, self.max_budget, seq_len, **kw)
        elif kv_dtype_of(kv_cache) == "e4m3":
            ops.tail_update_e4m3(kv_cache.e4m3, self.key_store, self.value_store, self.prefill, self.max_budget, seq_len, **kw)
        else:
            ops.tail_update(kv_cache.key_store, kv_cache.value_store, self.key_store, self.value_store, self.prefill,
                            self.max_budget, seq_len, **kw)

    def update(self, new_k_cache: torch.Tensor, new_v_cache: torch.Tensor, layer_idx: int):
        """Reference-compatible spec-slot write (cache.py:184-189); the engine writes them through the RoPE kernel."""
        if self.e4m3 is not None:
            raise NotImplementedError("RetrievalCache.update writes fp16 rows; an e4m3 retrieval cache is written by rope_append_e4m3")
        self.key_cache[layer_idx][:, self.real_budget - self.gamma - 1:] = new_k_cache
        self.value_cache[layer_idx][:, self.real_budget - self.gamma - 1:] = new_v_cache
        return self.key_cache[layer_idx][:, :self.real_budget], self.value_cache[layer_idx][:, :self.real_budget]

    def update_graph_cache_retrieval(self, kv_cache, query_states, layer_idx):
        """cache.py:191-194: rebuild + per-layer tail copy (taken from the 2nd prompt on, because `reset` leaves
        `init_graph` set)."""
        self.init_graph_cache(kv_cache, query_states, layer_idx)
        self.copy_tail_layer(kv_cache, kv_cache.seq_len, layer_idx)

    def copy_tail_layer(self, kv_cache, seq_len: int, layer_idx: int):
        """The per-layer tail copy of a rebuild (cache.py:191-194): full-KV rows [prefill, seq_len) of one layer go to the
        budget tail."""
        n = seq_len - self.prefill
        if n <= 0:
            return
        if self.e4m3 is None and kv_dtype_of(kv_cache) == "fp16":  # a slice copy: tf_tail_update has no layer range
            self.key_store[layer_idx, :, self.max_budget - n:self.max_budget] = kv_cache.key_store[layer_idx, :, self.prefill:seq_len]
            self.value_store[layer_idx, :, self.max_budget - n:self.max_budget] = kv_cache.value_store[layer_idx, :, self.prefill:seq_len]
        else:
            self._tail_copy(kv_cache, seq_len, layer0=layer_idx, n_layers=1)


class RetrievalCacheSeqouia(RetrievalCache):
    """DistributedRetrievalCache_Seqouia (reference cache.py:385-483): the retrieval budget followed by `tree_size` slots
    for the nodes of the speculation tree (instead of gamma+1 slots)."""

    def __init__(self, model, max_budget=1024, prefill=1024, chunk_size=8, tree_size=128, kv_dtype: str = "fp16",
                 max_context: Optional[int] = None) -> None:
        """`max_context`: as in RetrievalCache (the longest context `reselect` may select from; default `prefill`)."""
        if kv_dtype != "fp16":
            raise NotImplementedError(f"the Sequoia tree path keeps an fp16 retrieval cache (its tree growth needs a tree mode the "
                                      f"e4m3 verify attention does not have); kv_dtype={kv_dtype!r} is not supported")
        super().__init__(model, max_budget=max_budget, prefill=prefill, chunk_size=chunk_size, gamma=tree_size - 1,
                         max_context=max_context)
        self.tree_size = tree_size
        assert self.real_budget == max_budget + tree_size

    def init_graph_cache(self, kv_cache, query_states, layer_idx):
        require_fp16_store(kv_cache, "the Sequoia retrieval cache")
        if self.init_graph:
            raise ValueError("Graph is already initialized")  # cache.py:420-421
        super().init_graph_cache(kv_cache, query_states, layer_idx)

    def update(self, key_states, value_states, layer_idx, storage_ids):
        """Reference-compatible index_copy_ (cache.py:456-463); the engine writes tree slots through the RoPE kernel."""
        assert len(storage_ids) == key_states.shape[1] == value_states.shape[1]
        self.key_cache[layer_idx].index_copy_(dim=1, index=storage_ids, source=key_states)
        self.value_cache[layer_idx].index_copy_(dim=1, index=storage_ids, source=value_states)
        return self.key_cache[layer_idx], self.value_cache[layer_idx]

    def reset(self):
        super().reset()
        self.init_graph = False  # unlike RetrievalCache.reset (cache.py:476-479)


class StreamingLLMEvictionCache(_HeadMajorStore):
    """Draft cache (reference cache.py:200-265): `start_size` sink slots + `recent_size` window + gamma+3 slots for the
    tokens of the current round.  Keys are stored UN-rotated; the draft attention kernel rotates them at their slot index.

    `strict_reference_quirks=True` (default) reproduces `reset()` NOT resetting `seq_len` (cache.py:247-250): from the second
    prompt on the 16 sink slots stay all-zero, exactly as in the reference's timed runs (SURVEY §7 hard part 3)."""

    def __init__(self, model, gamma=6, start_size=16, recent_size=496, strict_reference_quirks: bool = True) -> None:
        self.gamma = gamma
        self.start_size = start_size
        self.recent_size = recent_size
        self.real_budget = self.start_size + self.recent_size + self.gamma + 1 + 1 + 1
        self.seq_len = 0  # just for prefill usage
        self.strict_reference_quirks = strict_reference_quirks
        L, H, d = _model_geometry(model)
        self.hidden_size = model.config.hidden_size
        self._alloc(L, H, self.real_budget, d, model.device)

    def print_status(self):
        print("[StreamingLLM Cache] Start Size:", self.start_size, "| Recent Size:", self.recent_size, "| Gamma:", self.gamma,
              "| Real Budget:", self.real_budget, "| Cached:", self.seq_len)

    def update(self, key_states, value_states, layer_idx):
        incoming = key_states.shape[-3]
        assert self.seq_len + incoming <= self.start_size + self.recent_size
        self.key_cache[layer_idx][:, self.seq_len:self.seq_len + incoming] = key_states
        self.value_cache[layer_idx][:, self.seq_len:self.seq_len + incoming] = value_states
        key = self.key_cache[layer_idx][:, :self.seq_len + incoming]
        value = self.value_cache[layer_idx][:, :self.seq_len + incoming]
        if layer_idx == self.layers - 1:
            self.seq_len += incoming
        return key, value

    def spec_update(self, new_k_cache, new_v_cache, layer_idx, gamma_offset=0):
        start = self.real_budget - self.gamma - 3
        end = start + new_k_cache.shape[-3]
        self.key_cache[layer_idx][:, start:end] = new_k_cache
        self.value_cache[layer_idx][:, start:end] = new_v_cache
        return self.key_cache[layer_idx][:, :end], self.value_cache[layer_idx][:, :end]

    def reset(self):
        super().reset()
        if not self.strict_reference_quirks:
            self.seq_len = 0

    def evict_prefill(self, incoming):
        if self.seq_len + incoming <= self.start_size + self.recent_size:
            return
        size_keep = self.recent_size - incoming
        ops.window_slide(self.key_store, self.value_store, self.seq_len - size_keep, self.start_size, size_keep)
        self.seq_len = self.start_size + self.recent_size - incoming

    def evict_for_spec(self, current_seq_len):
        ops.window_slide(self.key_store, self.value_store, current_seq_len - self.recent_size, self.start_size, self.recent_size)
