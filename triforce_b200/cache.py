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
    def _alloc(self, L, H, slots, d, device):
        self.key_store = torch.zeros((L, H, slots, d), dtype=torch.float16, device=device)
        self.value_store = torch.zeros((L, H, slots, d), dtype=torch.float16, device=device)
        self.layers, self.num_heads, self.head_dim, self.slots = L, H, d, slots
        self._maps: Optional[ops.KVTensorMaps] = None

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


class _GatherMixin:
    def gather_kv_incremental(self, indices, offset: int):
        """DistributedSimpleCache.gather_kv_incremental (reference cache.py:333-343): after a tree verify the KV rows of the
        accepted nodes (`offset + i` for i in `indices`) are packed to `offset ..` in every layer; `seq_len` follows."""
        idx = torch.tensor([int(i) + offset for i in indices], dtype=torch.int32, device=self.key_store.device)
        ops.kv_compact(self.key_store, self.value_store, idx, offset)
        self.seq_len = offset + len(indices)


KV_DTYPES = ("fp16", "e4m3")


def kv_dtype_of(cache) -> str:
    return getattr(cache, "kv_dtype", "fp16")


def require_fp16_store(cache, what: str) -> None:
    if kv_dtype_of(cache) != "fp16":
        raise NotImplementedError(f"{what} needs an fp16 full-KV store; this one is {kv_dtype_of(cache)}")


class FlashSimpleCache(_HeadMajorStore, _GatherMixin):
    """Full KV of the target (reference cache.py:20-61).

    kv_dtype="e4m3" stores the full KV in FP8 E4M3 with one power-of-two exponent per (layer, KV head, slot) row
    (include/triforce_b200.h): `e4m3` holds codes and exponents, `key_store` / `value_store` are the uint8 codes and the slot
    count is rounded up to a multiple of 64.  Every kernel reading it computes what its fp16 counterpart computes on the
    dequantized rows, so the target's numerics change with the store."""

    def __init__(self, model, max_budget=1024, kv_dtype: str = "fp16") -> None:
        if kv_dtype not in KV_DTYPES:
            raise ValueError(f"kv_dtype must be one of {KV_DTYPES}, got {kv_dtype!r}")
        self.kv_dtype = kv_dtype
        self.seq_len = 0
        self.max_budget = max_budget
        L, H, d = _model_geometry(model)
        self.hidden_size = model.config.hidden_size
        self.e4m3: Optional[ops.E4m3Store] = None
        if kv_dtype == "e4m3":
            slots = -(-max_budget // ops.VERIFY_BOX_KEYS) * ops.VERIFY_BOX_KEYS
            self.e4m3 = ops.E4m3Store.empty(L, H, slots, d, model.device)
            self.key_store, self.value_store = self.e4m3.k_codes, self.e4m3.v_codes
            self.layers, self.num_heads, self.head_dim, self.slots = L, H, d, slots
            self._maps = self.e4m3
        else:
            self._alloc(L, H, max_budget, d, model.device)
        self.seq_len_dev = torch.zeros(1, dtype=torch.int32, device=model.device)
        self._dev_mirror = 0  # value `seq_len_dev` holds once everything enqueued so far has run
        self.scores = []

    def print_status(self):
        print("[Full Cache] Cached:", self.seq_len, "| Budget:", self.max_budget)

    def reset(self):
        self.seq_len = 0
        self.key_store.zero_()
        self.value_store.zero_()
        if self.e4m3 is not None:
            self.e4m3.k_exp.zero_()
            self.e4m3.v_exp.zero_()

    def gather_kv_incremental(self, indices, offset: int):
        require_fp16_store(self, "gather_kv_incremental")
        super().gather_kv_incremental(indices, offset)

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
    full KV, followed by gamma+1 slots for the tokens being verified."""

    def __init__(self, model, max_budget=1024, prefill=1024, chunk_size=8, gamma=6) -> None:
        self.chunk_size = chunk_size
        self.prefill = prefill
        self.chunks = prefill // self.chunk_size
        self.select_sets = max_budget // self.chunk_size
        self.gamma = gamma
        self.max_budget = max_budget
        assert prefill % self.chunk_size == 0, f"prefill should be multiple of chunk_size, got {prefill} % {self.chunk_size}"
        assert max_budget % self.chunk_size == 0, f"max_budget should be multiple of chunk_size, got {max_budget} % {self.chunk_size}"
        self.real_budget = max_budget + gamma + 1
        L, H, d = _model_geometry(model)
        self.hidden_size = model.config.hidden_size
        self._alloc(L, H, self.real_budget, d, model.device)
        self.init_graph = False
        # last build's selection, kept for inspection / parity tests: int32 [L, H, select_sets], fp16 [L, H, chunks]
        self.topk_idx = torch.zeros((L, H, self.select_sets), dtype=torch.int32, device=model.device)
        self.chunk_scores = torch.zeros((L, H, self.chunks), dtype=torch.float16, device=model.device)

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
        if kv_dtype_of(kv_cache) == "e4m3":  # the dequantized rows of the E4M3 store
            if use_device_len:
                ops.tail_update_e4m3(kv_cache.e4m3, self.key_store, self.value_store, self.prefill, self.max_budget, 0,
                                     kv_cache.seq_len_dev, max_new)
            else:
                ops.tail_update_e4m3(kv_cache.e4m3, self.key_store, self.value_store, self.prefill, self.max_budget, kv_cache.seq_len)
            return
        if use_device_len:
            ops.tail_update(kv_cache.key_store, kv_cache.value_store, self.key_store, self.value_store, self.prefill,
                            self.max_budget, 0, kv_cache.seq_len_dev, max_new)
        else:
            ops.tail_update(kv_cache.key_store, kv_cache.value_store, self.key_store, self.value_store, self.prefill,
                            self.max_budget, kv_cache.seq_len)

    def update(self, new_k_cache: torch.Tensor, new_v_cache: torch.Tensor, layer_idx: int):
        """Reference-compatible spec-slot write (cache.py:184-189); the engine writes them through the RoPE kernel."""
        self.key_cache[layer_idx][:, self.real_budget - self.gamma - 1:] = new_k_cache
        self.value_cache[layer_idx][:, self.real_budget - self.gamma - 1:] = new_v_cache
        return self.key_cache[layer_idx][:, :self.real_budget], self.value_cache[layer_idx][:, :self.real_budget]

    def update_graph_cache_retrieval(self, kv_cache, query_states, layer_idx):
        """cache.py:191-194: rebuild + per-layer tail copy (taken from the 2nd prompt on, because `reset` leaves
        `init_graph` set)."""
        self.init_graph_cache(kv_cache, query_states, layer_idx)
        n = kv_cache.seq_len - self.prefill
        if n > 0 and kv_dtype_of(kv_cache) == "e4m3":
            ops.tail_update_e4m3(kv_cache.e4m3, self.key_store, self.value_store, self.prefill, self.max_budget, kv_cache.seq_len,
                                 layer0=layer_idx, n_layers=1)
        elif n > 0:
            self.key_store[layer_idx, :, self.max_budget - n:self.max_budget] = kv_cache.key_store[layer_idx, :, self.prefill:kv_cache.seq_len]
            self.value_store[layer_idx, :, self.max_budget - n:self.max_budget] = kv_cache.value_store[layer_idx, :, self.prefill:kv_cache.seq_len]

    def reset(self):  # NB: like the reference, does not clear `init_graph`
        self.key_store.zero_()
        self.value_store.zero_()


class RetrievalCacheSeqouia(RetrievalCache):
    """DistributedRetrievalCache_Seqouia (reference cache.py:385-483): the retrieval budget followed by `tree_size` slots
    for the nodes of the speculation tree (instead of gamma+1 slots)."""

    def __init__(self, model, max_budget=1024, prefill=1024, chunk_size=8, tree_size=128) -> None:
        super().__init__(model, max_budget=max_budget, prefill=prefill, chunk_size=chunk_size, gamma=tree_size - 1)
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
        self.key_store.zero_()
        self.value_store.zero_()
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
        self.key_store.zero_()
        self.value_store.zero_()
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
