"""Head-sharded tensor parallelism — the reference's `models/TP_llama.py` (DistributedLlama :27-388, distributed_init
:19-25), `models/TP_layers.py:126-147` (weight split) and `models/tensor_op.py:121-181,276-360` (TP attention / MLP with one
all-reduce after o_proj and one after down_proj) behind the same class and method names.

One process per GPU (`torchrun`), NCCL over NVLink/NVSwitch for the two all-reduces per layer; everything inside
attention — full KV, retrieval cache, per-head top-k selection, draft — is rank-local (SURVEY §8e).  The reference's
rank-0-samples-then-broadcast (+barrier) protocol (decoding.py:230-239,350-351) is replaced by identically seeded
replicated sampling: the logits are bit-identical on every rank after the all-reduce, so every rank draws the same token
with no communication.  KV offloading (`kv_offload`, `on_chip_layers`) is accepted and ignored: the whole KV stays in
HBM — split over the ranks' GPUs — (SURVEY §2a marks the offload path out of scope).
"""
from __future__ import annotations

import os
from typing import Dict, Optional

import torch
import torch.distributed as dist

from .cache import FlashSimpleCache, RetrievalCache, RetrievalCacheSeqouia, StreamingLLMEvictionCache
from .config import LlamaShape, named_config
from .engine import GraphInferenceEngine
from .llama import LlamaModel
from .sampling import norm_logits

_NAME_TO_SHAPE = {
    "NousResearch/Yarn-Llama-2-13b-128k": "llama-13B-128K",
    "NousResearch/Yarn-Llama-2-7b-128k": "llama-7B-128K",
    "LargeWorldModel/LWM-Text-Chat-128K": "lwm-128K",
    "LargeWorldModel/LWM-Text-128K": "lwm-128K",
}


def distributed_init(backend: str = "nccl"):
    """reference TP_llama.py:19-25 (single node: local rank == global rank)."""
    if not dist.is_initialized():
        dist.init_process_group(backend=backend)
    local_rank = dist.get_rank()
    world_size = dist.get_world_size()
    if backend == "nccl":
        torch.cuda.set_device(local_rank)
    return local_rank, world_size


def _symmetric_buffer(nbytes: int, device: torch.device, rank: int, world: int):
    """A zero-filled buffer of `nbytes` on every rank, mapped into every peer: returns (keep-alive objects, list of the
    `world` device pointers as seen from THIS process, transport name).  torch's symmetric memory when available, else
    plain CUDA IPC handles of an ordinary allocation exchanged over the process group."""
    keep, ptrs = [], None
    _symmetric_buffer.last_multicast_ptr = 0
    try:
        import torch.distributed._symmetric_memory as symm_mem
        buf = symm_mem.empty(nbytes, dtype=torch.uint8, device=device)
        buf.zero_()
        torch.cuda.synchronize(device)
        hdl = symm_mem.rendezvous(buf, dist.group.WORLD.group_name)
        ptrs = [int(p) for p in hdl.buffer_ptrs]
        keep += [buf, hdl]
        transport = "torch symmetric memory"
        try:  # NVLS multicast mapping of the same allocation (0 when the fabric / driver does not offer it)
            _symmetric_buffer.last_multicast_ptr = int(getattr(hdl, "multicast_ptr", 0) or 0)
        except Exception:
            _symmetric_buffer.last_multicast_ptr = 0
    except Exception:
        buf = torch.zeros(nbytes, dtype=torch.uint8, device=device)
        torch.cuda.synchronize(device)
        handle = buf.untyped_storage()._share_cuda_()
        handles = [None] * world
        dist.all_gather_object(handles, handle)
        ptrs = []
        for p, h in enumerate(handles):
            if p == rank:
                ptrs.append(buf.data_ptr())
            else:
                st = torch.UntypedStorage._new_shared_cuda(*h)
                keep.append(st)
                ptrs.append(st.data_ptr())
        keep.append(buf)
        transport = "CUDA IPC"
    dist.barrier()
    torch.cuda.synchronize(device)
    return keep, ptrs, transport


class PeerAllReduce:
    """One-shot NVLink all-reduce for the small decode-time messages of the TP seams (tf_allreduce_oneshot)."""

    def __init__(self, device: torch.device, rank: int, world: int, max_message_bytes: int = 1 << 20):
        import ctypes

        from . import _C
        self.rank, self.world, self.device = rank, world, device
        self.max_bytes = max_message_bytes
        # "LL" exchange (data and flag in one 8-byte slot, polled locally) by default; TRIFORCE_ALLREDUCE_LL=0 = push + flags
        self.ll = os.environ.get("TRIFORCE_ALLREDUCE_LL", "1") == "1"
        nbytes = _C.lib().tf_allreduce_ll_buffer_bytes(max_message_bytes) if self.ll else _C.lib().tf_allreduce_buffer_bytes(max_message_bytes)
        self._keep, ptrs, self.transport = _symmetric_buffer(nbytes, device, rank, world)
        self.multicast_ptr = _symmetric_buffer.last_multicast_ptr if os.environ.get("TRIFORCE_MULTICAST", "1") == "1" else 0
        if self.multicast_ptr:
            self.transport += " + NVLS multicast stores"
        self.transport += ", LL slots" if self.ll else ", push + flags"
        self._ptr_array = (ctypes.c_void_p * world)(*ptrs)
        self._local_ptr = ptrs[rank]
        # TRIFORCE_LL_SEAM=0: keep the all-reduce as its own kernel between the projection and the add+RMSNorm
        self.fused_seam = self.ll and os.environ.get("TRIFORCE_LL_SEAM", "1") == "1"
        if self.fused_seam:
            self.transport += ", pushed by the projection and folded into add+RMSNorm"
        self.state = torch.zeros(2, dtype=torch.int32, device=device)

    def all_reduce(self, t: torch.Tensor) -> torch.Tensor:
        """In-place SUM over ranks of a contiguous fp16 tensor (numel % 8 == 0, <= max_message_bytes)."""
        from . import _C, ops
        assert t.is_contiguous() and t.dtype == torch.float16
        fn = _C.lib().tf_allreduce_ll if self.ll else _C.lib().tf_allreduce_oneshot
        _C.check(fn(self._ptr_array, self.multicast_ptr or None, self.rank, self.world, t.data_ptr(), t.data_ptr(), t.numel(), self.max_bytes,
                    self.state.data_ptr(), _C.stream_ptr()), "tf_allreduce_ll" if self.ll else "tf_allreduce_oneshot")
        ops.COUNTER.n += 1
        return t

    def fits(self, t: torch.Tensor) -> bool:
        return t.dtype == torch.float16 and t.is_contiguous() and t.numel() % 8 == 0 and t.numel() * 2 <= self.max_bytes

    # --- the seam without a stand-alone collective: the projection pushes, the next add+RMSNorm polls ---------------------------
    def fits_seam(self, x: torch.Tensor, wmap) -> bool:
        """The LL seam applies: LL slots in use, a TMA-mapped weight, a decode-sized x whose [M, N] message fits the inbox."""
        from . import ops
        return (self.ll and self.fused_seam and wmap is not None and x.dtype == torch.float16 and x.stride(1) == 1 and x.shape[1] == wmap.K
                and x.shape[0] <= ops.STREAM_MAX_ROWS and wmap.N % 8 == 0 and x.shape[0] * wmap.N * 2 <= self.max_bytes)

    def linear_push(self, x: torch.Tensor, wmap, workspace: torch.Tensor) -> None:
        """x_r @ w_r.T of this rank, pushed as LL slots into every rank's inbox (tf_stream_linear_ll_push); nothing is returned —
        the sum over ranks materialises in the `add_rmsnorm` below."""
        from . import _C, ops
        M, K = x.shape
        _C.check(_C.lib().tf_stream_linear_ll_push(x.data_ptr(), x.stride(0), wmap.ptr, M, wmap.N, K, workspace.data_ptr(), workspace.numel(),
                                                   self._ptr_array, self.multicast_ptr or None, self.rank, self.world, self.max_bytes,
                                                   self.state.data_ptr(), _C.stream_ptr()), "tf_stream_linear_ll_push")
        ops.COUNTER.n += 1

    def add_rmsnorm(self, h: torch.Tensor, weight: torch.Tensor, eps: float, out: torch.Tensor) -> None:
        """h += sum over ranks of the pushed partials (rank order, fp32, rounded to fp16); out = RMSNorm(h) * weight."""
        from . import _C, ops
        rows, hidden = h.shape
        assert h.is_contiguous() and out.is_contiguous() and h.dtype == torch.float16
        _C.check(_C.lib().tf_add_rmsnorm_ll(h.data_ptr(), self._local_ptr, self.world, self.max_bytes, self.state.data_ptr(), weight.data_ptr(),
                                            eps, out.data_ptr(), rows, hidden, _C.stream_ptr()), "tf_add_rmsnorm_ll")
        ops.COUNTER.n += 1


class PeerFusedLinear:
    """Row-parallel linear + all-reduce as ONE kernel over NVLink peer memory (tf_skinny_gemm_allreduce): the o_proj /
    down_proj seams of the TP decode path (reference tensor_op.py:176-179, 357-359)."""

    MAX_ROWS, MAX_N = 16, 8192

    def __init__(self, device: torch.device, rank: int, world: int):
        import ctypes

        from . import _C
        self.rank, self.world, self.device = rank, world, device
        nbytes = _C.lib().tf_skinny_gemm_allreduce_buffer_bytes()
        self._keep, ptrs, self.transport = _symmetric_buffer(nbytes, device, rank, world)
        self._ptr_array = (ctypes.c_void_p * world)(*ptrs)
        self.state = torch.zeros(2, dtype=torch.int32, device=device)

    def fits(self, x: torch.Tensor, w: torch.Tensor) -> bool:
        return (x.dtype == torch.float16 and x.shape[0] <= self.MAX_ROWS and w.shape[0] <= self.MAX_N and w.shape[0] % 16 == 0
                and w.shape[1] % 32 == 0 and x.stride(1) == 1 and x.stride(0) % 8 == 0)

    def linear_allreduce(self, x: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
        """sum over ranks of x_r @ w_r.T  (x_r [M, K_local], w_r [N, K_local]) → [M, N], identical on every rank."""
        from . import _C, ops
        M, K = x.shape
        N = w.shape[0]
        y = torch.empty((M, N), dtype=torch.float16, device=x.device)
        _C.check(_C.lib().tf_skinny_gemm_allreduce(x.data_ptr(), x.stride(0), w.data_ptr(), w.stride(0), M, N, K, y.data_ptr(),
                                                   y.stride(0), self._ptr_array, self.rank, self.world, self.state.data_ptr(),
                                                   _C.stream_ptr()), "tf_skinny_gemm_allreduce")
        ops.COUNTER.n += 1
        return y


class PeerStreamLinear:
    """Row-parallel linear + all-reduce as ONE weight-streaming kernel over NVLink (tf_stream_linear_allreduce): the o_proj /
    down_proj seams of the TP decode path (reference tensor_op.py:176-179, 357-359).  Tiles are exchanged through NVLS multicast
    stores (`multimem.st`) when torch's symmetric memory exposes a multicast mapping, else through per-peer stores."""

    MAX_ROWS, MAX_N = 24, 8192

    def __init__(self, device: torch.device, rank: int, world: int):
        import ctypes

        from . import _C
        self.rank, self.world, self.device = rank, world, device
        nbytes = _C.lib().tf_stream_linear_allreduce_buffer_bytes()
        self._keep, ptrs, self.transport = _symmetric_buffer(nbytes, device, rank, world)
        self.multicast_ptr = _symmetric_buffer.last_multicast_ptr if os.environ.get("TRIFORCE_MULTICAST", "1") == "1" else 0
        if self.multicast_ptr:
            self.transport += " + NVLS multicast stores"
        self._ptr_array = (ctypes.c_void_p * world)(*ptrs)
        self.state = torch.zeros(2, dtype=torch.int32, device=device)

    def fits(self, x: torch.Tensor, wmap) -> bool:
        return wmap is not None and x.dtype == torch.float16 and x.shape[0] <= self.MAX_ROWS and wmap.N <= self.MAX_N and x.stride(1) == 1

    def linear_allreduce(self, x: torch.Tensor, wmap, workspace: torch.Tensor) -> torch.Tensor:
        """sum over ranks of x_r @ w_r.T  (x_r [M, K_local], w_r [N, K_local]) → [M, N] fp16, identical on every rank."""
        from . import _C, ops
        M, K = x.shape
        y = torch.empty((M, wmap.N), dtype=torch.float16, device=x.device)
        _C.check(_C.lib().tf_stream_linear_allreduce(x.data_ptr(), x.stride(0), wmap.ptr, M, wmap.N, K, y.data_ptr(), y.stride(0),
                                                     workspace.data_ptr(), workspace.numel(), self._ptr_array,
                                                     self.multicast_ptr or None, self.rank, self.world, self.state.data_ptr(),
                                                     _C.stream_ptr()), "tf_stream_linear_allreduce")
        ops.COUNTER.n += 1
        return y


def shard_bounds(total: int, rank: int, world: int):
    """Contiguous equal shards (heads for q/k/v/o, intermediate columns for gate/up/down) — TP_layers.py:126-147."""
    if total % world:
        raise ValueError(f"{total} is not divisible by the tensor-parallel world size {world}")
    per = total // world
    return rank * per, (rank + 1) * per


class DistributedLlama:
    def __init__(self, model_name_or_path: str, dtype=torch.float16, kv_offload=False, on_chip_layers=32, local_rank=0, world_size=1,
                 prefill=32768, bsz=1, gen_len=256, retrieval_budget=4096, retrieval_chunk_size=8, gamma=6, temperature=0.6,
                 top_p=0.9, ssl=0, draft=None, draft_cache=None, flash_attn=True, config: Optional[LlamaShape] = None,
                 tree_size: int = 0, kv_dtype: str = "fp16", weight_dtype: str = "fp16") -> None:
        assert bsz == 1
        if kv_dtype != "fp16":
            raise NotImplementedError(f"DistributedLlama (tensor parallel) keeps an fp16 full-KV store; kv_dtype={kv_dtype!r} is not supported")
        if weight_dtype != "fp16":
            raise NotImplementedError(f"DistributedLlama (tensor parallel) keeps fp16 weights; weight_dtype={weight_dtype!r} is not supported")
        self.device = torch.device("cuda", local_rank)
        self.dtype = dtype
        self.local_rank, self.world_size = local_rank, world_size
        self.kv_offload, self.on_chip_layers = kv_offload, on_chip_layers  # accepted, ignored: everything lives in HBM
        self.config = config or named_config(_NAME_TO_SHAPE.get(model_name_or_path, model_name_or_path))
        self.vocab_size = self.config.vocab_size
        self.prefill_len, self.gen_len = prefill, gen_len
        self.retrieval_budget, self.retrieval_chunk_size = retrieval_budget, retrieval_chunk_size
        self.temperature, self.top_p, self.gamma = temperature, top_p, gamma
        self.draft, self.draft_cache = draft, draft_cache
        self.tree_size = tree_size  # > 0: Sequoia mode (models/TP_llama_tree.py), retrieval cache reserves tree slots
        self.hidden_size = self.config.hidden_size
        self.num_heads = self.config.num_attention_heads
        self.head_dim = self.config.head_dim
        self.local_num_heads = self.num_heads // world_size
        self.local_num_key_value_heads = self.config.num_key_value_heads // world_size
        self.model: Optional[LlamaModel] = None
        self.graph_engine: Optional[GraphInferenceEngine] = None
        self.kv_cache = self.retrieval_cache = None

    def init_parameters(self, hf_model=None, state_dict: Optional[Dict[str, torch.Tensor]] = None, cuda_graphs: bool = True):
        """`hf_model`: an HF LlamaForCausalLM (its state_dict is sliced for this rank, TP_layers.py:126-147)."""
        sd = state_dict if state_dict is not None else hf_model.state_dict()
        self.model = LlamaModel(self.config, sd, device=self.device, tp_rank=self.local_rank, tp_world=self.world_size)
        self.num_layers = self.config.num_hidden_layers
        self.kv_cache = FlashSimpleCache(self.model, self.prefill_len + self.gen_len + 32 + self.tree_size)  # TP_llama.py:73
        budget = self.retrieval_budget if self.retrieval_budget > 0 else self.retrieval_chunk_size
        if self.tree_size > 0:
            self.retrieval_cache = RetrievalCacheSeqouia(self.model, max_budget=budget, prefill=self.prefill_len,
                                                         chunk_size=self.retrieval_chunk_size, tree_size=self.tree_size)
        else:
            self.retrieval_cache = RetrievalCache(self.model, max_budget=budget, prefill=self.prefill_len,
                                                  chunk_size=self.retrieval_chunk_size, gamma=self.gamma)
        if self.draft is not None:
            self.graph_engine = GraphInferenceEngine(self.model, self.kv_cache, self.retrieval_cache, self.draft, self.draft_cache)
            self.graph_engine.engine.draft_prefill_chunk = 128  # TP_llama.py:118-126
            if self.world_size > 1:
                t = torch.zeros(1, device=self.device)
                dist.all_reduce(t)  # create the NCCL communicator before any graph capture
                self.model.enable_peer_allreduce()
            if cuda_graphs:
                self.graph_engine.initialize_cuda_graph(self.gamma, probs=True, temperature=self.temperature, top_p=self.top_p)
            else:
                self.graph_engine.gamma = self.gamma

    # ---- reference API -------------------------------------------------------------------------------------------------
    def reset(self):
        self.kv_cache.reset()
        self.retrieval_cache.reset()
        if self.draft_cache is not None:
            self.draft_cache.reset()

    @torch.inference_mode()
    def inference(self, input_ids, position_ids=None, attention_mask=None, retrieval_cache=None):
        return self.model.forward_target(input_ids, self.kv_cache, retrieval_cache, position_ids, spec=False)

    @torch.inference_mode()
    def prefill(self, input_ids):
        import math
        c = 128
        for i in range(math.ceil(input_ids.shape[1] / c)):
            logits = self.inference(input_ids=input_ids[:, i * c:(i + 1) * c])
        return logits

    @torch.inference_mode()
    def build_retrieval_cache(self, input_ids):
        assert input_ids.shape[-1] == 1
        return self.inference(input_ids=input_ids, retrieval_cache=self.retrieval_cache)

    @torch.inference_mode()
    def retrieval_tree_inference(self, input_ids, position_ids, mask_bits, storage_start: int, storage_ids=None, attention_mask=None):
        """models/TP_llama_tree.py:406-425.  The reference's additive `attention_mask` / `storage_ids` are replaced by the packed
        512-bit ancestor masks of the rows and the first tree slot they occupy (slots are always a contiguous range)."""
        return self.model.forward_tree_retrieval(input_ids, self.retrieval_cache, position_ids, mask_bits, storage_start)

    @torch.inference_mode()
    def tree_verify_inference(self, input_ids, position_ids, mask_bits):
        """The masked full-KV forward of SpecTree.verify (SpecTree_TP.py:168-175)."""
        return self.model.forward_tree_verify(input_ids, self.kv_cache, position_ids, mask_bits)

    @torch.inference_mode()
    def retrieval_verify(self, input_ids, position_ids, temperature=0.6, top_p=0.9):
        return self.graph_engine.graph_verify(input_ids, position_ids)

    @torch.inference_mode()
    def draft_run(self, input_ids, gamma_offset: int = 0, probs=True, temperature=0.6, top_p=0.9):
        if input_ids.shape[-1] > 64:
            return self.graph_engine.graph_draft_prefill(input_ids)
        return self.graph_engine.graph_draft_inference(input_ids, gamma_offset)
