"""Llama target / draft forward passes around the sm_90a hot-path kernels.

Restates the dataflow of the reference's `models/modeling_llama.py:200-414` (target, YaRN RoPE, full / retrieval cache
routing) and `models/modeling_llama_68m.py:129-357` (Llama-68M draft, StreamingLLM cache, RoPE re-applied at slot
positions), and the head-sharded variant of `models/TP_llama.py` + `models/tensor_op.py:121-181,276-360` (column-split
q/k/v/gate/up, row-split o/down, one all-reduce after each).  Decode-time projections (<= 24 rows: q|k|v, o_proj, gate|up with
the SiLU·mul epilogue, down_proj, lm_head with the fp32 epilogue) run on this repo's weight-streaming kernel
(`tf_stream_linear`, SURVEY §8 row f-1), so a decode / verify forward launches nothing but this library's kernels and chains
them with programmatic dependent launch; prefill-sized GEMMs (> 24 rows) stay on cuBLAS through `F.linear` (plain library GEMMs).
The long-prompt PREFILL attention (q_len > 32) runs on this repo's wgmma kernel in causal mode for head_dim 128
(`tf_tree_attn_tc`, SURVEY §8 row f-2); the 64-wide heads of the parity-sized models keep the library call (flash-attn / SDPA).
"""
from __future__ import annotations

import math
import os
from types import SimpleNamespace
from typing import Dict, Optional

import torch
import torch.nn.functional as F

from . import ops
from ._C import lib as _C_lib
from .cache import FlashSimpleCache, RetrievalCache, StreamingLLMEvictionCache, kv_dtype_of
from .config import LlamaShape
from .rope import softmax_scale, tables_for


class _LayerWeights:
    __slots__ = ("wqkv", "wo", "wgu", "wd", "ln1", "ln2", "m_qkv", "m_o", "m_gu", "m_d")

    def __init__(self):
        self.m_qkv = self.m_o = self.m_gu = self.m_d = None


def _prefill_attention_library(q, key_layer, value_layer, kv_len: int, scale: float) -> torch.Tensor:
    """q [n,H,d]; key_layer/value_layer [Hkv,cap,d] (H % Hkv == 0, query head h reads KV head h // (H/Hkv)).  Bottom-right
    causal attention of n new rows over kv_len keys."""
    n, H, d = q.shape
    grp = H // key_layer.shape[0]
    try:
        from flash_attn import flash_attn_with_kvcache  # library kernel, prefill only; takes GQA natively
        k = key_layer.permute(1, 0, 2)[None, :kv_len]
        v = value_layer.permute(1, 0, 2)[None, :kv_len]
        return flash_attn_with_kvcache(q[None], k, v, softmax_scale=scale, causal=True)[0]
    except Exception:
        qh = q.transpose(0, 1)[None]  # [1,H,n,d]
        k = key_layer[None, :, :kv_len]
        v = value_layer[None, :, :kv_len]
        if grp > 1:
            k, v = k.repeat_interleave(grp, dim=1), v.repeat_interleave(grp, dim=1)
        i = torch.arange(n, device=q.device)[:, None]
        j = torch.arange(kv_len, device=q.device)[None, :]
        mask = j <= i + (kv_len - n)
        o = F.scaled_dot_product_attention(qh, k, v, attn_mask=mask, scale=scale)
        return o[0].transpose(0, 1).contiguous()


def shard_layer_weights(state_dict: Dict[str, torch.Tensor], config: LlamaShape, layer: int, tp_rank: int, tp_world: int,
                        device=None):
    """Megatron-style shard of one decoder layer (reference models/TP_layers.py:126-147): q/k/v/gate/up are split by
    OUTPUT rows (heads / intermediate columns), o/down by INPUT columns; returns fused (wqkv, wo, wgu, wd).  q rows are
    sliced by query head and k/v rows by KV head, so wqkv is [Hq·d | Hkv·d | Hkv·d] / world."""
    H, Hkv, d = config.num_attention_heads, config.num_key_value_heads, config.head_dim
    if H % tp_world or config.intermediate_size % tp_world:
        raise ValueError(f"heads ({H}) and intermediate size ({config.intermediate_size}) must be divisible by world size {tp_world}")
    if Hkv % tp_world:
        raise ValueError(f"key/value heads ({Hkv}) must be divisible by world size {tp_world}")
    Hl, Il = H // tp_world, config.intermediate_size // tp_world
    h0, h1 = tp_rank * Hl * d, (tp_rank + 1) * Hl * d
    Hkvl = Hkv // tp_world
    k0, k1 = tp_rank * Hkvl * d, (tp_rank + 1) * Hkvl * d
    i0, i1 = tp_rank * Il, (tp_rank + 1) * Il
    p = f"model.layers.{layer}."

    def g(name):
        t = state_dict[p + name]
        return t.to(device=device, dtype=torch.float16) if device is not None else t

    wqkv = torch.cat([g("self_attn.q_proj.weight")[h0:h1], g("self_attn.k_proj.weight")[k0:k1], g("self_attn.v_proj.weight")[k0:k1]], 0).contiguous()
    wo = g("self_attn.o_proj.weight")[:, h0:h1].contiguous()
    wgu = torch.cat([g("mlp.gate_proj.weight")[i0:i1], g("mlp.up_proj.weight")[i0:i1]], 0).contiguous()
    wd = g("mlp.down_proj.weight")[:, i0:i1].contiguous()
    return wqkv, wo, wgu, wd


_PUSHED = object()  # a seam whose sum over ranks is still sitting in the LL inboxes (see LlamaModel._seam)
WEIGHT_DTYPES = ("fp16", "e4m3")


class LlamaModel:
    """Weights + forward of one Llama (target or draft) on one GPU (optionally one tensor-parallel shard)."""

    def __init__(self, config: LlamaShape, state_dict: Dict[str, torch.Tensor], device="cuda", is_draft: bool = False,
                 tp_rank: int = 0, tp_world: int = 1, prefill_chunk: int = 128, weight_dtype: str = "fp16"):
        """weight_dtype="e4m3" stores the projection weights (q|k|v, o_proj, gate|up, down_proj, lm_head) in FP8 E4M3 with one
        power-of-two exponent per row (ops.E4m3WeightMap); embeddings and norms stay fp16.  This changes the target's numerics:
        the model computed is the one whose weights are D = code * 2^e, exactly as an fp16 model holding D would compute it."""
        if weight_dtype not in WEIGHT_DTYPES:
            raise ValueError(f"weight_dtype must be one of {WEIGHT_DTYPES}, got {weight_dtype!r}")
        if weight_dtype == "e4m3":
            if is_draft:
                raise ValueError("the draft keeps fp16 weights (weight_dtype='e4m3' is for the target)")
            if tp_world > 1:
                raise NotImplementedError("E4M3 weights are not supported under tensor parallelism (the TP seams are fp16)")
            if os.environ.get("TRIFORCE_STREAM_LINEAR", "1") != "1":
                raise NotImplementedError("E4M3 weights run their decode projections on tf_stream_linear_e4m3; "
                                          "TRIFORCE_STREAM_LINEAR=0 has no E4M3 path")
        self.weight_dtype = weight_dtype
        self.config = config
        self.device = torch.device(device)
        self.dtype = torch.float16
        self.is_draft = is_draft
        self.tp_rank, self.tp_world = tp_rank, tp_world
        H, d = config.num_attention_heads, config.head_dim
        assert H % tp_world == 0, "num_attention_heads must be divisible by the TP world size"
        assert config.intermediate_size % tp_world == 0
        assert config.num_key_value_heads % tp_world == 0, "num_key_value_heads must be divisible by the TP world size"
        self.local_num_heads = H // tp_world
        self.local_num_kv_heads = config.num_key_value_heads // tp_world
        self.gqa = self.local_num_kv_heads != self.local_num_heads
        assert not (self.gqa and is_draft), "the draft is multi-head attention"
        self.head_dim = d
        self.prefill_chunk = prefill_chunk
        Hl, Il = self.local_num_heads, config.intermediate_size // tp_world
        self.local_inter = Il

        def g(name):
            return state_dict[name].to(device=self.device, dtype=torch.float16)

        e4m3 = weight_dtype == "e4m3"
        q8 = ops.E4m3WeightMap.quantize
        self.embed_tokens = g("model.embed_tokens.weight")
        self.lm_head = g("lm_head.weight")
        self.m_lm_head = None
        if e4m3:  # quantize each matrix as soon as it exists and keep no fp16 copy
            self.m_lm_head, self.lm_head = q8(self.lm_head), None
        self.norm = g("model.norm.weight")
        self.layers = []
        for l in range(config.num_hidden_layers):
            p = f"model.layers.{l}."
            w = _LayerWeights()
            w.wqkv, w.wo, w.wgu, w.wd = shard_layer_weights(state_dict, config, l, tp_rank, tp_world, device=self.device)
            if e4m3:
                w.m_qkv, w.m_o, w.m_gu, w.m_d = q8(w.wqkv), q8(w.wo), q8(w.wgu, silu=True), q8(w.wd)
                w.wqkv = w.wo = w.wgu = w.wd = None
            w.ln1 = g(p + "input_layernorm.weight")
            w.ln2 = g(p + "post_attention_layernorm.weight")
            self.layers.append(w)
        cos, sin = tables_for(config, is_draft=is_draft)
        self.cos, self.sin = cos.to(self.device), sin.to(self.device)
        self.scale = softmax_scale(d)
        self._attn_ws: Optional[torch.Tensor] = None
        self.attn_variant = 0
        # decode-time linears (<= 24 rows): tf_stream_linear on every projection (SURVEY §8 row f-1).  TRIFORCE_STREAM_LINEAR=0
        # falls back to cuBLAS + tf_skinny_gemm + the stand-alone SiLU·mul kernel (the round-1 stack, kept for A/B timing).
        self.use_stream_linear = os.environ.get("TRIFORCE_STREAM_LINEAR", "1") == "1" and self.device.type == "cuda"
        self.use_skinny_gemm = os.environ.get("TRIFORCE_SKINNY_GEMM", "1") == "1"
        self._linear_ws = None
        self._dense_buf, self._dense_of = None, None  # E4M3 weights: the one-layer fp16 scratch of > 24-row forwards
        if e4m3:
            self._linear_ws = torch.zeros(_C_lib().tf_stream_linear_workspace_bytes(), dtype=torch.uint8, device=self.device)
            self._act_pad = None
        elif self.use_stream_linear:
            self._build_weight_maps()
        self.peer_allreduce = None  # set by enable_peer_allreduce() on TP ranks
        self.peer_linear = None     # fused row-parallel linear + all-reduce (one kernel over NVLink peer memory)
        self.peer_stream = None     # the same on tf_stream_linear (exchange of tile t hidden behind the weights of tile t+1)
        self.prefill_tc = os.environ.get("TRIFORCE_PREFILL_TC", "1") == "1" and self.device.type == "cuda"
        # retrieval-verify attention prefetching the o_proj weights into L2 while it is latency-bound (tf_verify_attn_prefetch).
        # OPT-IN (not measured faster on H100): the requests
        # compete with the K/V tiles of the attention they ride on, and o_proj's own ring fill under PDL already covers its start.
        # It has no e4m3 path: over an E4M3 retrieval cache the verify attention never prefetches.
        self.attn_prefetch = os.environ.get("TRIFORCE_ATTN_PREFETCH", "0") == "1" and self.use_stream_linear
        self._tc_ws, self._tc_ws_key = None, None

    # --- helpers ------------------------------------------------------------------------------------------------------
    def eval(self):
        return self

    def _build_weight_maps(self):
        WM = ops.WeightMap
        self._linear_ws = torch.zeros(_C_lib().tf_stream_linear_workspace_bytes(), dtype=torch.uint8, device=self.device)
        mk = lambda w, silu=False: WM(w, silu=silu) if WM.supported(w) else None
        self._act_pad = None
        for w in self.layers:
            w.m_qkv, w.m_o, w.m_gu, w.m_d = mk(w.wqkv), mk(w.wo), mk(w.wgu, True), mk(w.wd)
            # A down_proj shard whose K is not a multiple of 64 (7B over 8 GPUs: 11008 / 8 = 1376) is stored zero-padded to the
            # next multiple, and the SiLU epilogue of gate|up writes into a persistent activation buffer of that width whose pad
            # columns stay zero — the seam keeps the weight-streaming kernel instead of falling back to the skinny GEMV.
            K = int(w.wd.shape[1])
            if w.m_d is None and w.m_gu is not None and K % 8 == 0 and os.environ.get("TRIFORCE_PAD_DOWN_K", "1") == "1":
                Kp = (K + 63) // 64 * 64
                wd_pad = torch.zeros((w.wd.shape[0], Kp), dtype=w.wd.dtype, device=w.wd.device)
                wd_pad[:, :K].copy_(w.wd)
                w.wd = wd_pad[:, :K]  # the unpadded view for the GEMM fallbacks (prefill): same storage, row stride Kp
                w.m_d = WM(wd_pad)
                if self._act_pad is None:
                    self._act_pad = torch.zeros((ops.STREAM_MAX_ROWS, Kp), dtype=torch.float16, device=self.device)
        self.m_lm_head = mk(self.lm_head)

    def _dense(self, which):
        """E4M3 weights, forwards of more than 24 rows: D of layer `which` (wqkv, wo, wgu, wd) or of lm_head (`which` = "head") in a
        one-layer fp16 scratch, dequantized only when the layer it holds changes (lm_head reuses the same memory)."""
        maps = (self.m_lm_head,) if which == "head" else tuple(getattr(self.layers[which], n) for n in ("m_qkv", "m_o", "m_gu", "m_d"))
        if self._dense_buf is None:
            per_layer = sum(m.N * m.K for m in (self.layers[0].m_qkv, self.layers[0].m_o, self.layers[0].m_gu, self.layers[0].m_d))
            self._dense_buf = torch.empty(max(per_layer, self.m_lm_head.N * self.m_lm_head.K), dtype=torch.float16, device=self.device)
        out, off = [], 0
        for m in maps:
            out.append(self._dense_buf[off:off + m.N * m.K].view(m.N, m.K))
            off += m.N * m.K
        if self._dense_of != which:
            for m, t in zip(maps, out):
                ops.weight_dequantize_e4m3(m.codes, m.exps, out=t)
            self._dense_of = which
        return out

    def _tc_workspace(self, rows: int, maps) -> torch.Tensor:
        """Split-partial workspace of the wgmma attention (tf_tree_attn_tc) for `rows` query rows over this store."""
        key = (rows, self.local_num_heads, int(maps.shape[2]))
        if self._tc_ws_key != key:
            self._tc_ws = None  # release the old one first
            self._tc_ws, self._tc_ws_key = ops.tree_attn_tc_workspace(rows, self.local_num_heads, key[2], self.device), key
        return self._tc_ws

    def _workspace(self) -> torch.Tensor:
        if self._attn_ws is None:
            if self.gqa:
                self._attn_ws = ops.verify_attn_gqa_workspace(self.local_num_heads, self.local_num_kv_heads, self.head_dim, self.device)
            else:
                self._attn_ws = ops.verify_attn_workspace(ops.VERIFY_MAX_ROWS, self.local_num_heads, self.head_dim, self.device)
        return self._attn_ws

    # --- attention entry points: MHA, or grouped-query (Hkv < Hq) through the *_gqa kernels -----------------------------
    def _rope_append(self, qkv, q_out, key_layer, value_layer, **kw):
        if self.gqa:
            ops.rope_append_gqa(qkv, self.local_num_heads, self.local_num_kv_heads, self.head_dim, self.cos, self.sin, q_out,
                                key_layer, value_layer, **kw)
        else:
            ops.rope_append(qkv, self.local_num_heads, self.head_dim, self.cos, self.sin, q_out, key_layer, value_layer, **kw)

    def _verify_attn(self, q_out, maps, layer, kv_len, n, out, ws, kv_len_dev=None, clean_keys=0, next_weights=None):
        Hl, d = self.local_num_heads, self.head_dim
        if self.gqa:  # no L2 prefetch for GQA launches
            ops.verify_attn_gqa(q_out, maps, layer, kv_len, n, Hl, self.local_num_kv_heads, d, self.scale, out, ws,
                                kv_len_dev=kv_len_dev, clean_keys=clean_keys)
        else:
            ops.verify_attn(q_out, maps, layer, kv_len, n, Hl, d, self.scale, out, ws, kv_len_dev=kv_len_dev,
                            variant=self.attn_variant, clean_keys=clean_keys, next_weights=next_weights)

    def _tree_attn_tc(self, q_out, maps, layer, kv_len, n, mask_bits, tree_cols, out, causal=False):
        Hl, d = self.local_num_heads, self.head_dim
        ws = self._tc_workspace(n, maps)
        if self.gqa:
            ops.tree_attn_tc_gqa(q_out, maps, layer, kv_len, n, Hl, self.local_num_kv_heads, d, self.scale, mask_bits, tree_cols,
                                 out, ws, causal=causal)
        else:
            ops.tree_attn_tc(q_out, maps, layer, kv_len, n, Hl, d, self.scale, mask_bits, tree_cols, out, ws, causal=causal)

    # --- over a cache of either format: its `e4m3` store, or its fp16 layers through the entry points above ---------------
    def _append(self, cache, layer, qkv, q_out, **pos):
        """RoPE + append of the rows' K/V into `layer` of the cache (quantized into an E4M3 store); `pos`: the positions and
        slots of rope_append."""
        if cache.e4m3 is not None:
            ops.rope_append_e4m3(qkv, self.local_num_heads, self.local_num_kv_heads, self.head_dim, self.cos, self.sin, q_out,
                                 cache.e4m3, layer, **pos)
        else:
            self._rope_append(qkv, q_out, cache.key_store[layer], cache.value_store[layer], **pos)

    def _attend_workspace(self, cache, n):
        """The workspace `_attend` takes for n rows over the cache: the verify kernels', or None for prompt rows over an fp16
        store."""
        return self._workspace() if n <= ops.VERIFY_MAX_ROWS or cache.e4m3 is not None else None

    def _attend(self, cache, layer, q_out, kv_len, out, ws, kv_len_dev=None, clean_keys=0, next_weights=None):
        """Causal attention of the rows of q_out over the first kv_len keys of the cache, the rows' own keys last (see
        ops.verify_attn for `kv_len_dev`, `clean_keys` and `next_weights`).  An E4M3 store has no L2 prefetch.  More than 32
        rows over an fp16 store are prompt rows: they take the prefill split."""
        n = q_out.shape[0]
        if cache.e4m3 is not None:
            ops.verify_attn_e4m3(q_out, cache.e4m3, layer, kv_len, n, self.local_num_heads, self.local_num_kv_heads, self.head_dim,
                                 self.scale, out, ws, kv_len_dev=kv_len_dev, clean_keys=clean_keys)
            return out
        if n > ops.VERIFY_MAX_ROWS:
            return self._prefill_attention(q_out, cache.tensor_maps, cache.key_store[layer], cache.value_store[layer], layer, kv_len,
                                           n, out, ws)
        self._verify_attn(q_out, cache.tensor_maps, layer, kv_len, n, out, ws, kv_len_dev=kv_len_dev, clean_keys=clean_keys,
                          next_weights=next_weights)
        return out

    def _tree_attention(self, cache, layer, q_out, kv_len, mask_bits, tree_cols, out):
        """Attention of the n rows of q_out over the cache's first kv_len keys, of which the last tree_cols are seen through
        the rows' tree mask."""
        Hl, d = self.local_num_heads, self.head_dim
        n = q_out.shape[0]
        if cache.e4m3 is not None:  # forward_tree_verify admits only the shapes of this kernel
            ops.tree_attn_tc_e4m3(q_out, cache.e4m3, layer, kv_len, n, Hl, self.local_num_kv_heads, d, self.scale, mask_bits,
                                  tree_cols, out, self._tc_workspace(n, cache.e4m3))
            return
        maps = cache.tensor_maps
        if d == 128 and n >= 128 and n % 128 == 0 and os.environ.get("TRIFORCE_TREE_TC", "1") == "1":
            # the whole tree in ONE pass over the KV on the tensor cores (wgmma, variant 2; reads each KV byte n/128 times
            # instead of n/32 times)
            self._tree_attn_tc(q_out, maps, layer, kv_len, n, mask_bits, tree_cols, out)
            return
        ws = self._workspace()
        if self.gqa:  # blocks of VERIFY_MAX_ROWS / group-size rows (ops.verify_attn_gqa)
            ops.verify_attn_gqa(q_out, maps, layer, kv_len, n, Hl, self.local_num_kv_heads, d, self.scale, out, ws,
                                tree_mask=mask_bits[:n], tree_cols=tree_cols)
            return
        for r0 in range(0, n, ops.VERIFY_MAX_ROWS):  # blocks of <= 32 rows (tf_verify_attn_tree)
            r1 = min(n, r0 + ops.VERIFY_MAX_ROWS)
            ops.verify_attn_tree(q_out[r0:r1], maps, layer, kv_len, r1 - r0, Hl, d, self.scale, mask_bits[r0:r1], tree_cols,
                                 out[r0:r1], ws)

    def calibrate_attention(self, kv_cache, rows: int = 7, rounds: int = 4) -> Optional[dict]:
        """Init-time load balancing of the verify attention on this GPU (tf_verify_attn_calibrate): the kernel's per-CTA key
        ranges are re-cut in proportion to the HBM rate each CTA actually gets.  `rows` <= 16 calibrates the grid of the
        decode / verify launches, 17..32 the one-CTA-per-SM grid of the 32-row tree blocks.  OPT-IN (TRIFORCE_ATTN_CALIBRATE=1):
        on an H100 the equal split is faster (full-KV verify at 124 944 keys: 0.684 ms equal vs 0.721-0.726 ms calibrated per
        layer) and, unlike a split measured at start-up, bit-reproducible across processes.  Short stores (< 16K keys) are left
        alone — there is nothing to balance."""
        if os.environ.get("TRIFORCE_ATTN_CALIBRATE", "0") != "1" or self.is_draft or self.gqa or kv_dtype_of(kv_cache) != "fp16":
            return None  # no calibrated split for GQA or E4M3 launches
        maps = kv_cache.tensor_maps
        cap = int(maps.shape[2])
        if cap < 16384:
            return None
        Hl, d = self.local_num_heads, self.head_dim
        q = torch.zeros((rows, Hl, d), dtype=torch.float16, device=self.device)
        out = torch.empty_like(q)
        try:
            rep = ops.verify_attn_calibrate(q, maps, 0, cap, rows, Hl, d, self.scale, out, self._workspace(), rounds=rounds)
        except Exception as e:  # an optional optimisation must never take the engine down: back to the equal split
            try:
                ops.verify_attn_calibrate(q, maps, 0, cap, rows, Hl, d, self.scale, out, self._workspace(), rounds=0)
            except Exception:
                pass
            rep = {"error": repr(e)}
        self.attn_balance = rep
        return rep

    def enable_peer_allreduce(self, max_rows: int = 0):
        """NVLink seam exchange for decode-sized messages (PeerAllReduce: LL slots pushed through NVLS multicast stores, by default
        straight from the seam projection's epilogue and summed inside the following add+RMSNorm).  `max_rows` = largest message
        in rows of `hidden` (0 = automatic: 24 rows = every tf_stream_linear launch, so cfg4's gamma+1 = 17-row verifies stay on
        it; 8 rows for the round-1 pull kernel, which is meant for small messages).
        Larger messages (prefill) go through NCCL.  The older fused GEMV + all-reduce kernels stay opt-in
        (TRIFORCE_FUSED_LINEAR_ALLREDUCE=1, TRIFORCE_STREAM_ALLREDUCE=1)."""
        if max_rows <= 0:
            max_rows = ops.STREAM_MAX_ROWS if os.environ.get("TRIFORCE_ALLREDUCE_LL", "1") == "1" else 8
        if self.tp_world > 1 and os.environ.get("TRIFORCE_PEER_ALLREDUCE", "1") == "1":
            from .tp import PeerAllReduce, PeerFusedLinear, PeerStreamLinear
            self.peer_allreduce = PeerAllReduce(self.device, self.tp_rank, self.tp_world, max_rows * self.config.hidden_size * 2)
            if os.environ.get("TRIFORCE_FUSED_LINEAR_ALLREDUCE", "0") == "1":
                self.peer_linear = PeerFusedLinear(self.device, self.tp_rank, self.tp_world)
            # the seams as one kernel each: tf_stream_linear with the all-reduce in its epilogue.  OPT-IN: the seam projections
            # have ~1 tile per CTA (N = 4096, K long), so the exchange of a tile has no next tile to hide behind, and the
            # separate PDL-chained one-shot kernel is expected to be faster (not measured on H100).
            if self.use_stream_linear and os.environ.get("TRIFORCE_STREAM_ALLREDUCE", "0") == "1":
                self.peer_stream = PeerStreamLinear(self.device, self.tp_rank, self.tp_world)

    def _linear_allreduce(self, x: torch.Tensor, w: torch.Tensor, wmap=None) -> torch.Tensor:
        """Row-parallel projection followed by the TP all-reduce (o_proj / down_proj seams)."""
        if self.tp_world > 1 and self.peer_stream is not None and self.peer_stream.fits(x, wmap):
            return self.peer_stream.linear_allreduce(x, wmap, self._linear_ws)
        if self.tp_world > 1 and self.peer_linear is not None and self.peer_linear.fits(x, w):
            return self.peer_linear.linear_allreduce(x, w)
        return self._all_reduce(self._linear(x, w, wmap))

    def _linear(self, x: torch.Tensor, w: torch.Tensor, wmap=None, out_fp32: bool = False) -> torch.Tensor:
        if wmap is not None and x.shape[0] <= ops.STREAM_MAX_ROWS:
            return ops.stream_linear(x, wmap, out_fp32=out_fp32, workspace=self._linear_ws)
        if self.use_skinny_gemm and x.is_cuda and x.shape[0] <= 16 and w.shape[0] <= 8192 and w.shape[1] % 32 == 0:
            y = ops.skinny_gemm(x, w)
        else:
            y = F.linear(x, w)
        return y.float() if out_fp32 else y

    def _all_reduce(self, t: torch.Tensor) -> torch.Tensor:
        if self.tp_world > 1:
            if self.peer_allreduce is not None and self.peer_allreduce.fits(t):
                return self.peer_allreduce.all_reduce(t)  # tf_allreduce_ll / tf_allreduce_oneshot (decode-time messages)
            torch.distributed.all_reduce(t)               # NCCL (prefill-sized messages)
        return t

    def _seam(self, x: torch.Tensor, w: torch.Tensor, wmap=None):
        """A TP seam (o_proj / down_proj).  Returns the all-reduced [n, hidden] tensor — or _PUSHED when the projection pushed its
        partial straight into the peers' inboxes and the sum will materialise inside the next `_add_norm` (the LL seam)."""
        if self.tp_world > 1 and self.peer_allreduce is not None and self.peer_stream is None and self.peer_linear is None \
                and self.peer_allreduce.fits_seam(x, wmap):
            self.peer_allreduce.linear_push(x, wmap, self._linear_ws)
            return _PUSHED
        return self._linear_allreduce(x, w, wmap)

    def _add_norm(self, h: torch.Tensor, delta, weight: torch.Tensor, x: torch.Tensor) -> None:
        if delta is _PUSHED:
            self.peer_allreduce.add_rmsnorm(h, weight, self.config.rms_norm_eps, x)
        else:
            ops.add_rmsnorm(h, delta, weight, self.config.rms_norm_eps, x)

    def _stack(self, input_ids: torch.Tensor, attn_fn) -> torch.Tensor:
        """Decoder stack on [n] token ids → fp32 logits [n, V].  Decode-sized calls (n <= 24) launch 8 kernels per layer, all of
        this library: add+RMSNorm, q|k|v, RoPE+append, attention, o_proj, add+RMSNorm, gate|up (+SiLU·mul), down_proj — on TP ranks
        the same 8: the two seam projections push their partials to the peers and the add+RMSNorm that follows sums them."""
        ids = input_ids.reshape(-1)
        n = ids.numel()
        h = self.embed_tokens[ids].contiguous()
        x = torch.empty_like(h)
        delta = None
        for l in range(len(self.layers)):
            delta = self._layer(l, h, delta, x, attn_fn)
        return self._head(h, delta, x)

    def _layer(self, l: int, h: torch.Tensor, delta, x: torch.Tensor, attn_fn):
        """Decoder layer l on the n rows of the residual stream h (updated in place; x is scratch of h's shape): `delta` is the
        previous layer's down_proj output (None before layer 0); returns this layer's."""
        w = self.layers[l]
        n = h.shape[0]
        stream = self.use_stream_linear and n <= ops.STREAM_MAX_ROWS  # per projection: a shard whose K is not a multiple of 64 keeps the fallback
        if self.weight_dtype == "e4m3" and not stream:
            wqkv, wo, wgu, wd = self._dense(l)  # cuBLAS on D
        else:
            wqkv, wo, wgu, wd = w.wqkv, w.wo, w.wgu, w.wd
        self._add_norm(h, delta, w.ln1, x)
        qkv = self._linear(x, wqkv, w.m_qkv if stream else None)
        attn = attn_fn(l, qkv, n)
        o = self._seam(attn.view(n, -1), wo, w.m_o if stream else None)
        self._add_norm(h, o, w.ln2, x)
        if stream and w.m_gu is not None:
            if w.m_d is not None and w.m_d.K != self.local_inter:  # zero-padded down_proj (see _build_weight_maps)
                act = self._act_pad[:n]
                ops.stream_linear(x, w.m_gu, silu=True, out=act[:, :self.local_inter], workspace=self._linear_ws)
            else:
                act = ops.stream_linear(x, w.m_gu, silu=True, workspace=self._linear_ws)
        else:
            gu = self._linear(x, wgu)
            act = torch.empty((n, self.local_inter), dtype=torch.float16, device=self.device)
            ops.silu_mul(gu, act)
        m_d = w.m_d if (stream and w.m_d is not None and w.m_d.K == act.shape[1]) else None
        return self._seam(act, wd, m_d)

    def _head(self, h: torch.Tensor, delta, x: torch.Tensor) -> torch.Tensor:
        """Final norm + lm_head (fp32 logits) on the rows of h."""
        stream = self.use_stream_linear and h.shape[0] <= ops.STREAM_MAX_ROWS
        lm_head = self._dense("head")[0] if (self.weight_dtype == "e4m3" and not stream) else self.lm_head
        self._add_norm(h, delta, self.norm, x)
        return self._linear(x, lm_head, self.m_lm_head if stream else None, out_fp32=True)

    def _prefill_attention(self, q_out, maps, key_layer, value_layer, layer: int, kv_len: int, n: int, out, ws):
        """Causal attention of n prompt rows over an fp16 store: verify kernel up to 32 rows, wgmma at d = 128, else library."""
        if n <= ops.VERIFY_MAX_ROWS:
            self._verify_attn(q_out, maps, layer, kv_len, n, out, ws)
            return out
        if self.head_dim == 128 and self.prefill_tc:
            # prompt chunks on the wgmma kernel in causal mode (SURVEY §8 row f-2): no library call on the 7B / 13B path
            self._tree_attn_tc(q_out, maps, layer, kv_len, n, None, 0, out, causal=True)
            return out
        return _prefill_attention_library(q_out, key_layer, value_layer, kv_len, self.scale)

    def _score_targets(self, ids: torch.Tensor, logprobs) -> Optional[torch.Tensor]:
        """The int32 ids[1:] that `logprobs` (fp32 [N-1], int32 [N-1]) receives the scores of, checked once for the whole call;
        None without `logprobs`."""
        if logprobs is None:
            return None
        lp, am = logprobs
        n = ids.numel() - 1
        here = lambda t: t.device.type == self.device.type and self.device.index in (None, t.device.index)  # "cuda" is cuda:k
        if lp.dtype != torch.float32 or am.dtype != torch.int32 or lp.shape != (n,) or am.shape != (n,) or not here(lp) \
                or not here(am):
            raise ValueError(f"logprobs is a (float32 [{n}], int32 [{n}]) pair on {self.device} for {n + 1} ids")
        targets = ids[1:].to(torch.int32)
        if n:
            lo, hi = (int(v) for v in torch.aminmax(targets))
            V = self.config.vocab_size
            if lo < 0 or hi >= V:
                raise ValueError(f"token ids must lie in [0, {V}); got ids in [{lo}, {hi}]")
        return targets

    @staticmethod
    def _score_piece(logits: torch.Tensor, c0: int, targets: Optional[torch.Tensor], logprobs) -> None:
        """Scores of the piece of rows starting at prompt row c0 (its logits [rows, V]): row c0 + j is scored against
        targets[c0 + j] = ids[c0 + j + 1], so a piece's last row takes the next piece's first id, and the prompt's last row
        (which has no next id) none."""
        if targets is None:
            return
        r = min(logits.shape[0], targets.numel() - c0)
        if r > 0:
            lp, am = logprobs
            ops.token_logprobs(logits[:r], targets[c0:c0 + r], lp[c0:c0 + r], am[c0:c0 + r], check_ids=False)

    def prefill(self, input_ids: torch.Tensor, kv_cache: FlashSimpleCache, chunk: int = 128, logprobs=None) -> torch.Tensor:
        """Prompt prefill into the full-KV store, `chunk` ids at a time; returns the logits of the last piece.

        `logprobs`: None, or a (float32 [N-1], int32 [N-1]) pair on the model's device that receives, for i < N-1, log p(ids[i+1] |
        ids[:i+1]) under the model's own distribution and the argmax of row i (ops.token_logprobs), reduced piece by piece as
        the prompt runs.  The returned logits, the store's rows and its length are the same with and without it.

        fp16 weights over an fp16 store: chunk-major, `forward_target` on each piece in turn (the reference's chunking, which
        fixes the fp16 summation order the golden logits were produced with).

        An E4M3 store or E4M3 weights: layer-major.  For each layer, every piece runs through the layer with the ops and shapes
        of the chunk-major prefill, so each layer's weights are dequantized once rather than once per piece.  On an E4M3 store
        the pieces append their K/V to a one-layer fp16 scratch store with the fp16 RoPE kernel and attend over it with the fp16
        kernels, so the prompt's causal attention never reads E4M3; then the layer's rows are quantized into the store.  On an
        fp16 store they append into, and attend over, the store's own layer.  The residual stream of all prompt rows is kept
        between layers; logits are computed for the last piece only.  The logits and the fp16 K/V rows are therefore
        bit-identical to the chunk-major prefill with the same capacity and the same weights.  With `logprobs` the head also runs
        on every other piece, one piece at a time after the last layer (E4M3 weights: lm_head dequantized once)."""
        e4m3_store = kv_dtype_of(kv_cache) == "e4m3"
        ids = input_ids.reshape(-1)
        targets = self._score_targets(ids, logprobs)
        if not e4m3_store and self.weight_dtype == "fp16":
            for c0 in range(0, ids.numel(), chunk):
                logits = self.forward_target(ids[c0:c0 + chunk], kv_cache)
                self._score_piece(logits[0], c0, targets, logprobs)
            return logits
        if kv_cache.seq_len != 0:
            raise NotImplementedError("the layer-major prefill starts from an empty full-KV store (reset the cache first)")
        N = ids.numel()
        cap = kv_cache.e4m3.shape[2] if e4m3_store else kv_cache.key_store.shape[2]
        if N > cap:
            raise ValueError(f"{N} prompt tokens exceed the {cap} slots of the full-KV store")
        return self._layer_major(ids, kv_cache, chunk, targets=targets, logprobs=logprobs)

    def extend(self, input_ids: torch.Tensor, kv_cache: FlashSimpleCache, chunk: int = 128,
               queries: Optional[torch.Tensor] = None, logprobs=None) -> torch.Tensor:
        """Append n prompt rows after the store's `seq_len` rows (a follow-up turn over a prefilled context); returns the logits
        of the last row, [1, 1, V].  `queries`: None, or [L, H, d] fp16 that receives each layer's post-RoPE query of the last
        row (what the retrieval cache scores chunks with, RetrievalCache.reselect).

        fp16 weights over an fp16 store: `forward_target` on `chunk`-id pieces, the calls `prefill` makes, so when the existing
        length is a multiple of `chunk`, prefill(A) then extend(B) equals prefill(A + B) bit for bit.
        An E4M3 store or E4M3 weights: layer-major, like `prefill` (each layer's weights dequantized once per call).  Over a
        non-empty E4M3 store each piece appends its rows with the E4M3 RoPE kernel and attends over the store: pieces of more than
        64 rows on the causal wgmma kernel at head_dim 128 (tf_tree_attn_tc_causal_e4m3), others on the E4M3 verify attention.
        Over an empty store the call is `prefill`.  `logprobs`: the scores of ids[1:] given the store's rows and the ids before
        them, as in `prefill`."""
        ids = input_ids.reshape(-1)
        N, start = ids.numel(), kv_cache.seq_len
        if N < 1:
            raise ValueError("extend needs at least one id")
        if start + N > kv_cache.slots:
            raise ValueError(f"appending {N} tokens after {start} exceeds the {kv_cache.slots} slots of the full-KV store")
        if queries is not None:
            assert queries.dtype == torch.float16 and queries.shape == (len(self.layers), self.local_num_heads, self.head_dim)
        targets = self._score_targets(ids, logprobs)
        if kv_dtype_of(kv_cache) == "fp16" and self.weight_dtype == "fp16":
            for c0 in range(0, N, chunk):
                logits = self.forward_target(ids[c0:c0 + chunk], kv_cache, queries=queries if c0 + chunk >= N else None)
                self._score_piece(logits[0], c0, targets, logprobs)
        else:
            logits = self._layer_major(ids, kv_cache, chunk, queries, targets=targets, logprobs=logprobs)
        return logits[:, -1:]

    def _layer_major(self, ids: torch.Tensor, kv_cache: FlashSimpleCache, chunk: int,
                     queries: Optional[torch.Tensor] = None, targets: Optional[torch.Tensor] = None, logprobs=None) -> torch.Tensor:
        """The N ids after the store's seq_len rows, layer by layer in `chunk`-id pieces (see `prefill` and `extend`); the
        caller has checked the capacity.  An empty E4M3 store takes the fp16 scratch of `prefill`.  `targets` (from
        `_score_targets`): the head also runs on every piece but the last, in turn, into x and one piece of logits."""
        start = kv_cache.seq_len
        e4m3_store = kv_dtype_of(kv_cache) == "e4m3"
        scratch = e4m3_store and start == 0
        N = ids.numel()
        L, Hkv, cap, d = kv_cache.e4m3.shape if e4m3_store else kv_cache.key_store.shape
        Hl = self.local_num_heads
        h = self.embed_tokens[ids].contiguous()
        delta = [None] * ((N + chunk - 1) // chunk)
        x = torch.empty((min(chunk, N), h.shape[1]), dtype=torch.float16, device=self.device)
        if scratch:
            scratch_k = torch.zeros((1, Hkv, cap, d), dtype=torch.float16, device=self.device)
            scratch_v = torch.zeros_like(scratch_k)
            maps = ops.KVTensorMaps(scratch_k, scratch_v)
        else:
            maps = kv_cache.tensor_maps
        ws = self._workspace()
        for l in range(L):
            if scratch:
                kl, vl, ml = scratch_k[0], scratch_v[0], 0
            elif not e4m3_store:
                kl, vl, ml = kv_cache.key_store[l], kv_cache.value_store[l], l
            for i, c0 in enumerate(range(0, N, chunk)):
                c1 = min(N, c0 + chunk)

                def attn_fn(_l, qkv, n, p0=start + c0, last=c1 == N):
                    q_out = torch.empty((n, Hl, d), dtype=torch.float16, device=self.device)
                    out = torch.empty((n, Hl, d), dtype=torch.float16, device=self.device)
                    if e4m3_store and not scratch:
                        self._append(kv_cache, l, qkv, q_out, pos0=p0, slot0=p0)
                        if n > 2 * ops.VERIFY_MAX_ROWS and d == 128:
                            ops.tree_attn_tc_causal_e4m3(q_out, maps, l, p0 + n, n, Hl, Hkv, d, self.scale, out,
                                                         self._tc_workspace(n, maps))
                        else:
                            self._attend(kv_cache, l, q_out, p0 + n, out, ws)
                    else:
                        self._rope_append(qkv, q_out, kl, vl, pos0=p0, slot0=p0)
                        out = self._prefill_attention(q_out, maps, kl, vl, ml, p0 + n, n, out, ws)
                    if queries is not None and last:
                        queries[l] = q_out[-1]
                    return out

                delta[i] = self._layer(l, h[c0:c1], delta[i], x[:c1 - c0], attn_fn)
            if scratch:
                ops.kv_quantize_e4m3(scratch_k[0], kv_cache.e4m3.k_codes[l], kv_cache.e4m3.k_exp[l], 0, N)
                ops.kv_quantize_e4m3(scratch_v[0], kv_cache.e4m3.v_codes[l], kv_cache.e4m3.v_exp[l], 0, N)
        if scratch:
            del scratch_k, scratch_v
        del maps
        c0 = (N - 1) // chunk * chunk
        if targets is not None:
            for i, p0 in enumerate(range(0, c0, chunk)):
                self._score_piece(self._head(h[p0:p0 + chunk], delta[i], x), p0, targets, logprobs)
        logits = self._head(h[c0:], delta[-1], x[:N - c0])
        self._score_piece(logits, c0, targets, logprobs)
        kv_cache.seq_len = start + N
        return logits.unsqueeze(0)

    # --- target --------------------------------------------------------------------------------------------------------
    def forward_target(self, input_ids: torch.Tensor, kv_cache: FlashSimpleCache, graph_cache: Optional[RetrievalCache] = None,
                       position_ids: Optional[torch.Tensor] = None, spec: bool = False, use_device_len: bool = False,
                       queries: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Mirrors LlamaForCausalLM.forward(input_ids, kv_cache, graph_cache, position_ids, spec) of the reference.
        `use_device_len`: take the committed length from `kv_cache.seq_len_dev` (CUDA-graph replay) instead of the int.
        `queries`: None, or [L, H, d] fp16 that receives each layer's post-RoPE query of the last row (full-KV forwards)."""
        Hl, d = self.local_num_heads, self.head_dim
        n = input_ids.numel()
        build = (not spec) and n == 1 and isinstance(graph_cache, RetrievalCache)
        assert not (build and use_device_len), "a device-length forward does not build the retrieval cache"
        assert queries is None or not spec, "a retrieval verify does not report queries"
        qs = queries if queries is not None else (
            torch.empty((len(self.layers), Hl, d), dtype=torch.float16, device=self.device) if build else None)
        old_len = kv_cache.seq_len
        if kv_dtype_of(kv_cache) == "e4m3" and not spec and n > 2 * ops.VERIFY_MAX_ROWS:
            raise ValueError(f"a {n}-row full-KV forward over an E4M3 store: prompts go through prefill")
        if spec:
            assert n == graph_cache.gamma + 1, "retrieval verify takes exactly gamma+1 rows (cache.py:186)"
            pos = dict(pos_ids=position_ids.reshape(-1).to(torch.int32), slot0=graph_cache.max_budget)
        elif use_device_len:
            pos = dict(pos0_dev=kv_cache.seq_len_dev, slot0_dev=kv_cache.seq_len_dev)
        elif position_ids is not None:
            pos = dict(pos_ids=position_ids.reshape(-1).to(torch.int32), slot0=old_len)
        else:
            pos = dict(pos0=old_len, slot0=old_len)
        ws = self._attend_workspace(graph_cache if spec else kv_cache, n)

        def attn_fn(l, qkv, n):
            q_out = torch.empty((n, Hl, d), dtype=torch.float16, device=self.device)
            out = torch.empty((n, Hl, d), dtype=torch.float16, device=self.device)
            if spec:
                self._append(graph_cache, l, qkv, q_out, **pos)
                return self._attend(graph_cache, l, q_out, graph_cache.real_budget, out, ws,
                                    clean_keys=graph_cache.max_budget,  # rope_append wrote slots >= budget only
                                    next_weights=self.layers[l].wo if self.attn_prefetch else None)  # o_proj's weights ride into L2
            self._append(kv_cache, l, qkv, q_out, **pos)
            if qs is not None:
                qs[l] = q_out[-1]
            return self._attend(kv_cache, l, q_out, n if use_device_len else old_len + n, out, ws,
                                kv_len_dev=kv_cache.seq_len_dev if use_device_len else None)

        logits = self._stack(input_ids, attn_fn)
        if not spec and not use_device_len:
            kv_cache.seq_len = old_len + n  # reference bumps it inside the last layer's update (cache.py:58-59)
        if build:
            first = not graph_cache.init_graph
            graph_cache.build_all_layers(kv_cache, qs)
            if not first:  # cache.py:191-194 per-layer tail copy (empty in the on-chip flow: seq_len <= prefill)
                L = len(self.layers)
                for l in range(L):
                    graph_cache.copy_tail_layer(kv_cache, old_len + (1 if l == L - 1 else 0), l)
        return logits.unsqueeze(0)

    # --- tree (Sequoia) ------------------------------------------------------------------------------------------------
    def forward_tree_retrieval(self, input_ids: torch.Tensor, graph_cache, position_ids: torch.Tensor, mask_bits: torch.Tensor,
                               storage_start: int) -> torch.Tensor:
        """`retrieval_tree_inference` of the reference (TP_llama_tree.py:406-425 → tensor_op.py:230-272): the n new tree nodes
        are written to retrieval slots [budget + storage_start, …) and attend to the whole budget plus their ancestors."""
        Hl, d = self.local_num_heads, self.head_dim
        pos32 = position_ids.reshape(-1).to(torch.int32)
        T = graph_cache.tree_size
        mask_bits = mask_bits.contiguous()

        def attn_fn(l, qkv, n):
            q_out = torch.empty((n, Hl, d), dtype=torch.float16, device=self.device)
            out = torch.empty((n, Hl, d), dtype=torch.float16, device=self.device)
            self._append(graph_cache, l, qkv, q_out, pos_ids=pos32, slot0=graph_cache.max_budget + storage_start)
            self._tree_attention(graph_cache, l, q_out, graph_cache.real_budget, mask_bits, T, out)
            return out

        return self._stack(input_ids, attn_fn).unsqueeze(0)

    def forward_tree_verify(self, input_ids: torch.Tensor, kv_cache, position_ids: torch.Tensor, mask_bits: torch.Tensor) -> torch.Tensor:
        """The masked verify of all T tree nodes over the FULL KV (SpecTree_TP.py:168-175 → TP_llama_tree `inference` with an
        attention mask): nodes are appended at slots [seq_len, seq_len + T) and see the whole prefix plus their ancestors.
        Over an E4M3 store the attention runs on tf_tree_attn_tc_e4m3, which computes what tf_tree_attn_tc computes on the
        dequantized store.  It has no other kernel, so other shapes are refused."""
        Hl, d = self.local_num_heads, self.head_dim
        T = input_ids.numel()
        if kv_dtype_of(kv_cache) == "e4m3":
            tc = os.environ.get("TRIFORCE_TREE_TC", "1")
            if d != 128 or T == 0 or T % 128 or tc != "1":
                raise NotImplementedError(f"tree verify over an E4M3 store runs only on the wgmma tree kernel (head_dim 128, "
                                          f"a multiple of 128 tree rows, TRIFORCE_TREE_TC=1); got head_dim {d}, {T} rows, "
                                          f"TRIFORCE_TREE_TC={tc}")
        pos32 = position_ids.reshape(-1).to(torch.int32)
        old_len = kv_cache.seq_len
        mask_bits = mask_bits.contiguous()

        def attn_fn(l, qkv, n):
            q_out = torch.empty((n, Hl, d), dtype=torch.float16, device=self.device)
            out = torch.empty((n, Hl, d), dtype=torch.float16, device=self.device)
            self._append(kv_cache, l, qkv, q_out, pos_ids=pos32, slot0=old_len)
            self._tree_attention(kv_cache, l, q_out, old_len + T, mask_bits, T, out)
            return out

        logits = self._stack(input_ids, attn_fn)
        kv_cache.seq_len = old_len + T
        return logits.unsqueeze(0)

    # --- draft ---------------------------------------------------------------------------------------------------------
    def forward_draft(self, input_ids: torch.Tensor, cache: StreamingLLMEvictionCache, gamma_offset: int = -1) -> torch.Tensor:
        """Mirrors modeling_llama_68m.LlamaForCausalLM.forward(input_ids, kv_cache, graph_cache, gamma_offset)."""
        Hl, d = self.local_num_heads, self.head_dim
        n = input_ids.numel()
        if gamma_offset >= 0:  # speculative step: rows go to the round slots after the window (:151-162)
            assert n == gamma_offset + 1
            start = cache.real_budget - cache.gamma - 3
            kv_len = start + n
        else:  # prefill chunk (:164-178)
            start = cache.seq_len
            assert start + n <= cache.start_size + cache.recent_size
            kv_len = start + n

        def attn_fn(l, qkv, n):
            q_out = torch.empty((n, Hl, d), dtype=torch.float16, device=self.device)
            out = torch.empty((n, Hl, d), dtype=torch.float16, device=self.device)
            ops.rope_append(qkv, Hl, d, self.cos, self.sin, q_out, cache.key_store[l], cache.value_store[l], pos0=start,
                            slot0=start, rotate_q=True, rotate_k=False)
            ops.draft_attn(q_out, cache.key_store[l], cache.value_store[l], self.cos, self.sin, kv_len, self.scale, out)
            return out

        logits = self._stack(input_ids, attn_fn)
        if gamma_offset < 0:
            cache.seq_len += n
        return logits.unsqueeze(0)

    # reference-style call: model(input_ids=…, kv_cache=…, graph_cache=…, position_ids=…, spec=…, gamma_offset=…).logits
    def __call__(self, input_ids, kv_cache=None, graph_cache=None, position_ids=None, spec=False, gamma_offset=None, **kw):
        if self.is_draft:
            logits = self.forward_draft(input_ids, kv_cache, -1 if gamma_offset is None else gamma_offset)
        else:
            logits = self.forward_target(input_ids, kv_cache, graph_cache, position_ids, spec)
        return SimpleNamespace(logits=logits)
