"""numpy restatement of the "group_sum" retrieval rule of grouped-query targets (LlamaShape.gqa_retrieval).

The reference scores retrieval chunks by broadcasting its query heads over the KV heads (models/cache.py:157), which
defines nothing when there are fewer KV heads than query heads.  The rule restated here is this project's own: for each
(layer, KV head kvh) and chunk c,

    score = fp16( q̄ · k̄_c ),  q̄[i] = sum over g < G of q[kvh·G + g][i]   (G = Hq / Hkv)

with q̄ summed in fp64 (exact for G <= 64 fp16 values), and k̄_c, the fp64 dot, the order and the gather exactly those of
oracle.triforce_oracle.retrieval_build.  Under exact arithmetic the score is the sum of the group's per-head scores; at
G = 1 it is the MHA arithmetic bit for bit."""
import numpy as np

from oracle import triforce_oracle as orc


def group_query(q: np.ndarray, n_kv_heads: int) -> np.ndarray:
    """q [Hq, d] fp16 → q̄ [Hkv, d] fp64, the sum of each group's query heads (query head h belongs to KV head h // G)."""
    Hq, d = q.shape
    assert Hq % n_kv_heads == 0 and Hq // n_kv_heads <= 64
    return q.astype(np.float64).reshape(n_kv_heads, Hq // n_kv_heads, d).sum(axis=1)


def retrieval_build_group_sum(K: np.ndarray, V: np.ndarray, q: np.ndarray, prefill: int, chunk: int, budget: int):
    """K / V [S, Hkv, d] fp16, q [Hq, d] fp16 → (retr_K [budget, Hkv, d], retr_V, idx [Hkv, budget/chunk] int32,
    scores [Hkv, prefill/chunk] fp16)."""
    kbar = orc.chunk_mean_keys(K, prefill, chunk)
    scores = orc.chunk_scores(group_query(q, K.shape[1]), kbar)
    idx = orc.topk_chunks(scores, budget // chunk)
    return orc.gather_chunks(K[:prefill], idx, chunk), orc.gather_chunks(V[:prefill], idx, chunk), idx, scores
