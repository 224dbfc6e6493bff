"""Model shape descriptions for the TriForce hot path.

Only the fields the hot path needs (the reference pulls the same ones out of HF's ``LlamaConfig``:
``/root/reference/models/cache.py:25-28``, ``models/modeling_llama.py:162-172``).
The BASELINE.json configs are available by name through :func:`named_config`.
"""
from __future__ import annotations

import dataclasses
import math
from typing import Optional


@dataclasses.dataclass
class LlamaShape:
    hidden_size: int = 4096
    intermediate_size: int = 11008
    num_hidden_layers: int = 32
    num_attention_heads: int = 32
    num_key_value_heads: Optional[int] = None
    vocab_size: int = 32000
    max_position_embeddings: int = 131072
    rms_norm_eps: float = 1e-5
    rope_theta: float = 10000.0
    # None → plain RoPE (reference `LlamaRotaryEmbedding`); dict(type="yarn", factor, original_max_position_embeddings)
    # → YaRN (reference `LlamaYaRNRotaryEmbedding`, models/modeling_llama.py:73-130)
    rope_scaling: Optional[dict] = None
    initializer_range: float = 0.02
    name: str = "llama"
    # How a grouped-query target (num_key_value_heads < num_attention_heads) scores retrieval chunks.  The reference defines
    # no rule (cache.py:157 broadcasts q over kv heads), so a GQA shape must name one.  "group_sum": each KV head scores a
    # chunk with the fp64 sum of its group's query heads (tf_retrieval_build_gqa).  Ignored for MHA shapes.
    gqa_retrieval: Optional[str] = None

    GQA_RETRIEVAL_RULES = ("group_sum",)

    def __post_init__(self):
        if self.num_key_value_heads is None:
            self.num_key_value_heads = self.num_attention_heads
        if self.num_key_value_heads != self.num_attention_heads:
            if self.gqa_retrieval is None:
                # The reference's retrieval scoring broadcasts q heads against kv heads (cache.py:157): MHA only, unless the
                # shape names a GQA retrieval rule.
                raise ValueError("TriForce hot path is MHA-only (reference models/cache.py:157 broadcasts q over kv heads); "
                                 f"a grouped-query shape must name a gqa_retrieval rule {self.GQA_RETRIEVAL_RULES}")
            if self.gqa_retrieval not in self.GQA_RETRIEVAL_RULES:
                raise ValueError(f"unknown gqa_retrieval rule {self.gqa_retrieval!r}; known: {self.GQA_RETRIEVAL_RULES}")
            if self.num_key_value_heads < 1 or self.num_attention_heads % self.num_key_value_heads:
                raise ValueError(f"num_attention_heads ({self.num_attention_heads}) must be a multiple of "
                                 f"num_key_value_heads ({self.num_key_value_heads})")
        if self.hidden_size % self.num_attention_heads:
            raise ValueError("hidden_size must be divisible by num_attention_heads")

    @property
    def head_dim(self) -> int:
        return self.hidden_size // self.num_attention_heads

    # HF-style aliases so reference-shaped code (`model.config.num_hidden_layers` …) keeps working
    @property
    def _name_or_path(self) -> str:
        return self.name

    def param_count(self) -> int:
        h, i, L, v = self.hidden_size, self.intermediate_size, self.num_hidden_layers, self.vocab_size
        hkv = self.num_key_value_heads * self.head_dim  # k_proj / v_proj rows
        return 2 * v * h + L * (2 * h * h + 2 * hkv * h + 3 * h * i + 2 * h) + h

    def kv_bytes_per_token_layer(self) -> int:
        return 2 * self.num_key_value_heads * self.head_dim * 2  # K+V, fp16


def named_config(name: str) -> LlamaShape:
    """Shapes of the checkpoints the reference's entry points load (test/on_chip.py:48-53, test/offloading_TP.py:55-62)."""
    yarn32 = {"type": "yarn", "factor": 32.0, "original_max_position_embeddings": 4096}
    table = {
        # NousResearch/Yarn-Llama-2-7b-128k
        "llama-7B-128K": dict(hidden_size=4096, intermediate_size=11008, num_hidden_layers=32, num_attention_heads=32,
                              max_position_embeddings=131072, rope_scaling=yarn32, rms_norm_eps=1e-5),
        # synthetic grouped-query geometry (no checkpoint): llama-7B-128K with 8 KV heads and a 14336-wide MLP
        "llama-7B-gqa8-128K": dict(hidden_size=4096, intermediate_size=14336, num_hidden_layers=32, num_attention_heads=32,
                                   num_key_value_heads=8, max_position_embeddings=131072, rope_scaling=yarn32, rms_norm_eps=1e-5,
                                   gqa_retrieval="group_sum"),
        # NousResearch/Yarn-Llama-2-13b-128k
        "llama-13B-128K": dict(hidden_size=5120, intermediate_size=13824, num_hidden_layers=40, num_attention_heads=40,
                               max_position_embeddings=131072, rope_scaling=yarn32, rms_norm_eps=1e-5),
        # LargeWorldModel/LWM-Text-Chat-128K: Llama-2-7B shapes, plain RoPE with a large theta
        "lwm-128K": dict(hidden_size=4096, intermediate_size=11008, num_hidden_layers=32, num_attention_heads=32,
                         max_position_embeddings=131072, rope_scaling=None, rope_theta=10000000.0, rms_norm_eps=1e-5),
        # JackFram/llama-68m (the draft)
        "llama-68M": dict(hidden_size=768, intermediate_size=3072, num_hidden_layers=2, num_attention_heads=12,
                          max_position_embeddings=2048, rope_scaling=None, rms_norm_eps=1e-6),
        # BASELINE cfg1 target: 68M-shaped target with a YaRN rope (SURVEY Appendix A)
        "tiny-yarn-target": dict(hidden_size=768, intermediate_size=3072, num_hidden_layers=2, num_attention_heads=12,
                                 max_position_embeddings=4096, rms_norm_eps=1e-6,
                                 rope_scaling={"type": "yarn", "factor": 2.0, "original_max_position_embeddings": 2048}),
        # BASELINE cfg3 analogue for the parity fixtures: 68M-shaped target with LWM's plain RoPE (large theta, no scaling)
        "tiny-plain-target": dict(hidden_size=768, intermediate_size=3072, num_hidden_layers=2, num_attention_heads=12,
                                  max_position_embeddings=4096, rms_norm_eps=1e-6, rope_scaling=None, rope_theta=10000000.0),
    }
    if name not in table:
        raise KeyError(f"unknown model shape {name!r}; known: {sorted(table)}")
    return LlamaShape(name=name, **table[name])


def yarn_mscale(scale: float) -> float:
    """reference models/modeling_llama.py:50-53"""
    if scale <= 1:
        return 1.0
    return 0.1 * math.log(scale) + 1.0
