"""`utils/sampling.py` of the reference (norm_logits :43-60, sample :63-65, max_fn :68-75) on the fused CUDA kernels.
Same names, argument meaning and return shapes."""
from __future__ import annotations

import torch

from . import ops
from .rng import TorchNoise


def _top_k_mask_(logits: torch.Tensor, top_k: int) -> torch.Tensor:
    """sampling.py:16-18, in place: everything below the k-th largest logit of its row becomes -inf.  Off the hot path (the
    reference's loops always pass top_k = -1), so this one is a library call (ATen topk)."""
    kth = torch.topk(logits, min(int(top_k), logits.size(-1)))[0][:, [-1]]
    logits[logits < kth] = float("-inf")
    return logits


def top_k_top_p_filter(logits: torch.Tensor, top_k: int = 0, top_p: float = 0.0) -> torch.Tensor:
    """utils/sampling.py:5-27 — same signature and in-place semantics: returns `logits` [batch, vocab] with the filtered entries
    set to -inf.  The nucleus part is the sort-free kernel behind `norm_logits` (identical keep set: first crossing of top_p kept,
    ties in ascending index order): tokens it gives probability 0 are the removed ones."""
    assert logits.dim() == 2
    if top_k > 0:
        _top_k_mask_(logits, top_k)
    if top_p > 0.0:
        x = logits if (logits.dtype == torch.float32 and logits.stride(-1) == 1) else logits.float().contiguous()
        probs = ops.norm_logits(x, 1.0, float(top_p))
        logits[probs == 0] = float("-inf")
    return logits


def norm_logits(logits: torch.Tensor, temperature=0.6, top_k=-1, top_p=0.9) -> torch.Tensor:
    """logits [rows, vocab] fp32 → probabilities after temperature and nucleus filtering (one kernel, one CTA per row).
    top_k > 0 (never used by the reference's loops) masks with ATen first, then takes the same kernel.
    temperature 0 is greedy decoding: each row is one-hot at torch.argmax of its logits (top_k and top_p change nothing)."""
    assert logits.dim() == 2
    if logits.dtype != torch.float32:
        logits = logits.float()
    if logits.stride(-1) != 1:
        logits = logits.contiguous()
    if top_k is not None and top_k > 0:
        if temperature == 0:
            return ops.norm_logits(_top_k_mask_(logits.clone(), top_k), 0.0, float(top_p))
        return ops.norm_logits(_top_k_mask_(logits / temperature, top_k), 1.0, float(top_p))
    return ops.norm_logits(logits, float(temperature), float(top_p))


def sample(probs: torch.Tensor, num_samples=1, noise=None) -> torch.Tensor:
    """`torch.multinomial(probs, 1)` semantics on CUDA: argmax(p / Exp(1)).  The exponential noise is drawn with torch's
    generator exactly as ATen does (`empty_like(p).exponential_(1)`), so the Philox stream matches the reference's."""
    assert num_samples == 1
    noise = noise or TorchNoise(probs.device)
    p2 = probs.reshape(-1, probs.shape[-1])
    expo = torch.empty_like(p2)
    noise.exponential_into(expo)
    idx = ops.sample_argmax(p2, expo)
    return idx.reshape(*probs.shape[:-1], 1)


def max_fn(x: torch.Tensor) -> torch.Tensor:
    """norm(max(x, 0)) — the residual distribution of speculative sampling."""
    flat = x.reshape(-1).contiguous().float()
    return ops.residual_probs(flat, torch.zeros_like(flat)).reshape(x.shape)
