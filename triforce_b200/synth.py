"""Synthetic weights / prompts (there are no checkpoints or tokenizers offline).

Two generators:
  * ``numpy_state_dict``  – PCG64-seeded, bit-reproducible on any host; used for the small parity models so that the
    committed golden fixtures (made from the reference on CPU) and the GPU tests see identical weights.
  * ``cuda_state_dict``   – torch CUDA generator; used by ``bench.py`` for the 7B/13B-shaped random-init weights.

Names follow HF Llama checkpoints (what ``from_pretrained`` in the reference's ``test/on_chip.py:48-53`` loads), so a
real checkpoint's ``state_dict`` can be passed to the same loaders.
"""
from __future__ import annotations

from typing import Dict

import numpy as np
import torch

from .config import LlamaShape


def _param_shapes(cfg: LlamaShape):
    h, i, v = cfg.hidden_size, cfg.intermediate_size, cfg.vocab_size
    hkv = cfg.num_key_value_heads * cfg.head_dim  # == h for MHA
    yield "model.embed_tokens.weight", (v, h), "normal"
    for l in range(cfg.num_hidden_layers):
        p = f"model.layers.{l}."
        yield p + "self_attn.q_proj.weight", (h, h), "normal"
        yield p + "self_attn.k_proj.weight", (hkv, h), "normal"
        yield p + "self_attn.v_proj.weight", (hkv, h), "normal"
        yield p + "self_attn.o_proj.weight", (h, h), "normal"
        yield p + "mlp.gate_proj.weight", (i, h), "normal"
        yield p + "mlp.up_proj.weight", (i, h), "normal"
        yield p + "mlp.down_proj.weight", (h, i), "normal"
        yield p + "input_layernorm.weight", (h,), "ones"
        yield p + "post_attention_layernorm.weight", (h,), "ones"
    yield "model.norm.weight", (h,), "ones"
    yield "lm_head.weight", (v, h), "normal"


def numpy_state_dict(cfg: LlamaShape, seed: int = 0, std: float | None = None, lm_head_std: float | None = None,
                     norm_jitter: float = 0.0) -> Dict[str, torch.Tensor]:
    """fp16 CPU tensors, reproducible everywhere. ``lm_head_std`` lets tests sharpen the output distribution."""
    rng = np.random.Generator(np.random.PCG64(seed))
    std = cfg.initializer_range if std is None else std
    out = {}
    for name, shape, kind in _param_shapes(cfg):
        if kind == "ones":
            w = np.ones(shape, dtype=np.float32)
            if norm_jitter:
                w = w + norm_jitter * rng.standard_normal(shape, dtype=np.float32)
        else:
            s = lm_head_std if (lm_head_std is not None and name == "lm_head.weight") else std
            w = rng.standard_normal(shape, dtype=np.float32) * np.float32(s)
        out[name] = torch.from_numpy(w.astype(np.float16))
    return out


def cuda_state_dict(cfg: LlamaShape, seed: int = 0, device="cuda", std: float | None = None,
                    lm_head_std: float | None = None, host: bool = False) -> Dict[str, torch.Tensor]:
    """Seeded random-init weights drawn on `device`.  host=True moves each tensor to host memory as soon as it is drawn (the same
    values; the device holds one tensor at a time)."""
    if host:
        return {k: v.cpu() for k, v in _cuda_state_dict_iter(cfg, seed, device, std, lm_head_std)}
    return dict(_cuda_state_dict_iter(cfg, seed, device, std, lm_head_std))


def _cuda_state_dict_iter(cfg: LlamaShape, seed: int, device, std: float | None, lm_head_std: float | None):
    g = torch.Generator(device=device)
    g.manual_seed(seed)
    std = cfg.initializer_range if std is None else std
    for name, shape, kind in _param_shapes(cfg):
        if kind == "ones":
            yield name, torch.ones(shape, dtype=torch.float16, device=device)
        else:
            s = lm_head_std if (lm_head_std is not None and name == "lm_head.weight") else std
            w = torch.empty(shape, dtype=torch.float16, device=device)
            w.normal_(0.0, s, generator=g)
            yield name, w


def numpy_prompt(length: int, vocab: int = 32000, seed: int = 0) -> torch.Tensor:
    """``[1, length]`` int64 token ids, reproducible everywhere (SURVEY §8d: prompt = randint(0, 32000))."""
    rng = np.random.Generator(np.random.PCG64(seed))
    return torch.from_numpy(rng.integers(0, vocab, size=(1, length), dtype=np.int64))


def agreement_state_dicts(cfg_t: LlamaShape, cfg_d: LlamaShape, alpha_t: float, alpha_d: float, seed: int = 0, device="cuda"):
    """ACCEPTANCE-CALIBRATED synthetic weights (bench.py --weights agreement:a_t,a_d).

    Random-init weights of unrelated models give ~5 % speculative acceptance (a random 68M draft, a random 7B target
    and a 4K-of-125K retrieval cache have nothing in common), which measures the kernels but not the hierarchy.  This
    builds the SAME architectures, shapes and byte traffic with a controllable degree of agreement between the three
    levels: both models share one token table (the target's embedding / lm_head carry the draft's in their first
    `hidden_d` columns, rescaled so the RMS-normalised logits coincide), and every decoder layer's output projections
    (o_proj, down_proj) are scaled by alpha, so the layers — the only place where draft vs target and retrieval vs
    full attention can disagree — perturb the shared residual stream by a tunable amount.  alpha = 0 → the three levels
    agree exactly (acceptance → 1); alpha = 1 → ordinary random init.  Kernel work per step is identical in all cases."""
    hd, ht = cfg_d.hidden_size, cfg_t.hidden_size
    assert ht >= hd and cfg_t.vocab_size == cfg_d.vocab_size
    dsd = cuda_state_dict(cfg_d, seed=seed + 2, device=device)
    tsd = cuda_state_dict(cfg_t, seed=seed + 1, device=device)
    for sd, cfg, a in ((dsd, cfg_d, alpha_d), (tsd, cfg_t, alpha_t)):
        for l in range(cfg.num_hidden_layers):
            sd[f"model.layers.{l}.self_attn.o_proj.weight"].mul_(a)
            sd[f"model.layers.{l}.mlp.down_proj.weight"].mul_(a)
    emb = tsd["model.embed_tokens.weight"]
    emb.zero_()
    emb[:, :hd] = dsd["model.embed_tokens.weight"]
    head = tsd["lm_head.weight"]
    head.zero_()
    # rmsnorm over ht dims of a vector with hd non-zeros is sqrt(ht/hd) larger than the draft's normalised vector
    head[:, :hd] = (dsd["lm_head.weight"].float() * (hd / ht) ** 0.5).half()
    return tsd, dsd


def retune_agreement(target, draft, alpha_t: float, alpha_d: float, state: dict) -> None:
    """In-place version of `agreement_state_dicts` on two live `LlamaModel`s (bench.py's acceptance sweep): the first call moves
    the target onto the draft's token table, every call rescales the layers' output projections from the alpha they currently
    carry (`state`) to the requested one.  Shapes, buffers (and therefore TMA descriptors and captured graphs) stay as they
    are.  alpha can only go down to 0 once (0 cannot be scaled back up): sweep in descending order."""
    import torch

    if getattr(target, "weight_dtype", "fp16") != "fp16":
        raise NotImplementedError("retune_agreement rescales fp16 projection weights in place; this target stores them in "
                                  f"{target.weight_dtype}")
    hd, ht = draft.config.hidden_size, target.config.hidden_size
    with torch.no_grad():
        if not state.get("shared_table"):
            target.embed_tokens.zero_()
            target.embed_tokens[:, :hd] = draft.embed_tokens
            target.lm_head.zero_()
            # rmsnorm over ht dims of a vector with hd non-zeros is sqrt(ht/hd) larger than the draft's normalised vector
            target.lm_head[:, :hd] = (draft.lm_head.float() * (hd / ht) ** 0.5).half()
            state["shared_table"] = True
        for model, key, alpha in ((target, "alpha_t", alpha_t), (draft, "alpha_d", alpha_d)):
            cur = state.get(key, 1.0)
            if cur == 0.0 and alpha != 0.0:
                raise ValueError("retune_agreement: alpha was already 0 (sweep in descending order)")
            f = alpha / cur if cur != 0.0 else 0.0
            if f != 1.0:
                for w in model.layers:
                    w.wo.mul_(f)
                    w.wd.mul_(f)
            state[key] = alpha
