"""`from_pretrained`-style constructors so the reference's entry scripts keep their model-loading lines
(test/on_chip.py:48-53, test/offloading_TP.py:88-100).

Offline there are no checkpoints: a local directory with `*.safetensors` / `pytorch_model*.bin` (HF layout) is loaded if
it exists; otherwise pass `synthetic=True` (or set TRIFORCE_SYNTHETIC=1) to get seeded random-init weights of the
named architecture — what `bench.py` and the parity tests use.
"""
from __future__ import annotations

import glob
import os
from typing import Dict, Optional

import torch

from .config import LlamaShape, named_config
from .llama import LlamaModel
from .synth import cuda_state_dict

_HUB_TO_SHAPE = {
    "NousResearch/Yarn-Llama-2-7b-128k": "llama-7B-128K",
    "NousResearch/Yarn-Llama-2-13b-128k": "llama-13B-128K",
    "LargeWorldModel/LWM-Text-Chat-128K": "lwm-128K",
    "LargeWorldModel/LWM-Text-128K": "lwm-128K",
    "JackFram/llama-68m": "llama-68M",
}


def _load_local_checkpoint(path: str) -> Dict[str, torch.Tensor]:
    sd: Dict[str, torch.Tensor] = {}
    files = sorted(glob.glob(os.path.join(path, "*.safetensors")))
    if files:
        from safetensors.torch import load_file
        for f in files:
            sd.update(load_file(f))
        return sd
    files = sorted(glob.glob(os.path.join(path, "pytorch_model*.bin")))
    if not files:
        raise FileNotFoundError(f"no *.safetensors or pytorch_model*.bin under {path}")
    for f in files:
        sd.update(torch.load(f, map_location="cpu"))
    return sd


def shape_from_hf_config(path: str, gqa_retrieval: Optional[str] = None) -> LlamaShape:
    """`LlamaShape` from an HF checkpoint directory's config.json (the fields the reference reads off `LlamaConfig`).
    A grouped-query checkpoint needs `gqa_retrieval` (see LlamaShape.gqa_retrieval); without it, it is refused."""
    import json
    with open(os.path.join(path, "config.json")) as f:
        c = json.load(f)
    rs = c.get("rope_scaling")
    if rs is not None:
        kind = rs.get("type", rs.get("rope_type"))
        if kind in (None, "default"):
            rs = None
        elif kind == "yarn":
            rs = {"type": "yarn", "factor": float(rs["factor"]),
                  "original_max_position_embeddings": int(rs.get("original_max_position_embeddings", c.get("max_position_embeddings", 4096)))}
        else:
            raise ValueError(f"{path}: rope_scaling type {kind!r} is not supported (reference: yarn or none, modeling_llama.py:176-198)")
    return LlamaShape(hidden_size=c["hidden_size"], intermediate_size=c["intermediate_size"], num_hidden_layers=c["num_hidden_layers"],
                      num_attention_heads=c["num_attention_heads"], num_key_value_heads=c.get("num_key_value_heads"),
                      vocab_size=c["vocab_size"], max_position_embeddings=c.get("max_position_embeddings", 4096),
                      rms_norm_eps=c.get("rms_norm_eps", 1e-5), rope_theta=float(c.get("rope_theta", 10000.0)), rope_scaling=rs,
                      name=c.get("_name_or_path") or os.path.basename(os.path.normpath(path)), gqa_retrieval=gqa_retrieval)


def _device_from_map(device_map) -> torch.device:
    if device_map is None:
        return torch.device("cuda", torch.cuda.current_device())
    if isinstance(device_map, dict):
        device_map = next(iter(device_map.values()))
    return torch.device(device_map)


class _Factory:
    is_draft = False

    @classmethod
    def from_pretrained(cls, name_or_path: str, torch_dtype=torch.float16, device_map=None, synthetic=None, seed: int = 0,
                        config: LlamaShape = None, gqa_retrieval: Optional[str] = None, weight_dtype: str = "fp16", **kw) -> LlamaModel:
        """weight_dtype="e4m3": the target's projection weights in FP8 E4M3 (see LlamaModel); the draft stays fp16."""
        if torch_dtype not in (None, torch.float16):
            raise ValueError("the TriForce hot path is fp16 (reference: torch_dtype=torch.float16)")
        if weight_dtype not in ("fp16", "e4m3"):
            raise ValueError(f"weight_dtype must be 'fp16' or 'e4m3', got {weight_dtype!r}")
        if weight_dtype != "fp16" and cls.is_draft:
            raise ValueError("the draft keeps fp16 weights (weight_dtype='e4m3' is for the target)")
        is_dir = os.path.isdir(name_or_path)
        if config is not None:
            shape = config
        elif is_dir:  # a local checkpoint: its own config.json describes it (hub ids are resolved by name)
            shape = shape_from_hf_config(name_or_path, gqa_retrieval=gqa_retrieval)
        else:
            shape = named_config(_HUB_TO_SHAPE.get(name_or_path, name_or_path))
        if (gqa_retrieval is not None and shape.num_key_value_heads != shape.num_attention_heads
                and gqa_retrieval != shape.gqa_retrieval):
            raise ValueError(f"{name_or_path}: gqa_retrieval={gqa_retrieval!r} conflicts with the shape's rule {shape.gqa_retrieval!r}")
        dev = _device_from_map(device_map)
        if synthetic is None:
            synthetic = os.environ.get("TRIFORCE_SYNTHETIC", "0") == "1"
        if synthetic:
            print(f"[triforce_b200] {name_or_path}: SYNTHETIC seeded random-init weights (seed {seed}), not a checkpoint", flush=True)
            sd = cuda_state_dict(shape, seed=seed, device=dev)
        elif is_dir:
            sd = _load_local_checkpoint(name_or_path)
        else:
            raise FileNotFoundError(f"{name_or_path}: not a local checkpoint directory and there is no network (HF_HUB_OFFLINE); "
                                    "pass synthetic=True or set TRIFORCE_SYNTHETIC=1 for seeded random-init weights")
        return cls._make(shape, sd, dev, weight_dtype)

    @classmethod
    def _make(cls, shape, sd, dev, weight_dtype="fp16"):
        return LlamaModel(shape, sd, device=dev, is_draft=cls.is_draft, weight_dtype=weight_dtype)


class TargetLlamaForCausalLM(_Factory):
    is_draft = False


class DraftLlamaForCausalLM(_Factory):
    is_draft = True
