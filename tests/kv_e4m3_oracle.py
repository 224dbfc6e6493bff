"""The E4M3 full-KV store format, restated on the CPU (include/triforce_b200.h, csrc/common.cuh).

A row x of d fp16 values (K after RoPE, or V) is stored as
    e    = the smallest integer with max|x| <= 448 * 2^e   (0 for an all-zero row; in [-32, 8] for finite fp16 x)
    code = e4m3_rn(x / 2^e)                               (round to nearest even; exact division, nothing saturates)
and stands for D = fp16_rn(code * 2^e).  Every kernel that reads the store computes what its fp16 counterpart computes on D.
torch's CPU cast to float8_e4m3fn rounds to nearest even, ties and e4m3 subnormals included, so it serves as e4m3_rn.
"""
from __future__ import annotations

import torch

E4M3_MAX = 448.0


def row_exponent(x: torch.Tensor) -> torch.Tensor:
    """int8 [...] exponents of fp16 rows x [..., d]."""
    amax = x.detach().to(torch.float64).abs().amax(dim=-1)
    e = torch.ceil(torch.log2(amax / E4M3_MAX)).clamp(min=-200)
    # log2 of a ratio of exact values can land one off at a power-of-two boundary: settle e against the definition
    e = torch.where(amax > E4M3_MAX * torch.exp2(e), e + 1, e)
    e = torch.where(amax <= E4M3_MAX * torch.exp2(e - 1), e - 1, e)
    return torch.where(amax > 0, e, torch.zeros_like(e)).to(torch.int8)


def quantize(x: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """fp16 rows [..., d] -> (codes uint8 [..., d], exponents int8 [...])."""
    assert x.dtype == torch.float16
    e = row_exponent(x)
    scaled = x.detach().cpu().to(torch.float64) * torch.exp2(-e.cpu().to(torch.float64)).unsqueeze(-1)
    assert scaled.abs().max() <= E4M3_MAX if scaled.numel() else True
    codes = scaled.to(torch.float32).to(torch.float8_e4m3fn).view(torch.uint8)
    return codes, e.cpu()


def dequantize(codes: torch.Tensor, e: torch.Tensor) -> torch.Tensor:
    """(codes uint8 [..., d], exponents int8 [...]) -> D fp16 [..., d]."""
    c = codes.cpu().view(torch.float8_e4m3fn).to(torch.float64)
    return (c * torch.exp2(e.cpu().to(torch.float64)).unsqueeze(-1)).to(torch.float16)


def roundtrip(x: torch.Tensor) -> torch.Tensor:
    """D of the fp16 rows x."""
    return dequantize(*quantize(x))
