"""The E4M3 projection-weight format, restated on the CPU (include/triforce_b200.h, csrc/stream_linear.cu).

Each row w of a projection matrix W [N, K] (one output feature) is stored as
    e    = max(-15, the smallest integer with max|w| <= 448 * 2^e)   (0 for an all-zero row)
    code = e4m3_rn(w / 2^e)                                         (round to nearest even; exact division)
and stands for D = code * 2^e.  With e >= -15 and codes multiples of 2^-9 with at most 4 significant bits, D is an exact fp16
value: nothing rounds.  Rows that are not finite or have max|w| > 61440 = 240 * 2^8 are refused.  This is the rule of the E4M3
KV store (kv_e4m3_oracle) with the exponent clamped below.
"""
from __future__ import annotations

import torch

import kv_e4m3_oracle as kvo

E_MIN = -15
W_MAX = 61440.0  # 240 * 2^8: above it D can round past the fp16 maximum


def refused_rows(w: torch.Tensor) -> torch.Tensor:
    """bool [N]: rows loading refuses (not finite, or max|w| > W_MAX)."""
    w64 = w.detach().cpu().to(torch.float64)
    return ~torch.isfinite(w64).all(dim=-1) | (w64.abs().amax(dim=-1) > W_MAX)


def row_exponent(w: torch.Tensor) -> torch.Tensor:
    """int8 [N] exponents of accepted fp16 rows w [N, K]."""
    return kvo.row_exponent(w.cpu()).clamp(min=E_MIN)


def quantize(w: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """fp16 W [N, K] -> (codes uint8 [N, K], exponents int8 [N]).  Raises ValueError on a refused row."""
    assert w.dtype == torch.float16 and w.dim() == 2
    bad = refused_rows(w)
    if bool(bad.any()):
        raise ValueError(f"{int(bad.sum())} rows cannot be stored in E4M3")
    e = row_exponent(w)
    scaled = w.detach().cpu().to(torch.float64) * torch.exp2(-e.to(torch.float64)).unsqueeze(-1)
    assert scaled.abs().max() <= kvo.E4M3_MAX if scaled.numel() else True
    codes = scaled.to(torch.float32).to(torch.float8_e4m3fn).view(torch.uint8)
    return codes, e


def dequantize_exact(codes: torch.Tensor, e: torch.Tensor) -> torch.Tensor:
    """D = code * 2^e in float64 (no rounding)."""
    c = codes.cpu().view(torch.float8_e4m3fn).to(torch.float64)
    return c * torch.exp2(e.cpu().to(torch.float64)).unsqueeze(-1)


def dequantize(codes: torch.Tensor, e: torch.Tensor) -> torch.Tensor:
    """D as fp16 [N, K]; asserts that the cast is exact."""
    d64 = dequantize_exact(codes, e)
    d16 = d64.to(torch.float16)
    assert torch.equal(d16.to(torch.float64), d64), "D is not an exact fp16 value"
    return d16
