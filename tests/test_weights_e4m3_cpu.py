"""E4M3 projection weights without a GPU: the quantization rule of tests/weights_e4m3_oracle.py (edge rows, exactness of
D = code * 2^e), the argument checks of the four C entry points, the refusals and the switches."""
from __future__ import annotations

import ctypes

import pytest
import torch

import weights_e4m3_oracle as wo
from triforce_b200 import _C


def _rows(*rows, K=64):
    w = torch.zeros((len(rows), K), dtype=torch.float16)
    for i, vals in enumerate(rows):
        w[i, : len(vals)] = torch.tensor(vals, dtype=torch.float16)
    return w


def test_zero_and_signed_zero_rows():
    w = _rows([], [-0.0, 0.0, -0.0])
    codes, e = wo.quantize(w)
    assert e.tolist() == [0, 0]
    assert torch.equal(wo.dequantize(codes, e).view(torch.int16), w.view(torch.int16))  # -0 stays -0


@pytest.mark.parametrize("e", [-15, -9, -1, 0, 1, 5, 7])
def test_amax_exactly_448_times_2e_and_one_ulp_above(e):
    at = _rows([448.0 * 2.0 ** e, -1.0 * 2.0 ** e])
    codes, ex = wo.quantize(at)
    assert int(ex[0]) == e and codes[0, 0].item() == 0x7E
    assert torch.equal(wo.dequantize(codes, ex), at)
    above = at.clone()
    above[0, 0] = torch.tensor(448.0 * 2.0 ** e, dtype=torch.float16).view(torch.int16).add(1).view(torch.float16)
    assert int(wo.row_exponent(above)[0]) == e + 1


def test_exponent_clamped_at_minus_15():
    # max|w| = 2^-10 would take e = -19 in the KV rule; the weight rule stops at -15, so the codes are small (some are e4m3
    # subnormals), and D = code * 2^-15 is still exact in fp16: its grid 2^-9 * 2^-15 is fp16's subnormal step, so these
    # rows (at most 4 significant bits) come back unchanged
    w = _rows([2.0 ** -10, 3 * 2.0 ** -14, -2.0 ** -20, 2.0 ** -24, 5 * 2.0 ** -24])
    codes, e = wo.quantize(w)
    assert int(e[0]) == -15 and int(wo.row_exponent(w[:, :1].repeat(1, 2))[0]) == -15
    assert int(codes[0, 3]) == 0x01  # 2^-24 / 2^-15 = 2^-9, the smallest e4m3 subnormal
    assert torch.equal(wo.dequantize(codes, e), w)  # dequantize also asserts that D is exact


def test_fp16_subnormals_only_row():
    w = _rows([2.0 ** -24, -3 * 2.0 ** -24, 2.0 ** -23])
    codes, e = wo.quantize(w)
    assert int(e[0]) == -15
    wo.dequantize(codes, e)


def test_largest_accepted_row_and_the_refused_ones():
    ok = _rows([61440.0, -61440.0, 1.0])
    codes, e = wo.quantize(ok)
    assert int(e[0]) == 8 and wo.dequantize(codes, e)[0, 0].item() == 61440.0
    for bad in ([61472.0], [65504.0], [float("inf")], [-float("inf")], [float("nan")]):
        w = _rows([1.0], bad)
        assert wo.refused_rows(w).tolist() == [False, True]
        with pytest.raises(ValueError):
            wo.quantize(w)


def test_d_is_exact_for_every_accepted_row():
    g = torch.Generator().manual_seed(0)
    scales = torch.exp2(torch.randint(-30, 16, (1024, 1), generator=g).double())
    w = (torch.randn(1024, 128, generator=g, dtype=torch.float64) * scales).clamp(-61440, 61440).half()
    codes, e = wo.quantize(w)
    assert int(e.min()) >= -15 and int(e.max()) <= 8
    d64 = wo.dequantize_exact(codes, e)
    assert torch.equal(d64.to(torch.float16).to(torch.float64), d64)
    amax = w.double().abs().amax(-1)
    nz = amax > 0
    assert bool((amax[nz] <= 448 * torch.exp2(e[nz].double())).all())
    # one e4m3 rounding per element: |D - w| <= half a code step (2^-4 relative for normal codes, 2^-10 * 2^e absolute below)
    err = (d64 - w.double()).abs()
    step = torch.maximum(w.double().abs() * 2.0 ** -3, 2.0 ** -9 * torch.exp2(e.double()).unsqueeze(-1))
    assert bool((err <= step / 2 + 0).all())


def test_weight_bytes_from_shapes():
    # 7B: 32 layers of q|k|v, o, gate|up, down and lm_head; codes are half the fp16 bytes and the exponents add a byte per row
    shapes = [(12288, 4096), (4096, 4096), (22016, 4096), (4096, 11008)]
    fp16 = 32 * sum(n * k * 2 for n, k in shapes) + 32000 * 4096 * 2
    e4m3 = 32 * sum(n * k + n for n, k in shapes) + 32000 * 4096 + 32000
    assert abs(fp16 / 1e9 - 13.21) < 0.01 and abs((fp16 - e4m3) / 1e9 - 6.61) < 0.01


def test_e4m3_weight_entry_points_check_their_arguments():
    lib = _C.lib()
    buf = (ctypes.c_uint8 * 512)()
    p = ctypes.addressof(buf)
    a = (p + 15) & ~15
    big = 1 << 30
    ws = lib.tf_stream_linear_workspace_bytes()
    # tf_weight_quantize_e4m3(W, row_stride, N, K, codes, codes_row_stride, exps, refused, stream)
    assert lib.tf_weight_quantize_e4m3(None, 64, 1, 64, a, 64, a, None, None) == -1
    assert lib.tf_weight_quantize_e4m3(a, 96, 1, 96, a, 96, a, None, None) == -1  # K % 64
    assert b"multiple" in lib.tf_last_error()
    assert lib.tf_weight_quantize_e4m3(a + 8, 64, 1, 64, a, 64, a, None, None) == -1  # misaligned W
    assert lib.tf_weight_quantize_e4m3(a, 64, 1, 64, a, 72, a, None, None) == -1  # codes stride % 16
    # tf_weight_dequantize_e4m3(codes, codes_row_stride, exps, N, K, D, d_row_stride, stream)
    assert lib.tf_weight_dequantize_e4m3(a, 64, None, 1, 64, a, 64, None) == -1
    assert lib.tf_weight_dequantize_e4m3(a, 64, a, 1, 0, a, 64, None) == -1
    assert lib.tf_weight_dequantize_e4m3(a, 64, a, 1, 64, a + 4, 64, None) == -1
    # tf_weight_tensormap_encode_e4m3(out, codes, N, K, row_stride)
    assert lib.tf_weight_tensormap_encode_e4m3(p, None, 16, 64, 64) == -1
    assert lib.tf_weight_tensormap_encode_e4m3(p, a, 16, 32, 32) == -1
    assert lib.tf_weight_tensormap_encode_e4m3(p, a, 16, 64, 72) == -1
    assert lib.tf_weight_tensormap_encode_e4m3(p, a + 8, 16, 64, 64) == -1
    # tf_stream_linear_e4m3(x, x_stride, wmap, w_exp, M, N, K, epilogue, y, y_stride, ws, ws_bytes, stream)
    assert lib.tf_stream_linear_e4m3(a, 64, p, None, 1, 16, 64, 0, a, 16, a, big, None) == -1
    assert b"NULL exponents" in lib.tf_last_error()
    assert lib.tf_stream_linear_e4m3(a, 64, p, a, 0, 16, 64, 0, a, 16, a, big, None) == -1
    assert lib.tf_stream_linear_e4m3(a, 64, p, a, 25, 16, 64, 0, a, 16, a, big, None) == -1
    assert b"M=25" in lib.tf_last_error()
    assert lib.tf_stream_linear_e4m3(a, 96, p, a, 1, 16, 96, 0, a, 16, a, big, None) == -1
    assert lib.tf_stream_linear_e4m3(a + 8, 64, p, a, 1, 16, 64, 0, a, 16, a, big, None) == -1  # misaligned x
    assert lib.tf_stream_linear_e4m3(a, 64, p, a, 1, 16, 64, 0, a, 16, a, ws - 1, None) == -1
    assert b"workspace" in lib.tf_last_error()
    for epi in (3, 4):
        assert lib.tf_stream_linear_e4m3(a, 64, p, a, 1, 16, 64, epi, a, 16, a, big, None) == -1
        assert b"epilogue" in lib.tf_last_error()
    assert lib.tf_stream_linear_e4m3(a, 64, p, a, 1, 15, 64, 1, a, 16, a, big, None) == -1  # odd N with SiLU


# ---------------------------------------------------------------------------------------------------------------------
# refusals and the switches (no device needed: every check runs before anything is allocated)
# ---------------------------------------------------------------------------------------------------------------------
def test_paths_that_keep_fp16_weights_refuse_e4m3(monkeypatch):
    from triforce_b200.config import named_config
    from triforce_b200.hf_compat import DraftLlamaForCausalLM
    from triforce_b200.llama import LlamaModel
    from triforce_b200.synth import retune_agreement
    from triforce_b200.tp import DistributedLlama

    cfg = named_config("llama-7B-128K")
    with pytest.raises(ValueError, match="weight_dtype"):
        LlamaModel(cfg, {}, device="cpu", weight_dtype="int8")
    with pytest.raises(NotImplementedError, match="tensor parallel"):
        LlamaModel(cfg, {}, device="cpu", tp_world=2, weight_dtype="e4m3")
    with pytest.raises(ValueError, match="draft"):
        LlamaModel(cfg, {}, device="cpu", is_draft=True, weight_dtype="e4m3")
    with pytest.raises(ValueError, match="draft"):
        DraftLlamaForCausalLM.from_pretrained("JackFram/llama-68m", weight_dtype="e4m3")
    monkeypatch.setenv("TRIFORCE_STREAM_LINEAR", "0")
    with pytest.raises(NotImplementedError, match="TRIFORCE_STREAM_LINEAR"):
        LlamaModel(cfg, {}, device="cpu", weight_dtype="e4m3")
    monkeypatch.delenv("TRIFORCE_STREAM_LINEAR")
    with pytest.raises(NotImplementedError, match="tensor parallel"):
        DistributedLlama("llama-7B-128K", weight_dtype="e4m3")
    model = object.__new__(LlamaModel)
    model.weight_dtype = "e4m3"
    with pytest.raises(NotImplementedError, match="retune_agreement"):
        retune_agreement(model, None, 0.5, 0.5, {})


def test_on_chip_takes_the_weight_dtype_switch():
    from triforce_b200.cli import build_parser

    assert build_parser("on_chip").parse_args([]).weight_dtype == "fp16"
    assert build_parser("on_chip").parse_args(["--weight_dtype", "e4m3"]).weight_dtype == "e4m3"
    with pytest.raises(SystemExit):
        build_parser("on_chip").parse_args(["--weight_dtype", "int4"])
