"""CPU-side checks of the Sequoia tree path over an E4M3 full-KV store and E4M3 weights: the argument checks of
tf_tree_attn_tc_e4m3 and tf_kv_compact_e4m3 (no launch), SingleGpuLlama's formats and refusals, the E4M3 tree verify's refusal
of shapes off the wgmma kernel, and the offloading_seqouia switches.  No device is needed: every check runs before anything is
allocated."""
import ctypes
from types import SimpleNamespace

import pytest
import torch

from triforce_b200 import _C


def _buf():
    buf = (ctypes.c_uint8 * 512)()
    p = ctypes.addressof(buf)
    return buf, p, (p + 15) & ~15


def test_tree_attn_tc_e4m3_checks_its_arguments():
    lib = _C.lib()
    _keep, p, a = _buf()
    f = lib.tf_tree_attn_tc_e4m3
    # (q, kmap, vmap, k_exp, v_exp, cap, layer, kv_len, R, Hq, Hkv, d, scale, mask, tree_cols, out, ws, ws_bytes, stream)
    R, H, S, cap = 512, 40, 4096, 4160
    ws = lib.tf_tree_attn_tc_workspace_bytes(R, H, S)
    assert f(a, p, p, None, a, cap, 0, S, R, H, H, 128, 0.1, p, 512, p, a, ws, None) == -1
    assert b"NULL exponent" in lib.tf_last_error()
    assert f(a, p, p, a, a, cap, 0, S, R, H, H, 64, 0.1, p, 512, p, a, ws, None) == -2                   # head_dim 64
    assert f(a, p, p, a, a, cap, 0, S, R, H, H, 128, 0.1, p, 500, p, a, ws, None) == -1                  # tree_cols % 32
    assert b"multiple of 32" in lib.tf_last_error()
    assert f(a, p, p, a, a, cap, 0, S, R, H, H, 128, 0.1, p, 512, p, a, ws - 1, None) == -1              # workspace 1 B short
    assert b"workspace" in lib.tf_last_error()
    assert f(a, p, p, a + 1, a, cap, 0, S, R, H, H, 128, 0.1, p, 512, p, a, ws, None) == -1              # misaligned exponents
    assert b"16-byte aligned" in lib.tf_last_error()
    assert f(a, p, p, a, a, 4100, 0, S, R, H, H, 128, 0.1, p, 512, p, a, ws, None) == -1                 # cap % 64
    assert b"cap" in lib.tf_last_error()
    assert f(a, p, p, a, a, 4032, 0, S, R, H, H, 128, 0.1, p, 512, p, a, ws, None) == -1                 # kv_len > cap
    assert b"exceeds cap" in lib.tf_last_error()
    assert f(a, p, p, a, a, cap, 0, S, R, 40, 6, 128, 0.1, p, 512, p, a, ws, None) == -1                 # Hq % Hkv
    # grouped-query heads and the exact workspace pass; the call stops at the next check (a misaligned q), before any launch
    assert f(a + 2, p, p, a, a, cap, 0, S, R, 32, 8, 128, 0.1, p, 512, p, a, ws, None) == -1
    assert b"q must be 16-byte aligned" in lib.tf_last_error()


def test_kv_compact_e4m3_checks_its_arguments():
    lib = _C.lib()
    _keep, p, a = _buf()
    f = lib.tf_kv_compact_e4m3
    # (k_codes, v_codes, k_exp, v_exp, cap, n_layers, H, d, src_idx, n, dst_start, stream)
    assert f(a, a, None, a, 1024, 2, 8, 128, p, 4, 0, None) == -1
    assert b"NULL exponent" in lib.tf_last_error()
    assert f(a, a, a, a, 1024, 2, 8, 96, p, 4, 0, None) == -1                                             # head_dim 96
    assert f(a, a, a, a, 1024, 2, 8, 128, p, 4, 1021, None) == -1                                        # past cap
    assert b"outside" in lib.tf_last_error()
    assert f(a, a, a, a, 1024, 2, 8, 128, p, 400, 0, None) == -2                                         # > 48 KB staged
    assert f(a, a, a, a, 1024, 2, 8, 128, p, 0, 5, None) == 0                                            # nothing to move


def test_tree_verify_over_an_e4m3_store_refuses_other_kernels(monkeypatch):
    from triforce_b200.llama import LlamaModel

    kv = SimpleNamespace(kv_dtype="e4m3")
    model = object.__new__(LlamaModel)
    model.local_num_heads, model.head_dim = 32, 128
    with pytest.raises(NotImplementedError, match="multiple of 128 tree rows"):
        model.forward_tree_verify(torch.zeros(96, dtype=torch.long), kv, None, None)
    model.head_dim = 64
    with pytest.raises(NotImplementedError, match="head_dim 64"):
        model.forward_tree_verify(torch.zeros(512, dtype=torch.long), kv, None, None)
    model.head_dim = 128
    monkeypatch.setenv("TRIFORCE_TREE_TC", "0")
    with pytest.raises(NotImplementedError, match="TRIFORCE_TREE_TC=0"):
        model.forward_tree_verify(torch.zeros(512, dtype=torch.long), kv, None, None)


def test_single_gpu_llama_takes_the_e4m3_formats():
    from triforce_b200.tp import DistributedLlama, SingleGpuLlama

    llm = SingleGpuLlama("llama-13B-128K", kv_dtype="e4m3", weight_dtype="e4m3", tree_size=512)
    assert (llm.kv_dtype, llm.weight_dtype, llm.world_size) == ("e4m3", "e4m3", 1) and llm.e4m3_formats
    assert not DistributedLlama.e4m3_formats
    with pytest.raises(NotImplementedError, match="one GPU"):
        SingleGpuLlama("llama-13B-128K", world_size=2, kv_dtype="e4m3")
    with pytest.raises(ValueError, match="kv_dtype"):
        SingleGpuLlama("llama-13B-128K", kv_dtype="int8")
    with pytest.raises(ValueError, match="weight_dtype"):
        SingleGpuLlama("llama-13B-128K", weight_dtype="fp8")


def test_offloading_seqouia_takes_the_dtype_switches():
    from triforce_b200.cli import build_parser

    args = build_parser("offloading_seqouia").parse_args([])
    assert (args.kv_dtype, args.weight_dtype) == ("fp16", "fp16")
    args = build_parser("offloading_seqouia").parse_args(["--kv_dtype", "e4m3", "--weight_dtype", "e4m3", "--prefill", "130048"])
    assert (args.kv_dtype, args.weight_dtype, args.prefill) == ("e4m3", "e4m3", 130048)
    for flag in ("--kv_dtype", "--weight_dtype"):
        with pytest.raises(SystemExit):
            build_parser("offloading_seqouia").parse_args([flag, "int8"])
    # offloading_TP keeps its fp16 full store and weights (its engine runs under tensor parallelism)
    assert not hasattr(build_parser("offloading_TP").parse_args([]), "kv_dtype")
