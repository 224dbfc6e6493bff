"""Grouped-query-attention targets on the CPU tier: the shape checks and the named GQA geometry, loading a GQA
config.json, the shard algebra of q/k/v, the "group_sum" retrieval rule (tests/gqa_oracle.py) and the argument checks of
the new C entry points (no launch)."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

import golden_inputs as gi
import gqa_oracle
from oracle import triforce_oracle as orc
from triforce_b200 import _C
from triforce_b200.config import LlamaShape, named_config
from triforce_b200.hf_compat import shape_from_hf_config
from triforce_b200.llama import shard_layer_weights
from triforce_b200.synth import numpy_state_dict


# ---------------------------------------------------------------------------------------------------------------------
# configuration
# ---------------------------------------------------------------------------------------------------------------------
def test_gqa_shape_needs_a_retrieval_rule():
    with pytest.raises(ValueError, match="MHA-only"):
        LlamaShape(num_attention_heads=32, num_key_value_heads=8)
    s = LlamaShape(num_attention_heads=32, num_key_value_heads=8, gqa_retrieval="group_sum")
    assert s.num_key_value_heads == 8 and s.head_dim == 128
    with pytest.raises(ValueError, match="multiple"):
        LlamaShape(num_attention_heads=32, num_key_value_heads=6, gqa_retrieval="group_sum")
    with pytest.raises(ValueError, match="unknown gqa_retrieval"):
        LlamaShape(num_attention_heads=32, num_key_value_heads=8, gqa_retrieval="max")
    # MHA: the field is ignored, and the shape is what it was
    assert LlamaShape(gqa_retrieval="anything").num_key_value_heads == 32
    assert LlamaShape().param_count() == LlamaShape(gqa_retrieval="group_sum").param_count()


def test_named_gqa_shape():
    s = named_config("llama-7B-gqa8-128K")
    ref = named_config("llama-7B-128K")
    assert (s.num_attention_heads, s.num_key_value_heads, s.head_dim) == (32, 8, 128)
    assert (s.hidden_size, s.num_hidden_layers, s.vocab_size, s.intermediate_size) == (4096, 32, 32000, 14336)
    assert s.rope_scaling == ref.rope_scaling and s.max_position_embeddings == ref.max_position_embeddings
    assert s.gqa_retrieval == "group_sum"
    assert s.kv_bytes_per_token_layer() == 8 * 128 * 2 * 2 == 4096
    assert ref.kv_bytes_per_token_layer() == 4 * s.kv_bytes_per_token_layer()
    h, i, L, v, kv = 4096, 14336, 32, 32000, 8 * 128
    assert s.param_count() == 2 * v * h + L * (2 * h * h + 2 * kv * h + 3 * h * i + 2 * h) + h


def test_from_pretrained_refuses_a_conflicting_rule():
    from triforce_b200.hf_compat import TargetLlamaForCausalLM
    s = named_config("llama-7B-gqa8-128K")
    with pytest.raises(ValueError, match="conflicts"):
        TargetLlamaForCausalLM.from_pretrained("x", config=s, gqa_retrieval="max")


def test_shape_from_hf_config_gqa(tmp_path):
    cfg = {"hidden_size": 4096, "intermediate_size": 14336, "num_hidden_layers": 32, "num_attention_heads": 32,
           "num_key_value_heads": 8, "vocab_size": 32000, "max_position_embeddings": 131072, "rms_norm_eps": 1e-5,
           "rope_theta": 10000.0, "rope_scaling": {"type": "yarn", "factor": 32.0, "original_max_position_embeddings": 4096}}
    (tmp_path / "config.json").write_text(json.dumps(cfg))
    with pytest.raises(ValueError, match="MHA-only"):
        shape_from_hf_config(str(tmp_path))
    s = shape_from_hf_config(str(tmp_path), gqa_retrieval="group_sum")
    assert s.num_key_value_heads == 8 and s.gqa_retrieval == "group_sum"
    assert s.rope_scaling == named_config("llama-7B-gqa8-128K").rope_scaling


# ---------------------------------------------------------------------------------------------------------------------
# weights
# ---------------------------------------------------------------------------------------------------------------------
def _small_gqa(Hq=8, Hkv=4):
    return LlamaShape(hidden_size=64 * Hq, intermediate_size=256, num_hidden_layers=1, num_attention_heads=Hq,
                      num_key_value_heads=Hkv, vocab_size=64, max_position_embeddings=64, gqa_retrieval="group_sum")


def test_synthetic_state_dict_shapes():
    s = _small_gqa(8, 2)
    sd = numpy_state_dict(s, seed=3)
    assert sd["model.layers.0.self_attn.q_proj.weight"].shape == (512, 512)
    assert sd["model.layers.0.self_attn.k_proj.weight"].shape == (128, 512)
    assert sd["model.layers.0.self_attn.v_proj.weight"].shape == (128, 512)


@pytest.mark.parametrize("world", [2, 4])
def test_gqa_shards_concatenate_to_the_fused_weight(world):
    s = _small_gqa(8, 4)
    sd = numpy_state_dict(s, seed=5)
    d, Hq, Hkv = s.head_dim, 8, 4
    p = "model.layers.0."
    full, _, _, _ = shard_layer_weights(sd, s, 0, 0, 1)
    assert full.shape == ((Hq + 2 * Hkv) * d, s.hidden_size)
    parts = [shard_layer_weights(sd, s, 0, r, world)[0] for r in range(world)]
    qn, kn = Hq * d // world, Hkv * d // world
    for r, w in enumerate(parts):
        assert w.shape == (qn + 2 * kn, s.hidden_size)
        assert torch.equal(w[:qn], sd[p + "self_attn.q_proj.weight"][r * qn:(r + 1) * qn])
        assert torch.equal(w[qn:qn + kn], sd[p + "self_attn.k_proj.weight"][r * kn:(r + 1) * kn])
        assert torch.equal(w[qn + kn:], sd[p + "self_attn.v_proj.weight"][r * kn:(r + 1) * kn])
    # the q, k and v blocks of the shards, concatenated over ranks, give the unsharded [q | k | v]
    q = torch.cat([w[:qn] for w in parts]); k = torch.cat([w[qn:qn + kn] for w in parts]); v = torch.cat([w[qn + kn:] for w in parts])
    assert torch.equal(torch.cat([q, k, v]), full)


def test_kv_heads_must_divide_the_world():
    s = _small_gqa(8, 2)
    sd = numpy_state_dict(s, seed=1)
    with pytest.raises(ValueError, match="key/value heads"):
        shard_layer_weights(sd, s, 0, 0, 4)


# ---------------------------------------------------------------------------------------------------------------------
# the "group_sum" retrieval rule
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", gi.RETRIEVAL_CASES, ids=[c[0] for c in gi.RETRIEVAL_CASES])
def test_group_rule_at_g1_is_the_mha_build(case, golden_dir):
    """G = 1: every output of the rule equals the MHA oracle's bit for bit, which the golden test pins to the reference."""
    name, H, d, P, chunk, budget, seed = case
    K, V, q = gi.retrieval_inputs(case)
    want = orc.retrieval_build(K, V, q, P, chunk, budget)
    got = gqa_oracle.retrieval_build_group_sum(K, V, q, P, chunk, budget)
    for a, b in zip(got, want):
        assert a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))
    ref_scores = np.load(os.path.join(golden_dir, "retrieval_build.npz"))[f"{name}.scores_rest"]
    ulp = got[3][:, 1:].view(np.int16).astype(np.int32) - ref_scores.view(np.int16).astype(np.int32)
    assert np.abs(ulp).max() <= 1


def test_group_rule_picks_the_chunk_the_group_agrees_on():
    """Two query heads over one KV head: head 0 alone ranks chunk 1 first, head 1 alone chunk 2; chunk 3 is second for
    both, and its summed score wins."""
    d, chunk = 8, 1
    e0, e1 = np.eye(d, dtype=np.float32)[0], np.eye(d, dtype=np.float32)[1]
    K = np.stack([0 * e0, 4 * e0 - 2 * e1, -2 * e0 + 4 * e1, 2.5 * e0 + 2.5 * e1])[:, None, :].astype(np.float16)
    q = np.stack([e0, e1]).astype(np.float16)
    per_head = [orc.retrieval_build(K, K, q[h:h + 1], 4, chunk, 2)[2][0, 1] for h in range(2)]
    assert per_head == [1, 2]
    _, _, idx, scores = gqa_oracle.retrieval_build_group_sum(K, K, q, 4, chunk, 2)
    assert idx.tolist() == [[0, 3]]
    assert scores.astype(np.float32).tolist() == [[0.0, 2.0, 2.0, 5.0]]


# ---------------------------------------------------------------------------------------------------------------------
# C ABI (argument checks only)
# ---------------------------------------------------------------------------------------------------------------------
def test_gqa_entry_points_check_their_arguments():
    lib = _C.lib()
    buf = (ctypes.c_uint8 * 256)()
    p = ctypes.addressof(buf)
    ws = lib.tf_verify_attn_gqa_workspace_bytes(8, 32, 8, 128)
    assert ws == lib.tf_verify_attn_workspace_bytes(8, 8, 128)
    assert lib.tf_verify_attn_gqa_workspace_bytes(8, 30, 8, 128) == 0
    big = 1 << 30
    # tf_verify_attn_gqa(q, kmap, vmap, layer, kv_len, kv_len_dev, kv_len_max, R, Hq, Hkv, d, scale, out, ws, ws_bytes, variant, clean, stream)
    assert lib.tf_verify_attn_gqa(p, p, p, 0, 64, None, 64, 9, 32, 8, 128, 0.1, p, p, big, 0, 0, None) == -1  # R·G = 36 > 32
    assert b"packed rows" in lib.tf_last_error()
    assert lib.tf_verify_attn_gqa(p, p, p, 0, 64, None, 64, 1, 64, 1, 128, 0.1, p, p, big, 0, 0, None) == -1  # G = 64
    assert lib.tf_verify_attn_gqa(p, p, p, 0, 64, None, 64, 4, 30, 8, 128, 0.1, p, p, big, 0, 0, None) == -1  # Hq % Hkv
    assert b"multiple" in lib.tf_last_error()
    assert lib.tf_verify_attn_gqa(p, p, p, 0, 64, None, 64, 8, 32, 8, 128, 0.1, p, p, ws - 1, 0, 0, None) == -1  # short ws
    assert b"workspace" in lib.tf_last_error()
    assert lib.tf_verify_attn_gqa(p, p, p, 0, 64, None, 64, 8, 32, 8, 96, 0.1, p, p, big, 0, 0, None) == -2  # head_dim 96
    tree = (p, 32)  # tree_mask, tree_cols
    assert lib.tf_verify_attn_tree_gqa(p, p, p, 0, 64, None, 64, 9, 32, 8, 128, 0.1, *tree, p, p, big, None) == -1
    assert lib.tf_verify_attn_tree_gqa(p, p, p, 0, 64, None, 64, 4, 30, 8, 128, 0.1, *tree, p, p, big, None) == -1
    assert lib.tf_verify_attn_tree_gqa(p, p, p, 0, 64, None, 64, 8, 32, 8, 128, 0.1, *tree, p, p, ws - 1, None) == -1
    assert lib.tf_verify_attn_tree_gqa(p, p, p, 0, 64, None, 64, 8, 32, 8, 96, 0.1, *tree, p, p, big, None) == -2
    # tf_tree_attn_tc_gqa(q, kmap, vmap, layer, kv_len, R, Hq, Hkv, d, scale, mask, cols, causal, out, ws, ws_bytes, stream)
    a = (p + 15) & ~15
    tcw = lib.tf_tree_attn_tc_workspace_bytes(128, 32, 4096)
    assert lib.tf_tree_attn_tc_gqa(p, p, p, 0, 4096, 128, 30, 8, 128, 0.1, None, 0, 1, p, a, tcw, None) == -1
    assert lib.tf_tree_attn_tc_gqa(p, p, p, 0, 4096, 128, 32, 8, 96, 0.1, None, 0, 1, p, a, tcw, None) == -2
    assert lib.tf_tree_attn_tc_gqa(p, p, p, 0, 4096, 128, 32, 8, 128, 0.1, None, 0, 1, p, a, tcw - 1, None) == -1
    # tf_rope_append_gqa(q, k, v, stride, cos, sin, max_pos, pos_ids, pos0, pos0_dev, slot0, slot0_dev, R, Hq, Hkv, d, ...)
    assert lib.tf_rope_append_gqa(p, p, p, 8, p, p, 4, None, 0, None, 0, None, 1, 30, 8, 128, 1, 1, p, p, p, 128, 4, None) == -1
    assert lib.tf_rope_append_gqa(p, p, p, 8, p, p, 4, None, 0, None, 0, None, 1, 32, 8, 96, 1, 1, p, p, p, 128, 4, None) == -2
    # tf_retrieval_build_gqa: Hq % Hkv, and more than 64 query heads per KV head
    assert lib.tf_retrieval_build_gqa(p, p, 8, 8, p, 1, 30, 8, 128, 64, 8, 8, p, p, 8, 8, None, None, p, 64, None) == -1
    assert lib.tf_retrieval_build_gqa(p, p, 8, 8, p, 1, 128, 1, 128, 64, 8, 8, p, p, 8, 8, None, None, p, 64, None) == -1
    assert lib.tf_retrieval_build_gqa(p, p, 8, 8, p, 1, 32, 8, 96, 64, 8, 8, p, p, 8, 8, None, None, p, 64, None) == -2
