"""Pins `oracle/triforce_oracle.py` (the numpy restatement) against the committed golden fixtures, which are outputs of
the REFERENCE's own code run on CPU (`tests/golden/make_golden.py`).  Runs without a GPU."""
import json
import os

import numpy as np
import pytest

import golden_inputs as gi
from oracle import triforce_oracle as orc
from triforce_b200.config import named_config
from triforce_b200.rng import CounterNoise
from triforce_b200.synth import numpy_prompt, numpy_state_dict


def _canon(scores_rest, idx):
    """Sort a reference top-k result to the canonical order (descending score, ascending index)."""
    key = orc._sortable_u16(scores_rest[idx - 1]).astype(np.int64)
    return idx[np.lexsort((idx, -key))]


@pytest.mark.parametrize("case", gi.RETRIEVAL_CASES, ids=[c[0] for c in gi.RETRIEVAL_CASES])
def test_retrieval_build_matches_reference(case, golden_dir):
    name, H, d, P, chunk, budget, seed = case
    g = np.load(os.path.join(golden_dir, "retrieval_build.npz"))
    ref_scores, ref_idx = g[f"{name}.scores_rest"], g[f"{name}.topk_idx_rest"]
    K, V, q = gi.retrieval_inputs(case)
    rK, rV, idx, scores = orc.retrieval_build(K, V, q, P, chunk, budget)
    # scores: the reference's fp32-accumulated fp16 matmul vs the oracle's correctly rounded value: <= 1 ulp, rarely
    ulp = scores[:, 1:].view(np.int16).astype(np.int32) - ref_scores.view(np.int16).astype(np.int32)
    assert np.abs(ulp).max() <= 1 and (ulp != 0).mean() < 5e-3
    # selection applied to the REFERENCE's scores must reproduce the reference's indices exactly (canonical order)
    idx_on_ref = orc.topk_chunks(np.concatenate([np.zeros((H, 1), np.float16), ref_scores], 1), budget // chunk)
    for h in range(H):
        assert set(idx_on_ref[h, 1:]) == set(ref_idx[h]) or _tie_only_difference(ref_scores[h], idx_on_ref[h, 1:], ref_idx[h])
        vals = ref_scores[h][idx_on_ref[h, 1:] - 1].astype(np.float32)
        assert np.all(np.diff(vals) <= 0)  # descending
        np.testing.assert_array_equal(np.sort(ref_scores[h][ref_idx[h] - 1]), np.sort(ref_scores[h][idx_on_ref[h, 1:] - 1]))
    assert (idx[:, 0] == 0).all()
    # gathered rows: digest of the reference cache == digest of the oracle's gather driven by the reference's order
    ref_order = np.concatenate([np.zeros((H, 1), np.int32), ref_idx], 1)
    dK = orc.gather_chunks(K[:P], ref_order, chunk).astype(np.float64).reshape(budget // chunk, chunk, H, d).sum((1, 3))
    np.testing.assert_array_equal(dK, g[f"{name}.retrK_digest"])
    dV = orc.gather_chunks(V[:P], ref_order, chunk).astype(np.float64).reshape(budget // chunk, chunk, H, d).sum((1, 3))
    np.testing.assert_array_equal(dV, g[f"{name}.retrV_digest"])


def _tie_only_difference(scores_rest, a, b):
    """Sets may differ only among candidates tied with the k-th score (torch.topk's tie order is unspecified)."""
    sa, sb = set(a.tolist()), set(b.tolist())
    kth = min(scores_rest[np.asarray(sorted(sa)) - 1].astype(np.float32))
    return all(float(scores_rest[i - 1]) == kth for i in sa ^ sb)


@pytest.mark.parametrize("case", gi.SAMPLING_CASES, ids=[c[0] for c in gi.SAMPLING_CASES])
def test_norm_logits_and_max_fn_match_reference(case, golden_dir):
    name = case[0]
    g = np.load(os.path.join(golden_dir, "sampling.npz"))
    logits = gi.sampling_logits(case)
    probs = orc.norm_logits(logits.copy(), case[4], -1, case[5])
    ref = g[f"{name}.probs"]
    np.testing.assert_array_equal(probs > 0, ref > 0)  # identical nucleus
    np.testing.assert_allclose(probs, ref, rtol=2e-6, atol=1e-9)
    p, q = gi.residual_pair(case)
    np.testing.assert_allclose(orc.max_fn(p - q), g[f"{name}.max_fn"], rtol=2e-6, atol=1e-12)


def test_rope_tables_match_reference_rows(golden_dir):
    from triforce_b200.rope import tables_for
    g = np.load(os.path.join(golden_dir, "forward.npz"))
    cos, sin = tables_for(named_config("tiny-yarn-target"))
    np.testing.assert_array_equal(cos[::97].numpy(), g["yarn_cos_rows"])  # same torch recipe → bit-identical
    np.testing.assert_array_equal(sin[::97].numpy(), g["yarn_sin_rows"])
    ocos, osin = orc.rope_tables_yarn(64, 4096, 2.0, 2048)
    assert (ocos[::97] != g["yarn_cos_rows"]).mean() < 0.02  # numpy's cos differs from torch's by an fp16 ulp, rarely
    assert np.abs(ocos[::97].astype(np.float32) - g["yarn_cos_rows"].astype(np.float32)).max() <= 2e-3


def test_rope_tables_match_reference_rows_7b_geometry(golden_dir):
    """The 7B / 13B YaRN tables (head_dim 128, 131 072 positions, factor 32 over 4096): strided rows over the whole table,
    every row of 124 900..124 999 and the last 64 rows must equal the reference's bit for bit.  Near position 125K the
    fp32 product t * inv_freq is off by several fp16 ulps of cos / sin from the exact angle, so only the reference's own
    recipe reproduces these rows."""
    from triforce_b200.rope import tables_for
    g = np.load(os.path.join(golden_dir, "yarn_7b_rows.npz"))
    rows = g["rows"]
    assert set(range(124900, 125000)) <= set(rows.tolist()) and rows.max() == 131071 and len(rows) > 200
    cos, sin = tables_for(named_config("llama-7B-128K"))
    assert tuple(cos.shape) == (131072, 128)
    np.testing.assert_array_equal(cos[rows].numpy(), g["cos"])
    np.testing.assert_array_equal(sin[rows].numpy(), g["sin"])
    assert tables_for(named_config("llama-13B-128K"))[0].shape == cos.shape  # same head_dim, positions and scaling


def assert_logits_close(actual, desired, what=""):
    """BASELINE north_star tolerance for verify logits is rtol 1e-2 / atol 1e-3 (fp16).  Logits are fp16 numbers of
    magnitude ~1-3 (ulp 1e-3..2e-3), produced by two different fp16 pipelines, so a sliver of elements sits one or two
    ulps apart: require >= 99.5 % of the elements inside the stated tolerance and every element within 5e-3."""
    actual, desired = np.asarray(actual, np.float32), np.asarray(desired, np.float32)
    bad = np.abs(actual - desired) > (1e-3 + 1e-2 * np.abs(desired))
    assert bad.mean() <= 5e-3, f"{what}: {bad.mean():.4%} of logits outside rtol 1e-2 / atol 1e-3"
    assert np.abs(actual - desired).max() <= 5e-3, f"{what}: max |diff| {np.abs(actual - desired).max()}"


def _oracle_models(case):
    from triforce_b200.rope import tables_for
    ts, ds = named_config(case["target"]), named_config(case["draft"])
    tsd = {k: v.numpy() for k, v in numpy_state_dict(ts, case["target_seed"]).items()}
    dsd = {k: v.numpy() for k, v in numpy_state_dict(ds, case["draft_seed"]).items()}
    ot, od = orc.LlamaOracle(ts, tsd, False), orc.LlamaOracle(ds, dsd, True)
    c, s = tables_for(ts)
    ot.set_tables(c.numpy(), s.numpy())
    c, s = tables_for(ds, is_draft=True)
    od.set_tables(c.numpy(), s.numpy())
    return ot, od


def test_forward_logits_match_reference(golden_dir):
    case = gi.FORWARD_CASE
    g = np.load(os.path.join(golden_dir, "forward.npz"))
    ot, od = _oracle_models(case)
    P, B, c, gam = case["prefill"], case["budget"], case["chunk"], case["gamma"]
    eng = orc.EngineOracle(ot, od, P, 32, B, c, gam, case["temperature"], case["top_p"])
    ids = numpy_prompt(P, seed=case["prompt_seed"]).numpy().reshape(-1)
    eng.inference(ids[:-1])
    last = eng.inference(ids[-1:])[-1]
    assert_logits_close(last, g["logits_last"], "last prompt token")
    vt = np.asarray(case["verify_tokens"])
    vl = ot.forward_target(vt, eng.kv_cache, eng.graph_cache, np.arange(P, P + gam + 1), spec=True)
    assert_logits_close(vl, g["verify_logits"], "retrieval verify")
    fl = eng.inference(vt)
    assert_logits_close(fl, g["full_verify_logits"], "full verify")
    eng.draft_prefill(ids)
    dl = od.forward_draft(vt[:3], eng.draft_cache, 2)
    assert_logits_close(dl, g["draft_logits"], "draft")


@pytest.mark.parametrize("name", [c["name"] for c in gi.E2E_CASES])
def test_e2e_trace_matches_reference(name, golden_dir):
    """Whole TriForce loop (first call AND second call — the draft-cache reset quirk) + the autoregressive baseline:
    every sampled token, uniform draw, Middle_Spec return and target input equal the reference's, event by event."""
    rec = json.load(open(os.path.join(golden_dir, f"e2e_{name}.json")))
    case = rec["case"]
    ot, od = _oracle_models(case)
    eng = orc.EngineOracle(ot, od, case["prefill"], case["gen_len"] + 16, case["budget"], case["chunk"], case["gamma"],
                           case["temperature"], case["top_p"])
    ids = numpy_prompt(case["prefill"], seed=case["prompt_seed"]).numpy().reshape(-1)
    for call, ref in enumerate(rec["calls"]):
        res = orc.triforce(eng, ids, case["gamma"], case["gen_len"], CounterNoise(case["noise_seed"]))
        got = [[e[0], e[1]] for e in res["trace"]]
        want = ref["trace"]
        n_pin = ref["oracle_matching_prefix"]  # recorded when the fixture was made (divergences = nucleus-boundary tokens)
        assert got[:n_pin] == [[a, (list(b) if isinstance(b, list) else b)] for a, b in want[:n_pin]]
        assert n_pin == len(want), f"call {call}: fixture pins only {n_pin}/{len(want)} events"
        assert abs(res["acceptance_rate"] - ref["acceptance_rate"]) < 1e-12
    toks = orc.autoregressive(eng, ids, case["ar_len"], CounterNoise(case["noise_seed"]))
    assert toks == rec["autoregressive"]["tokens"]
