"""Greedy decoding (temperature 0) on the GPU.

* `tf_norm_logits` at T = 0 is bit-exactly `one_hot(torch.argmax(row))`: ties, +-inf, NaN, odd widths, strided rows; T = 0.6 is
  unchanged against the fp64 oracle.
* Lossless, token for token: a greedy TriForce run and a greedy autoregressive run of the same engine, from the same prompt,
  emit the same tokens.  Targets: the tiny config (step-wise loop, whole-loop device graph, `DistributedLlama` at world size 1),
  two-layer 7B-wide targets on acceptance-calibrated weights (synth.agreement_state_dicts) with fp16, E4M3-store, E4M3-weight
  and E4M3-retrieval-cache variants, and a grouped-query target.
* Internal consistency: every token the step-wise loop emits is torch.argmax of the full-verify logits row that accepted or
  corrected it (or of the prompt's last row, for the first token).
* Sequoia: a greedy SpecTree on the 512-node tree at 13B width emits the target's greedy autoregressive sequence, and its
  accept walk equals a CPU restatement of the T = 0 walk on every round.

Near ties.  The full verify computes gamma+1 (or gamma+2) rows at once, the autoregressive decode one row; their attention
splits differ, so a logit may differ in its last bits.  The comparison therefore walks the two sequences until their first
difference and requires that position to be a near tie of the autoregressive run: top-2 logit margin below NEAR_TIE.  The
bound is backed by a measurement: wherever both runs computed a row from the same context, the largest logit difference must
stay below NEAR_TIE / 2, so no row with a larger margin can change its argmax.  Each test prints how many positions it compared
and the measured difference, and fails when too few positions were compared or no draft token was accepted."""
import dataclasses
import os

import numpy as np
import pytest
import torch

from attn_needles import report_time_and_memory  # noqa: F401  (autouse fixture: wall time and peak memory per test)
import golden_inputs as gi
from e2e_util import TokenizerStub
from oracle import triforce_oracle as orc
from triforce_b200 import ops
from triforce_b200._C import TriForceNativeError
from triforce_b200.cache import FlashSimpleCache, RetrievalCache, StreamingLLMEvictionCache
from triforce_b200.config import named_config
from triforce_b200.decoding import Autoregressive, Baseline_Dist, TriForce_Dist, TriForceRun
from triforce_b200.device_loop import DeviceLoopRun
from triforce_b200.engine import GraphInferenceEngine
from triforce_b200.llama import LlamaModel
from triforce_b200.sampling import norm_logits
from triforce_b200.spectree import SpecTree, load_grow_map
from triforce_b200.synth import agreement_state_dicts, numpy_prompt, numpy_state_dict, retune_agreement
from triforce_b200.tp import DistributedLlama

pytestmark = pytest.mark.gpu
DEV = "cuda"
TOK = TokenizerStub()
NEAR_TIE = 0.02   # logit units: a top-2 margin below this is a near tie
# An E4M3 full-KV store: the gamma+1-row verify and the one-row decode were measured to differ by up to 0.034 in a logit (an fp16
# store: 0.0015), so the near-tie bound is wider there.
NEAR_TIE_E4M3_STORE = 0.1
TINY = dict(target="tiny-yarn-target", draft="llama-68M", target_seed=1, draft_seed=2, prompt_seed=3, prefill=512, budget=64, chunk=8,
            gamma=4)
TINY_ALPHA = 0.05


# ---------------------------------------------------------------------------------------------------------------------
# the kernel
# ---------------------------------------------------------------------------------------------------------------------
def _one_hot_rows(x: torch.Tensor) -> torch.Tensor:
    want = torch.zeros_like(x)
    want.scatter_(1, torch.argmax(x, dim=1, keepdim=True), 1.0)
    return want


def _special_rows(V: int, g: torch.Generator) -> torch.Tensor:
    rows = [torch.randn(V, generator=g) * 3]
    r = torch.randn(V, generator=g)
    r[[0, V // 3, V - 1]] = 9.0                                   # the maximum at the first, a middle and the last column
    rows.append(r)
    r = torch.randn(V, generator=g)
    r[[V // 2, V - 1]] = 9.0                                      # tie not involving column 0
    rows.append(r)
    r = torch.randn(V, generator=g)
    r[V - 1] = 9.0                                                # the maximum only in the last column
    rows.append(r)
    r = torch.full((V,), -float("inf"))
    r[(V // 2 + 1) % V] = -3.5                                    # all -inf but one value
    rows.append(r)
    rows.append(torch.full((V,), -float("inf")))                  # all -inf: index 0
    r = torch.randn(V, generator=g)
    r[[7 % V, V - 2]] = float("inf")                              # +inf twice
    rows.append(r)
    r = torch.randn(V, generator=g)
    r[[V // 4, V - 1]] = float("nan")                             # NaN counts as maximal, first one wins
    r[0] = float("inf")
    rows.append(r)
    r = torch.randn(V, generator=g)
    r[V - 1] = float("nan")
    rows.append(r)
    rows.append(torch.zeros(V))                                   # all tied
    rows.append(torch.randint(-3, 3, (V,), generator=g).float())  # many exact ties
    r = -torch.rand(V, generator=g) * 1e-30                        # -0.0 vs +0.0 vs tiny negatives
    r[V // 5] = 0.0
    r[V // 6] = -0.0
    rows.append(r)
    return torch.stack(rows)


@pytest.mark.parametrize("V", [32000, 32768, 1, 7, 1001, 4097, 31999])
def test_norm_logits_at_zero_temperature_is_one_hot_argmax(V):
    g = torch.Generator().manual_seed(V)
    x = torch.cat([_special_rows(V, g), torch.randn(20, V, generator=g) * torch.rand(20, 1, generator=g) * 10]).to(DEV)
    want = _one_hot_rows(x)
    for top_p in (0.9, 1.0, 0.0, 1e-6):
        got = ops.norm_logits(x, 0.0, top_p)
        assert torch.equal(got, want), (V, top_p, (got != want).nonzero()[:4])
    # a strided view (row stride V + 13)
    big = torch.full((x.shape[0], V + 13), 123.0, device=DEV)
    big[:, :V] = x
    assert torch.equal(ops.norm_logits(big[:, :V], 0.0, 0.9), want)
    # the Python front end, including the top-k branch, passes T = 0 through
    assert torch.equal(norm_logits(x, temperature=0.0, top_k=-1, top_p=0.9), want)
    if V > 50:
        finite = x[torch.isfinite(x).all(1)]
        assert torch.equal(norm_logits(finite, temperature=0, top_k=40, top_p=0.9), _one_hot_rows(finite))


def test_norm_logits_rejects_a_negative_temperature():
    x = torch.randn(2, 100, device=DEV)
    for t in (-1e-6, -0.6, float("nan")):
        with pytest.raises(TriForceNativeError, match="temperature"):
            ops.norm_logits(x, t, 0.9)


def test_norm_logits_at_positive_temperature_is_unchanged(golden_dir):
    """T > 0 against the reference's probabilities and the fp64 oracle, as tests/test_kernels_gpu.py checks them (the T = 0 path
    leaves the T > 0 kernel's SASS untouched)."""
    g = np.load(os.path.join(golden_dir, "sampling.npz"))
    cases = [c for c in gi.SAMPLING_CASES if c[4] > 0]
    assert cases
    for case in cases:
        probs = ops.norm_logits(torch.from_numpy(gi.sampling_logits(case)).to(DEV), case[4], case[5]).cpu().numpy()
        ref = g[f"{case[0]}.probs"]
        np.testing.assert_array_equal(probs > 0, ref > 0)
        np.testing.assert_allclose(probs, ref, rtol=1e-5, atol=1e-10)
    x = np.zeros((1, 32000), np.float32)
    x[0, 100] = 30.0
    want = orc.norm_logits(x.copy(), 0.6, -1, 0.9)
    got = ops.norm_logits(torch.from_numpy(x).to(DEV), 0.6, 0.9).cpu().numpy()
    np.testing.assert_array_equal(got > 0, want > 0)
    np.testing.assert_allclose(got, want, rtol=1e-5, atol=1e-10)


# ---------------------------------------------------------------------------------------------------------------------
# the T = 0 accept walk
# ---------------------------------------------------------------------------------------------------------------------
def cpu_greedy_walk(probs: torch.Tensor, tokens, succ, max_accept=24):
    """The T = 0 walk restated: from the root, follow the child whose token is torch.argmax of the node's target row; stop when
    no child carries it (or at a leaf).  An accepted token 0 or 2 ends the generation.  Returns (accepted nodes, code,
    terminal, next token)."""
    cur, acc = 0, []
    while True:
        best = int(torch.argmax(probs[cur]))
        child = next((c for c in succ[cur] if int(tokens[c]) == best), None)
        if child is None:
            return acc, (-2 if not succ[cur] else -1), False, best
        acc.append(child)
        cur = child
        if best in (0, 2):
            return acc, 0, True, None


def _csr(succ):
    off, flat = [0], []
    for ch in succ:
        flat.extend(ch)
        off.append(len(flat))
    return torch.tensor(off, dtype=torch.int32, device=DEV), torch.tensor(flat, dtype=torch.int32, device=DEV)


def test_tree_accept_walk_at_zero_temperature_matches_the_restatement():
    gm = load_grow_map("512")
    succ = gm["Successors"]
    off, flat = _csr(succ)
    T, V = 512, 2048
    g = torch.Generator().manual_seed(3)
    paths = []
    for trial in range(16):
        draft = torch.randn(T, V, generator=g) * 2
        tgt = torch.softmax(draft * 1.5 + torch.randn(T, V, generator=g) * (0.3 if trial % 2 else 1.5), dim=-1)
        if trial % 4 == 0:
            tgt = _one_hot_rows(tgt)  # what norm_logits at T = 0 hands the walk
        tokens = torch.randint(3, V, (T,), generator=g)
        for n in range(T):  # children: the draft's top-k, as the T = 0 growth makes them
            ch = succ[n]
            if ch:
                tokens[ch] = torch.sort(draft[n], descending=True, stable=True).indices[:len(ch)]
        if trial == 5:  # an accepted EOS ends the walk
            c = succ[0][0]
            tokens[c] = 2
            tgt[0] = 0
            tgt[0, 2] = 1
        acc, code, terminal, nxt = cpu_greedy_walk(tgt, tokens, succ)
        out = torch.full((32,), -7, dtype=torch.int32, device=DEV)
        resid = torch.full((V,), -1.0, device=DEV)
        scratch = torch.zeros(V, device=DEV)
        d_dev = draft.to(DEV)
        uni = torch.full((128,), float("nan"), device=DEV)  # never read at T = 0
        ops.tree_accept_walk(tgt.to(DEV), d_dev, tokens.to(DEV), off, flat, uni, 0.0, out, resid, scratch)
        w = out.tolist()
        assert w[0] == len(acc) and w[8:8 + w[0]] == acc, (trial, w[:12], acc)
        assert w[2] == 0 and w[3] == int(terminal) and w[4] == 0
        assert torch.equal(d_dev.cpu(), draft)  # the draft rows are neither read nor written
        if not terminal:
            assert w[1] == code
            want = torch.zeros(V)
            want[nxt] = 1.0
            assert torch.equal(resid.cpu(), want)
        paths.append(len(acc))
    assert max(paths) >= 2 and min(paths) == 0, paths  # deep walks and immediate stops were both exercised


# ---------------------------------------------------------------------------------------------------------------------
# lossless against greedy autoregressive decoding
# ---------------------------------------------------------------------------------------------------------------------
@torch.inference_mode()
def greedy_ar(ge, ids, n):
    """Greedy autoregressive decoding on the engine (decoding.Autoregressive's calls: the prompt, then one-row decode steps)
    with the logits of every step kept.  Returns (tokens [n + 1], logits rows [n + 1, V])."""
    eng = ge.engine
    eng.kv_cache.reset()
    expo = torch.ones(eng.model.config.vocab_size, device=DEV)
    row = ge.inference(input_ids=ids)[:, -1, :].float()
    rows, toks = [], []
    for i in range(n + 1):
        rows.append(row[0].clone())
        tok = ops.sample_argmax(norm_logits(row, temperature=0.0, top_k=-1, top_p=0.9), expo)
        toks.append(int(tok))
        if i < n:
            row = ge.decode_step(tok.reshape(1, 1))[:, -1, :].float()
    return toks, torch.stack(rows)


def margins(rows: torch.Tensor):
    top = torch.topk(rows, 2, dim=-1).values
    return (top[:, 0] - top[:, 1]).tolist()


def compare_to_greedy(tri, ar, ar_rows, min_compared, what, verify_rows=None, near_tie=NEAR_TIE):
    """Walk both sequences to their first difference, which must be a near tie of the AR run.  `verify_rows` (position ->
    verify logits row) measures the verify-vs-AR logit difference on positions both computed from the same context."""
    m = margins(ar_rows)
    n = min(len(tri), len(ar))
    k = next((i for i in range(n) if tri[i] != ar[i]), n)
    diff = None
    if verify_rows:
        diff = max((verify_rows[i] - ar_rows[i]).abs().max().item() for i in verify_rows if i <= min(k, n - 1) and i < len(ar_rows))
    print(f"\n[{what}] compared {k} of {n} positions; smallest AR top-2 margin on them "
          f"{min(m[:max(k, 1)]):.4g}; verify vs AR logits max |diff| "
          f"{'not measured' if diff is None else f'{diff:.3g}'}"
          f"{'' if k == n else f'; first difference at {k}: {tri[k]} vs {ar[k]}, AR margin {m[k]:.4g}'}")
    if k < n:
        assert m[k] < near_tie, f"{what}: tokens differ at position {k} ({tri[k]} vs {ar[k]}) with AR top-2 margin {m[k]} >= {near_tie}"
    if diff is not None:
        assert diff < near_tie / 2, f"{what}: verify and AR logits differ by {diff}, the near-tie bound {near_tie} does not cover it"
    assert k >= min_compared, f"{what}: only {k} positions compared"
    return k


class VerifyRecorder:
    """Keeps the logits of every full-KV call of at most `max_rows` rows (the first-token row and each full verify)."""

    def __init__(self, ge, max_rows):
        self.calls = []
        orig = ge.inference

        def inference(input_ids):
            out = orig(input_ids=input_ids)
            if input_ids.shape[-1] <= max_rows:
                self.calls.append(out[0].float().clone())
            return out
        ge.inference = inference
        self.ge, self.orig = ge, orig

    def remove(self):
        self.ge.inference = self.orig


@torch.inference_mode()
def stepwise_greedy(ge, ids, gamma, gen):
    """The step-wise TriForce loop at T = 0 with each full verify's logits recorded; checks internal consistency.  Returns
    (tokens, run, position -> verify row)."""
    rec = VerifyRecorder(ge, gamma + 2)
    try:
        run = TriForceRun(TOK, ge, gamma=gamma, top_p=0.9, temperature=0.0)
        run.prefill(ids)
        first = rec.calls[-1]
        assert int(torch.argmax(first[-1])) == run.generated[0]
        rows = {0: first[-1]}
        while run.n < gen:
            before = len(run.generated)
            n_calls = len(rec.calls)
            run.step()
            assert len(rec.calls) == n_calls + 1
            L = rec.calls[-1]
            produced = run.generated[before:]
            assert 1 <= len(produced) <= L.shape[0]
            for j, t in enumerate(produced):  # accepted draft tokens, then the correction or bonus token
                assert int(torch.argmax(L[j])) == t, (before, j, t)
            for j in range(len(produced)):
                rows[before + j] = L[j]
    finally:
        rec.remove()
    return run.generated, run, rows


def _tokens_per_step(run):
    steps = len(run.acc_rate_middle_list) if hasattr(run, "acc_rate_middle_list") else run.steps
    return (len(run.generated) - 1) / steps


def _tiny_engine(alpha=TINY_ALPHA, budget=None):
    ts, ds = named_config(TINY["target"]), named_config(TINY["draft"])
    target = LlamaModel(ts, numpy_state_dict(ts, TINY["target_seed"]), device=DEV)
    draft = LlamaModel(ds, numpy_state_dict(ds, TINY["draft_seed"]), device=DEV, is_draft=True)
    retune_agreement(target, draft, alpha, alpha, {})
    P, B, c, g = TINY["prefill"], budget or TINY["budget"], TINY["chunk"], TINY["gamma"]
    cache = FlashSimpleCache(target, P + 256)
    graph_cache = RetrievalCache(target, max_budget=B, prefill=P, gamma=g, chunk_size=c)
    draft_cache = StreamingLLMEvictionCache(draft, start_size=16, recent_size=256 - 16 - g, gamma=g)
    ge = GraphInferenceEngine(target, cache, graph_cache, draft, draft_cache)
    ge.initialize_cuda_graph(g, probs=True, temperature=0.0, top_p=0.9)
    return ge


def test_tiny_stepwise_loop_is_greedy_ar():
    ge = _tiny_engine()
    ids = numpy_prompt(TINY["prefill"], seed=TINY["prompt_seed"]).cuda()
    gen = 48  # the tail copy of the 64-slot retrieval cache holds at most 64 generated tokens
    ar, ar_rows = greedy_ar(ge, ids, gen + 8)
    _, ar_public = Autoregressive(TOK, ge, ids, max_len=gen + 8, temperature=0.0, return_tokens=True)
    assert ar_public == ar  # the public loop at T = 0 is this greedy loop
    tri, run, rows = stepwise_greedy(ge, ids, TINY["gamma"], gen)
    tps = _tokens_per_step(run)
    print(f"tiny step-wise: {len(tri)} tokens in {len(run.acc_rate_middle_list)} steps ({tps:.2f} per step), "
          f"accepted {run.accepted_count} of {run.draft_count}, {run.resample_count} corrections")
    compare_to_greedy(tri, ar, ar_rows, 40, "tiny, step-wise loop", rows)
    assert tps > 1.0 and run.accepted_count > 0


def test_tiny_device_loop_with_a_128_row_tail_is_greedy_ar():
    ge = _tiny_engine(budget=128)  # 96 generated tokens need a retrieval tail of more than the case's 64 rows
    ids = numpy_prompt(TINY["prefill"], seed=TINY["prompt_seed"]).cuda()
    gen = 96
    ar, ar_rows = greedy_ar(ge, ids, gen + 8)
    run = DeviceLoopRun(TOK, ge, gamma=TINY["gamma"], top_p=0.9, temperature=0.0, seed=5)
    run.prefill(ids)
    while run.n < gen:
        run.step()
    tps = (len(run.generated) - 1) / run.steps
    print(f"tiny device loop: {len(run.generated)} tokens in {run.steps} launches ({tps:.2f} per step), "
          f"accepted {run.accepted_count} of {run.draft_count}")
    compare_to_greedy(run.generated, ar, ar_rows, 64, "tiny, whole-loop device graph")
    assert tps > 1.0 and run.accepted_count > 0
    # the noise stream does not matter at T = 0: another seed emits the same tokens
    run2 = DeviceLoopRun(TOK, ge, gamma=TINY["gamma"], top_p=0.9, temperature=0.0, seed=12345)
    run2.prefill(ids)
    while run2.n < gen:
        run2.step()
    n = min(len(run.generated), len(run2.generated))
    assert run2.generated[:n] == run.generated[:n]


def test_tiny_distributed_llama_world1_is_greedy_ar():
    ts, ds = named_config(TINY["target"]), named_config(TINY["draft"])
    P, B, c, g = TINY["prefill"], TINY["budget"], TINY["chunk"], TINY["gamma"]
    gen = 40  # the tail copy of the 64-slot retrieval cache holds at most 64 generated tokens
    draft = LlamaModel(ds, numpy_state_dict(ds, TINY["draft_seed"]), device=DEV, is_draft=True)
    dcache = StreamingLLMEvictionCache(draft, start_size=16, recent_size=256 - 16 - g, gamma=g)
    llm = DistributedLlama(TINY["target"], local_rank=0, world_size=1, prefill=P, gen_len=gen + 32, retrieval_budget=B,
                           retrieval_chunk_size=c, gamma=g, temperature=0.0, top_p=0.9, draft=draft, draft_cache=dcache, config=ts)
    llm.init_parameters(state_dict=numpy_state_dict(ts, TINY["target_seed"]))
    retune_agreement(llm.model, draft, TINY_ALPHA, TINY_ALPHA, {})
    ids = numpy_prompt(P, seed=TINY["prompt_seed"]).to(DEV)
    ar, ar_rows = greedy_ar(llm.graph_engine, ids, gen + 8)
    _, base = Baseline_Dist(TOK, llm, ids, max_len=gen + 8, temperature=0.0)
    compare_to_greedy([ar[0]] + base[0].tolist(), ar, ar_rows, 32, "tiny, DistributedLlama world 1: Baseline_Dist")
    stats = {}
    TriForce_Dist(TOK, llm, ids, gamma=g, max_len=gen, top_p=0.9, temperature=0.0, stats=stats)
    tps = (len(stats["tokens"]) - 1) / stats["outer_iterations"]
    print(f"tiny TP world 1: {len(stats['tokens'])} tokens in {stats['outer_iterations']} steps ({tps:.2f} per step)")
    compare_to_greedy(stats["tokens"], ar, ar_rows, 32, "tiny, DistributedLlama world 1: TriForce_Dist")
    assert tps > 1.0 and stats["accepted_count"] > 0


PROD = [  # (target shape, full-KV store, weights, retrieval cache, prefill)
    ("llama-7B-128K", "fp16", "fp16", "fp16", 124928),
    ("llama-7B-128K", "e4m3", "fp16", "fp16", 32768),
    ("llama-7B-128K", "fp16", "e4m3", "fp16", 32768),
    ("llama-7B-128K", "fp16", "fp16", "e4m3", 32768),
    ("llama-7B-gqa8-128K", "fp16", "fp16", "fp16", 32768),
]
PROD_ALPHA, PROD_GAMMA, PROD_BUDGET, PROD_GEN = 0.01, 6, 4096, 64


@pytest.mark.parametrize("name,kv,weights,retrieval,P", PROD, ids=[f"{p[0]}-kv_{p[1]}-w_{p[2]}-r_{p[3]}-P{p[4]}" for p in PROD])
def test_production_width_target_is_greedy_ar(name, kv, weights, retrieval, P):
    """Two-layer targets at the 7B width on acceptance-calibrated weights: the step-wise loop and the whole-loop device graph
    against greedy AR on the same engine."""
    cfg_t = dataclasses.replace(named_config(name), num_hidden_layers=2)
    cfg_d = named_config("llama-68M")
    tsd, dsd = agreement_state_dicts(cfg_t, cfg_d, PROD_ALPHA, PROD_ALPHA, seed=0, device=DEV)
    target = LlamaModel(cfg_t, tsd, device=DEV, weight_dtype=weights)
    draft = LlamaModel(cfg_d, dsd, device=DEV, is_draft=True)
    del tsd, dsd
    cache = FlashSimpleCache(target, P + 2 * PROD_GEN + 64, kv_dtype=kv)
    graph_cache = RetrievalCache(target, max_budget=PROD_BUDGET, prefill=P, gamma=PROD_GAMMA, chunk_size=8, kv_dtype=retrieval)
    draft_cache = StreamingLLMEvictionCache(draft, start_size=16, recent_size=256 - 16 - PROD_GAMMA, gamma=PROD_GAMMA)
    ge = GraphInferenceEngine(target, cache, graph_cache, draft, draft_cache)
    ge.initialize_cuda_graph(PROD_GAMMA, probs=True, temperature=0.0, top_p=0.9)
    ids = numpy_prompt(P, seed=5).cuda()
    what = f"{name} kv={kv} weights={weights} retrieval={retrieval} P={P}"
    ar, ar_rows = greedy_ar(ge, ids, PROD_GEN + 8)
    tri, run, rows = stepwise_greedy(ge, ids, PROD_GAMMA, PROD_GEN)
    tps = _tokens_per_step(run)
    print(f"{what}, step-wise: {tps:.2f} tokens per step, accepted {run.accepted_count} of {run.draft_count}")
    near_tie = NEAR_TIE_E4M3_STORE if kv == "e4m3" else NEAR_TIE
    compare_to_greedy(tri, ar, ar_rows, 32, what + ", step-wise loop", rows, near_tie)
    assert tps > 1.0 and run.accepted_count > 0
    dev = DeviceLoopRun(TOK, ge, gamma=PROD_GAMMA, top_p=0.9, temperature=0.0, seed=1, max_new=2 * PROD_GEN)
    dev.prefill(ids)
    while dev.n < PROD_GEN:
        dev.step()
    tps = (len(dev.generated) - 1) / dev.steps
    print(f"{what}, device loop: {tps:.2f} tokens per step")
    compare_to_greedy(dev.generated, ar, ar_rows, 32, what + ", whole-loop device graph", near_tie=near_tie)
    assert tps > 1.0


# ---------------------------------------------------------------------------------------------------------------------
# Sequoia
# ---------------------------------------------------------------------------------------------------------------------
@torch.inference_mode()
def test_greedy_spectree_is_greedy_ar_at_13b_width():
    cfg = dataclasses.replace(named_config("llama-13B-128K"), num_hidden_layers=2)
    # at T = 0 a node is accepted only when the retrieval level's argmax is the full target's, which the flat synthetic
    # distributions give much less often than a high acceptance at T > 0: hence a smaller alpha than PROD_ALPHA
    tsd, _ = agreement_state_dicts(cfg, named_config("llama-68M"), 0.001, 0.001, seed=0, device=DEV)
    P, B, rounds = 16384, 4096, 16
    gm = load_grow_map("512")
    llm = DistributedLlama("llama-13B-128K", local_rank=0, world_size=1, prefill=P, gen_len=rounds * 24 + 64, retrieval_budget=B,
                           retrieval_chunk_size=8, gamma=6, temperature=0.0, config=cfg, tree_size=gm["size"])
    llm.init_parameters(state_dict=tsd, cuda_graphs=False)
    del tsd
    ids = numpy_prompt(P, seed=9)[0].to(DEV)
    # greedy AR on the same engine: 128-row prefill chunks, then one-row steps over the full KV
    n_ar = rounds * 17 + 8
    llm.reset()
    row = llm.prefill(ids.unsqueeze(0))[:, -1, :].float()
    ar, ar_rows = [], []
    for i in range(n_ar + 1):
        ar_rows.append(row[0].clone())
        ar.append(int(torch.argmax(row[0])))
        if i < n_ar:
            row = llm.inference(torch.tensor([[ar[-1]]], device=DEV))[:, -1, :].float()
    ar_rows = torch.stack(ar_rows)

    st = SpecTree(engine=llm, temperature=0.0, top_p=0.9, max_length=P + 512, grow_map=gm, vocab_size=cfg.vocab_size)
    nt = st.prefill(prefix=ids)
    emitted = [int(nt.reshape(-1)[0])]
    counts = []
    for r in range(rounds):
        st.construct_grow_map(next_token=nt)
        tokens = st.verify_tokens.clone()
        # the T = 0 growth: each parent's children are its draft row's top-k, ties to the lower index
        for parent in (0, 1):
            ch = gm["Successors"][parent]
            want = torch.sort(st.draft_logits[parent], descending=True, stable=True).indices[:len(ch)]
            assert tokens[ch].tolist() == want.tolist()
        nt, acc, toks = st.verify()
        assert nt is not None, "an EOS was accepted"
        probs = st.target_logits.cpu()
        assert torch.equal(probs, _one_hot_rows(probs))
        walk, code, terminal, nxt = cpu_greedy_walk(probs, tokens.cpu(), gm["Successors"])
        toks = [int(t) for t in toks.tolist()]
        assert not terminal and st._walk_out[2].item() == 0
        assert acc == len(walk) + 1 and toks[1:-1] == tokens[walk].tolist() and toks[-1] == nxt, (r, walk, toks)
        emitted.extend(toks[1:])
        counts.append(acc)
        nt = nt.unsqueeze(0)
    print(f"Sequoia 13B width, greedy: tokens per round {counts}")
    compare_to_greedy(emitted, ar, ar_rows, rounds + 1, "SpecTree 512 nodes, 13B width")
    assert sum(counts) / len(counts) > 1.0
