"""Scoring a given continuation on the GPU: tf_token_logprobs, LlamaModel.prefill / extend with `logprobs`, Session.score and
TreeSession.score.

* The kernel against an fp64 reference at V = 1 000, 32 000 and 128 256 (ties, -inf entries, logits of magnitude 1e30 and 1e4,
  a row stride wider than V): |delta| <= 1e-5 (1 + |lp|), argmax equal to torch.argmax; two launches and a CUDA-graph replay
  give the same bits.
* Prefill with scoring computes what prefill without it computes (logits, store rows, codes and exponents, seq_len), for fp16,
  an E4M3 store, E4M3 weights and a grouped-query 7B.  Chunk-major scores are the kernel on the logits forward_target returns
  for the same pieces; E4M3-weight scores are those of an fp16 target holding D, and E4M3-store scores those over an fp16
  store, bit for bit.
* A score leaves no trace: the turns after it (step-wise loop, whole-loop graph, Sequoia tree over fp16 and over an E4M3 store
  with E4M3 weights) emit what a session that never scored emits.  Tokens a session emits at T = 0 score as greedy except at near ties."""
from __future__ import annotations

import dataclasses

import pytest
import torch

from attn_needles import report_time_and_memory  # noqa: F401  (autouse fixture: wall time and peak memory per test)
from e2e_util import TokenizerStub
from test_greedy_gpu import NEAR_TIE
from test_session_gpu import TINY, _tiny_engine
from test_tree_session_gpu import _engine as _tree_engine
from test_weights_e4m3_model_gpu import d_state_dict
from triforce_b200 import ops
from triforce_b200.cache import FlashSimpleCache
from triforce_b200.config import named_config
from triforce_b200.llama import LlamaModel
from triforce_b200.session import Session, TreeSession
from triforce_b200.synth import cuda_state_dict, numpy_prompt

pytestmark = pytest.mark.gpu
DEV = "cuda"
TOK = TokenizerStub()


# ---------------------------------------------------------------------------------------------------------------------
# the kernel
# ---------------------------------------------------------------------------------------------------------------------
def _rows(V, seed):
    """16 rows of V logits, written into a [16, V + 40] buffer (row stride wider than V), with the rows' special cases."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    buf = torch.randn((16, V + 40), generator=g, device=DEV) * 3
    x = buf[:, :V]
    x[1, :] = 0.5                                     # all tied: argmax 0, lp = -log V
    x[2, V // 3] = x[2, V // 2] = x[2, -1] = 50.0     # ties at the top, not at the start
    x[3, ::3] = -float("inf")                         # -inf entries (one of them scored below)
    x[4] *= 1e30                                      # very large logits: the max shift keeps exp finite
    x[5] += 1e4                                       # a large common offset
    x[6, :-1] = -float("inf")                         # one finite entry
    x[7, 7] = 1e30
    ids = torch.randint(0, V, (16,), generator=g, device=DEV, dtype=torch.int64)
    ids[3] = 0                                        # a -inf target: lp = -inf
    ids[6] = V - 1
    ids[2] = V // 2
    return x, ids.to(torch.int32)


@pytest.mark.parametrize("V", [1000, 32000, 128256])
def test_token_logprobs_against_fp64(V):
    x, ids = _rows(V, seed=V)
    assert x.stride(0) == V + 40
    lp, am = ops.token_logprobs(x, ids)
    torch.cuda.synchronize()
    x64 = x.double()
    want = x64.gather(1, ids.long()[:, None])[:, 0] - torch.logsumexp(x64, dim=1)
    got = lp.double()
    inf = torch.isinf(want)
    assert torch.equal(torch.isinf(got), inf) and (got[inf] == want[inf]).all()
    err = (got - want).abs()[~inf]
    tol = 1e-5 * (1 + want.abs()[~inf])
    assert (err <= tol).all(), f"V={V}: worst |delta| {err.max().item():.3g}, rows {torch.nonzero(err > tol).flatten().tolist()}"
    assert torch.equal(am.long(), torch.argmax(x, dim=1))
    assert am[1] == 0 and am[2] == V // 3 and am[6] == V - 1 and am[7] == 7
    assert abs(lp[1].item() + torch.log(torch.tensor(float(V))).item()) < 1e-5 * (1 + lp[1].abs().item())
    # two launches: the same bits
    lp2, am2 = ops.token_logprobs(x, ids)
    assert torch.equal(lp, lp2) and torch.equal(am, am2)
    # captured in a graph (ids already checked): the replay equals the eager call
    glp, gam = torch.empty_like(lp), torch.empty_like(am)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.token_logprobs(x, ids, glp, gam, check_ids=False)  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    glp.zero_(), gam.zero_()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.token_logprobs(x, ids, glp, gam, check_ids=False)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(glp, lp) and torch.equal(gam, am)


def test_token_logprobs_refuses_ids_out_of_range():
    x = torch.zeros((3, 100), device=DEV)
    for bad in (100, -1):
        with pytest.raises(ValueError, match=r"\[0, 100\)"):
            ops.token_logprobs(x, torch.tensor([0, bad, 5], dtype=torch.int32, device=DEV))


# ---------------------------------------------------------------------------------------------------------------------
# LlamaModel.prefill with logprobs
# ---------------------------------------------------------------------------------------------------------------------
PREFILL_CASES = [("llama-7B-128K", "fp16", "fp16"), ("llama-7B-128K", "e4m3", "fp16"), ("llama-7B-128K", "fp16", "e4m3"),
                 ("llama-7B-gqa8-128K", "fp16", "fp16")]


def _store_state(kv):
    if kv.e4m3 is not None:
        st = kv.e4m3
        return [st.k_codes.clone(), st.k_exp.clone(), st.v_codes.clone(), st.v_exp.clone()]
    return [kv.key_store.clone(), kv.value_store.clone()]


@pytest.mark.parametrize("name,kv_dtype,weights", PREFILL_CASES, ids=[f"{a}-kv_{b}-w_{c}" for a, b, c in PREFILL_CASES])
@torch.inference_mode()
def test_prefill_with_scores_computes_the_same_prefill(name, kv_dtype, weights):
    N, chunk = 1500, 128  # 11 pieces of 128 and one of 92
    cfg = dataclasses.replace(named_config(name), num_hidden_layers=2)
    sd = cuda_state_dict(cfg, seed=3, lm_head_std=0.01)
    model = LlamaModel(cfg, sd, device=DEV, weight_dtype=weights)
    ids = numpy_prompt(N, seed=8).cuda()[0]
    kv = FlashSimpleCache(model, N + 64, kv_dtype=kv_dtype)
    want = model.prefill(ids, kv, chunk=chunk)
    want_store, want_len = _store_state(kv), kv.seq_len
    kv.reset()
    lp = torch.full((N - 1,), float("nan"), device=DEV)
    am = torch.full((N - 1,), -1, dtype=torch.int32, device=DEV)
    got = model.prefill(ids, kv, chunk=chunk, logprobs=(lp, am))
    torch.cuda.synchronize()
    assert torch.equal(got, want) and kv.seq_len == want_len == N
    for a, b in zip(_store_state(kv), want_store):
        assert torch.equal(a, b)
    assert torch.isfinite(lp).all() and (lp <= 0).all() and (am >= 0).all()
    print(f"\n{name} kv={kv_dtype} w={weights}: mean logprob {lp.mean().item():.4f}, greedy share "
          f"{(am.long() == ids[1:]).float().mean().item():.4f}")
    if kv_dtype == "fp16" and weights == "fp16":
        # chunk-major: the kernel on the logits forward_target returns for the same pieces
        ref = FlashSimpleCache(model, N + 64)
        tg = ids[1:].to(torch.int32)
        for c0 in range(0, N, chunk):
            lg = model.forward_target(ids[c0:c0 + chunk], ref)[0]
            r = min(lg.shape[0], N - 1 - c0)
            p, a = ops.token_logprobs(lg[:r], tg[c0:c0 + r])
            assert torch.equal(p, lp[c0:c0 + r]) and torch.equal(a, am[c0:c0 + r]), f"piece at {c0}"
    if kv_dtype == "e4m3":
        # the prompt attends over an fp16 scratch, so a prefill over an E4M3 store scores what it scores over an fp16 store
        k16 = FlashSimpleCache(model, N + 64)
        lp16, am16 = torch.empty_like(lp), torch.empty_like(am)
        model.prefill(ids, k16, chunk=chunk, logprobs=(lp16, am16))
        assert torch.equal(lp16, lp) and torch.equal(am16, am)
    if weights == "e4m3":
        # the fp16 target holding D (chunk-major over an fp16 store) scores the same bits
        del model
        torch.cuda.empty_cache()
        mD = LlamaModel(cfg, d_state_dict(cfg, sd), device=DEV)
        kD = FlashSimpleCache(mD, N + 64)
        lpD, amD = torch.empty_like(lp), torch.empty_like(am)
        mD.prefill(ids, kD, chunk=chunk, logprobs=(lpD, amD))
        assert torch.equal(lpD, lp) and torch.equal(amD, am)


@torch.inference_mode()
def test_extend_scores_continue_the_prefill_scores():
    """prefill(A) then extend(B) scores ids[1:] of B as prefill(A + B) scores them (fp16, A a multiple of the chunk)."""
    cfg = dataclasses.replace(named_config("llama-7B-128K"), num_hidden_layers=2)
    model = LlamaModel(cfg, cuda_state_dict(cfg, seed=4, lm_head_std=0.01), device=DEV)
    A, Bn = 1024, 300
    ids = numpy_prompt(A + Bn, seed=2).cuda()[0]
    one, two = FlashSimpleCache(model, A + Bn + 64), FlashSimpleCache(model, A + Bn + 64)
    lp, am = torch.empty(A + Bn - 1, device=DEV), torch.empty(A + Bn - 1, dtype=torch.int32, device=DEV)
    model.prefill(ids, one, logprobs=(lp, am))
    model.prefill(ids[:A], two)
    lpe, ame = torch.empty(Bn - 1, device=DEV), torch.empty(Bn - 1, dtype=torch.int32, device=DEV)
    model.extend(ids[A:], two, logprobs=(lpe, ame))
    assert torch.equal(lpe, lp[A:]) and torch.equal(ame, am[A:])


# ---------------------------------------------------------------------------------------------------------------------
# Session.score / TreeSession.score
# ---------------------------------------------------------------------------------------------------------------------
def _chain_turns(ids, scored, device_loop):
    P = TINY["prefill"]
    ge = _tiny_engine()
    kv = ge.engine.kv_cache
    s = Session(ge, gamma=TINY["gamma"], tokenizer=TOK, pad_full_verify=True)
    s.prefill(ids[:P])
    scores = []

    def score(x):
        before = (s.length, int(kv.seq_len_dev.item()), list(s.ids), s.pending, None if s._logits is None else s._logits.clone())
        scores.append(s.score(x))
        after = (s.length, int(kv.seq_len_dev.item()), list(s.ids), s.pending)
        assert after == before[:4] and (before[4] is None or torch.equal(s._logits, before[4]))

    if scored:
        score(ids[P:P + 40])           # on the held logits of the prefill
    t1 = s.generate(20, seed=5, device_loop=device_loop)
    r1 = s.last_run
    if scored:
        score(ids[P + 40:P + 140])     # the pending token forwarded first
    s.append(ids[P:P + 60])
    if scored:
        score(ids[P + 60:P + 61])      # one id: the held logits only
    t2 = s.generate(30, seed=6, device_loop=device_loop)
    r2 = s.last_run
    counts = [(r.accepted_count, r.draft_count, r.resample_count) for r in (r1, r2)]
    return (t1, t2, counts, s.length, list(s.ids), s.pending), scores


@pytest.mark.parametrize("device_loop", [False, True], ids=["step_wise", "device_loop"])
@torch.inference_mode()
def test_chain_score_leaves_no_trace(device_loop):
    ids = numpy_prompt(TINY["prefill"] + 200, seed=3).cuda()[0]
    plain, _ = _chain_turns(ids, False, device_loop)
    scored, scores = _chain_turns(ids, True, device_loop)
    assert scored == plain
    assert [sc.logprobs.numel() for sc in scores] == [40, 100, 1]
    for sc in scores:
        assert torch.isfinite(sc.logprobs).all() and (sc.logprobs <= 0).all()
    print(f"\n{'device loop' if device_loop else 'step-wise'}: turns of {len(plain[0])} and {len(plain[1])} tokens, identical "
          f"with and without three scores")


@pytest.mark.parametrize("fmt", ["fp16", "e4m3"], ids=["fp16", "e4m3_store_and_weights"])
@torch.inference_mode()
def test_tree_score_leaves_no_trace(fmt):
    """E4M3: the scores run the layer-major extend over a non-empty E4M3 store with E4M3 weights."""
    P, B = 8192, 4096
    llm, _, _ = _tree_engine("llama-7B-128K", fmt, fmt, P, B, 0.6)
    ids = numpy_prompt(P + 400, seed=12)[0].to(DEV)
    out = []
    for scored in (False, True):
        s = TreeSession(llm)
        s.prefill(ids[:P])
        if scored:
            sc = s.score(ids[P:P + 64])
            assert torch.isfinite(sc.logprobs).all() and (sc.logprobs <= 0).all()
        t1 = s.generate(40, temperature=0.6, seed=3)
        a1 = list(s.last_turn.accepted)
        if scored:
            n0, rc = s.length, llm.retrieval_cache.prefill
            s.score(ids[P + 64:P + 300])
            assert s.length == n0 and llm.retrieval_cache.prefill == rc
        s.append(ids[P:P + 100])
        t2 = s.generate(40, temperature=0.6, seed=4)
        out.append((t1, a1, t2, list(s.last_turn.accepted), s.length, list(s.ids), s.pending))
    assert out[0] == out[1]


@torch.inference_mode()
def test_greedy_output_scores_as_greedy():
    P = TINY["prefill"]
    ge = _tiny_engine(temperature=0.0)
    ids = numpy_prompt(P, seed=3).cuda()[0]
    s = Session(ge, gamma=TINY["gamma"], tokenizer=TOK)
    s.prefill(ids)
    toks = s.generate(64, temperature=0.0)
    s.prefill(ids)  # the same context again: the held logits of the same prefill
    sc = s.score(toks)
    off = torch.nonzero(~sc.greedy).flatten().tolist()
    for i in off:  # the emitted token and the argmax at a non-greedy position are a near tie of that row
        alt = s.score(toks[:i] + [int(sc.argmax[i])])
        gap = alt.logprobs[i].item() - sc.logprobs[i].item()
        assert 0 <= gap < NEAR_TIE, f"position {i}: emitted {toks[i]}, argmax {int(sc.argmax[i])}, logit gap {gap:.4g}"
    print(f"\n{len(toks)} greedy tokens scored: {len(toks) - len(off)} greedy, {len(off)} near ties")
    assert len(off) <= 2
