"""The kernels and the chain decode loops at the ends of their caches.

Kernels, against a plain reference at the rows where a cache ends:
  * the tail copies (tf_tail_update, tf_tail_update_e4m3, tf_tail_update_to_e4m3) into a retrieval store carved out of a larger
    allocation with sentinel guard rows around every (layer, head) run: bit-exact, and the guards untouched, also when a
    device length claims up to G rows more than the budget (the kernels copy the last `budget` rows, never more);
  * the full-store attention at kv_len == cap, on stores whose capacity is not a multiple of the key tile, so the last key
    tile meets the end of the tensor map (fp64 reference of tests/attn_needles.py, a needle at the last slot);
  * the RoPE append at the last slots of a store and the last positions of the RoPE table (bit-exact).

Loops, step-wise (decoding.TriForceRun) and whole-loop graph (device_loop.DeviceLoopRun) from the same Philox seed, driven until
the room check refuses: they agree token for token, the retrieval cache holds what it should at the edge, and the refused step
changes nothing."""
from __future__ import annotations

from types import SimpleNamespace

import pytest
import torch

import kv_e4m3_oracle as eo
from attn_needles import Needles, base_logit, excess, reference, visibility, report_time_and_memory  # noqa: F401
from oracle import triforce_oracle as orc
from triforce_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda"

# ---------------------------------------------------------------------------------------------------------------------
# tail copies into a guarded retrieval store
# ---------------------------------------------------------------------------------------------------------------------
L_, H_, P_, B_, GAMMA_, GUARD = 2, 3, 256, 64, 4, 8
SRC_CAP = 384                     # >= P + B + GUARD, a multiple of 64 (an E4M3 store's rule)
RCAP = B_ + GAMMA_ + 1            # the retrieval store's rows: budget + gamma + 1 speculation slots
SENT_F16, SENT_CODE, SENT_EXP = 1000.0, 0xA5, 77  # no fp16 normal sample is 1000; 77 is no E4M3 row exponent


def _src(kind: str, d: int):
    """(the full store as the entry point takes it, its K and V rows as fp16 readers see them, the E4m3Store or None)."""
    g = torch.Generator(device=DEV).manual_seed(d)
    K = torch.randn((L_, H_, SRC_CAP, d), generator=g, device=DEV, dtype=torch.float16)
    V = torch.randn((L_, H_, SRC_CAP, d), generator=g, device=DEV, dtype=torch.float16)
    if kind == "fp16":
        return (K, V), K, V, None
    st = ops.E4m3Store.empty(L_, H_, SRC_CAP, d, DEV)
    for l in range(L_):
        ops.kv_quantize_e4m3(K[l], st.k_codes[l], st.k_exp[l], 0, SRC_CAP)
        ops.kv_quantize_e4m3(V[l], st.v_codes[l], st.v_exp[l], 0, SRC_CAP)
    Kd = eo.dequantize(st.k_codes.cpu(), st.k_exp.cpu()).to(DEV)
    Vd = eo.dequantize(st.v_codes.cpu(), st.v_exp.cpu()).to(DEV)
    return st, Kd, Vd, st


def _guarded(dst: str, d: int):
    """The retrieval store as views [L, H, RCAP, d] into [L, H, GUARD + RCAP + GUARD, d] allocations filled with sentinels.
    Returns (whole allocations, views): fp16 (K, V), or E4M3 (K codes, V codes, K exps, V exps)."""
    rows = GUARD + RCAP + GUARD
    if dst == "fp16":
        bufs = [torch.full((L_, H_, rows, d), SENT_F16, dtype=torch.float16, device=DEV) for _ in range(2)]
    else:
        bufs = [torch.full((L_, H_, rows, d), SENT_CODE, dtype=torch.uint8, device=DEV) for _ in range(2)]
        bufs += [torch.full((L_, H_, rows), SENT_EXP, dtype=torch.int8, device=DEV) for _ in range(2)]
    return bufs, [b[:, :, GUARD:GUARD + RCAP] for b in bufs]


def _tail(path: str, src, views, seq_len: int, dev_len: bool, max_new: int):
    kw = dict(seq_len_dev=torch.tensor([seq_len], dtype=torch.int32, device=DEV), max_new=max_new) if dev_len else {}
    host = 0 if dev_len else seq_len
    if path == "tail_update":
        ops.tail_update(src[0], src[1], views[0], views[1], P_, B_, host, **kw)
    elif path == "tail_update_e4m3":
        ops.tail_update_e4m3(src, views[0], views[1], P_, B_, host, **kw)
    else:  # the cache argument is read through .shape and its four tensors, so strided views stand in for an E4m3Store
        cache = SimpleNamespace(k_codes=views[0], v_codes=views[1], k_exp=views[2], v_exp=views[3], shape=tuple(views[0].shape))
        ops.tail_update_to_e4m3(src, cache, P_, B_, host, **kw)


# (entry point, source store, retrieval store)
TAIL_PATHS = [("tail_update", "fp16", "fp16"), ("tail_update_e4m3", "e4m3", "fp16"),
              ("tail_update_to_e4m3", "fp16", "e4m3"), ("tail_update_to_e4m3", "e4m3", "e4m3")]


@pytest.mark.parametrize("path,src_kind,dst", TAIL_PATHS)
@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("dev_len", [False, True], ids=["host_len", "dev_len"])
def test_tail_copy_at_the_budget_keeps_its_guards(path, src_kind, dst, d, dev_len):
    src, K, V, st = _src(src_kind, d)
    cases = [(n, m) for n in (0, 1, B_ - 1, B_) for m in ((1, B_) if dev_len else (0,))]
    if dev_len:  # a device length past the budget: the last B rows, nothing before slot 0 (k <= GUARD keeps a stray row inside)
        cases += [(B_ + k, m) for k in (1, 3, GUARD) for m in (1, B_)]
    for n_new, max_new in cases:
        bufs, views = _guarded(dst, d)
        before = [b.clone() for b in bufs]
        _tail(path, src, views, P_ + n_new, dev_len, max_new)
        torch.cuda.synchronize()
        n = min(n_new, B_)
        s0 = P_ + n_new - n  # the copied source rows: [seq_len - n, seq_len)
        what = f"{path} {src_kind}->{dst} d={d} n_new={n_new} max_new={max_new}"
        if dst == "fp16":
            want = [K[:, :, s0:s0 + n], V[:, :, s0:s0 + n]]
        elif st is not None:  # E4M3 into E4M3: the store's codes and exponents
            want = [st.k_codes[:, :, s0:s0 + n], st.v_codes[:, :, s0:s0 + n], st.k_exp[:, :, s0:s0 + n], st.v_exp[:, :, s0:s0 + n]]
        else:  # fp16 rows quantized by the oracle
            kc, ke = eo.quantize(K[:, :, s0:s0 + n].cpu())
            vc, ve = eo.quantize(V[:, :, s0:s0 + n].cpu())
            want = [kc, vc, ke, ve]
        for b, b0, w in zip(bufs, before, want):
            lo, hi = GUARD + B_ - n, GUARD + B_
            assert torch.equal(b[:, :, lo:hi].cpu(), w.cpu()), f"{what}: tail rows differ"
            assert torch.equal(b[:, :, :GUARD], b0[:, :, :GUARD]), f"{what}: guard rows before the store overwritten"
            assert torch.equal(b[:, :, GUARD:lo], b0[:, :, GUARD:lo]), f"{what}: rows before the tail overwritten"
            assert torch.equal(b[:, :, hi:], b0[:, :, hi:]), f"{what}: speculation slots or guard rows after the store overwritten"
    if not dev_len:  # a host length past the budget is refused before the launch
        bufs, views = _guarded(dst, d)
        with pytest.raises(RuntimeError, match="exceed budget"):
            _tail(path, src, views, P_ + B_ + 1, False, 0)


# ---------------------------------------------------------------------------------------------------------------------
# full-store attention at kv_len == cap
# ---------------------------------------------------------------------------------------------------------------------
def _needle_inputs(Hkv: int, d: int, cap: int, R: int, groups: int = 1, seed: int = 0):
    """K / V [1, Hkv, cap, d] with needles at the first key, the middle, the first key every row sees (cap - R) and the last
    slot (cap - 1, seen by the last row only); q [R, Hkv * groups, d], query head h reading KV head h // groups."""
    nd = Needles(Hkv, seed=seed + cap + d, d=d)
    K, V = nd.store(1, cap), nd.store(1, cap)
    keys = [0, cap // 2, cap - R, cap - 1]
    nd.plant(K, V, 0, keys, [base_logit(cap)] * len(keys))
    q = torch.stack([nd.queries(R) for _ in range(groups)], dim=2).reshape(R, Hkv * groups, d).contiguous()
    return nd, K, V, q


def _check_against_fp64(out, q, K, V, kv_len: int, groups: int, what: str):
    R, Hq, _ = q.shape
    vis = visibility(R, kv_len, kv_len, causal=True)
    for h in range(Hq):
        want = reference(q[:, h], K[0, h // groups], V[0, h // groups], vis)
        e = excess(out[:, h], want)
        assert e <= 1.0, f"{what}: head {h} off the fp64 reference by {e:.3g} of the tolerance"


def _dev_len(n: int) -> torch.Tensor:
    return torch.tensor([n], dtype=torch.int32, device=DEV)


def _in_graph(fn):
    """fn captured into a CUDA graph (after a warm-up on a side stream) and replayed once."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    g.replay()
    torch.cuda.synchronize()


@pytest.mark.parametrize("cap,H,d", [(259, 4, 64), (259, 4, 128), (4103, 4, 128), (124936, 8, 128)])
@pytest.mark.parametrize("mode", ["host_len", "dev_len", "graph"])
def test_verify_attn_reads_the_last_key_tile(cap, H, d, mode):
    R = GAMMA_ + 2
    nd, K, V, q = _needle_inputs(H, d, cap, R)
    maps = ops.KVTensorMaps(K, V)
    out = torch.full((R, H, d), float("nan"), dtype=torch.float16, device=DEV)
    ws = ops.verify_attn_workspace(R, H, d, DEV)
    if mode == "host_len":
        ops.verify_attn(q, maps, 0, cap, R, H, d, nd.scale, out, ws)
    else:  # the committed length on the device, the grid sized for the whole store (what a captured verify launches)
        dev = _dev_len(cap - R)
        call = lambda: ops.verify_attn(q, maps, 0, R, R, H, d, nd.scale, out, ws, kv_len_dev=dev)
        call() if mode == "dev_len" else _in_graph(call)
    _check_against_fp64(out, q, K, V, cap, 1, f"verify_attn cap={cap} d={d} {mode}")


@pytest.mark.parametrize("cap", [259, 4103])
@pytest.mark.parametrize("mode", ["host_len", "dev_len"])
def test_verify_attn_gqa_reads_the_last_key_tile(cap, mode):
    Hq, Hkv, d, R = 32, 8, 128, 13  # two row blocks of gqa_row_block(32, 8) = 8 rows
    nd, K, V, q = _needle_inputs(Hkv, d, cap, R, groups=Hq // Hkv)
    out = torch.full((R, Hq, d), float("nan"), dtype=torch.float16, device=DEV)
    ws = ops.verify_attn_gqa_workspace(Hq, Hkv, d, DEV)
    maps = ops.KVTensorMaps(K, V)
    if mode == "host_len":
        ops.verify_attn_gqa(q, maps, 0, cap, R, Hq, Hkv, d, nd.scale, out, ws)
    else:
        ops.verify_attn_gqa(q, maps, 0, R, R, Hq, Hkv, d, nd.scale, out, ws, kv_len_dev=_dev_len(cap - R))
    _check_against_fp64(out, q, K, V, cap, Hq // Hkv, f"verify_attn_gqa cap={cap} {mode}")


@pytest.mark.parametrize("slots,Hq,Hkv,d", [(320, 4, 4, 64), (320, 4, 4, 128), (4160, 32, 8, 128)])
@pytest.mark.parametrize("mode", ["host_len", "dev_len"])
def test_verify_attn_e4m3_reads_the_last_key_tile(slots, Hq, Hkv, d, mode):
    """An E4M3 store's slots are a multiple of VERIFY_BOX_KEYS, so its end is tile-aligned: kv_len == slots."""
    R = GAMMA_ + 2
    nd, K, V, q = _needle_inputs(Hkv, d, slots, R, groups=Hq // Hkv)
    st = ops.E4m3Store.empty(1, Hkv, slots, d, DEV)
    ops.kv_quantize_e4m3(K[0], st.k_codes[0], st.k_exp[0], 0, slots)
    ops.kv_quantize_e4m3(V[0], st.v_codes[0], st.v_exp[0], 0, slots)
    Kd = eo.dequantize(st.k_codes.cpu(), st.k_exp.cpu()).to(DEV)
    Vd = eo.dequantize(st.v_codes.cpu(), st.v_exp.cpu()).to(DEV)
    out = torch.full((R, Hq, d), float("nan"), dtype=torch.float16, device=DEV)
    ws = ops.verify_attn_gqa_workspace(Hq, Hkv, d, DEV)
    if mode == "host_len":
        ops.verify_attn_e4m3(q, st, 0, slots, R, Hq, Hkv, d, nd.scale, out, ws)
    else:
        ops.verify_attn_e4m3(q, st, 0, R, R, Hq, Hkv, d, nd.scale, out, ws, kv_len_dev=_dev_len(slots - R))
    _check_against_fp64(out, q, Kd, Vd, slots, Hq // Hkv, f"verify_attn_e4m3 slots={slots} {mode}")


@pytest.mark.parametrize("cap,R", [(259, 128), (4103, 200)])
def test_tree_attn_tc_causal_chunk_ending_at_the_last_slot(cap, R):
    H, d = 4, 128
    nd, K, V, q = _needle_inputs(H, d, cap, R)
    out = torch.full((R, H, d), float("nan"), dtype=torch.float16, device=DEV)
    ws = ops.tree_attn_tc_workspace(R, H, cap, DEV)
    ops.tree_attn_tc(q, ops.KVTensorMaps(K, V), 0, cap, R, H, d, nd.scale, None, 0, out, ws, causal=True)
    _check_against_fp64(out, q, K, V, cap, 1, f"tree_attn_tc causal cap={cap} R={R}")


# ---------------------------------------------------------------------------------------------------------------------
# RoPE append at the last slots and the last positions
# ---------------------------------------------------------------------------------------------------------------------
MAX_POS = 4096


@pytest.mark.parametrize("kind,Hq,Hkv,d,cap", [("fp16", 4, 4, 64, 259), ("fp16", 4, 4, 128, 259), ("gqa", 8, 2, 128, 259),
                                               ("e4m3", 8, 2, 128, 320), ("e4m3", 4, 4, 64, 320)])
@pytest.mark.parametrize("dev_len", [False, True], ids=["host_len", "dev_len"])
def test_rope_append_at_the_last_slots_and_positions(kind, Hq, Hkv, d, cap, dev_len):
    R = GAMMA_ + 2
    g = torch.Generator(device=DEV).manual_seed(cap + d + Hq)
    qkv = torch.randn((R, (Hq + 2 * Hkv) * d), generator=g, device=DEV, dtype=torch.float16)
    cos_np, sin_np = orc.rope_tables_plain(d, MAX_POS)
    cos, sin = torch.from_numpy(cos_np).to(DEV), torch.from_numpy(sin_np).to(DEV)
    q_out = torch.empty((R, Hq, d), dtype=torch.float16, device=DEV)
    slot0, pos0 = cap - R, MAX_POS - R  # the last R slots, at positions up to MAX_POS - 1
    pos = dict(pos0_dev=_dev_len(pos0), slot0_dev=_dev_len(slot0)) if dev_len else dict(pos0=pos0, slot0=slot0)
    if kind == "e4m3":
        st = ops.E4m3Store.empty(1, Hkv, cap, d, DEV)
        for t, v in ((st.k_codes, SENT_CODE), (st.v_codes, SENT_CODE), (st.k_exp, SENT_EXP), (st.v_exp, SENT_EXP)):
            t.fill_(v)
        ops.rope_append_e4m3(qkv, Hq, Hkv, d, cos, sin, q_out, st, 0, **pos)
        stores = [st.k_codes[0], st.v_codes[0], st.k_exp[0], st.v_exp[0]]
    else:
        Kl = torch.full((Hkv, cap, d), SENT_F16, dtype=torch.float16, device=DEV)
        Vl = torch.full_like(Kl, SENT_F16)
        if kind == "gqa":
            ops.rope_append_gqa(qkv, Hq, Hkv, d, cos, sin, q_out, Kl, Vl, **pos)
        else:
            ops.rope_append(qkv, Hq, d, cos, sin, q_out, Kl, Vl, **pos)
        stores = [Kl, Vl]
    torch.cuda.synchronize()
    x = qkv.cpu().numpy()
    p = pos0 + torch.arange(R).numpy()
    want_q = orc.apply_rope(x[:, :Hq * d].reshape(R, Hq, d), cos_np, sin_np, p)
    want_k = torch.from_numpy(orc.apply_rope(x[:, Hq * d:(Hq + Hkv) * d].reshape(R, Hkv, d), cos_np, sin_np, p)).transpose(0, 1)
    want_v = torch.from_numpy(x[:, (Hq + Hkv) * d:].reshape(R, Hkv, d)).transpose(0, 1)
    assert torch.equal(q_out.cpu(), torch.from_numpy(want_q)), "rotated queries differ"
    if kind == "e4m3":
        kc, ke = eo.quantize(want_k.contiguous())
        vc, ve = eo.quantize(want_v.contiguous())
        want, sent = [kc, vc, ke, ve], [SENT_CODE, SENT_CODE, SENT_EXP, SENT_EXP]
    else:
        want, sent = [want_k, want_v], [SENT_F16, SENT_F16]
    for t, w, s in zip(stores, want, sent):
        assert torch.equal(t[:, slot0:].cpu(), w), f"{kind}: appended rows differ"
        assert bool((t[:, :slot0] == s).all()), f"{kind}: rows before slot0 written"


# ---------------------------------------------------------------------------------------------------------------------
# the chain loops at the edge
# ---------------------------------------------------------------------------------------------------------------------
# (golden e2e case's shapes: target, prefill, budget, gamma; the full-KV store's and the retrieval cache's format)
LOOP_CASES = {"tiny": (512, 64, 4, "fp16"), "g16": (1024, 128, 16, "fp16"), "e4m3": (512, 64, 4, "e4m3")}
SAMPLING = dict(top_p=0.9, temperature=0.6)


def _engine(kind: str, slots: int):
    from triforce_b200.cache import FlashSimpleCache, RetrievalCache, StreamingLLMEvictionCache
    from triforce_b200.config import named_config
    from triforce_b200.engine import GraphInferenceEngine
    from triforce_b200.llama import LlamaModel
    from triforce_b200.synth import numpy_state_dict

    P, B, g, fmt = LOOP_CASES[kind]
    ts, ds = named_config("tiny-yarn-target"), named_config("llama-68M")
    target = LlamaModel(ts, numpy_state_dict(ts, 1), device=DEV)
    draft = LlamaModel(ds, numpy_state_dict(ds, 2), device=DEV, is_draft=True)
    cache = FlashSimpleCache(target, slots, kv_dtype=fmt)
    graph_cache = RetrievalCache(target, max_budget=B, prefill=P, gamma=g, chunk_size=8, kv_dtype=fmt, max_context=cache.slots)
    draft_cache = StreamingLLMEvictionCache(draft, start_size=16, recent_size=256 - 16 - g, gamma=g)
    ge = GraphInferenceEngine(target, cache, graph_cache, draft, draft_cache)
    ge.initialize_cuda_graph(g, probs=True, **SAMPLING)
    return ge


def _prompt(kind: str, seed: int):
    from triforce_b200.synth import numpy_prompt
    return numpy_prompt(LOOP_CASES[kind][0], seed=seed).cuda()


def _retrieval_rows(gc, B: int):
    """The retrieval cache's budget rows [L, H, B, ...] of K and V (E4M3: codes and exponents)."""
    ts = [gc.key_store, gc.value_store] + ([gc.e4m3.k_exp, gc.e4m3.v_exp] if gc.e4m3 is not None else [])
    return [t[:, :, :B] for t in ts]


def _store_rows(kv, a: int, b: int):
    ts = [kv.key_store, kv.value_store] + ([kv.e4m3.k_exp, kv.e4m3.v_exp] if kv.e4m3 is not None else [])
    return [t[:, :, a:b] for t in ts]


def _check_tail(eng, snapshot, what: str):
    """Budget rows [0, B - n) as the selection after the prompt left them, rows [B - n, B) the store's rows [P, S): bit-exact
    (both stores of a case have one format, so the tail copy moves fp16 rows or E4M3 codes and exponents unchanged)."""
    kv, gc = eng.kv_cache, eng.graph_cache
    B, P, S = gc.max_budget, gc.prefill, kv.seq_len
    n = S - P
    for got, snap, src in zip(_retrieval_rows(gc, B), snapshot, _store_rows(kv, P, S)):
        assert torch.equal(got[:, :, :B - n], snap[:, :, :B - n]), f"{what}: selected rows changed at S={S}"
        assert torch.equal(got[:, :, B - n:], src), f"{what}: tail rows differ from the store's rows [{P}, {S})"


def _state(eng, rng):
    """Everything a refused step must leave as it was."""
    kv, gc, dc = eng.kv_cache, eng.graph_cache, eng.draft_cache
    ts = [kv.key_store, kv.value_store, kv.seq_len_dev, gc.key_store, gc.value_store, dc.key_store, dc.value_store, rng]
    for c in (kv, gc):
        if c.e4m3 is not None:
            ts += [c.e4m3.k_exp, c.e4m3.v_exp]
    return (kv.seq_len, gc.prefill, dc.seq_len), [t.clone() for t in ts]


def _assert_refused_without_trace(run, eng, rng, limit: str):
    ints, before = _state(eng, rng)
    with pytest.raises(ValueError, match=rf"\({limit}\)"):
        run.step()
    torch.cuda.synchronize()
    ints_after, after = _state(eng, rng)
    assert ints_after == ints
    for i, (a, b) in enumerate(zip(before, after)):
        assert torch.equal(a, b), f"state tensor {i} changed by the refused step"


def _drive(run, eng, each_step=None, max_steps: int = 400):
    """Steps until the room check refuses; returns (tokens per step, committed length at the start of each step)."""
    steps, starts = [], []
    while run.room() is None:
        assert len(steps) < max_steps
        starts.append(eng.kv_cache.seq_len)
        before = len(run.generated)
        run.step()
        steps.append(run.generated[before:])
        if each_step is not None:
            each_step()
    return steps, starts


def _run_both(kind: str, slots: int, seed: int, prompt_seed: int, check_tail: bool):
    """The step-wise loop, then the device loop on a fresh engine (both see a first prompt), from one Philox seed, each until
    the room check refuses and then once more (refused without a trace).  Returns what each did."""
    from e2e_util import TokenizerStub
    from triforce_b200.decoding import TriForceRun
    from triforce_b200.device_loop import DeviceLoopRun, PhiloxNoise

    P, B, gamma, _ = LOOP_CASES[kind]
    ids, tok, out = _prompt(kind, prompt_seed), TokenizerStub(), {}
    for loop in ("step-wise", "device"):
        ge = _engine(kind, slots)
        eng = ge.engine
        if loop == "step-wise":
            run = TriForceRun(tok, ge, gamma=gamma, noise=PhiloxNoise(torch.device(DEV), seed), pad_full_verify=True, **SAMPLING)
            rng = run.noise.state
        else:
            run = DeviceLoopRun(tok, ge, gamma=gamma, seed=seed, **SAMPLING)
            rng = run.loop.rng
        run.prefill(ids)
        snapshot = [t.clone() for t in _retrieval_rows(eng.graph_cache, B)]
        each = (lambda: _check_tail(eng, snapshot, f"{kind} step-wise")) if check_tail and loop == "step-wise" else None
        steps, starts = _drive(run, eng, each)
        if check_tail:
            _check_tail(eng, snapshot, f"{kind} {loop}, last step")
        stop = run.room()
        _assert_refused_without_trace(run, eng, rng, stop)
        out[loop] = dict(tokens=list(run.generated), steps=steps, starts=starts, stop=stop, length=eng.kv_cache.seq_len,
                         counts=(run.accepted_count, run.draft_count, run.inner_iterations), slots=eng.kv_cache.slots,
                         last_row=eng.kv_cache.key_store[0, 0, eng.kv_cache.slots - 1].clone())
        del run, ge, eng
    h, d = out["step-wise"], out["device"]
    assert d["tokens"] == h["tokens"], (d["steps"][-4:], h["steps"][-4:])
    assert d["steps"] == h["steps"] and d["starts"] == h["starts"]
    assert d["length"] == h["length"] and d["counts"] == h["counts"] and d["stop"] == h["stop"]
    return h


@pytest.mark.parametrize("kind,seed", [("tiny", 3), ("g16", 7), ("e4m3", 5)])
def test_loops_agree_up_to_the_retrieval_tail(kind, seed):
    P, B, gamma, _ = LOOP_CASES[kind]
    h = _run_both(kind, P + B + 64, seed, prompt_seed=seed + 100, check_tail=True)
    assert h["stop"] == "tail"
    assert B - (h["length"] - P) < gamma + 2, "the loops stopped before the edge of the retrieval tail"
    print(f"{kind}: {len(h['tokens'])} tokens in {len(h['steps'])} steps; stopped with the tail at {h['length'] - P} of {B}")


def test_loops_agree_up_to_the_last_slot_of_the_store():
    """The store fills before the tail (slots < P + B).  A first run on a store of X0 slots finds the length S at which its last
    step started; on a store of S + gamma + 2 slots the same steps run and the last one writes slot slots - 1."""
    from e2e_util import TokenizerStub
    from triforce_b200.decoding import TriForceRun
    from triforce_b200.device_loop import PhiloxNoise

    kind, seed = "tiny", 11
    P, B, gamma, _ = LOOP_CASES[kind]
    x0 = P + 56  # 9 key tiles, like every store a few slots shorter: the verify's grid does not change
    ge = _engine(kind, x0)
    run = TriForceRun(TokenizerStub(), ge, gamma=gamma, noise=PhiloxNoise(torch.device(DEV), seed), pad_full_verify=True, **SAMPLING)
    run.prefill(_prompt(kind, 200))
    _, starts0 = _drive(run, ge.engine)
    assert run.room() == "slots"
    del run, ge
    slots = starts0[-1] + gamma + 2
    h = _run_both(kind, slots, seed, prompt_seed=200, check_tail=False)
    assert h["stop"] == "slots" and h["slots"] == slots
    assert h["starts"] == starts0 and h["starts"][-1] + gamma + 2 == slots, "the last step did not reach the store's last slot"
    assert bool(h["last_row"].ne(0).any()), "the last slot of the store was not written"


def test_session_stops_at_the_tail_and_goes_on_after_an_append():
    from e2e_util import TokenizerStub
    from triforce_b200.session import Session

    kind = "tiny"
    P, B, gamma, _ = LOOP_CASES[kind]
    ids, question = _prompt(kind, 300), list(range(1000, 1012))
    turns = {}
    for device_loop in (False, True):
        s = Session(_engine(kind, P + 3 * B), gamma=gamma, tokenizer=TokenizerStub(), pad_full_verify=True)
        s.prefill(ids)
        first = s.generate(10 * B, seed=4, device_loop=device_loop, **SAMPLING)
        assert s.last_stop == "tail" and len(first) < 10 * B
        end = s.length
        s.append(question)
        assert s.eng.graph_cache.prefill == (end + 1 + len(question)) // 8 * 8  # re-selected at the new boundary
        second = s.generate(16, seed=5, device_loop=device_loop, **SAMPLING)
        assert s.last_stop == "max_new" and len(second) >= 16
        turns[device_loop] = (first, second, s.length)
        del s
    assert turns[True] == turns[False]
    print(f"first turn {len(turns[False][0])} tokens (stopped at the tail), second turn {len(turns[False][1])} tokens")
