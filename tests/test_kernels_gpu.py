"""GPU parity tests: every sm_90a kernel, called THROUGH THE C ABI (triforce_b200.ops → ctypes), against the CPU oracle
on the same seeded inputs.  Bit-exact for index / byte / fp16-elementwise work, stated tolerances for attention."""
import os

import numpy as np
import pytest
import torch

import golden_inputs as gi
from oracle import triforce_oracle as orc
from triforce_b200 import _C, ops

pytestmark = pytest.mark.gpu
DEV = "cuda"


def head_major(x: np.ndarray, cap: int = None) -> torch.Tensor:
    """[S,H,d] numpy → [1,H,cap,d] cuda store."""
    S, H, d = x.shape
    cap = cap or S
    t = torch.zeros((1, H, cap, d), dtype=torch.float16, device=DEV)
    t[0, :, :S] = torch.from_numpy(x).to(DEV).permute(1, 0, 2)
    return t


def from_head_major(t: torch.Tensor, S: int) -> np.ndarray:
    return t[0, :, :S].permute(1, 0, 2).contiguous().cpu().numpy()


# ---------------------------------------------------------------------------------------------------------------------
# (i) retrieval build
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", gi.RETRIEVAL_CASES, ids=[c[0] for c in gi.RETRIEVAL_CASES])
def test_retrieval_build_bit_exact(case, golden_dir):
    name, H, d, P, chunk, budget, seed = case
    K, V, q = gi.retrieval_inputs(case)
    oK, oV, oidx, osc = orc.retrieval_build(K, V, q, P, chunk, budget)
    Ks, Vs = head_major(K, P + 16), head_major(V, P + 16)
    rK = torch.zeros((1, H, budget + 8, d), dtype=torch.float16, device=DEV)
    rV = torch.zeros_like(rK)
    idx = torch.zeros((1, H, budget // chunk), dtype=torch.int32, device=DEV)
    sc = torch.zeros((1, H, P // chunk), dtype=torch.float16, device=DEV)
    ops.retrieval_build(Ks, Vs, torch.from_numpy(q).to(DEV)[None].contiguous(), rK, rV, P, chunk, budget, out_idx=idx, out_scores=sc)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(sc[0].cpu().numpy().view(np.uint16), osc.view(np.uint16))  # bit-exact scores
    np.testing.assert_array_equal(idx[0].cpu().numpy(), oidx)                                # bit-exact top-k indices
    np.testing.assert_array_equal(from_head_major(rK, budget), oK)
    np.testing.assert_array_equal(from_head_major(rV, budget), oV)
    # and against the REFERENCE's own scores/indices (golden): same selected set, ties aside
    g = np.load(os.path.join(golden_dir, "retrieval_build.npz"))
    ref_idx = g[f"{name}.topk_idx_rest"]
    got = idx[0].cpu().numpy()
    same = sum(set(got[h, 1:]) == set(ref_idx[h]) for h in range(H))
    assert same >= H - 1, f"only {same}/{H} heads select the reference's chunk set"


def test_retrieval_build_full_size_properties():
    """BASELINE cfg2 geometry for a few layers (H=32, d=128, prefill=124928, budget=4096): size-independent properties."""
    L, H, d, P, chunk, budget = 2, 32, 128, 124928, 8, 4096
    g = torch.Generator(device=DEV).manual_seed(5)
    Ks = torch.randn((L, H, P + 64, d), generator=g, device=DEV, dtype=torch.float16)
    Vs = torch.randn((L, H, P + 64, d), generator=g, device=DEV, dtype=torch.float16)
    q = torch.randn((L, H, d), generator=g, device=DEV, dtype=torch.float16)
    rK = torch.zeros((L, H, budget + 7, d), dtype=torch.float16, device=DEV)
    rV = torch.zeros_like(rK)
    sel, chunks = budget // chunk, P // chunk
    idx = torch.zeros((L, H, sel), dtype=torch.int32, device=DEV)
    sc = torch.zeros((L, H, chunks), dtype=torch.float16, device=DEV)
    ops.retrieval_build(Ks, Vs, q, rK, rV, P, chunk, budget, out_idx=idx, out_scores=sc)
    torch.cuda.synchronize()
    # scores against an fp64 torch evaluation of the same formula
    kbar = Ks[:, :, :P].float().view(L, H, chunks, chunk, d).sum(3).mul(1.0 / chunk).half()
    ref = torch.einsum("lhcd,lhd->lhc", kbar.double(), q.double()).half()
    assert (ref.view(torch.int16) != sc.view(torch.int16)).float().mean().item() < 1e-4
    assert (idx[..., 0] == 0).all()
    li = idx.long()
    assert (li[..., 1:] >= 1).all() and (li[..., 1:] < chunks).all()
    vals = torch.gather(sc.float(), 2, li)[..., 1:]
    assert (vals[..., :-1] >= vals[..., 1:]).all(), "slots must be in descending score order"
    ties = vals[..., :-1] == vals[..., 1:]
    assert (li[..., 1:-1][ties] < li[..., 2:][ties]).all(), "ties must be in ascending chunk order"
    for l in range(L):
        for h in (0, 13, 31):
            assert len(set(li[l, h].tolist())) == sel
            kth = vals[l, h, -1].item()
            rest = sc[l, h, 1:].float()
            assert (rest > kth).sum().item() <= sel - 1 <= (rest >= kth).sum().item()
    # gather: slot s of head h holds chunk idx[h, s]
    src = Ks[:, :, :P].view(L, H, chunks, chunk * d)
    want = torch.gather(src, 2, li[..., None].expand(-1, -1, -1, chunk * d)).view(L, H, budget, d)
    assert torch.equal(rK[:, :, :budget], want)
    srcv = Vs[:, :, :P].view(L, H, chunks, chunk * d)
    wantv = torch.gather(srcv, 2, li[..., None].expand(-1, -1, -1, chunk * d)).view(L, H, budget, d)
    assert torch.equal(rV[:, :, :budget], wantv)
    assert (rK[:, :, budget:] == 0).all()


# ---------------------------------------------------------------------------------------------------------------------
# RoPE + append
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d,H,R", [(128, 4, 7), (64, 12, 5), (128, 2, 1)])
def test_rope_append_bit_exact(d, H, R):
    rng = np.random.Generator(np.random.PCG64(31))
    qkv = rng.standard_normal((R, 3 * H * d), dtype=np.float32).astype(np.float16)
    cos, sin = orc.rope_tables_yarn(d, 512, 4.0, 128)
    pos = np.array([300, 301, 17, 5, 511, 0, 42][:R])
    cap = 64
    Kc = torch.zeros((H, cap, d), dtype=torch.float16, device=DEV)
    Vc = torch.zeros_like(Kc)
    q_out = torch.empty((R, H, d), dtype=torch.float16, device=DEV)
    t = lambda a: torch.from_numpy(a).to(DEV)
    ops.rope_append(t(qkv), H, d, t(cos), t(sin), q_out, Kc, Vc, pos_ids=t(pos.astype(np.int32)), slot0=9)
    q = qkv[:, :H * d].reshape(R, H, d)
    k = qkv[:, H * d:2 * H * d].reshape(R, H, d)
    v = qkv[:, 2 * H * d:].reshape(R, H, d)
    np.testing.assert_array_equal(q_out.cpu().numpy().view(np.uint16), orc.apply_rope(q, cos, sin, pos).view(np.uint16))
    np.testing.assert_array_equal(Kc[:, 9:9 + R].permute(1, 0, 2).cpu().numpy().view(np.uint16),
                                  orc.apply_rope(k, cos, sin, pos).view(np.uint16))
    np.testing.assert_array_equal(Vc[:, 9:9 + R].permute(1, 0, 2).cpu().numpy(), v)
    assert (Kc[:, :9] == 0).all() and (Kc[:, 9 + R:] == 0).all()
    # device-side offsets + un-rotated keys (draft layout)
    Kc.zero_(); Vc.zero_()
    off = torch.tensor([20], dtype=torch.int32, device=DEV)
    ops.rope_append(t(qkv), H, d, t(cos), t(sin), q_out, Kc, Vc, pos0=3, pos0_dev=off, slot0=1, slot0_dev=off, rotate_k=False)
    np.testing.assert_array_equal(q_out.cpu().numpy().view(np.uint16),
                                  orc.apply_rope(q, cos, sin, 23 + np.arange(R)).view(np.uint16))
    np.testing.assert_array_equal(Kc[:, 21:21 + R].permute(1, 0, 2).cpu().numpy(), k)


# ---------------------------------------------------------------------------------------------------------------------
# (iii) verify attention
# ---------------------------------------------------------------------------------------------------------------------
def _attn_case(R, H, d, S, seed, cap_extra=70, scale=None):
    rng = np.random.Generator(np.random.PCG64(seed))
    q = rng.standard_normal((R, H, d), dtype=np.float32).astype(np.float16)
    K = rng.standard_normal((S, H, d), dtype=np.float32).astype(np.float16)
    V = rng.standard_normal((S, H, d), dtype=np.float32).astype(np.float16)
    scale = scale or orc.softmax_scale_fp16(d)
    return q, K, V, scale


def assert_attn_close(got: np.ndarray, want: np.ndarray):
    # fp16 outputs of an fp32-accumulated softmax·V; P is rounded to fp16 before the PV MMA as in FlashAttention-2
    np.testing.assert_allclose(got.astype(np.float32), want.astype(np.float32), rtol=1e-2, atol=2e-3)


@pytest.mark.parametrize("R,H,d,S", [(1, 4, 128, 64), (7, 4, 128, 100), (7, 3, 128, 4103), (8, 2, 128, 777), (16, 2, 128, 300),
                                     (5, 12, 64, 261), (1, 12, 64, 2049), (18, 2, 128, 500), (32, 1, 128, 129), (20, 3, 64, 333),
                                     (3, 2, 128, 3), (7, 32, 128, 4103)])
def test_verify_attn_matches_oracle(R, H, d, S):
    q, K, V, scale = _attn_case(R, H, d, S, seed=100 + R + S)
    want = orc.attention(q, K, V, scale, causal=True)
    Ks, Vs = head_major(K, S + 70), head_major(V, S + 70)
    Ks[0, :, S:] = 77.0  # stale rows beyond kv_len must be ignored
    Vs[0, :, S:] = -55.0
    maps = ops.KVTensorMaps(Ks, Vs)
    ws = ops.verify_attn_workspace(R, H, d, DEV)
    out = torch.empty((R, H, d), dtype=torch.float16, device=DEV)
    ops.verify_attn(torch.from_numpy(q).to(DEV), maps, 0, S, R, H, d, scale, out, ws)
    torch.cuda.synchronize()
    assert_attn_close(out.cpu().numpy(), want)
    # same launch with the length coming from device memory (CUDA-graph path): kv_len = host R + dev (S-R)
    out2 = torch.zeros_like(out)
    dev_len = torch.tensor([S - R], dtype=torch.int32, device=DEV)
    ops.verify_attn(torch.from_numpy(q).to(DEV), maps, 0, R, R, H, d, scale, out2, ws, kv_len_dev=dev_len, kv_len_max=S)
    torch.cuda.synchronize()
    assert torch.equal(out, out2)  # same split → bit-identical (the in-CTA merge is ordered, no atomics)
    # grid sized for the whole cache capacity (what a captured graph does): different split, same answer within rounding
    out3 = torch.zeros_like(out)
    ops.verify_attn(torch.from_numpy(q).to(DEV), maps, 0, R, R, H, d, scale, out3, ws, kv_len_dev=dev_len)
    torch.cuda.synchronize()
    assert_attn_close(out3.cpu().numpy(), want)


def test_verify_attn_layer_coordinate():
    L, H, d, S, R = 3, 2, 128, 200, 4
    rng = np.random.Generator(np.random.PCG64(7))
    Ks = torch.from_numpy(rng.standard_normal((L, H, S + 8, d), dtype=np.float32)).half().to(DEV)
    Vs = torch.from_numpy(rng.standard_normal((L, H, S + 8, d), dtype=np.float32)).half().to(DEV)
    q = rng.standard_normal((R, H, d), dtype=np.float32).astype(np.float16)
    maps = ops.KVTensorMaps(Ks, Vs)
    ws = ops.verify_attn_workspace(R, H, d, DEV)
    scale = orc.softmax_scale_fp16(d)
    for l in range(L):
        out = torch.empty((R, H, d), dtype=torch.float16, device=DEV)
        ops.verify_attn(torch.from_numpy(q).to(DEV), maps, l, S, R, H, d, scale, out, ws)
        want = orc.attention(q, Ks[l, :, :S].permute(1, 0, 2).cpu().numpy(), Vs[l, :, :S].permute(1, 0, 2).cpu().numpy(), scale)
        assert_attn_close(out.cpu().numpy(), want)


def test_verify_attn_full_128k_against_torch():
    """BASELINE cfg2 geometry: 7B heads, 124928-token prefix + gamma+2 = 8 rows; reference = torch fp32 on the GPU."""
    R, H, d, S = 8, 32, 128, 124928 + 8
    g = torch.Generator(device=DEV).manual_seed(11)
    Ks = torch.randn((1, H, S + 56, d), generator=g, device=DEV, dtype=torch.float16)
    Vs = torch.randn((1, H, S + 56, d), generator=g, device=DEV, dtype=torch.float16)
    q = torch.randn((R, H, d), generator=g, device=DEV, dtype=torch.float16)
    scale = orc.softmax_scale_fp16(d)
    maps = ops.KVTensorMaps(Ks, Vs)
    ws = ops.verify_attn_workspace(R, H, d, DEV)
    out = torch.empty((R, H, d), dtype=torch.float16, device=DEV)
    ops.verify_attn(q, maps, 0, S, R, H, d, scale, out, ws)
    torch.cuda.synchronize()
    for h in (0, 7, 31):
        s = (q[:, h].float() @ Ks[0, h, :S].float().T) * scale
        i = torch.arange(R, device=DEV)[:, None]
        j = torch.arange(S, device=DEV)[None, :]
        s = s.masked_fill(j > i + S - R, float("-inf"))
        want = (torch.softmax(s, -1) @ Vs[0, h, :S].float()).half()
        torch.testing.assert_close(out[:, h].float(), want.float(), rtol=1e-2, atol=2e-3)
    # linearity in V: attention(q, K, 2V) == 2 attention(q, K, V) exactly in fp16 (power-of-two scaling)
    Vs.mul_(2)
    out2 = torch.empty_like(out)
    ops.verify_attn(q, ops.KVTensorMaps(Ks, Vs), 0, S, R, H, d, scale, out2, ws)
    # (exact for normal fp16 outputs; outputs in the fp16 subnormal range round differently after doubling)
    torch.testing.assert_close(out2.float(), 2 * out.float(), rtol=0, atol=1.3e-7)


@pytest.mark.parametrize("R,H,S", [(8, 4, 124928 + 8), (7, 2, 50000), (1, 4, 70001), (12, 4, 60000)])
def test_verify_attn_head_sharded_long_store(R, H, S):
    """A tensor-parallel rank's view of the full store (4 of 32 heads at 8 GPUs): each head is cut into dozens of partials, which the
    last CTA of the head folds in two independent streams when R <= 8 (one stream otherwise); reference = torch fp32 on the GPU."""
    d = 128
    g = torch.Generator(device=DEV).manual_seed(300 + R + H)
    Ks = torch.randn((1, H, S + 56, d), generator=g, device=DEV, dtype=torch.float16)
    Vs = torch.randn((1, H, S + 56, d), generator=g, device=DEV, dtype=torch.float16)
    q = torch.randn((R, H, d), generator=g, device=DEV, dtype=torch.float16)
    scale = orc.softmax_scale_fp16(d)
    maps = ops.KVTensorMaps(Ks, Vs)
    ws = ops.verify_attn_workspace(R, H, d, DEV)
    out = torch.empty((R, H, d), dtype=torch.float16, device=DEV)
    ops.verify_attn(q, maps, 0, S, R, H, d, scale, out, ws)
    out_b = torch.empty_like(out)
    ops.verify_attn(q, maps, 0, S, R, H, d, scale, out_b, ws)
    torch.cuda.synchronize()
    assert torch.equal(out, out_b)  # ordered merge: same launch twice is bit-identical
    for h in range(H):
        s = (q[:, h].float() @ Ks[0, h, :S].float().T) * scale
        i = torch.arange(R, device=DEV)[:, None]
        j = torch.arange(S, device=DEV)[None, :]
        s = s.masked_fill(j > i + S - R, float("-inf"))
        want = (torch.softmax(s, -1) @ Vs[0, h, :S].float()).half()
        torch.testing.assert_close(out[:, h].float(), want.float(), rtol=1e-2, atol=2e-3)


def test_verify_attn_calibrated_split():
    """tf_verify_attn_calibrate re-cuts the per-CTA key ranges by measured rate: same answer (fp32 partial merges re-associate,
    so equal within fp16 rounding, not bitwise), deterministic for a given table, still correct for other lengths / rows."""
    R, H, d, S = 7, 32, 128, 65536 + 7
    g = torch.Generator(device=DEV).manual_seed(12)
    Ks = torch.randn((1, H, S + 57, d), generator=g, device=DEV, dtype=torch.float16)
    Vs = torch.randn((1, H, S + 57, d), generator=g, device=DEV, dtype=torch.float16)
    q = torch.randn((R, H, d), generator=g, device=DEV, dtype=torch.float16)
    scale = orc.softmax_scale_fp16(d)
    maps = ops.KVTensorMaps(Ks, Vs)
    ws = ops.verify_attn_workspace(R, H, d, DEV)
    out_eq = torch.empty((R, H, d), dtype=torch.float16, device=DEV)
    ops.verify_attn(q, maps, 0, S, R, H, d, scale, out_eq, ws)
    scratch = torch.empty_like(out_eq)
    rep = ops.verify_attn_calibrate(q, maps, 0, S, R, H, d, scale, scratch, ws, rounds=3)
    assert rep["spread_before"] >= 1.0 and rep["spread_after"] >= 1.0 and rep["median_ns_after"] > 0
    tab = ws.view(torch.int32)  # the table header somewhere in the workspace now carries the grid size
    assert int((tab == 2 * torch.cuda.get_device_properties(0).multi_processor_count).sum()) >= 1
    out_a, out_b = torch.empty_like(out_eq), torch.empty_like(out_eq)
    ops.verify_attn(q, maps, 0, S, R, H, d, scale, out_a, ws)
    ops.verify_attn(q, maps, 0, S, R, H, d, scale, out_b, ws)
    torch.cuda.synchronize()
    assert torch.equal(out_a, out_b)
    torch.testing.assert_close(out_a.float(), out_eq.float(), rtol=2e-3, atol=2e-5)
    for h in (0, 13, 31):
        sc = (q[:, h].float() @ Ks[0, h, :S].float().T) * scale
        i = torch.arange(R, device=DEV)[:, None]
        j = torch.arange(S, device=DEV)[None, :]
        sc = sc.masked_fill(j > i + S - R, float("-inf"))
        want = (torch.softmax(sc, -1) @ Vs[0, h, :S].float()).half()
        torch.testing.assert_close(out_a[:, h].float(), want.float(), rtol=1e-2, atol=2e-3)
    # other lengths and row counts under the same table (device-side length as in a captured graph), and a short one
    # that falls back to the equal split
    for (S2, R2) in [(40000, 1), (S, 7), (3000, 5), (300, 2)]:
        o1, o2 = torch.empty((R2, H, d), dtype=torch.float16, device=DEV), torch.empty((R2, H, d), dtype=torch.float16, device=DEV)
        ws_plain = ops.verify_attn_workspace(R2, H, d, DEV)
        ops.verify_attn(q[:R2].contiguous(), maps, 0, S2, R2, H, d, scale, o1, ws_plain)
        dev_len = torch.tensor([S2 - R2], dtype=torch.int32, device=DEV)
        ops.verify_attn(q[:R2].contiguous(), maps, 0, R2, R2, H, d, scale, o2, ws, kv_len_dev=dev_len)
        torch.testing.assert_close(o2.float(), o1.float(), rtol=2e-3, atol=2e-5)
    # rounds = 0 removes the table: back to the bit pattern of the equal split
    ops.verify_attn_calibrate(q, maps, 0, S, R, H, d, scale, scratch, ws, rounds=0)
    out_c = torch.empty_like(out_eq)
    ops.verify_attn(q, maps, 0, S, R, H, d, scale, out_c, ws)
    assert torch.equal(out_c, out_eq)
    print("calibration report:", rep)


# ---------------------------------------------------------------------------------------------------------------------
# (ii) draft attention with RoPE-on-read
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("R,kv_len", [(1, 253), (3, 255), (7, 259), (64, 252), (64, 64), (40, 300)])
def test_draft_attn_matches_oracle(R, kv_len):
    H, d = 12, 64
    rng = np.random.Generator(np.random.PCG64(900 + R))
    q = rng.standard_normal((R, H, d), dtype=np.float32).astype(np.float16)
    K = rng.standard_normal((kv_len, H, d), dtype=np.float32).astype(np.float16)
    V = rng.standard_normal((kv_len, H, d), dtype=np.float32).astype(np.float16)
    K[:16] = 0  # zero sinks (the reference's reset quirk)
    V[:16] = 0
    cos, sin = orc.rope_tables_plain(d, 2048)
    scale = orc.softmax_scale_fp16(d)
    want = orc.attention(q, orc.apply_rope(K, cos, sin, np.arange(kv_len)), V, scale, causal=True)
    Ks, Vs = head_major(K, kv_len + 5), head_major(V, kv_len + 5)
    out = torch.empty((R, H, d), dtype=torch.float16, device=DEV)
    t = lambda a: torch.from_numpy(a).to(DEV)
    ops.draft_attn(t(q), Ks[0], Vs[0], t(cos), t(sin), kv_len, scale, out)
    torch.cuda.synchronize()
    np.testing.assert_allclose(out.cpu().numpy().astype(np.float32), want.astype(np.float32), rtol=5e-3, atol=1e-3)


# ---------------------------------------------------------------------------------------------------------------------
# cache maintenance + elementwise glue
# ---------------------------------------------------------------------------------------------------------------------
def test_tail_update_and_window_slide():
    L, H, d, P, B = 3, 4, 128, 96, 32
    g = torch.Generator(device=DEV).manual_seed(3)
    Ks = torch.randn((L, H, P + 40, d), generator=g, device=DEV, dtype=torch.float16)
    Vs = torch.randn((L, H, P + 40, d), generator=g, device=DEV, dtype=torch.float16)
    rK = torch.randn((L, H, B + 5, d), generator=g, device=DEV, dtype=torch.float16)
    rV = torch.randn((L, H, B + 5, d), generator=g, device=DEV, dtype=torch.float16)
    for seq_len, use_dev in [(P + 7, False), (P + 19, True), (P, False), (P - 1, False)]:
        wK, wV = rK.clone(), rV.clone()
        n = seq_len - P
        if n > 0:
            wK[:, :, B - n:B] = Ks[:, :, P:seq_len]
            wV[:, :, B - n:B] = Vs[:, :, P:seq_len]
        if use_dev:
            dev = torch.tensor([seq_len], dtype=torch.int32, device=DEV)
            ops.tail_update(Ks, Vs, rK, rV, P, B, 0, dev, max_new=B)
        else:
            ops.tail_update(Ks, Vs, rK, rV, P, B, seq_len)
        assert torch.equal(rK, wK) and torch.equal(rV, wV)
    # overlapping slide with clone semantics (evict_for_spec, cache.py:263-265)
    C = torch.randn((2, 12, 259, 64), generator=g, device=DEV, dtype=torch.float16)
    D_ = torch.randn((2, 12, 259, 64), generator=g, device=DEV, dtype=torch.float16)
    wc, wd = C.clone(), D_.clone()
    wc[:, :, 16:16 + 234] = C[:, :, 19:19 + 234].clone()
    wd[:, :, 16:16 + 234] = D_[:, :, 19:19 + 234].clone()
    ops.window_slide(C, D_, 19, 16, 234)
    assert torch.equal(C, wc) and torch.equal(D_, wd)


@pytest.mark.parametrize("rows,hidden", [(1, 4096), (7, 768), (130, 5120)])
def test_add_rmsnorm_and_silu_mul(rows, hidden):
    rng = np.random.Generator(np.random.PCG64(rows))
    h = rng.standard_normal((rows, hidden), dtype=np.float32).astype(np.float16)
    dl = (rng.standard_normal((rows, hidden), dtype=np.float32) * 0.3).astype(np.float16)
    w = (1 + 0.1 * rng.standard_normal(hidden, dtype=np.float32)).astype(np.float16)
    t = lambda a: torch.from_numpy(a).to(DEV)
    ht, out = t(h.copy()), torch.empty((rows, hidden), dtype=torch.float16, device=DEV)
    ops.add_rmsnorm(ht, t(dl), t(w), 1e-5, out)
    hs = (h.astype(np.float32) + dl.astype(np.float32)).astype(np.float16)
    np.testing.assert_array_equal(ht.cpu().numpy().view(np.uint16), hs.view(np.uint16))  # residual add is exact fp16
    want = orc._rmsnorm(hs, w, 1e-5)
    # rsqrtf (GPU, 2 ulp) vs 1/sqrt (numpy) feeds two fp16 roundings: allow <= 2 fp16 ulps on a sliver of elements
    diff = np.abs(out.cpu().numpy().view(np.int16).astype(np.int32) - want.view(np.int16).astype(np.int32))
    assert diff.max() <= 2 and (diff != 0).mean() < 0.02 and (diff > 1).mean() < 1e-3
    inter = hidden * 2
    gu = rng.standard_normal((rows, 2 * inter), dtype=np.float32).astype(np.float16)
    act = torch.empty((rows, inter), dtype=torch.float16, device=DEV)
    ops.silu_mul(t(gu), act)
    want = (orc._silu16(gu[:, :inter]).astype(np.float32) * gu[:, inter:].astype(np.float32)).astype(np.float16)
    diff = np.abs(act.cpu().numpy().view(np.int16).astype(np.int32) - want.view(np.int16).astype(np.int32))
    assert diff.max() <= 2 and (diff != 0).mean() < 0.02 and (diff > 1).mean() < 1e-4  # expf (GPU) vs numpy exp


# ---------------------------------------------------------------------------------------------------------------------
# sampling
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", gi.SAMPLING_CASES, ids=[c[0] for c in gi.SAMPLING_CASES])
def test_norm_logits_matches_reference_fixture(case, golden_dir):
    name = case[0]
    g = np.load(os.path.join(golden_dir, "sampling.npz"))
    logits = gi.sampling_logits(case)
    probs = ops.norm_logits(torch.from_numpy(logits).to(DEV), case[4], case[5]).cpu().numpy()
    ref = g[f"{name}.probs"]
    np.testing.assert_array_equal(probs > 0, ref > 0)  # identical nucleus, ties in ascending index order
    np.testing.assert_allclose(probs, ref, rtol=1e-5, atol=1e-10)
    np.testing.assert_allclose(probs.sum(-1), 1.0, rtol=1e-5)
    p, q = gi.residual_pair(case)
    got = ops.residual_probs(torch.from_numpy(p).to(DEV), torch.from_numpy(q).to(DEV)).cpu().numpy()
    np.testing.assert_allclose(got, g[f"{name}.max_fn"], rtol=1e-5, atol=1e-12)


def test_norm_logits_tie_quota_and_strided_rows():
    """Massive exact ties at the nucleus boundary: the kept set must be the canonical one — everything above the
    threshold value plus the FIRST tied tokens in ascending index order (what a stable descending sort gives) — and its
    size must agree with the oracle's up to cumulative-sum rounding (32000 equal addends: order-of-summation noise)."""
    V = 32000
    x = np.zeros((3, V), np.float32)
    x[0, ::2] = 1.0          # half of the tokens tie at the top
    x[1, :] = 0.5            # everything ties
    x[2, 100] = 30.0         # one dominant token
    want = orc.norm_logits(x.copy(), 0.6, -1, 0.9)
    big = torch.zeros((3, V + 13), dtype=torch.float32, device=DEV)
    big[:, :V] = torch.from_numpy(x).to(DEV)
    got = ops.norm_logits(big[:, :V], 0.6, 0.9).cpu().numpy()
    np.testing.assert_allclose(got.sum(-1), 1.0, rtol=1e-5)
    kept, okept = got > 0, want > 0
    assert abs(int(kept[0].sum()) - int(okept[0].sum())) <= 16 and abs(int(kept[1].sum()) - int(okept[1].sum())) <= 16
    assert kept[0, ::2].all()                                   # the whole top group survives
    odd = kept[0, 1::2]
    assert odd[:odd.sum()].all() and not odd[odd.sum():].any()  # tied group: a prefix in index order
    assert kept[1, :kept[1].sum()].all() and not kept[1, kept[1].sum():].any()
    np.testing.assert_array_equal(kept[2], okept[2])
    assert kept[2].sum() == 1 and kept[2, 100]
    nz = kept & okept
    np.testing.assert_allclose(got[2], want[2], rtol=1e-5, atol=1e-10)
    np.testing.assert_allclose(got[nz], want[nz], rtol=2e-3)


def test_top_k_top_p_filter_and_top_k_norm_logits_follow_the_reference_formulas():
    """utils/sampling.py:5-27 (top_k_top_p_filter) and norm_logits with top_k > 0 — not on the hot path (the loops pass top_k = -1)
    but part of the reference's call surface: checked against the reference's own formulas restated with torch on the CPU."""
    from triforce_b200.sampling import norm_logits, top_k_top_p_filter

    def ref_filter(logits, top_k, top_p):  # the reference's code, with the stable sort its CUDA path has
        logits = logits.clone()
        if top_k > 0:
            f = torch.topk(logits, min(top_k, logits.size(-1)))[0]
            logits[logits < f[:, [-1]]] = float("-inf")
        if top_p > 0.0:
            sl, si = torch.sort(logits, descending=True, stable=True)
            cp = torch.cumsum(torch.softmax(sl, dim=-1), dim=-1)
            flt = cp > top_p
            flt[..., 1:] = flt[..., :-1].clone()
            flt[..., 0] = 0
            logits[flt.scatter(1, si, flt)] = float("-inf")
        return logits

    g = torch.Generator().manual_seed(3)
    x = (torch.randn((4, 32000), generator=g) * 3).float()
    for top_k, top_p in ((50, 0.9), (0, 0.8), (5, 0.0), (1000, 0.95)):
        want = ref_filter(x, top_k, top_p)
        got = top_k_top_p_filter(x.clone().to(DEV), top_k=top_k, top_p=top_p).cpu()
        assert torch.equal(torch.isinf(got), torch.isinf(want)), (top_k, top_p)
        assert torch.equal(got[~torch.isinf(got)], want[~torch.isinf(want)])
    want = torch.softmax(ref_filter(x / 0.6, 40, 0.9), dim=-1)
    got = norm_logits(x.to(DEV), temperature=0.6, top_k=40, top_p=0.9).cpu()
    assert torch.equal(got > 0, want > 0)
    torch.testing.assert_close(got, want, rtol=1e-5, atol=1e-10)


def test_sample_argmax_bit_exact():
    from triforce_b200.rng import CounterNoise
    rng = np.random.Generator(np.random.PCG64(77))
    V = 32000
    noise = CounterNoise(5)
    for trial in range(6):
        p = rng.random(V, dtype=np.float32) ** (1 + trial)
        p[rng.random(V) < 0.4] = 0
        p = (p / p.sum()).astype(np.float32)
        e = noise.exponential(V)
        want = orc.sample_from_noise(p, e)
        got = ops.sample_argmax(torch.from_numpy(p).to(DEV), torch.from_numpy(e).to(DEV))
        assert int(got.item()) == want
    # ties → first index; all-zero row → index 0
    p = np.zeros(V, np.float32); p[[5, 9]] = 0.5
    e = np.ones(V, np.float32)
    assert int(ops.sample_argmax(torch.from_numpy(p).to(DEV), torch.from_numpy(e).to(DEV)).item()) == 5
    assert int(ops.sample_argmax(torch.zeros(V, device=DEV), torch.ones(V, device=DEV)).item()) == 0


def _prob_rows(rng, rows, V, zero_frac=0.3):
    a = rng.random((rows, V), dtype=np.float32) ** 3
    a[rng.random((rows, V)) < zero_frac] = 0
    return (a / a.sum(-1, keepdims=True, dtype=np.float32)).astype(np.float32)


def test_middle_accept_matches_reference_semantics():
    """decoding.py:192-220 on random probabilities: accept flag, emitted ids, proposal rows, slot update — exact."""
    from triforce_b200.rng import CounterNoise
    rng = np.random.Generator(np.random.PCG64(123))
    V, gamma = 4096, 4
    noise = CounterNoise(99)
    t = lambda a: torch.from_numpy(a).to(DEV)
    for trial in range(40):
        n = int(rng.integers(0, gamma))
        k = int(rng.integers(0, 3))
        sp = _prob_rows(rng, 1, V)[0]
        vp = _prob_rows(rng, gamma + 1, V)
        vt = rng.integers(0, V, gamma + 1).astype(np.int64)
        tok = int(rng.choice(np.nonzero(sp)[0]))
        vt[n + 1] = tok
        if trial % 3 == 0:
            vp[n, tok] = 0.0  # certain reject
        r = noise.uniform()
        e = noise.exponential(V)
        with np.errstate(divide="ignore", invalid="ignore"):
            ok = np.float32(r) < np.minimum(np.float32(1), vp[n, tok] / sp[tok])
        st = torch.tensor([n, k, 0, 10, 20, 0, 0, 0], dtype=torch.int32, device=DEV)
        out_ids = torch.full((gamma + 2,), -1, dtype=torch.int64, device=DEV)
        spec = torch.zeros((gamma + 2, V), dtype=torch.float32, device=DEV)
        vtd = t(vt.copy())
        ops.middle_accept(t(sp), t(vp), vtd, torch.tensor([r], device=DEV), t(e), gamma, st, out_ids, spec)
        st_h, ids_h, vt_h = st.tolist(), out_ids.tolist(), vtd.tolist()
        if ok:
            t2 = orc.sample_from_noise(vp[n + 1], e)
            assert st_h[:5] == [n + 2, k + 2, 1, 11, 21]
            assert ids_h[k] == tok and ids_h[k + 1] == t2
            np.testing.assert_array_equal(spec[k].cpu().numpy(), vp[n])
            np.testing.assert_array_equal(spec[k + 1].cpu().numpy(), vp[n + 1])
            if n + 2 <= gamma:
                assert vt_h[n + 2] == t2
        else:
            t2 = orc.sample_from_noise(vp[n], e)
            assert st_h[:5] == [n + 1, k + 1, 0, 10, 21]
            assert ids_h[k] == t2 and vt_h[n + 1] == t2
            np.testing.assert_array_equal(spec[k].cpu().numpy(), vp[n])


def test_verify_accept_and_resample_match_oracle():
    """decoding.py:97-134: accept mask, count, residual / bonus token, pass_tokens — exact, incl. EOS and NaN ratios."""
    from triforce_b200.rng import CounterNoise
    rng = np.random.Generator(np.random.PCG64(321))
    V = 4096
    noise = CounterNoise(42)
    t = lambda a: torch.from_numpy(a).to(DEV)
    for trial in range(60):
        g2 = int(rng.integers(1, 8))
        p = _prob_rows(rng, g2 + 1, V)
        qrows = _prob_rows(rng, g2, V)
        gen = np.array([int(rng.choice(np.nonzero(qrows[i])[0])) for i in range(g2)], dtype=np.int64)
        if trial % 4 == 0:  # make acceptance likely
            for i in range(g2):
                p[i, gen[i]] = max(p[i, gen[i]], qrows[i, gen[i]] * 2)
        eos = int(gen[g2 // 2]) if trial % 7 == 0 else 2
        u = np.array([noise.uniform() for _ in range(g2)], dtype=np.float32)
        e = noise.exponential(V)
        strict = trial % 5 != 0
        # oracle walk (with the reference's EOS break)
        count, rejected, examined, hit = 0, False, 0, False
        for i in range(g2):
            examined += 1
            c, rj = orc.accept_walk([gen[i]], [qrows[i]], p[i:i + 1], [u[i]], strict_less=strict)
            if rj:
                rejected = True
                break
            count += 1
            if gen[i] == eos:
                hit = True
                break
        res = torch.zeros(4, dtype=torch.int32, device=DEV)
        pt = torch.zeros(g2 + 2, dtype=torch.int64, device=DEV)
        ot = torch.zeros(1, dtype=torch.int64, device=DEV)
        ops.verify_accept(t(p), t(qrows), t(gen), g2, t(u), strict, eos, 1234, res, pt)
        assert res.tolist() == [count, int(rejected), examined, int(hit)]
        ops.verify_resample(t(p), t(qrows), t(gen), g2, t(e), res, ot, pt)
        want_pass = [1234] + [100] * (g2 + 1)
        for i in range(count):
            want_pass[1 + i] = int(gen[i])
        if rejected:
            tok = orc.sample_from_noise(orc.max_fn(p[count] - qrows[count]), e)
            want_pass[count + 1] = tok
            assert res.tolist()[0] == count
        elif count == g2:
            tok = orc.sample_from_noise(p[g2], e)
            want_pass[count + 1] = tok
            assert res.tolist()[0] == count + 1
        else:
            tok = int(gen[count - 1])
        assert int(ot.item()) == tok
        assert pt.tolist() == want_pass


# ---------------------------------------------------------------------------------------------------------------------
# decode-time linear layers (row f-1)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,N,K", [(1, 4096, 4096), (7, 12288, 4096), (8, 4096, 11008), (16, 22016, 4096), (5, 32000, 4096),
                                   (7, 768, 768), (3, 130, 96), (7, 2304, 768), (2, 768, 3072)])
def test_skinny_gemm_matches_fp32_reference(M, N, K):
    g = torch.Generator(device=DEV).manual_seed(M * 1000 + N)
    x = torch.randn((M, K), generator=g, device=DEV, dtype=torch.float16)
    W = (torch.randn((N, K), generator=g, device=DEV, dtype=torch.float16) * 0.05)
    y = ops.skinny_gemm(x, W)
    ref = (x.float() @ W.float().T)
    # fp32 accumulate, one rounding to fp16 at the end: within half an fp16 ulp of the fp32 result (+ accumulation noise)
    torch.testing.assert_close(y.float(), ref.half().float(), rtol=2e-3, atol=2e-3)
    assert (y.float() - ref).abs().max().item() <= 2e-3 * max(1.0, ref.abs().max().item())
    # strided x (a slice of a wider activation) and determinism
    xw = torch.randn((M, K + 64), generator=g, device=DEV, dtype=torch.float16)
    y1 = ops.skinny_gemm(xw[:, :K], W)
    y2 = ops.skinny_gemm(xw[:, :K].contiguous(), W)
    assert torch.equal(y1, y2)
    assert torch.equal(ops.skinny_gemm(x, W), y)


@pytest.mark.parametrize("M,N,K", [(1, 4096, 4096), (7, 12288, 4096), (8, 4096, 11008), (16, 22016, 4096), (9, 4096, 4096), (17, 12288, 4096),
                                   (24, 4096, 5504), (5, 32000, 4096), (7, 768, 768), (3, 130, 128), (7, 40, 64), (2, 768, 3072), (8, 4096, 5504),
                                   (7, 5120, 13824), (18, 2304, 768)])
def test_stream_linear_matches_fp32_reference(M, N, K):
    g = torch.Generator(device=DEV).manual_seed(M * 1000 + N + 1)
    x = torch.randn((M, K), generator=g, device=DEV, dtype=torch.float16)
    W = (torch.randn((N, K), generator=g, device=DEV, dtype=torch.float16) * 0.05)
    y = ops.stream_linear(x, W)
    ref = (x.float() @ W.float().T)
    # fp32 accumulate, one rounding to fp16 at the end: within half an fp16 ulp of the fp32 result (+ accumulation noise)
    torch.testing.assert_close(y.float(), ref.half().float(), rtol=2e-3, atol=2e-3)
    assert (y.float() - ref).abs().max().item() <= 2e-3 * max(1.0, ref.abs().max().item())
    xw = torch.randn((M, K + 64), generator=g, device=DEV, dtype=torch.float16)
    assert torch.equal(ops.stream_linear(xw[:, :K], W), ops.stream_linear(xw[:, :K].contiguous(), W))  # strided rows
    assert torch.equal(ops.stream_linear(x, W), y)                                                       # deterministic
    # fp32 epilogue (lm_head + .float() of the reference): exactly the fp16 result, widened
    assert torch.equal(ops.stream_linear(x, W, out_fp32=True), y.float())


def test_stream_linear_under_programmatic_dependent_launch():
    """With tf_set_pdl the kernels of a chain start before their predecessor has finished (weight ring filled before
    griddepcontrol.wait).  A chain x -> W1 -> W2 -> W3 replayed from a CUDA graph must give the bits of the serial launches."""
    g = torch.Generator(device=DEV).manual_seed(5)
    x = torch.randn((7, 4096), generator=g, device=DEV, dtype=torch.float16)
    Ws = [ops.WeightMap(torch.randn((4096, 4096), generator=g, device=DEV, dtype=torch.float16) * 0.02) for _ in range(6)]

    def chain():
        y = x
        for w in Ws:
            y = ops.stream_linear(y, w)
        return y

    want = chain().clone()
    lib = _C.lib()
    try:
        lib.tf_set_pdl(255)
        got = chain().clone()
        assert torch.equal(got, want)
        torch.cuda.synchronize()
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr):
            out = chain()
        for _ in range(3):
            gr.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, want)
    finally:
        lib.tf_set_pdl(int(os.environ.get("TRIFORCE_PDL", str(_C.DEFAULT_PDL_MASK))))  # the mask _C.lib() loaded with


@pytest.mark.parametrize("M,inter,K", [(1, 11008, 4096), (7, 11008, 4096), (8, 13824, 5120), (16, 5504, 4096), (8, 24, 64), (5, 1376, 4096),
                                       (7, 3072, 768), (17, 2752, 4096)])
def test_stream_linear_silu_epilogue_is_bit_identical_to_silu_mul(M, inter, K):
    g = torch.Generator(device=DEV).manual_seed(M + inter)
    x = torch.randn((M, K), generator=g, device=DEV, dtype=torch.float16)
    W = (torch.randn((2 * inter, K), generator=g, device=DEV, dtype=torch.float16) * 0.05)
    # The SiLU launch tiles the stack as (8 gate rows, their 8 up rows).  The plain launch on the weights re-stacked in that
    # tile order has the same tiles and the same k-splits, so its product — un-permuted — followed by tf_silu_mul must give
    # the same bits.
    assert inter % 8 == 0
    perm = torch.stack([torch.arange(inter, device=DEV).view(-1, 8), inter + torch.arange(inter, device=DEV).view(-1, 8)], dim=1).reshape(-1)
    gu_perm = ops.stream_linear(x, W[perm].contiguous())
    gu = torch.empty_like(gu_perm)
    gu[:, perm] = gu_perm
    want = torch.empty((M, inter), dtype=torch.float16, device=DEV)
    ops.silu_mul(gu, want)
    got = ops.stream_linear(x, W, silu=True)
    assert torch.equal(got, want)
    # and within fp16 rounding of the product in natural row order (only tiles cut by a CTA boundary re-associate)
    gu_nat = ops.stream_linear(x, W)
    assert (gu_nat != gu).float().mean().item() < 0.2
    torch.testing.assert_close(gu_nat.float(), gu.float(), rtol=2e-3, atol=2e-3)
    ref = torch.nn.functional.silu(gu[:, :inter].float()) * gu[:, inter:].float()
    torch.testing.assert_close(got.float(), ref, rtol=2e-3, atol=2e-3)


@pytest.mark.parametrize("M,N,K,world", [(7, 4096, 512, 2), (1, 4096, 1408, 4), (8, 768, 384, 2), (17, 4096, 2752, 2), (24, 5120, 640, 8), (3, 4096, 512, 3)])
def test_ll_seam_matches_allreduce_then_add_rmsnorm(M, N, K, world):
    """The LL seam (tf_stream_linear_ll_push -> tf_add_rmsnorm_ll) with `world` ranks emulated on ONE GPU: every rank has its own
    inbox and epoch (as on its own GPU) and sees the others' inboxes as peer pointers (no multicast mapping here, so the per-peer
    store path runs).  Must be bit-identical to: fp16 partials, summed in rank order in fp32, rounded to fp16, tf_add_rmsnorm."""
    import ctypes
    lib = _C.lib()
    g = torch.Generator(device=DEV).manual_seed(M * 31 + N + K + world)
    xs = [torch.randn((M, K), generator=g, device=DEV, dtype=torch.float16) for _ in range(world)]
    Ws = [torch.randn((N, K), generator=g, device=DEV, dtype=torch.float16) * 0.05 for _ in range(world)]
    maps = [ops.WeightMap(W) for W in Ws]
    ln = torch.randn((N,), generator=g, device=DEV, dtype=torch.float16)
    h0 = torch.randn((M, N), generator=g, device=DEV, dtype=torch.float16)
    max_bytes = 24 * N * 2
    bufs = [torch.zeros(lib.tf_allreduce_ll_buffer_bytes(max_bytes), dtype=torch.uint8, device=DEV) for _ in range(world)]
    states = [torch.zeros(2, dtype=torch.int32, device=DEV) for _ in range(world)]
    ptrs = (ctypes.c_void_p * world)(*[b.data_ptr() for b in bufs])
    ws = ops.stream_linear_workspace(DEV)
    for rounds in range(3):  # three exchanges: both inbox parities and a reused one
        want_h = h0.clone()
        partial = [ops.stream_linear(xs[r], maps[r]) for r in range(world)]
        acc = torch.zeros((M, N), dtype=torch.float32, device=DEV)
        for r in range(world):
            acc += partial[r].float()
        want_x = torch.empty_like(h0)
        ops.add_rmsnorm(want_h, acc.half(), ln, 1e-6, want_x)
        for r in range(world):
            _C.check(lib.tf_stream_linear_ll_push(xs[r].data_ptr(), xs[r].stride(0), maps[r].ptr, M, N, K, ws.data_ptr(), ws.numel(), ptrs, None, r,
                                                  world, max_bytes, states[r].data_ptr(), _C.stream_ptr()), "tf_stream_linear_ll_push")
        for r in range(world):
            h = h0.clone()
            x = torch.empty_like(h)
            _C.check(lib.tf_add_rmsnorm_ll(h.data_ptr(), bufs[r].data_ptr(), world, max_bytes, states[r].data_ptr(), ln.data_ptr(), 1e-6,
                                           x.data_ptr(), M, N, _C.stream_ptr()), "tf_add_rmsnorm_ll")
            torch.cuda.synchronize()
            assert torch.equal(h, want_h) and torch.equal(x, want_x), f"rank {r}, exchange {rounds}"
            assert int(states[r][0]) == rounds + 1 and int(states[r][1]) == 0
        xs = [x_ * 0.5 + 0.25 for x_ in xs]  # new payloads for the next exchange
    # the consumer launched BEFORE the pushes (side stream): it must spin on stale flags, re-poll, and finish once the slots arrive
    import time
    want_h = h0.clone()
    acc = torch.zeros((M, N), dtype=torch.float32, device=DEV)
    for r in range(world):
        acc += ops.stream_linear(xs[r], maps[r]).float()
    want_x = torch.empty_like(h0)
    ops.add_rmsnorm(want_h, acc.half(), ln, 1e-6, want_x)
    h_early, x_early = h0.clone(), torch.empty_like(h0)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        _C.check(lib.tf_add_rmsnorm_ll(h_early.data_ptr(), bufs[0].data_ptr(), world, max_bytes, states[0].data_ptr(), ln.data_ptr(), 1e-6,
                                       x_early.data_ptr(), M, N, _C.stream_ptr()), "tf_add_rmsnorm_ll")
    time.sleep(0.05)
    assert not side.query()  # still waiting for its peers
    for r in range(world):
        _C.check(lib.tf_stream_linear_ll_push(xs[r].data_ptr(), xs[r].stride(0), maps[r].ptr, M, N, K, ws.data_ptr(), ws.numel(), ptrs, None, r,
                                              world, max_bytes, states[r].data_ptr(), _C.stream_ptr()), "tf_stream_linear_ll_push")
    side.synchronize()
    torch.cuda.synchronize()
    assert torch.equal(h_early, want_h) and torch.equal(x_early, want_x)
    for r in range(1, world):  # the other ranks consume the same exchange (keeps every epoch in step)
        h, x = h0.clone(), torch.empty_like(h0)
        _C.check(lib.tf_add_rmsnorm_ll(h.data_ptr(), bufs[r].data_ptr(), world, max_bytes, states[r].data_ptr(), ln.data_ptr(), 1e-6,
                                       x.data_ptr(), M, N, _C.stream_ptr()), "tf_add_rmsnorm_ll")
        torch.cuda.synchronize()
        assert torch.equal(h, want_h) and torch.equal(x, want_x)
    with pytest.raises(_C.TriForceNativeError):  # a message larger than the inbox is refused, not truncated
        _C.check(lib.tf_stream_linear_ll_push(xs[0].data_ptr(), xs[0].stride(0), maps[0].ptr, M, N, K, ws.data_ptr(), ws.numel(), ptrs, None, 0, world,
                                              64, states[0].data_ptr(), _C.stream_ptr()), "tf_stream_linear_ll_push")


@pytest.mark.parametrize("rows,hidden,world", [(1, 4096, 2), (7, 4096, 8), (17, 768, 4), (24, 5120, 3)])
def test_allreduce_ll_emulated_ranks(rows, hidden, world):
    """tf_allreduce_ll (stand-alone LL exchange) with `world` ranks emulated on ONE GPU, one stream per rank so that the kernels
    run concurrently (each pushes, then polls for all the others): rank-order fp32 sum rounded to fp16, identical on every rank,
    over three exchanges (both inbox parities)."""
    import ctypes
    lib = _C.lib()
    g = torch.Generator(device=DEV).manual_seed(rows + hidden + world)
    max_bytes = 24 * hidden * 2
    bufs = [torch.zeros(lib.tf_allreduce_ll_buffer_bytes(max_bytes), dtype=torch.uint8, device=DEV) for _ in range(world)]
    states = [torch.zeros(2, dtype=torch.int32, device=DEV) for _ in range(world)]
    ptrs = (ctypes.c_void_p * world)(*[b.data_ptr() for b in bufs])
    streams = [torch.cuda.Stream() for _ in range(world)]
    for exchange in range(3):
        ts = [torch.randn((rows, hidden), generator=g, device=DEV, dtype=torch.float16) for _ in range(world)]
        acc = torch.zeros((rows, hidden), dtype=torch.float32, device=DEV)
        for t in ts:
            acc += t.float()
        want = acc.half()
        torch.cuda.synchronize()
        for r in range(world):
            with torch.cuda.stream(streams[r]):
                _C.check(lib.tf_allreduce_ll(ptrs, None, r, world, ts[r].data_ptr(), ts[r].data_ptr(), ts[r].numel(), max_bytes,
                                             states[r].data_ptr(), _C.stream_ptr()), "tf_allreduce_ll")
        torch.cuda.synchronize()
        for r in range(world):
            assert torch.equal(ts[r], want), f"rank {r}, exchange {exchange}"
            assert int(states[r][0]) == exchange + 1


def test_stream_linear_zero_padded_k():
    """A weight shard whose K is not a multiple of 64 (7B down_proj over 8 GPUs: K = 1376) runs zero-padded: W and x padded to
    1408 columns give the unpadded product (the pad columns contribute exact zeros)."""
    M, N, K, Kp = 7, 4096, 1376, 1408
    g = torch.Generator(device=DEV).manual_seed(77)
    Wp = torch.zeros((N, Kp), dtype=torch.float16, device=DEV)
    Wp[:, :K] = torch.randn((N, K), generator=g, device=DEV, dtype=torch.float16) * 0.05
    xp = torch.zeros((24, Kp), dtype=torch.float16, device=DEV)
    xp[:M, :K] = torch.randn((M, K), generator=g, device=DEV, dtype=torch.float16)
    y = ops.stream_linear(xp[:M], ops.WeightMap(Wp))
    ref = xp[:M, :K].float() @ Wp[:, :K].float().T
    torch.testing.assert_close(y.float(), ref.half().float(), rtol=2e-3, atol=2e-3)
    torch.testing.assert_close(y.float(), ops.skinny_gemm(xp[:M, :K], Wp[:, :K]).float(), rtol=2e-3, atol=2e-3)  # the strided fallback
    # the SiLU epilogue writing into the padded activation buffer leaves the pad columns untouched
    inter = K
    Wgu = torch.randn((2 * inter, 256), generator=g, device=DEV, dtype=torch.float16) * 0.05
    x = torch.randn((M, 256), generator=g, device=DEV, dtype=torch.float16)
    act = torch.zeros((24, Kp), dtype=torch.float16, device=DEV)
    ops.stream_linear(x, ops.WeightMap(Wgu, silu=True), silu=True, out=act[:M, :inter])
    assert torch.equal(act[:M, :inter], ops.stream_linear(x, ops.WeightMap(Wgu, silu=True), silu=True))
    assert not act[:, inter:].any() and not act[M:].any()


def test_stream_linear_rejects_bad_shapes():
    with pytest.raises(_C.TriForceNativeError):
        ops.WeightMap(torch.zeros((64, 96), dtype=torch.float16, device=DEV))  # K % 64 != 0
    with pytest.raises(_C.TriForceNativeError):
        ops.stream_linear(torch.zeros((25, 128), dtype=torch.float16, device=DEV), torch.zeros((64, 128), dtype=torch.float16, device=DEV))


# ---------------------------------------------------------------------------------------------------------------------
# tree (Sequoia) attention + KV compaction — SURVEY §8 row a18
# ---------------------------------------------------------------------------------------------------------------------
def _random_tree_visibility(rng, R, T, row0):
    """Ancestor-closed visibility like grow_map["mask"]: node n sees itself and a random chain of earlier nodes."""
    vis = np.zeros((R, T), dtype=bool)
    for i in range(R):
        n = row0 + i
        vis[i, n] = True
        p = n
        while p > 0:
            p = int(rng.integers(0, p))
            vis[i, p] = True
    return vis


@pytest.mark.parametrize("R,H,d,S,T,row0", [(1, 4, 128, 600, 64, 0), (7, 4, 128, 600, 64, 5), (32, 2, 128, 8704, 512, 200),
                                              (22, 3, 64, 390, 128, 40), (32, 2, 128, 1100, 512, 480)])
def test_verify_attn_tree_matches_oracle(R, H, d, S, T, row0):
    rng = np.random.Generator(np.random.PCG64(S + R))
    q = rng.standard_normal((R, H, d), dtype=np.float32).astype(np.float16)
    K = rng.standard_normal((S, H, d), dtype=np.float32).astype(np.float16)
    V = rng.standard_normal((S, H, d), dtype=np.float32).astype(np.float16)
    vis = _random_tree_visibility(rng, R, T, row0)
    scale = orc.softmax_scale_fp16(d)
    want = orc.attention_tree(q, K, V, scale, vis)
    Ks, Vs = head_major(K, S + 30), head_major(V, S + 30)
    maps = ops.KVTensorMaps(Ks, Vs)
    ws = ops.verify_attn_workspace(R, H, d, DEV)
    out = torch.empty((R, H, d), dtype=torch.float16, device=DEV)
    mask = torch.from_numpy(orc.pack_tree_mask(vis).view(np.int32)).to(DEV)
    ops.verify_attn_tree(torch.from_numpy(q).to(DEV), maps, 0, S, R, H, d, scale, mask, T, out, ws)
    torch.cuda.synchronize()
    assert_attn_close(out.cpu().numpy(), want)


@pytest.mark.parametrize("R,H,S,T", [(128, 2, 1000, 0), (128, 3, 1024 + 128, 128), (256, 2, 3000, 256), (512, 2, 5000 + 512, 512), (128, 1, 128, 0)])
def test_tree_attn_tcgen05_matches_oracle(R, H, S, T):
    """The wgmma tree-verify kernel (variant 2) against the oracle's attention_tree, and its raw first score tile
    against an fp32 Q·K^T (which checks the wgmma shared-memory descriptors in isolation)."""
    d = 128
    rng = np.random.Generator(np.random.PCG64(S + R + T))
    q = rng.standard_normal((R, H, d), dtype=np.float32).astype(np.float16)
    K = rng.standard_normal((S, H, d), dtype=np.float32).astype(np.float16)
    V = rng.standard_normal((S, H, d), dtype=np.float32).astype(np.float16)
    vis = _random_tree_visibility(rng, R, T, 0) if T else np.ones((R, 0), dtype=bool)
    scale = orc.softmax_scale_fp16(d)
    want = orc.attention_tree(q, K, V, scale, vis) if T else orc.attention(q, K, V, scale, causal=False)
    Ks, Vs = head_major(K, S + 30), head_major(V, S + 30)
    maps = ops.KVTensorMaps(Ks, Vs)
    ws = ops.tree_attn_tc_workspace(R, H, S, DEV)
    out = torch.empty((R, H, d), dtype=torch.float16, device=DEV)
    mask = torch.from_numpy(orc.pack_tree_mask(vis).view(np.int32)).to(DEV) if T else None
    dbg = torch.zeros((128, 128), dtype=torch.float32, device=DEV)
    ops.tree_attn_tc(torch.from_numpy(q).to(DEV), maps, 0, S, R, H, d, scale, mask, T, out, ws, debug_scores=dbg)
    torch.cuda.synchronize()
    s_ref = q[:128, 0].astype(np.float32) @ K[:128, 0].astype(np.float32).T
    n = min(128, S)
    np.testing.assert_allclose(dbg.cpu().numpy()[:, :n], s_ref[:, :n], rtol=1e-3, atol=1e-2)
    assert_attn_close(out.cpu().numpy(), want)


@pytest.mark.parametrize("R,H,S", [(128, 2, 128), (128, 2, 1000), (1024, 2, 1024), (1024, 2, 3000), (1023, 1, 2500), (200, 3, 777), (40, 2, 333)])
def test_prefill_attention_tcgen05_causal_matches_oracle(R, H, S):
    """Causal mode of the wgmma kernel = the prefill attention of a prompt chunk (row i sees keys <= S - R + i), any R."""
    d = 128
    rng = np.random.Generator(np.random.PCG64(S * 7 + R))
    q = rng.standard_normal((R, H, d), dtype=np.float32).astype(np.float16)
    K = rng.standard_normal((S, H, d), dtype=np.float32).astype(np.float16)
    V = rng.standard_normal((S, H, d), dtype=np.float32).astype(np.float16)
    scale = orc.softmax_scale_fp16(d)
    want = orc.attention(q, K, V, scale, causal=True)
    Ks, Vs = head_major(K, S + 30), head_major(V, S + 30)
    maps = ops.KVTensorMaps(Ks, Vs)
    ws = ops.tree_attn_tc_workspace(R, H, S, DEV)
    out = torch.empty((R, H, d), dtype=torch.float16, device=DEV)
    ops.tree_attn_tc(torch.from_numpy(q).to(DEV), maps, 0, S, R, H, d, scale, None, 0, out, ws, causal=True)
    torch.cuda.synchronize()
    assert_attn_close(out.cpu().numpy(), want)


def test_kv_compact_clone_semantics():
    L, H, d, cap = 3, 4, 128, 300
    g = torch.Generator(device=DEV).manual_seed(9)
    K = torch.randn((L, H, cap, d), generator=g, device=DEV, dtype=torch.float16)
    V = torch.randn((L, H, cap, d), generator=g, device=DEV, dtype=torch.float16)
    offset = 200
    accept = [0, 3, 4, 17, 1, 60]  # tree nodes, relative to `offset`; overlaps the destination range on purpose
    idx = torch.tensor([offset + a for a in accept], dtype=torch.int32, device=DEV)
    wK, wV = K.clone(), V.clone()
    wK[:, :, offset:offset + len(accept)] = K[:, :, idx.long()].clone()
    wV[:, :, offset:offset + len(accept)] = V[:, :, idx.long()].clone()
    ops.kv_compact(K, V, idx, offset)
    assert torch.equal(K, wK) and torch.equal(V, wV)
