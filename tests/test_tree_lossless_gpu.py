"""Sampled Sequoia tree verification (T > 0) emits the target's distribution, on the kernels and through `SpecTree`.

Each trial grows a tree with the product's sampling callables and gather indices on fresh race noise, walks it with
`tf_tree_accept_walk` on fresh uniforms, and samples the residual with `tf_sample_argmax` on fresh exponentials.  The
draft and target rows are synthetic and depend on the node only (tests/tree_lossless_util.py), so:
  * the first emitted token must follow the root's target row p (chi-square at the 10^-6 level, and never a token with
    p = 0), on a 64-node depth-3 tree (branches 4/3/4) at V = 1000 and on the committed 512-node map at V = 32 000;
  * given the walk accepted node c, the next emitted token must follow c's target row, whether it is an accepted child
    of c or the residual sample at c;
  * the same counts must reject the root's q, p with 2 % moved between its top two tokens, and the same trials walked
    with the root's children in reverse order (a walk whose child order is not the race order).
Deterministic edges are compared with the oracle's walk.  The last test runs the same property through `SpecTree` on a
stub engine, with the production fp16 race noise.
"""
import time

import numpy as np
import pytest
import torch

from chi2_util import chi2, chi2_threshold
from oracle import triforce_oracle as orc
from triforce_b200 import ops
from triforce_b200.rng import TorchNoise
from triforce_b200.spectree import SpecTree, build_sampling, load_grow_map
from tree_lossless_util import SMALL_TREE, StubEngine, csr, grow_batch, grow_map_of, perturbed, softmax64, synthetic_logits

pytestmark = pytest.mark.gpu
DEV = "cuda"
SETTINGS = [(0.6, 0.9), (1.0, 1.0)]


def _t(a) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _spectree(gm, V, T, top_p, seed):
    draft, target = synthetic_logits(gm["size"], V, seed)
    st = SpecTree(StubEngine(_t(draft), _t(target)), temperature=T, top_p=top_p, grow_map=gm, vocab_size=V,
                  noise=TorchNoise(DEV))
    return st, draft, target


def _walk_trials(st, draft, P, trials, fresh_levels, seed, per_graph=500):
    """`trials` independent rounds of growth + walk + residual sample, with SpecTree's own successor CSR ("product") and
    with the root's children reversed ("reversed_root") on the same trees and noise.  Levels below `fresh_levels` are grown
    once per graph of `per_graph` trials (shared by its trials); the first token depends on the root's children only.  After
    each walk, the draft entries it may have set to -FLT_MAX (the parent row at each child's token) are restored.
    Returns, per walk, numpy arrays: n_acc, code, terminal, nan, nodes [N, 3] (accepted node ids), em [N, 3] (tokens)."""
    gm = st.grow_map
    size, V, T = gm["size"], P.shape[1], st.temperature
    levels = len(gm["roots"]) - 1
    off_r, flat_r = csr(gm["Successors"], reverse_root=True)
    walks = {"product": (st.succ_off, st.succ),
             "reversed_root": (torch.tensor(off_r, dtype=torch.int32, device=DEV), torch.tensor(flat_r, dtype=torch.int32, device=DEV))}
    parent = [0] * size
    for p, ch in enumerate(gm["Successors"]):
        for c in ch:
            parent[c] = p
    par = torch.tensor(parent[1:], dtype=torch.long, device=DEV)
    depth = st.depth
    draft_dev = _t(draft)
    dl = draft_dev.clone()
    B = per_graph
    toks = torch.ones((B, size), dtype=torch.long, device=DEV)
    vals = torch.empty((B, size - 1), dtype=torch.float32, device=DEV)
    uni = torch.empty((B, st._uniforms.numel()), dtype=torch.float32, device=DEV)
    expo = torch.empty((B, V), dtype=torch.float32, device=DEV)
    outs = {k: torch.full((B, 32), -1, dtype=torch.int32, device=DEV) for k in walks}
    smp = {k: torch.zeros(B, dtype=torch.long, device=DEV) for k in walks}
    resid = torch.zeros(V, dtype=torch.float32, device=DEV)
    scratch = torch.zeros(V, dtype=torch.float32, device=DEV)

    def body(name):
        off, flat = walks[name]
        for t in range(B):
            ops.tree_accept_walk(P, dl, toks[t], off, flat, uni[t], T, outs[name][t], resid, scratch)
            ops.sample_argmax(resid, expo[t], out=smp[name][t:t + 1])
            dl.index_put_((par, toks[t, 1:]), vals[t])  # undo this walk's -FLT_MAX writes before the next trial

    toks.copy_(grow_batch(gm, st.sampling_callables, st.sample_gather_indices, draft_dev, B, levels, lambda shape: torch.rand(shape, device=DEV)))
    vals.copy_(draft_dev[par[None, :].expand(B, -1), toks[:, 1:]])
    uni.zero_()
    expo.fill_(1.0)
    graphs = {}
    for name in walks:
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            body(name)
        torch.cuda.current_stream().wait_stream(side)
        graphs[name] = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graphs[name]):
            body(name)

    dl.copy_(draft_dev)
    g = torch.Generator(device=DEV).manual_seed(seed)
    race = lambda shape: 1 - torch.rand(shape, device=DEV, generator=g)  # (0, 1]: no log(0)
    rec = {k: [] for k in walks}
    j = torch.arange(3, device=DEV)
    for _ in range(trials // B):
        grown = grow_batch(gm, st.sampling_callables, st.sample_gather_indices, draft_dev, B, fresh_levels, race)
        if fresh_levels < levels:
            shared = grow_batch(gm, st.sampling_callables, st.sample_gather_indices, draft_dev, 1, levels, race)
            grown = torch.where(depth[None, :] > fresh_levels, shared, grown)
        toks.copy_(grown)
        vals.copy_(draft_dev[par[None, :].expand(B, -1), toks[:, 1:]])
        uni.copy_(torch.rand(uni.shape, device=DEV, generator=g))
        expo.exponential_(1.0, generator=g)
        for name in walks:
            outs[name].fill_(-1)
            graphs[name].replay()
            o = outs[name].long()
            n = o[:, 0:1]
            nodes = o[:, 8:11]
            tk = toks.gather(1, nodes.clamp(min=0))
            em = torch.where(j < n, tk, torch.where(j == n, smp[name][:, None], -1))
            rec[name].append(torch.cat([o[:, :5], nodes, em], 1))
    res = {}
    for name, parts in rec.items():
        a = torch.cat(parts).cpu().numpy()
        res[name] = dict(n_acc=a[:, 0], code=a[:, 1], terminal=a[:, 3], nan=a[:, 4], nodes=a[:, 5:8], em=a[:, 8:11])
    return res


def _check_walk_outputs(r, N):
    assert len(r["n_acc"]) == N
    assert (r["terminal"] == 0).all() and (r["nan"] == 0).all()
    assert np.isin(r["code"], [-1, -2]).all()


def _assert_follows(tag, tokens, p, V, controls=()):
    """chi-square of `tokens` against p (below the 10^-6 threshold), no token with p = 0, and every control rejected."""
    counts = np.bincount(tokens, minlength=V)
    assert counts[p == 0].sum() == 0, (tag, np.flatnonzero((p == 0) & (counts > 0))[:10])
    if (p > 0).sum() == 1:  # one token carries all of p: the zero-count check above is the whole test
        print(f"\n[tree lossless] {tag}, N {counts.sum()}: p is one-hot, every count on its token")
        return
    stat, df = chi2(counts, p)
    msg = [f"vs p {stat:.1f} (df {df}, 1e-6 threshold {chi2_threshold(df):.1f})"]
    rejected = {}
    for name, c, ref in controls:
        s, d = chi2(c, ref)
        rejected[name] = s > chi2_threshold(d)
        msg.append(f"vs {name} {s:.1f} (df {d}, threshold {chi2_threshold(d):.1f})")
    print(f"\n[tree lossless] {tag}, N {counts.sum()}: " + "; ".join(msg))
    assert stat < chi2_threshold(df), tag
    for name, ok in rejected.items():
        assert ok, f"{tag}: control {name} not rejected"


def _first_token_with_controls(tag, res, P, draft, T, V, moved_control=True):
    p = P[0].astype(np.float64)
    q = softmax64(draft[0], T)
    first = res["product"]["em"][:, 0]
    counts = np.bincount(first, minlength=V)
    r = res["reversed_root"]
    # the mis-wired walk can end on a residual of zero mass (NaN), where the product ends the generation: not counted
    mis = np.bincount(r["em"][r["nan"] == 0, 0], minlength=V)
    print(f"\n[tree lossless] {tag}: reversed-root walk, {int((r['nan'] != 0).sum())} of {len(r['nan'])} trials end on a NaN residual")
    controls = [("q_root", counts, q), ("reversed_root_walk", mis, p)]
    if moved_control:
        controls.append(("p_2pct_moved", counts, perturbed(p)))
    _assert_follows(tag + " first token", first, p, V, controls)


@pytest.mark.parametrize("T,top_p", SETTINGS)
def test_small_tree_walk_is_lossless(T, top_p):
    t0 = time.perf_counter()
    gm = grow_map_of(SMALL_TREE)
    V, N = 1000, 200_000
    st, draft, target = _spectree(gm, V, T, top_p, seed=27)
    P_dev = ops.norm_logits(_t(target), T, top_p)
    P = P_dev.cpu().numpy()
    np.testing.assert_array_equal(P > 0, orc.norm_logits(target, T, -1, top_p) > 0)
    res = _walk_trials(st, draft, P_dev, N, fresh_levels=3, seed=1000 + int(T * 10))
    _check_walk_outputs(res["product"], N)
    tag = f"4/3/4 tree V {V} T {T} top_p {top_p}"
    _first_token_with_controls(tag, res, P, draft, T, V)
    r = res["product"]
    n, nodes, em = r["n_acc"], r["nodes"], r["em"]
    root_children = gm["Successors"][0]
    hits = [(int(((n >= 1) & (nodes[:, 0] == c)).sum()), c) for c in root_children]
    for cnt, c in sorted(hits, reverse=True)[:2]:
        sel = (n >= 1) & (nodes[:, 0] == c)
        _assert_follows(f"{tag} next token after root child {c} ({cnt} trials)", em[sel, 1], P[c].astype(np.float64), V)
    sel2 = n >= 2
    c2 = int(np.bincount(nodes[sel2, 1]).argmax())
    sel = sel2 & (nodes[:, 1] == c2)
    assert int(gm["depth"][c2]) == 2 and sel.sum() >= 5000
    _assert_follows(f"{tag} next token after depth-2 node {c2} ({sel.sum()} trials)", em[sel, 2], P[c2].astype(np.float64), V)
    print(f"[tree lossless] {tag}: {time.perf_counter() - t0:.1f} s")


@pytest.mark.parametrize("T,top_p", SETTINGS)
def test_512_map_first_token_is_lossless(T, top_p):
    t0 = time.perf_counter()
    gm = load_grow_map("512")
    V = 32000
    N = 50_000 if top_p < 1 else 200_000  # p is flat at T = 1: 10^4 pooled bins, a wider threshold
    st, draft, target = _spectree(gm, V, T, top_p, seed=22)
    P_dev = ops.norm_logits(_t(target), T, top_p)
    P = P_dev.cpu().numpy()
    res = _walk_trials(st, draft, P_dev, N, fresh_levels=1, seed=2000 + int(T * 10))
    _check_walk_outputs(res["product"], N)
    tag = f"512-node map V {V} T {T} top_p {top_p}"
    # with p spread over 32 000 tokens (T = 1, no nucleus) 2 % moved between two tokens stays under the threshold of
    # ~10^4 degrees of freedom at 2*10^5 trials; the 4/3/4 tree rejects that control at T = 1
    _first_token_with_controls(tag, res, P, draft, T, V, moved_control=top_p < 1)
    print(f"[tree lossless] {tag}: {time.perf_counter() - t0:.1f} s")


# ---------------------------------------------------------------------------------------------------------------------
# deterministic edges, against the oracle's walk
# ---------------------------------------------------------------------------------------------------------------------
def _walk_once(P, draft, toks, gm, uni, T):
    off, flat = csr(gm["Successors"])
    V = P.shape[1]
    out = torch.zeros(32, dtype=torch.int32, device=DEV)
    resid = torch.zeros(V, device=DEV)
    scratch = torch.zeros(V, device=DEV)
    d_dev = _t(draft.copy())
    ops.tree_accept_walk(_t(P), d_dev, _t(toks), torch.tensor(off, dtype=torch.int32, device=DEV),
                         torch.tensor(flat, dtype=torch.int32, device=DEV), _t(uni), T, out, resid, scratch)
    w = out.tolist()
    return w, resid.cpu().numpy(), d_dev.cpu().numpy()


def _grow_once(gm, draft, T, seed):
    callables, gather = build_sampling(gm, T, DEV)
    g = torch.Generator(device=DEV).manual_seed(seed)
    return grow_batch(gm, callables, gather, _t(draft), 1, len(gm["roots"]) - 1,
                      lambda shape: 1 - torch.rand(shape, device=DEV, generator=g))[0].cpu().numpy()


def test_p_equal_q_accepts_down_to_a_leaf():
    """top_p = 1 and target logits = draft logits: p = q at every node, so with uniforms <= 0.999 every walk accepts the
    first child at each level and ends at a leaf (code -2), like the oracle."""
    gm = grow_map_of(SMALL_TREE)
    V, T = 1000, 0.6
    draft, _ = synthetic_logits(gm["size"], V, seed=23)
    P = ops.norm_logits(_t(draft), T, 1.0).cpu().numpy()
    rng = np.random.Generator(np.random.PCG64(23))
    for trial in range(16):
        toks = _grow_once(gm, draft, T, seed=trial)
        uni = (rng.random(16, dtype=np.float32) * np.float32(0.999)).astype(np.float32)
        if trial == 0:
            uni[:] = np.float32(0.999)
        acc, code, used, terminal, res = orc.tree_accept_walk(P, draft.copy(), toks, gm["Successors"], uni, T)
        w, resid, _ = _walk_once(P, draft, toks, gm, uni, T)
        want = [gm["Successors"][0][0]]
        while gm["Successors"][want[-1]]:
            want.append(gm["Successors"][want[-1]][0])
        assert acc == want and code == -2 and used == 3 and not terminal
        assert w[0] == 3 and w[8:11] == want and w[1] == -2 and w[2] == 3 and w[3] == 0 and w[4] == 0, (trial, w[:12])
        np.testing.assert_array_equal(resid, P[want[-1]])


@pytest.mark.parametrize("T", [0.6, 1.0])
def test_draft_row_with_fewer_nonzero_entries_than_branches(T):
    """The root's draft row has 2 tokens of nonzero fp32 probability at T and 4 branches.  What happens: the race gives the
    2 supported tokens first; the other 2 children come from top-k among exact ties (log(u) / 0 = -inf for every token
    outside the support), so which tokens they are is top-k's choice.  The walk rejects the supported children here (the
    target gives them p = 0) and sets their draft logits to -FLT_MAX; at T = 0.6, -FLT_MAX / T overflows to -inf.  The
    next q is the softmax of the remaining floor logits, so the third child is tested against a q it was not drawn from
    (the floor is uniform).  Losslessness is claimed only for rows with at least `branches` nonzero entries; here the
    kernel must equal the oracle's walk: accepted nodes, uniforms used, code, `terminal` and the residual's NaN flag."""
    gm = grow_map_of(SMALL_TREE)
    V = 1000
    draft, target = synthetic_logits(gm["size"], V, seed=24)
    support = [5, 9]
    draft[0, :] = -1e4
    draft[0, support] = [0.0, 0.5]
    target[0, support] = -1e4
    assert (softmax64(draft[0], T).astype(np.float32) > 0).sum() == 2
    P = ops.norm_logits(_t(target), T, 0.9).cpu().numpy()
    rng = np.random.Generator(np.random.PCG64(24))
    seen = set()
    for trial in range(24):
        toks = _grow_once(gm, draft, T, seed=100 + trial)
        root_toks = [int(toks[c]) for c in gm["Successors"][0]]
        assert sorted(root_toks[:2]) == support, root_toks
        uni = rng.random(16, dtype=np.float32)
        d_ref = draft.copy()
        acc, code, used, terminal, res = orc.tree_accept_walk(P, d_ref, toks, gm["Successors"], uni, T)
        w, resid, d_dev = _walk_once(P, draft, toks, gm, uni, T)
        assert w[0] == len(acc) and w[8:8 + w[0]] == acc, (trial, w[:12], acc)
        assert w[2] == used and w[3] == int(terminal) and w[1] == code
        assert w[4] == int(np.isnan(res).any())
        np.testing.assert_array_equal(d_dev == np.finfo(np.float32).min, d_ref == np.finfo(np.float32).min)
        seen.add((tuple(root_toks[2:]), len(acc) > 0 and acc[0] in gm["Successors"][0][2:], w[4]))
    print(f"\n[tree edge] T {T}: root children past the support {sorted({s[0] for s in seen})}; "
          f"accepted one of them: {any(s[1] for s in seen)}; NaN residual: {any(s[2] for s in seen)}")


# ---------------------------------------------------------------------------------------------------------------------
# through SpecTree
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("race_dtype", [torch.float16, torch.float32])
def test_spectree_first_token_is_lossless(race_dtype):
    """`construct_grow_map` + `verify` on a stub engine, the production path: race noise redrawn before every trial
    (`tree_uniform_into`, as `prefill` does), `self.rand[idx_list]`, the draft-logit row assignment and the uniform rewind.
    float16 is the production race noise; float32 (the buffer swapped in by the test) separates its rounding from the
    wiring."""
    t0 = time.perf_counter()
    gm = grow_map_of(SMALL_TREE)
    V, T, top_p, N = 1000, 0.6, 0.9, 20_000
    torch.manual_seed(31)
    st, draft, target = _spectree(gm, V, T, top_p, seed=25)
    st.rand = torch.empty((gm["size"], V), dtype=race_dtype, device=DEV)
    P = ops.norm_logits(_t(target), T, top_p).cpu().numpy()
    nt = torch.ones((1, 1), dtype=torch.long, device=DEV)
    first = []
    for _ in range(N):
        st.noise.tree_uniform_into(st.rand)
        st.construct_grow_map(next_token=nt)
        nxt, acc, toks = st.verify()
        assert nxt is not None
        first.append(toks[1])
    first = torch.stack(first).cpu().numpy()
    p = P[0].astype(np.float64)
    counts = np.bincount(first, minlength=V)
    if race_dtype == torch.float16:
        # float16 race noise is rejected at this N (DESIGN.md section 7); only the support and the q control are asserted
        assert counts[p == 0].sum() == 0
        stat, df = chi2(counts, p)
        sq, dq = chi2(counts, softmax64(draft[0], T))
        print(f"\n[tree lossless] SpecTree, float16 race noise, first token, N {N}: vs p {stat:.1f} (df {df}, 1e-6 threshold "
              f"{chi2_threshold(df):.1f}, not asserted); vs q_root {sq:.1f} (df {dq}, threshold {chi2_threshold(dq):.1f})")
        assert sq > chi2_threshold(dq)
        return
    _assert_follows(f"SpecTree, {race_dtype} race noise, 4/3/4 tree V {V} T {T} top_p {top_p} first token", first, p, V,
                    [("q_root", counts, softmax64(draft[0], T))])
    print(f"[tree lossless] SpecTree {race_dtype}: {time.perf_counter() - t0:.1f} s")
