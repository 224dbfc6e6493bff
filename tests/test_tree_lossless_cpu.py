"""Sequoia tree wiring and the losslessness harness on the CPU.

  * wiring: for the committed 512-node map and hand-written trees, the children of the parents of level i, concatenated
    in `roots[i]` order, are exactly `roots[i+1]`, and the gather indices of `build_sampling` put race position j of parent
    p on p's j-th successor.  The walk visits children in `Successors[p]` order and the growth writes them in race order,
    so this is what makes the two orders the same.
  * statistics: a Monte Carlo of the product's growth (on CPU tensors), the oracle's accept walk and a residual draw emits
    a first token that passes chi-square against the root's target p, while the counts reject q, a p with 2 % moved, and
    the same trials walked with the root's children in reverse order.  This is the harness the GPU test runs on the
    kernels, checked where it costs nothing.
"""
import numpy as np
import pytest
import torch

from chi2_util import chi2, chi2_threshold
from oracle import triforce_oracle as orc
from triforce_b200.spectree import build_sampling, load_grow_map
from tree_lossless_util import (CHAIN_TREE, IRREGULAR_TREE, SMALL_TREE, grow_batch, grow_map_of, perturbed, softmax64,
                                synthetic_logits)

MAPS = {"512": None, "small": SMALL_TREE, "irregular": IRREGULAR_TREE, "chain": CHAIN_TREE}


def _map(name):
    return load_grow_map("512") if MAPS[name] is None else grow_map_of(MAPS[name])


@pytest.mark.parametrize("name", list(MAPS))
def test_successors_concatenate_to_the_next_level(name):
    gm = _map(name)
    succ, roots = gm["Successors"], gm["roots"]
    assert sum(len(r) for r in roots) == gm["size"]
    for i in range(len(roots) - 1):
        assert [c for p in roots[i] for c in succ[p]] == roots[i + 1], i
        assert gm["branches"][i] == [len(succ[p]) for p in roots[i]]
    assert all(not succ[p] for p in roots[-1])


def test_committed_map_children_are_consecutive_and_ascending():
    gm = load_grow_map("512")
    nxt = 1
    for p in range(gm["size"]):
        ch = gm["Successors"][p]
        assert ch == list(range(nxt, nxt + len(ch))), p
        nxt += len(ch)


@pytest.mark.parametrize("name", list(MAPS))
def test_gather_indices_put_race_position_j_on_successor_j(name):
    gm = _map(name)
    _, gather = build_sampling(gm, 0.6, "cpu")
    succ, roots = gm["Successors"], gm["roots"]
    for i in range(len(roots) - 1):
        k = max(gm["branches"][i])
        want = [pi * k + j for pi, p in enumerate(roots[i]) for j in range(len(succ[p]))]
        assert gather[i].tolist() == want, i


@pytest.mark.parametrize("name", list(MAPS))
def test_growth_writes_each_child_token_on_its_node(name):
    """`SpecTree.collective_grow_static`'s own steps (callable, gather, scatter to roots[i+1]) at T = 0, where the race is
    the top-k of each row: parent n's row ranks tokens 10 n + j first for j = 0, 1, ..., so child j of n must carry 10 n + j."""
    gm = _map(name)
    size = gm["size"]
    V = 10 * size + 10
    draft = torch.full((size, V), -1.0)
    for n in range(size):
        draft[n, 10 * n:10 * n + 10] = torch.arange(10, 0, -1, dtype=torch.float32)
    callables, gather = build_sampling(gm, 0.0, "cpu")
    toks = grow_batch(gm, callables, gather, draft, 1, len(gm["roots"]) - 1, lambda shape: torch.rand(shape))[0]
    for n, ch in enumerate(gm["Successors"]):
        for j, c in enumerate(ch):
            assert int(toks[c]) == 10 * n + j, (n, j, c)


# ---------------------------------------------------------------------------------------------------------------------
# the statistics, on the oracle
# ---------------------------------------------------------------------------------------------------------------------
def _first_tokens(gm, draft, P, T, trials, reverse_root, seed):
    succ = [list(c) for c in gm["Successors"]]
    if reverse_root:
        succ[0] = succ[0][::-1]
    callables, gather = build_sampling(gm, T, "cpu")
    g = torch.Generator().manual_seed(seed)
    toks = grow_batch(gm, callables, gather, torch.from_numpy(draft), trials, len(gm["roots"]) - 1,
                      lambda shape: 1 - torch.rand(shape, generator=g)).numpy()
    rng = np.random.Generator(np.random.PCG64(seed))
    uni = rng.random((trials, 16), dtype=np.float32)
    V = draft.shape[1]
    first = np.empty(trials, dtype=np.int64)
    for t in range(trials):
        acc, code, used, terminal, res = orc.tree_accept_walk(P, draft.copy(), toks[t], succ, uni[t], T)
        assert not terminal
        first[t] = toks[t, acc[0]] if acc else orc.sample_from_noise(res, rng.standard_exponential(V, dtype=np.float32))
    return first


@pytest.mark.parametrize("T,top_p", [(0.6, 0.9), (1.0, 1.0)])
def test_oracle_walk_first_token_follows_the_target(T, top_p):
    gm = grow_map_of(SMALL_TREE)
    V, N = 64, 40_000
    draft, target = synthetic_logits(gm["size"], V, seed=8)
    P = orc.norm_logits(target, T, -1, top_p)
    p, q = P[0].astype(np.float64), softmax64(draft[0], T)
    counts = np.bincount(_first_tokens(gm, draft, P, T, N, False, seed=1), minlength=V)
    mis = np.bincount(_first_tokens(gm, draft, P, T, N, True, seed=1), minlength=V)
    assert counts.sum() == N and counts[p == 0].sum() == 0
    stat, df = chi2(counts, p)
    controls = dict(q=chi2(counts, q), p_2pct=chi2(counts, perturbed(p)), reversed_root=chi2(mis, p))
    print(f"\n[tree lossless, oracle] T {T} top_p {top_p} V {V} N {N}: chi2 vs p {stat:.1f} (df {df}, 1e-6 threshold "
          f"{chi2_threshold(df):.1f}); " + "; ".join(f"vs {k} {s:.1f} (df {d}, threshold {chi2_threshold(d):.1f})"
                                                   for k, (s, d) in controls.items()))
    assert stat < chi2_threshold(df)
    for k, (s, d) in controls.items():
        assert s > chi2_threshold(d), k
