"""Shared pieces of the Sequoia losslessness tests (tests/test_tree_lossless_cpu.py, tests/test_tree_lossless_gpu.py).

Sampled tree verification is lossless when the three parts that live in different places agree:
  * growth (`spectree.create_sampling_callable` + `build_sampling`) draws each parent's children WITHOUT replacement from
    softmax(draft_logits[parent] / T) with the exponential race, and the gather indices put race position j of parent p at
    `verify_tokens[roots[i+1][...]]`;
  * the walk (`tf_tree_accept_walk`, `orc.tree_accept_walk`) visits the children of p in `Successors[p]` order, recomputes q
    at the same T and removes every rejected token from it;
  * the residual at the node where the walk stops is sampled with `tf_sample_argmax`.
Sampling without replacement is not exchangeable, so a walk whose child order is not the race order is biased.

The synthetic rows here depend on the NODE, not on its token: node n's draft row is q_n and its target row p_n whatever
token it carries.  Then, given the walk reached node c, the next emitted token must follow p_c.
"""
from __future__ import annotations

import json
import os
import tempfile
from typing import Dict, List

import numpy as np
import torch

from triforce_b200.spectree import load_grow_map


def _level_tree(branches: List[int]) -> List[List[int]]:
    """Successors of a regular tree: every node at depth i has branches[i] children, numbered level by level."""
    succ: List[List[int]] = [[]]
    level, nxt = [0], 1
    for b in branches:
        new = []
        for n in level:
            succ[n] = list(range(nxt, nxt + b))
            new.extend(succ[n])
            nxt += b
            succ.extend([] for _ in range(b))
        level = new
    return succ


# depth 3: 4 children at the root, 3 under each of those, 4 under each of those but the last, which has 3: 64 nodes
# (`SpecTree` packs the ancestor mask in 32-bit words, so the tree size is a multiple of 32)
SMALL_TREE = _level_tree([4, 3, 4])[:-1]
SMALL_TREE[16].pop()

# parents of one level with different branch counts, and leaves above the last level
IRREGULAR_TREE = [[1, 2, 3], [4, 5, 6], [], [7], [8], [], [9, 10], [11, 12, 13], [], [], [], [], [], []]
CHAIN_TREE = [[1], [2], [3], []]


def grow_map_of(successors: List[List[int]]) -> Dict:
    """The grow_map `load_grow_map` builds from a Successors file, for a hand-written tree."""
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "tree.json")
        with open(path, "w") as f:
            json.dump(dict(size=len(successors), Successors=successors), f)
        return load_grow_map(path)


def csr(successors: List[List[int]], reverse_root: bool = False):
    """(offsets, flat) of the successor lists, the layout `SpecTree` hands to the walk; `reverse_root` visits the root's
    children in the opposite order (a mis-wired walk)."""
    off, flat = [0], []
    for n, ch in enumerate(successors):
        flat.extend(ch[::-1] if (reverse_root and n == 0) else ch)
        off.append(len(flat))
    return off, flat


def synthetic_logits(size: int, V: int, seed: int):
    """Per-node draft and target logits [size, V] fp32.  Each draft row has 4 dominant tokens on a N(0, 1) floor (so the
    draft proposes a few tokens most of the time and the order of the walk matters); the target row is the draft row plus
    N(0, 1) noise, so p and q differ everywhere.  Tokens 0 and 2 (which end a generation) get logit -1e4: probability 0 in
    both, so no walk is terminal.  The boost grows with log V to keep q's dominant mass similar across vocabularies."""
    rng = np.random.Generator(np.random.PCG64(seed))
    boost = 4.0 + np.log(V / 1000.0)
    draft = rng.standard_normal((size, V), dtype=np.float32)
    for n in range(size):
        top = rng.permutation(np.arange(3, V))[:4]
        draft[n, top] += np.float32(boost) + np.float32(0.5) * np.arange(4, dtype=np.float32)
    target = (draft + rng.standard_normal((size, V), dtype=np.float32)).astype(np.float32)
    draft[:, [0, 2]] = -1e4
    target[:, [0, 2]] = -1e4
    return draft.astype(np.float32), target


def softmax64(x: np.ndarray, T: float) -> np.ndarray:
    z = x.astype(np.float64) / T
    e = np.exp(z - z.max(-1, keepdims=True))
    return e / e.sum(-1, keepdims=True)


def perturbed(p: np.ndarray, mass: float = 0.02) -> np.ndarray:
    """p with `mass` moved from its most likely token to the second one."""
    a, b = np.argsort(-p, kind="stable")[:2]
    p2 = p.astype(np.float64).copy()
    p2[a] -= mass
    p2[b] += mass
    return p2


def grow_batch(grow_map, callables, gather, draft_rows: torch.Tensor, trials: int, levels: int, rand_fn) -> torch.Tensor:
    """verify_tokens [trials, size] of `trials` independent growths of the first `levels` levels, with the product's
    sampling callables and gather indices and fresh race noise `rand_fn(shape)` per trial.  Batched over trials: the
    synthetic draft rows depend on the node only.  Deeper levels stay 1 (never read by a walk that ends above them)."""
    size = grow_map["size"]
    dev = draft_rows.device
    toks = torch.ones((trials, size), dtype=torch.long, device=dev)
    for i in range(levels):
        idx = torch.tensor(grow_map["roots"][i], dtype=torch.long, device=dev)
        nxt = torch.tensor(grow_map["roots"][i + 1], dtype=torch.long, device=dev)
        rows = draft_rows[idx]
        n, V = rows.shape
        logits = rows.unsqueeze(0).expand(trials, n, V).reshape(trials * n, V)
        new = callables[i](logits, rand_fn((trials * n, V))).view(trials, -1)
        toks[:, nxt] = new[:, gather[i]]
    return toks


class StubEngine:
    """The members `SpecTree` reads from its engine, serving fixed per-node logits: the draft logits of the nodes being
    grown (nodes `storage_start + arange(n)`, numbered level by level) and the target logits of the whole tree."""

    class _KV:
        seq_len = 100

        def gather_kv_incremental(self, accept_list, offset):
            pass

    class _Retrieval:
        max_budget = 256

        def __init__(self, tree_size):
            self.real_budget = self.max_budget + tree_size

        def update_graph_cache(self, kv_cache):
            pass

    def __init__(self, draft: torch.Tensor, target: torch.Tensor):
        self.device = draft.device
        self.draft, self.target = draft, target
        self.kv_cache = self._KV()
        self.retrieval_cache = self._Retrieval(draft.shape[0])

    def retrieval_tree_inference(self, input_ids, position_ids, mask_bits, storage_start):
        n = input_ids.shape[-1]
        return self.draft[storage_start:storage_start + n].unsqueeze(0)

    def tree_verify_inference(self, input_ids, position_ids, mask_bits):
        return self.target.unsqueeze(0)
