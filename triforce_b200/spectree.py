"""Sequoia tree self-speculation on top of the retrieval cache — the reference's `utils/SpecTree_TP.py` (SpecTree :31-236)
with `test/offloading_seqouia.py:24-39,119-133` (residual, sampling without replacement, gather indices), BASELINE cfg 5.

The target model with its RETRIEVAL cache grows a static 512-node token tree in 16 masked forward passes
(`retrieval_tree_inference`, tree mask over the cache's tree slots), then ONE masked forward of all 512 nodes over the FULL
KV verifies it; the accepted root-to-leaf path is walked with recursive rejection sampling and the accepted nodes' KV rows
are compacted into the cache (`gather_kv_incremental`).

GPU mapping: both masked attentions run on `tf_verify_attn_tree` (prefix fully visible + a 512-bit ancestor mask per
row, 32 query rows per launch); the accept walk (SpecTree.accept_step :147-165 + verify :181-197) is ONE kernel
(`tf_tree_accept_walk`) instead of ~5 host round-trips per examined child; top-p + softmax of the 512 target rows is
`tf_norm_logits`; the KV compaction is `tf_kv_compact`.  The reference's 5 broadcast+barrier pairs per verify (:205-223)
disappear: every rank computes the same walk from identical probabilities and identically seeded noise.

The tree topology (`tree/512.pt` of the reference: 16 levels, widths 1,7,14,…) ships as a data fixture
(`triforce_b200/data/tree_512.json`, the `Successors` lists); roots / branches / mask / depth are rebuilt from it.
"""
from __future__ import annotations

import json
import os
from typing import Dict, List, Optional

import numpy as np
import torch

from . import ops
from .rng import TorchNoise
from .sampling import norm_logits

_DATA = os.path.join(os.path.dirname(os.path.abspath(__file__)), "data")


def load_grow_map(name_or_path: str = "512") -> Dict:
    """Rebuild the reference's grow_map dict (keys roots, branches, Successors, mask, depth, size) from the Successors lists."""
    path = name_or_path if os.path.exists(name_or_path) else os.path.join(_DATA, f"tree_{name_or_path}.json")
    raw = json.load(open(path))
    succ: List[List[int]] = raw["Successors"]
    size = raw["size"]
    parent = [-1] * size
    for p, ch in enumerate(succ):
        for c in ch:
            parent[c] = p
    depth = [0] * size
    for n in range(1, size):  # nodes are numbered level by level, parents before children
        depth[n] = depth[parent[n]] + 1
    levels = max(depth) + 1
    roots = [[n for n in range(size) if depth[n] == lv] for lv in range(levels)]
    branches = [[len(succ[n]) for n in roots[lv]] for lv in range(levels)]
    mask = torch.zeros((size, size), dtype=torch.int64)
    for n in range(size):
        a = n
        while a >= 0:
            mask[n, a] = 1
            a = parent[a]
    return dict(roots=roots, branches=branches, Successors=succ, mask=mask, depth=torch.tensor(depth, dtype=torch.int64), size=size)


def pack_mask_bits(mask: torch.Tensor) -> torch.Tensor:
    """[n, T] 0/1 → int32 [n, T/32] (bit c of word c//32 = column c), the layout `tf_verify_attn_tree` takes."""
    n, T = mask.shape
    assert T % 32 == 0
    m = mask.to(torch.int64).reshape(n, T // 32, 32)
    words = (m << torch.arange(32, dtype=torch.int64)[None, None, :]).sum(-1)
    words = torch.where(words >= 2 ** 31, words - 2 ** 32, words)  # reinterpret as int32
    return words.to(torch.int32).contiguous()


def get_residual(p: torch.Tensor, q: torch.Tensor) -> torch.Tensor:
    """test/offloading_seqouia.py:24-27"""
    residual = (p - q).relu_()
    return residual / (residual.sum(dim=-1).unsqueeze(-1))


def create_sampling_callable(num_samples: int, temperature: float = 0.6):
    """Sampling WITHOUT replacement of `num_samples` children per parent row: the Gumbel/exponential-race trick of
    test/offloading_seqouia.py:29-39 — `(rand.log() / softmax(logits / T)).topk(k)` (rank-0 + broadcast in the reference;
    here every rank evaluates it on identical inputs).

    temperature 0 (greedy): the T -> 0 limit of the race, the `num_samples` largest logits of each row, ties to the lower
    index (a stable descending sort; NaN sorts first, as torch.argmax counts it maximal).  The noise is not read."""
    if temperature == 0:
        def greedy_children(sampling_logits: torch.Tensor, static_rand: torch.Tensor) -> torch.Tensor:
            return torch.sort(sampling_logits, dim=-1, descending=True, stable=True).indices[:, :num_samples].flatten()
        return greedy_children

    def sampling_without_replacement(sampling_logits: torch.Tensor, static_rand: torch.Tensor) -> torch.Tensor:
        sampling_q = torch.softmax(sampling_logits / temperature, dim=-1)
        return (static_rand.log() / sampling_q).topk(k=num_samples).indices.flatten()
    return sampling_without_replacement


def build_sampling(grow_map: Dict, temperature: float, device):
    """test/offloading_seqouia.py:119-133"""
    branch_lists = grow_map["branches"]
    draft_step = len(grow_map["roots"])
    callables, gather = {}, {}
    for i in range(draft_step - 1):
        k = max(branch_lists[i])
        callables[i] = create_sampling_callable(k, temperature)
        idx = [torch.arange(b, device=device, dtype=torch.long) + j * k for j, b in enumerate(branch_lists[i])]
        gather[i] = torch.cat(idx)
    return callables, gather


class SpecTree:
    def __init__(self, engine, temperature: float = 0.6, top_p: float = 0.9, max_length=256, vocab_size=32000, grow_map=None,
                 residual_graph=None, sampling_callables=None, sample_gather_indices=None, tokenizer=None, noise=None,
                 race_dtype=torch.float16) -> None:
        """`race_dtype`: the uniform race noise `self.rand` of the growth, fp16 like the reference's buffer (SpecTree_TP.py:86)
        or fp32 (what session.TreeSession uses: fp16 uniforms bias the race, DESIGN.md section 7)."""
        self.graph_engine = engine
        self.temperature, self.top_p = temperature, top_p
        self.residual_graph = residual_graph or get_residual
        self.tokenizer = tokenizer
        self.device = engine.device
        self.dtype = race_dtype
        self.grow_map = grow_map or load_grow_map("512")
        if sampling_callables is None:
            sampling_callables, sample_gather_indices = build_sampling(self.grow_map, temperature, self.device)
        self.sampling_callables, self.sample_gather_indices = sampling_callables, sample_gather_indices
        self.draft_step = len(self.grow_map["roots"])
        self.grow_map_roots_gpu = [torch.tensor(x, dtype=torch.long, device=self.device) for x in self.grow_map["roots"]]
        self.Successors = self.grow_map["Successors"]
        self.tree_size = self.grow_map["size"]
        self.vocab_size = vocab_size
        self.noise = noise or TorchNoise(self.device)
        rc = engine.retrieval_cache
        assert rc.real_budget - rc.max_budget == self.tree_size, "retrieval cache must reserve tree_size slots"
        # 512-bit ancestor masks (the reference builds additive fp16 masks [rows, budget+tree] / [tree, seq_len+tree])
        self.mask_bits = pack_mask_bits(self.grow_map["mask"]).to(self.device)  # [tree, tree/32]
        self.depth = self.grow_map["depth"].to(self.device)
        self.level_start = []
        start = 1
        for i in range(self.draft_step - 1):
            self.level_start.append(start)
            start += sum(self.grow_map["branches"][i])
        # CSR of the successor lists for the fused accept walk
        off = [0]
        flat: List[int] = []
        for ch in self.Successors:
            flat.extend(ch)
            off.append(len(flat))
        self.succ_off = torch.tensor(off, dtype=torch.int32, device=self.device)
        self.succ = torch.tensor(flat if flat else [0], dtype=torch.int32, device=self.device)
        self.max_children_on_path = sum(max((len(self.Successors[n]) for n in lv), default=0) for lv in self.grow_map["roots"])

        self.draft_logits = torch.zeros((self.tree_size, vocab_size), dtype=torch.float32, device=self.device)
        self.rand = torch.empty((self.tree_size, vocab_size), dtype=self.dtype, device=self.device)
        self.noise.tree_uniform_into(self.rand)  # SpecTree_TP.py:86 draws it at construction and again in every prefill (:93)
        self.verify_tokens = torch.zeros(self.tree_size, dtype=torch.long, device=self.device)
        self._uniforms = torch.empty(self.max_children_on_path + 1, dtype=torch.float32, device=self.device)
        self._walk_out = torch.zeros(32, dtype=torch.int32, device=self.device)
        self._residual = torch.zeros(vocab_size, dtype=torch.float32, device=self.device)
        self._scratch = torch.zeros(vocab_size, dtype=torch.float32, device=self.device)
        self._expo = torch.empty(vocab_size, dtype=torch.float32, device=self.device)

    @torch.inference_mode()
    def prefill(self, prefix: torch.LongTensor):
        self.draft_logits.zero_()
        self.verify_tokens.zero_()
        self.noise.tree_uniform_into(self.rand)
        eng = self.graph_engine
        eng.reset()
        eng.prefill(input_ids=prefix.unsqueeze(0)[:, :-1])
        logits = eng.build_retrieval_cache(input_ids=prefix.unsqueeze(0)[:, -1:])
        probs = norm_logits(logits[:, -1, :], temperature=self.temperature, top_k=-1, top_p=self.top_p)
        self.noise.exponential_into(self._expo)
        return ops.sample_argmax(probs, self._expo).reshape(1, 1)

    @torch.inference_mode()
    def construct_grow_map(self, next_token):
        eng = self.graph_engine
        self.verify_tokens[0] = next_token.reshape(-1)[0]
        seq_len = eng.kv_cache.seq_len
        position_ids = torch.arange(seq_len, seq_len + 1, device=self.device)
        draft_logits = eng.retrieval_tree_inference(input_ids=next_token.reshape(1, 1), position_ids=position_ids.unsqueeze(0),
                                                    mask_bits=self.mask_bits[0:1], storage_start=0)[0]
        self.draft_logits[0] = draft_logits
        for i in range(self.draft_step - 1):
            draft_logits = self.collective_grow_static(self.grow_map_roots_gpu[i], self.grow_map_roots_gpu[i + 1],
                                                       self.grow_map["branches"][i], grow_step=i)
            self.draft_logits[self.grow_map_roots_gpu[i + 1]] = draft_logits

    @torch.inference_mode()
    def collective_grow_static(self, idx_list, next_idx_list, n_branch_list, grow_step=None, draft_logits=None):
        total_branch = sum(n_branch_list)
        new_tokens_set = self.sampling_callables[grow_step](self.draft_logits[idx_list], self.rand[idx_list])
        new_tokens_set = new_tokens_set[self.sample_gather_indices[grow_step]]
        self.verify_tokens[next_idx_list] = new_tokens_set
        new_tokens_set = new_tokens_set.view(1, total_branch)
        eng = self.graph_engine
        position_ids = (self.depth[next_idx_list] + eng.kv_cache.seq_len).unsqueeze(0)
        start = self.level_start[grow_step]
        return eng.retrieval_tree_inference(input_ids=new_tokens_set, position_ids=position_ids,
                                            mask_bits=self.mask_bits[start:start + total_branch], storage_start=start)[0]

    @torch.inference_mode()
    def verify(self):
        eng = self.graph_engine
        offset = eng.kv_cache.seq_len
        position_ids = (self.depth + offset).unsqueeze(0)
        logits = eng.tree_verify_inference(input_ids=self.verify_tokens.unsqueeze(0), position_ids=position_ids, mask_bits=self.mask_bits)[0]
        # get_sampling_logits + softmax(/T) (SpecTree_TP.py:8-21,175-176) == norm_logits with top-p
        self.target_logits = norm_logits(logits, temperature=self.temperature, top_k=-1, top_p=self.top_p)

        # fused accept walk (accept_step :147-165 driven by verify :181-197)
        mark = self.noise.mark()
        self.noise.uniform_block_into(self._uniforms)
        ops.tree_accept_walk(self.target_logits, self.draft_logits, self.verify_tokens, self.succ_off, self.succ, self._uniforms,
                             self.temperature, self._walk_out, self._residual, self._scratch)
        w = self._walk_out.tolist()
        n_accept, code, used, terminal, nan_residual = w[0], w[1], w[2], w[3], w[4]
        self.noise.rewind(mark, used)
        accept_list = [0] + w[8:8 + n_accept]
        acc_count = n_accept
        next_token = torch.zeros((1,), dtype=torch.long, device=self.device)
        if not terminal:
            if nan_residual:
                terminal = 1
            else:
                self.noise.exponential_into(self._expo)
                next_token = ops.sample_argmax(self._residual, self._expo).reshape(1)
                acc_count += 1
        accept_list = accept_list[:acc_count]  # SpecTree_TP.py:217 (keeps reference semantics incl. its truncation)
        if terminal:
            return None, acc_count, []
        accept_tokens = self.verify_tokens[torch.tensor(accept_list, dtype=torch.long, device=self.device)]
        accept_tokens = torch.cat([accept_tokens, next_token], dim=-1)
        eng.kv_cache.gather_kv_incremental(accept_list, offset)
        eng.retrieval_cache.update_graph_cache(eng.kv_cache)
        self.draft_logits.zero_()
        self.verify_tokens.zero_()
        return next_token, acc_count, accept_tokens
