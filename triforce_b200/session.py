"""Follow-up turns over one prefilled long context: the engine answers several questions about the same document without
prefilling it again.  `Session` runs the chain path (`GraphInferenceEngine`: draft model, retrieval verify, full-KV verify);
`TreeSession` runs the Sequoia tree path (`tp.SingleGpuLlama` with `tree_size > 0`).

    s = Session(ge, gamma=6)
    s.prefill(document_and_question_ids)          # today's TriForce prompt phase
    answer = s.generate(256, temperature=0.6, top_p=0.9, seed=0)
    s.append(next_question_ids)                   # extend the full KV, re-select the retrieval cache, feed the draft
    answer2 = s.generate(256, temperature=0.6, top_p=0.9, seed=1)
    s.truncate(n); s.append(other_question_ids)   # roll back to a saved length and ask something else
    sc = s.score(candidate_answer_ids)            # log p(each id | context, earlier ids); the session does not change

`score` runs between turns and leaves no trace: see `_Turns.score`.

A turn is prefill or append followed by one generate.  The turn's first token is drawn when generate starts, from the logits
prefill or append left, because that is where the turn's temperature, top_p and seed are given; the events and draws are those
of `decoding.TriForce` (the first turn replays it event for event).  The last token a turn samples is pending: it is not in
the full KV until the next append forwards it (keep_pending=True) or drops it.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import torch

from . import ops
from .decoding import TriForceRun, prompt_phase
from .device_loop import DeviceLoopRun, PhiloxNoise
from .sampling import norm_logits
from .spectree import SpecTree, load_grow_map


@dataclass
class Score:
    """What `score(ids)` returns, one entry per id, on the model's device: `logprobs` (fp32), log p(ids[i] | context, ids[:i])
    under the model's own distribution (temperature 1, no top-p); `argmax` (int32), the id greedy decoding would emit there
    (torch.argmax's rule); `greedy` (bool), argmax == ids."""
    logprobs: torch.Tensor
    argmax: torch.Tensor
    greedy: torch.Tensor


class _Turns:
    """The turn bookkeeping both sessions share: the committed ids, the pending token, the logits a turn starts from, the order
    of calls, the rollback of the full KV's length and `score`.  A subclass sets `_kv` (the full-KV cache), `_model` (the
    target), `_positions` (its RoPE positions) and `_score_extend` (its LlamaModel.extend call)."""

    def __init__(self):
        self.ids: List[int] = []            # the ids whose K/V rows the full KV holds, in order
        self.pending: Optional[int] = None  # the last sampled token, not yet forwarded
        self._logits = None                 # last-row logits of the current turn's input, until generate samples from them
        self._queries = None

    @property
    def _kv(self):
        raise NotImplementedError

    @property
    def _model(self):
        raise NotImplementedError

    @property
    def _positions(self) -> int:
        return self._model.config.max_position_embeddings

    def _score_extend(self, ids: torch.Tensor, logprobs) -> None:
        raise NotImplementedError

    @property
    def length(self) -> int:
        """The committed length: tokens in the full KV."""
        return self._kv.seq_len

    @torch.inference_mode()
    def score(self, ids) -> Score:
        """Score `ids` as a continuation of the committed context: the first id on the row the next token would be drawn from
        (the held logits of prefill or append, or the pending token's row, which is forwarded first), each later id on the row
        of the id before it.  The rows go into the full KV after its committed length (LlamaModel.extend with `logprobs`) and
        the length is rolled back: the ids, the pending token, the turn's logits, the retrieval cache, the draft and the
        captured graphs are as they were.  Refused, before anything changes, before prefill, after a truncate (no row to
        condition on) and past the full KV's slots or the model's RoPE positions."""
        if not self.ids:
            raise RuntimeError("score before prefill: the session has no context")
        if self.pending is None:
            self._check_turn()
        new = [int(i) for i in _as_ids(ids)[0].tolist()]
        if not new:
            raise ValueError("score needs at least one id")
        m = self._model
        V = m.config.vocab_size
        if not all(0 <= i < V for i in new):
            raise ValueError(f"token ids must lie in [0, {V}); got ids in [{min(new)}, {max(new)}]")
        # rows forwarded: the pending token and every id (the last id's row is forwarded too: extend scores within its ids)
        rows = [self.pending] + new if self.pending is not None else new
        kv = self._kv
        if len(rows) > 1:
            if kv.seq_len + len(rows) > kv.slots:
                raise ValueError(f"appending {len(rows)} tokens after {kv.seq_len} exceeds the {kv.slots} slots of the full-KV store")
            if kv.seq_len + len(rows) > self._positions:
                raise ValueError(f"appending {len(rows)} tokens after {kv.seq_len} reaches past the model's "
                                 f"{self._positions} RoPE positions")
        n = len(new)
        target = torch.tensor(new, dtype=torch.int32, device=m.device)
        lp = torch.empty(n, dtype=torch.float32, device=m.device)
        am = torch.empty(n, dtype=torch.int32, device=m.device)
        k = 0
        if self.pending is None:  # the first id on the held last-row logits
            ops.token_logprobs(self._logits.reshape(-1, V)[-1:], target[:1], lp[:1], am[:1], check_ids=False)
            k = 1
        if len(rows) > 1:
            start = kv.seq_len
            try:
                self._score_extend(torch.tensor([rows], dtype=torch.int64, device=m.device), (lp[k:], am[k:]))
            finally:
                kv.seq_len = start  # extend moved only the host length; the device copy the graphs read is untouched
        return Score(logprobs=lp, argmax=am, greedy=am == target)

    def _new_ids(self, ids, keep_pending: bool) -> List[int]:
        """The ids an append forwards: the pending token (if kept) and `ids`."""
        if not self.ids:
            raise RuntimeError("append before prefill: the session has no context")
        new = ([self.pending] if keep_pending and self.pending is not None else []) + [int(i) for i in _as_ids(ids)[0].tolist()]
        if not new:
            raise ValueError("append needs at least one id")
        return new

    def _check_turn(self) -> None:
        """generate needs the logits of a prefill or an append: a turn starts with one of them."""
        if not self.ids:
            raise RuntimeError("generate before prefill: the session has no context")
        if self._logits is None:
            raise RuntimeError("a turn starts with prefill or append; after a generate or a truncate, call append")

    def truncate(self, n: int) -> None:
        """Roll the committed length back to n (the host length and the device copy the graphs read); the pending token is
        dropped.  The next call must be append (or prefill)."""
        if not self.ids:
            raise RuntimeError("truncate before prefill: the session has no context")
        if not 1 <= n <= self.length:
            raise ValueError(f"truncate to {n}: the committed length is {self.length}")
        kv = self._kv
        kv.seq_len = n
        kv.sync_seq_len_to_device()
        del self.ids[n:]
        self.pending, self._logits = None, None
        self._truncated()

    def _truncated(self) -> None:
        pass


class Session(_Turns):
    def __init__(self, graph_engine, gamma: int = 6, tokenizer=None, trace: Optional[list] = None, strict_less: bool = True,
                 pad_full_verify: bool = False):
        """`trace`: a list that receives the ("target_in" | "sample" | "rand" | "middle", value) events of every turn.
        `strict_less`, `pad_full_verify`: as in decoding.TriForceRun (the step-wise loop)."""
        self.ge = graph_engine
        self.eng = graph_engine.engine
        self.gamma = gamma
        self.tokenizer, self.trace = tokenizer, trace
        self.strict_less, self.pad_full_verify = strict_less, pad_full_verify
        super().__init__()
        self.last_run = None                # the TriForceRun / DeviceLoopRun of the last turn (its counts)
        self.last_stop: Optional[str] = None  # why the last turn stopped (see generate)
        self._draft_stale = False

    @property
    def _kv(self):
        return self.eng.kv_cache

    @property
    def _model(self):
        return self.eng.model

    def _score_extend(self, ids: torch.Tensor, logprobs) -> None:
        self.eng.model.extend(ids, self.eng.kv_cache, chunk=self.eng.target_prefill_chunk, logprobs=logprobs)

    @torch.inference_mode()
    def prefill(self, ids) -> None:
        """A new context: the three caches are reset and the prompt goes through TriForce's prompt phase."""
        ids = _as_ids(ids).to(self.eng.model.device)
        if ids.shape[1] < 2:
            raise ValueError("a prompt needs at least two ids")
        self._logits = prompt_phase(self.ge, ids, trace=self.trace)
        self.ids = ids[0].tolist()
        self.pending, self._draft_stale = None, False

    @torch.inference_mode()
    def append(self, ids, keep_pending: bool = True) -> None:
        """The next question: the pending token (if kept) and `ids` are appended to the full KV (LlamaModel.extend), the retrieval
        cache re-selects its budget with the last id's queries (RetrievalCache.reselect), and the draft's window takes the
        appended ids.  Refused, before anything changes, past the full KV's capacity or when the new boundary would leave less
        than the retrieval budget."""
        new = self._new_ids(ids, keep_pending)
        kv = self.eng.kv_cache
        if kv.seq_len + len(new) > kv.slots:
            raise ValueError(f"appending {len(new)} tokens after {kv.seq_len} exceeds the {kv.slots} slots of the full-KV store")
        self.eng.graph_cache.boundary(kv.seq_len + len(new))
        if self.trace is not None:
            self.trace.append(("target_in", list(new)))
        self._logits = self._extend(new)
        self._reselect()
        self.ids += new
        self.pending = None
        self._feed_draft(new)

    @torch.inference_mode()
    def generate(self, max_new: int, temperature: float = 0.6, top_p: float = 0.9, seed: int = 0, device_loop: bool = False,
                 noise=None) -> List[int]:
        """Draw the turn's first token, then run TriForce steps until at least `max_new` tokens: step-wise (decoding.TriForceRun)
        or one whole-loop graph launch per step (device_loop.DeviceLoopRun, re-captured when a re-selection moved the retrieval
        boundary).  Noise: the device Philox stream of `seed`, or for the step-wise loop any noise source (`noise`).  Returns
        the turn's tokens; all but the last are committed, the last is pending.
        The turn stops early, before a step that would not fit (decoding.chain_room), and `last_stop` says why: "max_new",
        "slots", "tail" or "positions".  After "tail" an append re-selects the retrieval boundary and the next turn goes on."""
        self._check_turn()
        if device_loop:
            if noise is not None:
                raise ValueError("the device loop draws from the Philox stream of `seed`; it takes no noise source")
            run = DeviceLoopRun(self.tokenizer, self.ge, gamma=self.gamma, top_p=top_p, temperature=temperature, seed=seed,
                                strict_less=self.strict_less)
        else:
            run = TriForceRun(self.tokenizer, self.ge, gamma=self.gamma, top_p=top_p, temperature=temperature,
                              noise=noise if noise is not None else PhiloxNoise(self.eng.model.device, seed), trace=self.trace,
                              strict_less=self.strict_less, pad_full_verify=self.pad_full_verify)
        run.start(self._logits)
        self._logits = None
        self.last_stop = "max_new"
        while run.n < max_new:
            stop = run.room()
            if stop is not None:
                self.last_stop = stop
                break
            run.step()
        self.ids += run.generated[:-1]
        self.pending = run.generated[-1]
        self.last_run = run
        return list(run.generated)

    def _truncated(self) -> None:
        self._draft_stale = True

    # --- the three parts of append (tools/bench_session.py times each) ----------------------------------------------------
    def _extend(self, new: List[int]):
        m = self.eng.model
        self._queries = torch.empty((len(m.layers), m.local_num_heads, m.head_dim), dtype=torch.float16, device=m.device)
        ids = torch.tensor([new], dtype=torch.int64, device=m.device)
        return m.extend(ids, self.eng.kv_cache, chunk=self.eng.target_prefill_chunk, queries=self._queries)

    def _reselect(self):
        self.eng.graph_cache.reselect(self.eng.kv_cache, self._queries)
        self._queries = None

    def _feed_draft(self, new: List[int]):
        """The appended ids go through the draft's prompt path.  After a rollback the window's rows belong to tokens that are gone,
        so it is cleared (sinks kept) and re-filled from the kept ids — the last `recent_size` of them, the appended ids included;
        the rows the re-fill does not reach stay zero, as after a prompt."""
        dc = self.eng.draft_cache
        feed = new
        if self._draft_stale:
            keep = 0 if len(self.ids) <= dc.start_size + dc.recent_size else dc.start_size
            dc.key_store[:, :, keep:].zero_()
            dc.value_store[:, :, keep:].zero_()
            dc.seq_len, feed = keep, (self.ids if keep == 0 else self.ids[-dc.recent_size:])
            self._draft_stale = False
        self.eng.draft_prefill(torch.tensor([feed], dtype=torch.int64, device=self.eng.draft.device))


@dataclass
class TreeTurn:
    """What one TreeSession turn did: its tokens, the tokens each tree round emitted (accepted nodes + the residual or bonus
    sample), and why it stopped: "max_new", "eos" (an accepted end token or an empty residual ended the generation),
    "slots" (the next verify would not fit the full-KV store), "tail" (the next round could carry the committed rows past the
    boundary beyond the retrieval budget) or "positions" (the next tree would reach past the model's RoPE positions)."""
    tokens: List[int] = field(default_factory=list)
    accepted: List[int] = field(default_factory=list)
    stop: str = "max_new"

    @property
    def rounds(self) -> int:
        return len(self.accepted)

    @property
    def tokens_per_round(self) -> float:
        return sum(self.accepted) / max(len(self.accepted), 1)


def tree_round(st: SpecTree, next_token: torch.Tensor):
    """One round of the Sequoia tree as a TreeSession runs it: fresh race noise from `st.noise` (at T > 0; the greedy tree does
    not read it), the growth (`construct_grow_map`), then `verify` (the walk's uniform block, then the residual exponential).
    Returns what `SpecTree.verify` returns."""
    if st.temperature > 0:
        st.noise.tree_uniform_into(st.rand)
    st.construct_grow_map(next_token=next_token)
    return st.verify()


class TreeSession(_Turns):
    """Follow-up turns on the Sequoia tree path: a `tp.SingleGpuLlama` (or a one-GPU `tp.DistributedLlama`) with `tree_size > 0`,
    over an fp16 or E4M3 full-KV store, fp16 or E4M3 weights, MHA or grouped-query attention.

        llm = SingleGpuLlama(name, prefill=P, max_context=P + 4096, tree_size=512, kv_dtype="e4m3", weight_dtype="e4m3", ...)
        llm.init_parameters(state_dict=sd)
        s = TreeSession(llm)
        s.prefill(document_ids)                        # P ids: SpecTree's prompt phase
        answer = s.generate(256, temperature=0.6, top_p=0.9, seed=0)
        s.append(question_ids)                         # extend the full KV, re-select the retrieval cache
        answer2 = s.generate(256, seed=1)

    The turn semantics are `Session`'s.  `prefill` resets the caches, prefills all ids but the last and runs the last one, which
    builds the retrieval cache (SpecTree.prefill's prompt phase).  `append` forwards the pending token and the new ids into the
    full KV (LlamaModel.extend) and re-selects the retrieval budget with the last id's queries (RetrievalCache.reselect).
    `generate` samples the turn's first token from the logits prefill or append left, then runs tree rounds (`tree_round`) until
    the turn has at least `max_new` tokens, an end token is accepted, or the next round would not fit (TreeTurn.stop).

    Noise: by default the device Philox stream of `seed`, restarted for every turn (`PhiloxNoise`), so a turn is reproducible and
    independent of torch's generator.  The draws, in order: one exponential draw [V] for the first token; then per round the
    race block [tree_size, V] (fp32, at T > 0 only), the walk's uniform block [max_children_on_path + 1] and, when the walk ends
    on a residual or a bonus sample, one exponential draw [V].  `noise` (any source of `rng`) replaces the stream.

    Unlike SpecTree's reference default, which draws the race once per prompt and reuses it in every round, the race is drawn
    again before every round: a round's candidates are a fresh sample from the draft given what earlier rounds emitted.
    One SpecTree (sampling callables, ~100 MB of buffers) is kept per (temperature, top_p) and reused across turns."""

    def __init__(self, llm, tokenizer=None, grow_map: Optional[Dict] = None):
        if getattr(llm, "world_size", 1) != 1:
            raise NotImplementedError(f"TreeSession runs on one GPU; world_size={llm.world_size} (tensor parallel) is not covered")
        if getattr(llm, "tree_size", 0) <= 0:
            raise ValueError("TreeSession needs a tree engine (tree_size > 0); the chain path has session.Session")
        self.llm, self.tokenizer = llm, tokenizer
        self.grow_map = grow_map
        super().__init__()
        self.last_turn: Optional[TreeTurn] = None
        self._trees: Dict[Tuple[float, float], SpecTree] = {}

    @property
    def _kv(self):
        return self.llm.kv_cache

    @property
    def _model(self):
        return self.llm.model

    @property
    def _rc(self):
        return self.llm.retrieval_cache

    @property
    def _positions(self) -> int:
        return self.llm.config.max_position_embeddings

    def _score_extend(self, ids: torch.Tensor, logprobs) -> None:
        self.llm.model.extend(ids, self._kv, logprobs=logprobs)

    def _tree(self, temperature: float, top_p: float) -> SpecTree:
        key = (float(temperature), float(top_p))
        if key not in self._trees:
            if self.grow_map is None:
                self.grow_map = load_grow_map("512")
            if self.grow_map["size"] != self.llm.tree_size:
                raise ValueError(f"the grow map has {self.grow_map['size']} nodes, the engine reserves {self.llm.tree_size}")
            # built on a throwaway stream (the constructor draws the race once): each turn sets its own source
            self._trees[key] = SpecTree(self.llm, temperature=temperature, top_p=top_p, grow_map=self.grow_map,
                                        vocab_size=self.llm.config.vocab_size, tokenizer=self.tokenizer,
                                        noise=PhiloxNoise(self.llm.device, 0), race_dtype=torch.float32)
        return self._trees[key]

    @torch.inference_mode()
    def prefill(self, ids) -> None:
        """A new context of exactly `prefill` ids (the retrieval cache's constructed boundary): SpecTree's prompt phase."""
        ids = _as_ids(ids)
        if ids.shape[1] != self.llm.prefill_len:
            raise ValueError(f"a tree-path prompt has the engine's prefill length {self.llm.prefill_len}, got {ids.shape[1]} ids; "
                             "longer contexts come through append")
        kv = self._kv
        if ids.shape[1] + self.llm.tree_size > kv.slots:
            raise ValueError(f"a {ids.shape[1]}-token prompt leaves fewer than the {self.llm.tree_size} slots a tree verify "
                             f"writes in the {kv.slots}-slot full-KV store")
        ids = ids.to(self.llm.device)
        self.llm.reset()
        self.llm.prefill(input_ids=ids[:, :-1])
        self._logits = self.llm.build_retrieval_cache(input_ids=ids[:, -1:])[:, -1:]
        self.ids = ids[0].tolist()
        self.pending = None

    @torch.inference_mode()
    def append(self, ids, keep_pending: bool = True) -> None:
        """The next question: the pending token (if kept) and `ids` go into the full KV (LlamaModel.extend) and the retrieval
        cache re-selects its budget with the last id's queries (RetrievalCache.reselect).  Refused, before anything changes,
        when fewer than `tree_size` slots of the full-KV store would stay free (every round's verify writes that many rows), or
        when the new boundary would leave less than the retrieval budget or pass `max_context`."""
        new = self._new_ids(ids, keep_pending)
        kv, T = self._kv, self.llm.tree_size
        if kv.seq_len + len(new) + T > kv.slots:
            raise ValueError(f"appending {len(new)} tokens after {kv.seq_len} leaves fewer than the {T} slots a tree verify "
                             f"writes in the {kv.slots}-slot full-KV store")
        if kv.seq_len + len(new) >= self._positions:
            raise ValueError(f"appending {len(new)} tokens after {kv.seq_len} reaches past the model's "
                             f"{self._positions} RoPE positions")
        self._rc.boundary(kv.seq_len + len(new))
        self._logits = self._extend(new)
        self._reselect()
        self.ids += new
        self.pending = None

    @torch.inference_mode()
    def generate(self, max_new: int, temperature: float = 0.6, top_p: float = 0.9, seed: int = 0, noise=None) -> List[int]:
        """Draw the turn's first token, then run tree rounds until the turn has at least `max_new` tokens or stops (see
        TreeTurn.stop).  Returns the turn's tokens; all but the last are committed, the last is pending.  `last_turn` holds
        the turn's rounds and tokens per round."""
        self._check_turn()
        st = self._tree(temperature, top_p)
        st.noise = noise if noise is not None else PhiloxNoise(self.llm.device, seed)
        turn = TreeTurn(tokens=[self._first_token(st, self._logits)])
        self._logits = None
        next_token = torch.tensor([[turn.tokens[0]]], dtype=torch.long, device=self.llm.device)
        while len(turn.tokens) < max_new:
            turn.stop = self._room(st)
            if turn.stop != "max_new":
                break
            offset = self._kv.seq_len
            nt, acc, toks = tree_round(st, next_token)
            if nt is None:
                turn.tokens += self._end(st, offset)
                turn.accepted.append(acc)
                turn.stop = "eos"
                break
            turn.tokens += [int(t) for t in toks[1:].tolist()]
            turn.accepted.append(acc)
            next_token = nt.reshape(1, 1)
        self.ids += turn.tokens[:-1]
        self.pending = turn.tokens[-1]
        self.last_turn = turn
        return list(turn.tokens)

    def _first_token(self, st: SpecTree, logits) -> int:
        """SpecTree.prefill's sample: top-p at the turn's temperature, one exponential draw."""
        probs = norm_logits(logits[:, -1, :], temperature=st.temperature, top_k=-1, top_p=st.top_p)
        st.noise.exponential_into(st._expo)
        return int(ops.sample_argmax(probs, st._expo).reshape(-1)[0])

    def _room(self, st: SpecTree) -> str:
        """"max_new" when the next round fits: its verify writes tree_size rows after the committed length, its nodes take
        positions up to seq_len + draft_step - 1, and it commits at most `draft_step` rows (the root and an accepted path), all
        of which the tail copy puts in the budget."""
        kv, rc = self._kv, self._rc
        if kv.seq_len + st.tree_size > kv.slots:
            return "slots"
        if kv.seq_len + st.draft_step > self._positions:
            return "positions"
        if kv.seq_len + st.draft_step - rc.prefill > rc.max_budget:
            return "tail"
        return "max_new"

    def _end(self, st: SpecTree, offset: int) -> List[int]:
        """The walk ended the generation (SpecTree.verify returned no next token): an end token was accepted, or the residual
        had no mass.  The accepted nodes are the turn's last tokens; the root's and all but the last accepted node's rows stay
        in the full KV (the last token is pending) and reach the retrieval tail."""
        w = st._walk_out.tolist()
        nodes = w[8:8 + w[0]]
        toks = st.verify_tokens[torch.tensor(nodes, dtype=torch.long, device=st.device)].tolist() if nodes else []
        keep = [0] + nodes[:-1] if nodes else []
        if keep:
            self._kv.gather_kv_incremental(keep, offset)
        else:
            self._kv.seq_len = offset
        self._rc.update_graph_cache(self._kv)
        st.draft_logits.zero_()
        st.verify_tokens.zero_()
        return [int(t) for t in toks]

    # --- the two parts of append (tools/bench_tree_session.py times each) -------------------------------------------------
    def _extend(self, new: List[int]):
        m = self.llm.model
        self._queries = torch.empty((len(m.layers), m.local_num_heads, m.head_dim), dtype=torch.float16, device=m.device)
        ids = torch.tensor([new], dtype=torch.int64, device=m.device)
        return m.extend(ids, self._kv, queries=self._queries)

    def _reselect(self):
        self._rc.reselect(self._kv, self._queries)
        self._queries = None


def _as_ids(ids) -> torch.Tensor:
    """[1, n] int64 ids from a list, a 1-D or a [1, n] tensor."""
    t = ids if torch.is_tensor(ids) else torch.tensor(list(ids), dtype=torch.int64)
    return t.reshape(1, -1).to(torch.int64)
