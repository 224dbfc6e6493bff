"""Follow-up turns over one prefilled long context: the on-chip engine (`GraphInferenceEngine`) answers several questions about
the same document without prefilling it again.

    s = Session(ge, gamma=6)
    s.prefill(document_and_question_ids)          # today's TriForce prompt phase
    answer = s.generate(256, temperature=0.6, top_p=0.9, seed=0)
    s.append(next_question_ids)                   # extend the full KV, re-select the retrieval cache, feed the draft
    answer2 = s.generate(256, temperature=0.6, top_p=0.9, seed=1)
    s.truncate(n); s.append(other_question_ids)   # roll back to a saved length and ask something else

A turn is prefill or append followed by one generate.  The turn's first token is drawn when generate starts, from the logits
prefill or append left, because that is where the turn's temperature, top_p and seed are given; the events and draws are those
of `decoding.TriForce` (the first turn replays it event for event).  The last token a turn samples is pending: it is not in
the full KV until the next append forwards it (keep_pending=True) or drops it.
"""
from __future__ import annotations

from typing import List, Optional

import torch

from .decoding import TriForceRun, prompt_phase
from .device_loop import DeviceLoopRun, PhiloxNoise


class Session:
    def __init__(self, graph_engine, gamma: int = 6, tokenizer=None, trace: Optional[list] = None, strict_less: bool = True,
                 pad_full_verify: bool = False):
        """`trace`: a list that receives the ("target_in" | "sample" | "rand" | "middle", value) events of every turn.
        `strict_less`, `pad_full_verify`: as in decoding.TriForceRun (the step-wise loop)."""
        self.ge = graph_engine
        self.eng = graph_engine.engine
        self.gamma = gamma
        self.tokenizer, self.trace = tokenizer, trace
        self.strict_less, self.pad_full_verify = strict_less, pad_full_verify
        self.ids: List[int] = []            # the ids whose K/V rows the full KV holds, in order
        self.pending: Optional[int] = None  # the last sampled token, not yet forwarded
        self.last_run = None                # the TriForceRun / DeviceLoopRun of the last turn (its counts)
        self._logits = None                 # last-row logits of the current turn's input, until generate samples from them
        self._queries = None
        self._draft_stale = False

    @property
    def length(self) -> int:
        """The committed length: tokens in the full KV."""
        return self.eng.kv_cache.seq_len

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
        if not self.ids:
            raise RuntimeError("append before prefill: the session has no context")
        new = ([self.pending] if keep_pending and self.pending is not None else []) + [int(i) for i in _as_ids(ids)[0].tolist()]
        if not new:
            raise ValueError("append needs at least one id")
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
        the turn's tokens; all but the last are committed, the last is pending."""
        if not self.ids:
            raise RuntimeError("generate before prefill: the session has no context")
        if self._logits is None:
            raise RuntimeError("a turn starts with prefill or append; after a generate or a truncate, call append")
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
        while run.n < max_new:
            run.step()
        self.ids += run.generated[:-1]
        self.pending = run.generated[-1]
        self.last_run = run
        return list(run.generated)

    def truncate(self, n: int) -> None:
        """Roll the committed length back to n (the host length and the device copy the graphs read); the pending token is
        dropped.  The next call must be append (or prefill)."""
        if not self.ids:
            raise RuntimeError("truncate before prefill: the session has no context")
        if not 1 <= n <= self.length:
            raise ValueError(f"truncate to {n}: the committed length is {self.length}")
        kv = self.eng.kv_cache
        kv.seq_len = n
        kv.sync_seq_len_to_device()
        del self.ids[n:]
        self.pending, self._logits = None, None
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


def _as_ids(ids) -> torch.Tensor:
    """[1, n] int64 ids from a list, a 1-D or a [1, n] tensor."""
    t = ids if torch.is_tensor(ids) else torch.tensor(list(ids), dtype=torch.int64)
    return t.reshape(1, -1).to(torch.int64)
