"""CPU-side checks of follow-up turns on the Sequoia tree path (session.TreeSession): the refusals that run before anything
changes, the capacity and retrieval-tail limits at which generate stops, the draws of a turn in order on the device Philox
stream restated on the CPU (tests/philox_oracle.py), and the max_context plumbing of the Sequoia retrieval cache."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import philox_oracle as px
from triforce_b200 import device_loop, session
from triforce_b200.cache import RetrievalCache, RetrievalCacheSeqouia
from triforce_b200.session import TreeSession
from triforce_b200.tp import DistributedLlama, SingleGpuLlama

V, T = 96, 64  # vocabulary and tree size of the stubs


def _model_stub(L=2, H=4, hidden=512):
    cfg = SimpleNamespace(num_hidden_layers=L, num_key_value_heads=H, hidden_size=hidden, num_attention_heads=H)
    return SimpleNamespace(config=cfg, device=torch.device("cpu"))


class _Kv:
    def __init__(self, seq_len, slots):
        self.seq_len, self.slots = seq_len, slots

    def sync_seq_len_to_device(self):
        pass


class _Llm:
    """The members TreeSession reads from a tree engine; `calls` records every call that would change device state."""

    def __init__(self, seq_len=5000, slots=8192, budget=4096, prefill=4096, max_context=8192, world_size=1, tree_size=T):
        self.world_size, self.tree_size, self.prefill_len = world_size, tree_size, prefill
        self.device = torch.device("cpu")
        self.config = SimpleNamespace(vocab_size=V, max_position_embeddings=131072)
        self.kv_cache = _Kv(seq_len, slots)
        self.retrieval_cache = RetrievalCache(_model_stub(), max_budget=budget, prefill=prefill, chunk_size=8, gamma=tree_size - 1,
                                              max_context=max_context)
        self.calls = []

    def reset(self):
        self.calls.append("reset")

    def prefill(self, input_ids):
        self.calls.append("prefill")


def _session(**kw):
    return TreeSession(_Llm(**kw))


def test_tree_session_refuses_engines_it_does_not_cover():
    with pytest.raises(NotImplementedError, match="world_size=2"):
        TreeSession(_Llm(world_size=2))
    with pytest.raises(ValueError, match="tree_size > 0"):
        TreeSession(_Llm(tree_size=0))


def test_tree_session_refuses_calls_out_of_order():
    s = _session()
    with pytest.raises(RuntimeError, match="append before prefill"):
        s.append([1, 2, 3])
    with pytest.raises(RuntimeError, match="generate before prefill"):
        s.generate(16)
    with pytest.raises(RuntimeError, match="truncate before prefill"):
        s.truncate(10)
    s.ids = list(range(5000))  # as after a prefill whose turn was generated
    with pytest.raises(RuntimeError, match="call append"):
        s.generate(16)
    s.ids, s.pending = [], None
    with pytest.raises(ValueError, match="prefill length 4096, got 4000"):
        s.prefill(list(range(4000)))
    assert s.llm.calls == [] and s.ids == []


def test_tree_session_refuses_appends_past_the_store_or_the_boundary():
    s = _session()
    s.ids, s.pending = list(range(5000)), 7
    rc = s.llm.retrieval_cache
    # 5000 committed + 1 pending + n new + 64 tree rows must fit 8192 slots: n = 3127 fits, 3128 does not
    with pytest.raises(ValueError, match="fewer than the 64 slots a tree verify writes in the 8192-slot"):
        s.append(list(range(3128)))
    with pytest.raises(ValueError, match="at least one id"):
        s.append([], keep_pending=False)
    for n in (0, 5001, -3):
        with pytest.raises(ValueError, match="committed length is 5000"):
            s.truncate(n)
    assert s.ids == list(range(5000)) and s.pending == 7 and s.llm.kv_cache.seq_len == 5000 and rc.prefill == 4096
    # the boundary: beyond max_context (8192 slots but max_context 6000), below the budget
    s = _session(max_context=6000)
    s.ids = list(range(5000))
    with pytest.raises(ValueError, match="beyond max_context 6000"):
        s.append(list(range(1008)))  # 6008 tokens: boundary 6008 > 6000
    s = _session(seq_len=4000, prefill=4000, budget=4096)
    s.ids = list(range(4000))
    with pytest.raises(ValueError, match="fewer than the retrieval budget"):
        s.append(list(range(95)))  # 4095 tokens: a boundary of 4088 < 4096
    assert s.ids == list(range(4000)) and s.pending is None and s.llm.kv_cache.seq_len == 4000


class _Tree:
    """The members of SpecTree a TreeSession turn touches.  A round emits two tokens (its verify commits the root and one node)
    and records the race buffer the growth saw and the noise verify drew."""
    draft_step = 4

    def __init__(self, kv, temperature=0.6, top_p=0.9, k=5):
        self.kv, self.temperature, self.top_p = kv, temperature, top_p
        self.tree_size = T
        self.rand = torch.zeros((T, V), dtype=torch.float32)
        self._uniforms = torch.zeros(k, dtype=torch.float32)
        self._expo = torch.zeros(V, dtype=torch.float32)
        self.noise = None
        self.seen = []

    def construct_grow_map(self, next_token):
        assert self.kv.seq_len + T <= self.kv.slots, "a verify past the store"
        self.seen.append(("race", self.rand.clone()))

    def verify(self):
        self.noise.uniform_block_into(self._uniforms)
        self.seen.append(("walk", self._uniforms.clone()))
        self.noise.exponential_into(self._expo)
        self.seen.append(("residual", self._expo.clone()))
        self.kv.seq_len += 2
        return torch.tensor([5]), 2, torch.tensor([4, 9, 5])


def _cpu_philox_fill(log):
    """tf_philox_fill restated with tests/philox_oracle.py: element i of draw state[1] of stream state[0]."""
    def fill(state, kind, out):
        seed, draw = int(state[0]), int(state[1])
        w = px.words(seed, draw, out.numel())
        vals = px.uniform(w) if kind == 0 else px.exponential(w).astype(np.float32)
        out.copy_(torch.from_numpy(vals).view_as(out))
        state[1] += 1
        log.append((draw, kind, out.numel()))
        return out
    return fill


def _turn_on_stubs(monkeypatch, s, tree, max_new, seed=0, logits_row=None):
    """generate on CPU: the first token's top-p and argmax sampler are stubbed (they are kernels); the noise is the session's."""
    log = []
    monkeypatch.setattr(device_loop.ops, "philox_fill", _cpu_philox_fill(log))
    monkeypatch.setattr(session, "norm_logits", lambda x, **k: x)
    firsts = []

    def sample_argmax(probs, expo):
        firsts.append(expo.clone())
        return torch.tensor([int(torch.argmax(probs / expo))])
    monkeypatch.setattr(session.ops, "sample_argmax", sample_argmax)
    s._trees[(tree.temperature, tree.top_p)] = tree
    s.ids = list(range(s.llm.kv_cache.seq_len))
    s._logits = torch.ones((1, 1, V)) if logits_row is None else logits_row
    toks = s.generate(max_new, temperature=tree.temperature, top_p=tree.top_p, seed=seed)
    return toks, log, firsts


def test_turn_draws_in_the_documented_order_on_the_philox_stream(monkeypatch):
    """First-token exponential; then per round the race block, the walk's uniform block and the residual exponential — each one
    draw of the stream restarted at `seed`, holding the values tf_philox_fill writes."""
    seed = 0x5EED
    s = _session()
    tree = _Tree(s.llm.kv_cache)
    toks, log, firsts = _turn_on_stubs(monkeypatch, s, tree, max_new=7, seed=seed)
    k = tree._uniforms.numel()
    assert s.last_turn.rounds == 3 and toks[1:] == [9, 5] * 3 and s.last_turn.accepted == [2, 2, 2]
    assert log == [(0, 1, V)] + [e for r in range(3) for e in ((1 + 3 * r, 0, T * V), (2 + 3 * r, 0, k), (3 + 3 * r, 1, V))]
    np.testing.assert_array_equal(firsts[0].numpy(), px.exponential(px.words(seed, 0, V)).astype(np.float32))
    for r in range(3):
        (n0, race), (n1, walk), (n2, res) = tree.seen[3 * r:3 * r + 3]
        assert (n0, n1, n2) == ("race", "walk", "residual")
        want = px.uniform(px.words(seed, 1 + 3 * r, T * V)).reshape(T, V)
        np.testing.assert_array_equal(race.numpy(), want)
        assert (race > 0).all() and (race < 1).all()
        np.testing.assert_array_equal(walk.numpy(), px.uniform(px.words(seed, 2 + 3 * r, k)))
        np.testing.assert_array_equal(res.numpy(), px.exponential(px.words(seed, 3 + 3 * r, V)).astype(np.float32))
    # the last token is pending, the others committed
    assert s.pending == toks[-1] and s.ids[-len(toks) + 1:] == toks[:-1]


def test_greedy_turn_draws_no_race(monkeypatch):
    s = _session()
    tree = _Tree(s.llm.kv_cache, temperature=0.0)
    _, log, _ = _turn_on_stubs(monkeypatch, s, tree, max_new=3)
    assert [kind for _, kind, n in log] == [1, 0, 1] and all(n != T * V for *_, n in log)
    assert [d for d, *_ in log] == [0, 1, 2]


def test_generate_stops_before_the_store_overflows(monkeypatch):
    # 5000 committed, 5070 slots, 64 tree rows: rounds at 5000, 5002, 5004, 5006; 5008 + 64 > 5070
    s = _session(slots=5070)
    tree = _Tree(s.llm.kv_cache)
    toks, *_ = _turn_on_stubs(monkeypatch, s, tree, max_new=100)
    assert s.last_turn.stop == "slots" and s.last_turn.rounds == 4 and len(toks) == 9
    assert s.llm.kv_cache.seq_len == 5008 and s.length == len(s.ids) == 5008 and s.pending == toks[-1]


def test_generate_stops_before_the_retrieval_tail_overflows(monkeypatch):
    # boundary 4096, budget 4096: a round commits up to draft_step = 4 rows, so it runs while seq_len + 4 - 4096 <= 4096
    s = _session(seq_len=8180, slots=9000, max_context=9000)
    tree = _Tree(s.llm.kv_cache)
    _turn_on_stubs(monkeypatch, s, tree, max_new=100)
    assert s.last_turn.stop == "tail" and s.length == 8190
    assert s.length + tree.draft_step - 4096 > 4096 >= s.length - 2 + tree.draft_step - 4096


def test_append_and_generate_stay_inside_the_rope_positions(monkeypatch):
    s = _session(seq_len=5000, slots=140000, max_context=140000)
    s.llm.config.max_position_embeddings = 5100
    s.ids = list(range(5000))
    with pytest.raises(ValueError, match="past the model's 5100 RoPE positions"):
        s.append(list(range(100)))
    assert s.length == 5000 and s.ids == list(range(5000))
    # rounds while seq_len + draft_step <= 5100: from 5090 the rounds start at 5090, 5092, 5094 and 5096
    s = _session(seq_len=5090, slots=140000, max_context=140000)
    s.llm.config.max_position_embeddings = 5100
    _turn_on_stubs(monkeypatch, s, _Tree(s.llm.kv_cache), max_new=100)
    assert s.last_turn.stop == "positions" and s.last_turn.rounds == 4 and s.length == 5098


def test_generate_keeps_max_new_as_its_target(monkeypatch):
    s = _session()
    _turn_on_stubs(monkeypatch, s, _Tree(s.llm.kv_cache), max_new=1)
    assert s.last_turn.rounds == 0 and s.last_turn.stop == "max_new" and s.length == 5000
    with pytest.raises(RuntimeError, match="call append"):
        s.generate(4)


def test_sequoia_retrieval_cache_takes_max_context():
    rc = RetrievalCacheSeqouia(_model_stub(), max_budget=4096, prefill=124928, chunk_size=8, tree_size=512, max_context=131072)
    assert rc.max_context == 131072 and rc.boundary(130000) == 130000 and rc.real_budget == 4096 + 512
    assert rc._scores.numel() == 2 * 4 * (131072 // 8)
    assert RetrievalCacheSeqouia(_model_stub(), max_budget=64, prefill=1024, tree_size=128).max_context == 1024
    with pytest.raises(ValueError, match="beyond max_context"):
        RetrievalCacheSeqouia(_model_stub(), max_budget=64, prefill=1024, tree_size=128).boundary(1032)


def test_engine_max_context_defaults_to_prefill_and_is_checked():
    llm = SingleGpuLlama("llama-13B-128K", prefill=130048, tree_size=512)
    assert llm.max_context == 130048
    assert SingleGpuLlama("llama-13B-128K", prefill=8192, max_context=12288, tree_size=512).max_context == 12288
    with pytest.raises(ValueError, match="below prefill"):
        DistributedLlama("llama-13B-128K", prefill=8192, max_context=4096)
