"""The room check of the chain decode loops on stubs (no device): decoding.chain_room at "exactly fits" and "one row over" for
each of its three limits, the refusal of TriForceRun.step and DeviceLoopRun.step before the engine sees any call, and the stop
reasons of Session.generate."""
from types import SimpleNamespace

import pytest
import torch

from triforce_b200 import session as session_mod
from triforce_b200.decoding import TriForceRun, chain_room, check_room
from triforce_b200.device_loop import DeviceLoopRun
from triforce_b200.session import Session

BIG = 1 << 20
P = 4096  # the retrieval boundary of the stubs


def _eng(seq_len, slots=BIG, budget=BIG, positions=BIG, prefill=P):
    return SimpleNamespace(kv_cache=SimpleNamespace(seq_len=seq_len, slots=slots),
                           graph_cache=SimpleNamespace(prefill=prefill, max_budget=budget),
                           model=SimpleNamespace(config=SimpleNamespace(max_position_embeddings=positions, vocab_size=16),
                                                 device=torch.device("cpu")))


@pytest.mark.parametrize("gamma", [4, 6, 16])
@pytest.mark.parametrize("limit", ["slots", "tail", "positions"])
def test_room_fits_exactly_and_refuses_one_row_over(limit, gamma):
    # the committed length S at which a step's gamma + 2 rows end exactly at the limit
    size = {"slots": 6000, "tail": 512, "positions": 7000}[limit]
    S = (P + size if limit == "tail" else size) - gamma - 2
    fits = _eng(S, **{{"slots": "slots", "tail": "budget", "positions": "positions"}[limit]: size})
    assert chain_room(fits, gamma) is None
    check_room(fits, gamma)
    over = _eng(S + 1, **{{"slots": "slots", "tail": "budget", "positions": "positions"}[limit]: size})
    assert chain_room(over, gamma) == limit
    with pytest.raises(ValueError, match=rf"\({limit}\)"):
        check_room(over, gamma)


def test_room_names_the_first_limit_it_passes():
    e = _eng(P + 100, slots=P + 100, budget=64, positions=P + 100)
    assert chain_room(e, 6) == "slots"
    e.kv_cache.slots = BIG
    assert chain_room(e, 6) == "tail"
    e.graph_cache.max_budget = BIG
    assert chain_room(e, 6) == "positions"
    # the boundary moves with a re-selection: the same length fits again once `prefill` follows it
    e = _eng(P + 60, budget=64)
    assert chain_room(e, 6) == "tail"
    e.graph_cache.prefill = P + 56
    assert chain_room(e, 6) is None


class _Recorder:
    """Records every call made on it (and on what its calls return)."""

    def __init__(self, calls, name):
        self._calls, self._name = calls, name

    def __getattr__(self, attr):
        def call(*a, **k):
            self._calls.append(f"{self._name}.{attr}")
            raise AssertionError(f"{self._name}.{attr} called before the room check refused")
        return call


@pytest.mark.parametrize("limit", ["slots", "tail", "positions"])
def test_steps_refuse_before_the_engine_sees_a_call(limit):
    gamma = 6
    kw = {"slots": dict(slots=P + 40), "tail": dict(budget=32), "positions": dict(positions=P + 40)}[limit]
    eng = _eng(P + 40 - gamma - 1, **kw)
    calls = []
    ge = _Recorder(calls, "graph_engine")
    ge.engine, ge._loop_buffers = eng, None
    run = TriForceRun(None, ge, gamma=gamma, noise=_Recorder(calls, "noise"))
    run.next_token, run.generated = 5, [5]
    with pytest.raises(ValueError, match=rf"\({limit}\)"):
        run.step()
    dev = object.__new__(DeviceLoopRun)
    dev.eng, dev.gamma, dev.loop = eng, gamma, _Recorder(calls, "device_loop")
    with pytest.raises(ValueError, match=rf"\({limit}\)"):
        dev.step()
    assert calls == []
    assert eng.kv_cache.seq_len == P + 40 - gamma - 1 and run.n == 0 and run.generated == [5]


class _FakeRun:
    """Stands in for TriForceRun / DeviceLoopRun inside Session.generate: each step commits `per_step` tokens."""
    per_step = 3

    def __init__(self, tokenizer, ge, gamma, **kw):
        self.eng, self.gamma = ge.engine, gamma
        self.n, self.generated, self.steps = 0, [], 0

    def start(self, logits):
        self.generated = [7]

    def room(self):
        return chain_room(self.eng, self.gamma)

    def step(self):
        check_room(self.eng, self.gamma)
        self.eng.kv_cache.seq_len += self.per_step
        self.generated += [8] * self.per_step
        self.n += self.per_step
        self.steps += 1


@pytest.mark.parametrize("device_loop", [False, True])
@pytest.mark.parametrize("limit", ["max_new", "slots", "tail", "positions"])
def test_session_generate_stops_before_a_step_that_does_not_fit(monkeypatch, limit, device_loop):
    monkeypatch.setattr(session_mod, "TriForceRun", _FakeRun)
    monkeypatch.setattr(session_mod, "DeviceLoopRun", _FakeRun)
    gamma, S0 = 6, P + 1
    kw = {"max_new": {}, "slots": dict(slots=P + 30), "tail": dict(budget=24), "positions": dict(positions=P + 36)}[limit]
    eng = _eng(S0, **kw)
    s = Session(SimpleNamespace(engine=eng), gamma=gamma)
    s.ids, s._logits = list(range(S0)), object()
    toks = s.generate(40, device_loop=device_loop)
    assert s.last_stop == limit
    run = s.last_run
    assert toks == run.generated and len(toks) == 1 + 3 * run.steps
    if limit == "max_new":
        assert run.n >= 40
    else:
        assert run.n < 40 and chain_room(eng, gamma) == limit
        assert chain_room(_eng(eng.kv_cache.seq_len - 3, **kw), gamma) is None  # the last step taken did fit
    assert s.ids == list(range(S0)) + toks[:-1] and s.pending == toks[-1]
    assert eng.kv_cache.seq_len == S0 + 3 * run.steps
