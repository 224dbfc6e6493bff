"""CPU-side checks of scoring: the argument checks of tf_token_logprobs (no launch), the refusals of Session.score,
TreeSession.score and LlamaModel.prefill's `logprobs` that run before anything changes, the order of what score forwards and
its rollback (on stubs), and tools/perplexity.py's arguments and shape arithmetic."""
import ctypes
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from triforce_b200 import _C, session
from triforce_b200.llama import LlamaModel
from triforce_b200.session import Session, TreeSession

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import perplexity  # noqa: E402

V = 96


def test_token_logprobs_checks_its_arguments():
    lib = _C.lib()
    buf = (ctypes.c_uint8 * 64)()
    p = ctypes.addressof(buf)
    f = lib.tf_token_logprobs  # (logits, row_stride, rows, V, ids, logprob, argmax, stream)
    for args in ((None, 8, 1, 8, p, p, p), (p, 8, 1, 8, None, p, p), (p, 8, 1, 8, p, None, p), (p, 8, 1, 8, p, p, None)):
        assert f(*args, None) == -1
        assert b"NULL" in lib.tf_last_error()
    assert f(p, 8, -1, 8, p, p, p, None) == -1 and b"rows -1" in lib.tf_last_error()
    assert f(p, 8, 1, 0, p, p, p, None) == -1 and b"V 0" in lib.tf_last_error()
    assert f(p, 7, 2, 8, p, p, p, None) == -1 and b"row stride 7" in lib.tf_last_error()
    assert f(p, 8, 0, 8, p, p, p, None) == 0  # no rows: nothing to launch


class _Kv:
    def __init__(self, seq_len, slots):
        self.seq_len, self.slots = seq_len, slots


def _model(positions=131072):
    return SimpleNamespace(config=SimpleNamespace(vocab_size=V, max_position_embeddings=positions), device=torch.device("cpu"))


def _chain(seq_len=5000, slots=8192, positions=131072):
    eng = SimpleNamespace(kv_cache=_Kv(seq_len, slots), model=_model(positions), target_prefill_chunk=128)
    return Session(SimpleNamespace(engine=eng), gamma=6)


def _tree(seq_len=5000, slots=8192, positions=131072):
    llm = SimpleNamespace(world_size=1, tree_size=64, kv_cache=_Kv(seq_len, slots), model=_model(positions),
                          config=SimpleNamespace(vocab_size=V, max_position_embeddings=positions))
    return TreeSession(llm)


@pytest.mark.parametrize("make", [_chain, _tree], ids=["Session", "TreeSession"])
def test_score_refusals_leave_the_store_as_it_was(make):
    s = make()
    with pytest.raises(RuntimeError, match="score before prefill"):
        s.score([1, 2])
    s.ids = list(range(5000))  # as after a truncate: no pending token, no held logits
    with pytest.raises(RuntimeError, match="a turn starts with prefill or append; after a generate or a truncate, call append"):
        s.score([1, 2])
    s.pending = 7              # as after a generate
    with pytest.raises(ValueError, match="at least one id"):
        s.score([])
    with pytest.raises(ValueError, match=r"\[0, 96\)"):
        s.score([3, 96])
    # 5000 committed + the pending token + n ids must fit the 8192 slots: 3193 ids do not
    with pytest.raises(ValueError, match="appending 3194 tokens after 5000 exceeds the 8192 slots"):
        s.score([1] * 3193)
    s = make(slots=1 << 20, positions=6000)
    s.ids, s.pending = list(range(5000)), 7
    with pytest.raises(ValueError, match="appending 1001 tokens after 5000 reaches past the model's 6000 RoPE positions"):
        s.score([1] * 1000)
    assert s.length == 5000 and s.pending == 7 and s.ids == list(range(5000))


def _cpu_logprobs(logits, ids, lp, am, check_ids=True):
    x = logits.double()
    lp.copy_((x.gather(1, ids.long()[:, None])[:, 0] - torch.logsumexp(x, 1)).float())
    am.copy_(torch.argmax(logits, 1).to(torch.int32))


@pytest.mark.parametrize("pending", [None, 11], ids=["held_logits", "pending"])
def test_score_forwards_the_rows_it_scores_and_rolls_back(monkeypatch, pending):
    """What score forwards (the pending token first), where each id's score comes from, and the rollback of the host length."""
    s = _chain()
    s.ids, s.pending = list(range(5000)), pending
    held = torch.randn(1, 1, V)
    s._logits = None if pending is not None else held
    calls = []

    def fake_extend(ids, logprobs):
        calls.append(ids.tolist()[0])
        s._kv.seq_len += ids.numel()
        lp, am = logprobs
        lp.copy_(-torch.arange(1, lp.numel() + 1, dtype=torch.float32))
        am.copy_(ids[0, 1:].to(torch.int32))  # "greedy" on every forwarded row

    monkeypatch.setattr(s, "_score_extend", fake_extend)
    monkeypatch.setattr(session.ops, "token_logprobs", _cpu_logprobs)
    sc = s.score([4, 5, 6])
    assert s.length == 5000 and s.pending == pending and s.ids == list(range(5000))
    if pending is None:
        assert calls == [[4, 5, 6]] and s._logits is held
        want0 = (held[0, -1].double() - torch.logsumexp(held[0, -1].double(), 0))[4].float()
        assert sc.logprobs[0] == want0 and sc.argmax[0] == int(torch.argmax(held[0, -1]))
        assert sc.logprobs[1:].tolist() == [-1.0, -2.0] and sc.greedy[1:].tolist() == [True, True]
    else:
        assert calls == [[11, 4, 5, 6]]
        assert sc.logprobs.tolist() == [-1.0, -2.0, -3.0] and sc.greedy.all()
    assert sc.logprobs.dtype == torch.float32 and sc.argmax.dtype == torch.int32 and sc.greedy.dtype == torch.bool
    # an extend that fails still leaves the length where it was
    s._logits = held

    def failing(ids, logprobs):
        s._kv.seq_len += 3
        raise RuntimeError("boom")

    monkeypatch.setattr(s, "_score_extend", failing)
    with pytest.raises(RuntimeError, match="boom"):
        s.score([1, 2])
    assert s.length == 5000


def test_prefill_refuses_a_mis_shaped_logprobs_pair():
    model = object.__new__(LlamaModel)
    model.device, model.config = torch.device("cpu"), SimpleNamespace(vocab_size=V)
    ids = torch.arange(10)
    for pair in ((torch.empty(10), torch.empty(9, dtype=torch.int32)), (torch.empty(9, dtype=torch.float64), torch.empty(9, dtype=torch.int32)),
                 (torch.empty(9), torch.empty(9, dtype=torch.int64))):
        with pytest.raises(ValueError, match=r"float32 \[9\], int32 \[9\]"):
            model._score_targets(ids, pair)
    with pytest.raises(ValueError, match=r"\[0, 96\)"):
        model._score_targets(torch.tensor([0, 5, 96]), (torch.empty(2), torch.empty(2, dtype=torch.int32)))
    assert model._score_targets(ids, None) is None
    assert model._score_targets(ids, (torch.empty(9), torch.empty(9, dtype=torch.int32))).tolist() == list(range(1, 10))


def test_perplexity_arguments_and_dry_run(tmp_path, capsys):
    with pytest.raises(SystemExit):
        perplexity.parse_args(["--legs", "fp16,fp8"])
    with pytest.raises(SystemExit):
        perplexity.parse_args(["--tokens", "1"])
    a = perplexity.parse_args(["--legs", "fp16,both", "--layers", "2"])
    assert a.legs == ["fp16", "both"] and a.tokens == 124928 and a.chunk == 128
    cfg = perplexity.model_config(a)
    assert cfg.num_hidden_layers == 2 and cfg.vocab_size == 32000
    ids = perplexity.load_ids(a, cfg.vocab_size)
    assert ids.shape == (124928,) and ids.min() >= 0 and ids.max() < 32000
    assert np.array_equal(ids, perplexity.load_ids(a, cfg.vocab_size))  # the seed fixes the document
    arith = perplexity.shape_arithmetic(124928, cfg, 128)
    assert arith["pieces"] == 976 and arith["last_piece_rows"] == 128 and arith["scored_positions"] == 124927
    assert arith["logits_read_gb"] == round(124927 * 32000 * 4 / 1e9, 3)                  # ~16 GB of fp32 logits
    assert arith["layer_major_head_tflop"] == round(2 * 124800 * 4096 * 32000 / 1e12, 3)  # ~33 TFLOP
    assert perplexity.shape_arithmetic(1000, cfg, 128)["last_piece_rows"] == 104
    f = tmp_path / "doc.npy"
    np.save(f, np.array([[1, 2, 3]]))
    b = perplexity.parse_args(["--ids", str(f)])
    assert perplexity.load_ids(b, 32000).tolist() == [1, 2, 3]
    np.save(f, np.array([1, 32000]))
    with pytest.raises(SystemExit, match=r"\[0, 32000\)"):
        perplexity.load_ids(b, 32000)
    assert perplexity.main(["--dry-run", "--tokens", "1000", "--out", str(tmp_path / "o")]) == 0
    out = capsys.readouterr().out
    assert '"dry_run": true' in out and '"pieces": 8' in out
    assert not (tmp_path / "o").exists()  # a dry run writes nothing
