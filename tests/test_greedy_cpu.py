"""Greedy decoding (temperature 0) on the host side: the `--temp` flag of the three entry points, and the T = 0 growth of the
Sequoia tree (the top-k draft tokens of each parent, ties to the lower index)."""
import math

import pytest
import torch

from triforce_b200.cli import build_parser
from triforce_b200.spectree import build_sampling, create_sampling_callable, load_grow_map

ENTRIES = ("on_chip", "offloading_TP", "offloading_seqouia")
E4M3_FLAGS = {"on_chip": ["--kv_dtype", "e4m3", "--weight_dtype", "e4m3", "--retrieval_dtype", "e4m3"],
              "offloading_TP": ["--retrieval_dtype", "e4m3"], "offloading_seqouia": []}


@pytest.mark.parametrize("entry", ENTRIES)
def test_temp_zero_is_accepted(entry):
    p = build_parser(entry)
    assert p.parse_args(["--temp", "0"]).temp == 0.0
    assert p.parse_args(["--temp", "0.0"] + E4M3_FLAGS[entry]).temp == 0.0
    assert p.parse_args([]).temp == 0.6  # the default is unchanged
    assert p.parse_args(["--temp", "1.3"]).temp == 1.3


@pytest.mark.parametrize("entry", ENTRIES)
@pytest.mark.parametrize("bad", ["-0.1", "-1", "nan", "abc"])
def test_negative_temp_is_an_argparse_error(entry, bad, capsys):
    with pytest.raises(SystemExit) as e:
        build_parser(entry).parse_args([f"--temp={bad}"])
    assert e.value.code == 2
    assert "--temp" in capsys.readouterr().err


def test_greedy_growth_takes_top_k_with_ties_to_the_lower_index():
    f = create_sampling_callable(3, temperature=0.0)
    neg = -math.inf
    logits = torch.tensor([
        [0.0, 5.0, 1.0, 5.0, 2.0, 5.0, 5.0, 0.0],        # a four-way tie at the top: the three lowest indices
        [1.0, 2.0, 3.0, 4.0, 5.0, 6.0, 7.0, 8.0],        # strictly increasing: the last three, largest first
        [neg, neg, neg, 0.5, neg, neg, neg, neg],        # one finite value, then -inf ties in index order
        [3.0, 3.0, 3.0, 3.0, 3.0, 3.0, 3.0, 3.0],        # all tied
        [1.0, math.inf, 2.0, 2.0, -1.0, math.inf, 0.0, 2.0],  # +inf first, then the tie at 2
        [1.0, 2.0, math.nan, 0.0, 7.0, 0.0, 0.0, 0.0],   # NaN counts as maximal (torch.argmax's rule)
    ], dtype=torch.float32)
    rand = torch.full((logits.shape[0], logits.shape[1]), 0.5, dtype=torch.float16)
    got = f(logits, rand).view(-1, 3).tolist()
    assert got == [[1, 3, 5], [7, 6, 5], [3, 0, 1], [0, 1, 2], [1, 5, 2], [2, 4, 1]]
    # the first child is torch.argmax of the row
    assert [g[0] for g in got] == torch.argmax(logits, dim=-1).tolist()
    # the noise is not read: any draw gives the same children
    assert f(logits, torch.rand(rand.shape).half()).view(-1, 3).tolist() == got


def test_greedy_growth_on_random_rows_is_the_stable_top_k():
    g = torch.Generator().manual_seed(0)
    logits = torch.randint(-4, 5, (64, 1000), generator=g).float()  # many exact ties
    f = create_sampling_callable(7, temperature=0.0)
    got = f(logits, torch.empty(64, 1000, dtype=torch.float16)).view(64, 7)
    for r in range(64):
        row = logits[r].tolist()
        want = sorted(range(1000), key=lambda i: (-row[i], i))[:7]
        assert got[r].tolist() == want


def test_build_sampling_at_temperature_zero_covers_every_level():
    gm = load_grow_map("512")
    callables, gather = build_sampling(gm, 0.0, "cpu")
    assert len(callables) == len(gm["roots"]) - 1
    for i, f in callables.items():
        k = max(gm["branches"][i])
        rows = len(gm["roots"][i])
        logits = torch.arange(rows * 50, dtype=torch.float32).view(rows, 50)
        out = f(logits, None)
        assert out.shape == (rows * k,) and out.view(rows, k)[:, 0].tolist() == [49] * rows
