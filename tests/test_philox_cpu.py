"""The CPU restatement of the device Philox stream (tests/philox_oracle.py): Random123's known answers, and the word -> uniform
map over all 2^24 inputs, before and after mapping the round-to-even 1.0 inside (0, 1)."""
import numpy as np
import pytest

import philox_oracle as px


@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0), (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
])
def test_philox4x32_10_known_answers(ctr, key, want):
    assert tuple(int(v) for v in px.philox4x32_10(*ctr, *key)) == want
    # vectorised: the same answer in every position of a broadcast batch
    got = px.philox4x32_10(*(np.full(3, c, dtype=np.uint64) for c in ctr), *key)
    assert all((g == w).all() for g, w in zip(got, want))


def test_element_layout():
    """Element i of a draw is lane i % 4 of counter (i / 4, draw_lo, draw_hi, 0) under key (seed_lo, seed_hi)."""
    seed, draw = 0x0123456789ABCDEF, (7 << 32) | 5
    w = px.words(seed, draw, 11)
    for i in range(11):
        r = px.philox4x32_10(i // 4, draw & 0xFFFFFFFF, draw >> 32, 0, seed & 0xFFFFFFFF, seed >> 32)
        assert int(w[i]) == int(r[i % 4])
    assert (px.words(seed, [draw, draw + 1], 11)[0] == w).all()


def test_uniform_map_over_all_24_bit_words():
    x = np.arange(1 << 24, dtype=np.uint32) << np.uint32(8)
    cur = px.uniform_current(x)
    fixed = px.uniform(x)
    # the current map rounds exactly one word, 0xFFFFFF, onto 1.0
    assert np.flatnonzero(cur >= np.float32(1)).tolist() == [px.UNIT]
    assert (cur > 0).all()
    # the fixed map stays strictly inside (0, 1), and differs from the current one on that word only, bit for bit
    assert (fixed > 0).all() and (fixed < 1).all()
    same = fixed.view(np.uint32) == cur.view(np.uint32)
    assert np.flatnonzero(~same).tolist() == [px.UNIT]
    assert fixed[px.UNIT].view(np.uint32) == 0x3F7FFFFF
    # 1 - 2^-24 is new: the round-to-even sum never produces it, so no other stream value collides with it
    assert not (cur.view(np.uint32) == 0x3F7FFFFF).any()
    with np.errstate(divide="raise", invalid="raise"):
        e = -np.log(fixed)
    assert e.dtype == np.float32 and np.isfinite(e).all() and (e > 0).all()
    # the low 8 bits of the word never matter
    assert (px.uniform(x | np.uint32(0xFF)).view(np.uint32) == fixed.view(np.uint32)).all()


def test_unit_draws_of_seed_0():
    hits = px.unit_draws(0, 32000, 1300)
    assert (1229, 2648) in hits
    assert hits == [(1229, 2648)]
    assert int(px.words(0, 1229, 32000)[2648]) == 0xFFFFFF7A
    assert px.uniform_current(px.words(0, 1229, 2649))[2648] == 1.0
    # an explicit list of draws scans those draws only
    assert px.unit_draws(0, 32000, [1228, 1229, 1230]) == [(1229, 2648)]
    assert px.unit_draws(0, 2648, [1229]) == []
