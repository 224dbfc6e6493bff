"""The sampling side of the whole-loop graph (csrc/loop_graph.cu) against plain restatements, not against the step-wise loop
that reads the same noise:

  * the Philox stream `tf_philox_fill` replays equals the CPU restatement bit for bit (tests/philox_oracle.py), and its
    exponentials are -log(u) within 2 float32 ulps;
  * at a word whose uniform used to round to 1.0 (found by calculation with `unit_draws`), no sampler returns a token of
    probability zero: before the fix the exponential there was -0.0, p / e was NaN for p = 0, and NaN wins the argmax;
  * `loop_draft_sample`, `loop_middle_accept` and `loop_verify` equal the oracle (or the step-wise kernels) fed the same draws,
    at V = 32 000, 32 768 and 32 003 (odd V: the scalar copy path of `tf_middle_accept`, a ragged last Philox group);
  * draft sample + verify, replayed 2*10^5 times in CUDA graphs, emit a first token distributed as the target's p (chi-square,
    and zero counts on p = 0), and the same counts reject q and a slightly perturbed p."""
import functools

import numpy as np
import pytest
import torch

import philox_oracle as px
from oracle import triforce_oracle as orc
from triforce_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda"
F32 = np.float32


def _i64(x: int) -> int:
    x &= 0xFFFFFFFFFFFFFFFF
    return x - (1 << 64) if x >= 1 << 63 else x


def _rng_state(seed: int, draw: int) -> torch.Tensor:
    return torch.tensor([_i64(seed), _i64(draw)], dtype=torch.int64, device=DEV)


def _fill(seed: int, draw: int, kind: int, n: int) -> np.ndarray:
    st = _rng_state(seed, draw)
    out = ops.philox_fill(st, kind, torch.empty(n, dtype=torch.float32, device=DEV))
    assert st.tolist() == [_i64(seed), _i64(draw + 1)]
    return out.cpu().numpy()


def _t(a) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _prob_rows(rng, rows, V, zero_frac=0.3):
    a = rng.random((rows, V), dtype=np.float32) ** 3
    a[rng.random((rows, V)) < zero_frac] = 0
    return (a / a.sum(-1, keepdims=True, dtype=np.float32)).astype(np.float32)


@functools.lru_cache(maxsize=None)
def _first_unit_draw():
    """(draw, element) of the first word of stream 0 with x >> 8 == 0xFFFFFF among 32 000 elements."""
    hits = px.unit_draws(0, 32000, 1300)
    assert hits, "no unit word in the scanned draws"
    return hits[0]


# ---------------------------------------------------------------------------------------------------------------------
# (a) the stream
# ---------------------------------------------------------------------------------------------------------------------
STREAMS = [(0, 0), (0, 1229), (1, 7), (0x9E3779B97F4A7C15, 3), (12345, (1 << 32) + 5), (0xFFFFFFFF00000001, (1 << 32) - 1),
           (0x00000001FFFFFFFF, (3 << 32) + 17)]


@pytest.mark.parametrize("n", [1, 4, 32000, 32003])
def test_philox_fill_equals_the_restatement(n):
    for seed, draw in STREAMS:
        u = _fill(seed, draw, 0, n)
        want = px.uniform(px.words(seed, draw, n))
        assert np.array_equal(u.view(np.uint32), want.view(np.uint32)), (seed, draw, np.flatnonzero(u != want)[:8])
        e = _fill(seed, draw, 1, n)
        ref = px.exponential(px.words(seed, draw, n))
        assert np.isfinite(e).all() and (e > 0).all(), (seed, draw, np.flatnonzero(~(e > 0))[:8])
        ulp = np.spacing(ref.astype(np.float32)).astype(np.float64)
        err = np.abs(e.astype(np.float64) - ref)
        assert (err <= 2 * ulp).all(), (seed, draw, float((err / ulp).max()))


def test_philox_fill_advances_one_draw_per_fill():
    seed, draw = 0xDEADBEEF12345678, (1 << 32) - 2
    st = _rng_state(seed, draw)
    buf = torch.empty(32003, dtype=torch.float32, device=DEV)
    for i in range(5):  # uniform, exponential, uniform, ... across the 2^32 boundary of the draw index
        ops.philox_fill(st, i % 2, buf)
        assert st.tolist() == [_i64(seed), _i64(draw + i + 1)]
        w = px.words(seed, draw + i, buf.numel())
        got = buf.cpu().numpy()
        if i % 2 == 0:
            assert np.array_equal(got.view(np.uint32), px.uniform(w).view(np.uint32))
        else:
            ref = px.exponential(w)
            assert (np.abs(got - ref) <= 2 * np.spacing(ref.astype(np.float32))).all()


def test_unit_words_in_the_filled_stream():
    """Seed 0, V = 32 000: the filled uniforms equal 1 - 2^-24 exactly where `unit_draws` says, and at about V / 2^24 per row."""
    V, D = 32000, 20000
    scanned = 1300
    one_minus = float(px.ONE_MINUS_ULP)
    st = _rng_state(0, 0)
    buf = torch.empty((D, V), dtype=torch.float32, device=DEV)
    for d in range(D):
        ops.philox_fill(st, 0, buf[d])
    assert (buf < 1).all() and (buf > 0).all()
    hits = torch.nonzero(buf == one_minus).tolist()
    del buf
    assert [tuple(h) for h in hits if h[0] < scanned] == px.unit_draws(0, V, scanned)
    expected = D * V / 2 ** 24
    print(f"\n[philox] seed 0, V {V}: {len(hits)} unit words in {D} draws, V / 2^24 expects {expected:.1f}")
    assert abs(len(hits) - expected) < 6 * expected ** 0.5


# ---------------------------------------------------------------------------------------------------------------------
# (b) the unit draw: a token of probability zero is never sampled
# ---------------------------------------------------------------------------------------------------------------------
def _row_without(rng, V, el):
    p = _prob_rows(rng, 1, V)[0]
    p[el] = 0
    return (p / p.sum(dtype=np.float32)).astype(np.float32)


def test_unit_draw_fill_stays_inside_the_interval():
    draw, el = _first_unit_draw()
    u = _fill(0, draw, 0, 32000)
    e = _fill(0, draw, 1, 32000)
    assert u[el] < 1 and u[el].view(np.uint32) == 0x3F7FFFFF
    assert e[el] > 0 and np.isfinite(e[el]) and not np.signbit(e[el])


def test_unit_draw_sample_argmax():
    draw, el = _first_unit_draw()
    V = 32000
    p = _row_without(np.random.Generator(np.random.PCG64(1)), V, el)
    e = _fill(0, draw, 1, V)
    got = int(ops.sample_argmax(_t(p), _t(e)).item())
    assert got != el and p[got] > 0
    assert got == orc.sample_from_noise(p, e)


def test_unit_draw_loop_draft_sample():
    draw, el = _first_unit_draw()
    V, gamma, n = 32000, 4, 2
    rng = np.random.Generator(np.random.PCG64(2))
    dp = _prob_rows(rng, gamma, V)
    dp[n] = _row_without(rng, V, el)
    st = torch.tensor([n, 0, 0, 0, 0, 0, 0, 0], dtype=torch.int32, device=DEV)
    vt = torch.full((gamma + 1,), 100, dtype=torch.int64, device=DEV)
    ops.loop_draft_sample(_t(dp), st, _rng_state(0, draw), vt)
    got = int(vt[n + 1].item())
    assert got != el and dp[n, got] > 0
    assert got == orc.sample_from_noise(dp[n], _fill(0, draw, 1, V))


def test_unit_draw_loop_middle_accept_replacement():
    draw, el = _first_unit_draw()
    V, gamma, n, k = 32000, 4, 1, 1
    rng = np.random.Generator(np.random.PCG64(3))
    dp = _prob_rows(rng, gamma, V)
    vp = _prob_rows(rng, gamma + 1, V)
    vp[n] = _row_without(rng, V, el)
    tok = int(np.flatnonzero(dp[n])[0])
    vp[n, tok] = 0  # certain reject: the replacement is drawn from vp[n] at the unit draw (the uniform comes first)
    vt = torch.full((gamma + 1,), 100, dtype=torch.int64, device=DEV)
    vt[n + 1] = tok
    st = torch.tensor([n, k, 0, 0, 0, 0, 0, 0], dtype=torch.int32, device=DEV)
    out_ids = torch.full((gamma + 2,), -1, dtype=torch.int64, device=DEV)
    spec = torch.zeros((gamma + 2, V), dtype=torch.float32, device=DEV)
    ops.loop_middle_accept(_t(dp), _t(vp), vt, _rng_state(0, draw - 1), gamma, st, out_ids, spec)
    assert st.tolist()[:3] == [n + 1, k + 1, 0]
    got = int(out_ids[k].item())
    assert got != el and vp[n, got] > 0
    assert got == orc.sample_from_noise(vp[n], _fill(0, draw, 1, V))


def _verify(p, q, gen, seed, draw, strict_less=True, eos=-1, st_extra=(0, 0), first=1234, seq_len=500, pass_extra=1):
    """Runs loop_verify on fresh buffers; returns (res[:10], tokens[:res[0]], pass_tokens, first_token, seq_len, rng ctr)."""
    g2 = len(gen)
    st = torch.tensor([g2, g2, 0, st_extra[0], st_extra[1], 0, 0, 0], dtype=torch.int32, device=DEV)
    rng = _rng_state(seed, draw)
    ft = torch.tensor([first], dtype=torch.int64, device=DEV)
    res = torch.full((16,), -7, dtype=torch.int32, device=DEV)
    tokens = torch.full((g2 + 3,), -1, dtype=torch.int64, device=DEV)
    pt = torch.full((g2 + 2 + pass_extra,), -1, dtype=torch.int64, device=DEV)
    sl = torch.tensor([seq_len], dtype=torch.int32, device=DEV)
    ops.loop_verify(_t(p), _t(q), _t(np.asarray(gen, dtype=np.int64)), st, rng, strict_less, eos, ft, res, tokens, pt, sl)
    r = res.tolist()
    assert r[10:] == [-7] * 6
    return r[:10], tokens.tolist()[:r[0]], pt.tolist(), int(ft.item()), int(sl.item()), rng.tolist()[1]


def test_unit_draw_loop_verify_residual_and_bonus():
    draw, el = _first_unit_draw()
    V, g2 = 32000, 3
    rng = np.random.Generator(np.random.PCG64(4))
    q = _prob_rows(rng, g2 + 1, V)
    gen = [int(np.flatnonzero(q[i])[i]) for i in range(g2)]
    # residual: reject at 1; max(p - q, 0) is zero at `el` (p = q there), the rest of the mass elsewhere
    p = _prob_rows(rng, g2 + 1, V)
    p[0, gen[0]] = q[0, gen[0]] * 2
    p[1, gen[1]] = 0
    p[1, el] = q[1, el]
    r, toks, *_ = _verify(p, q, gen, 0, draw - 1)
    assert r[:3] == [2, 1, 1]
    res_row = orc.max_fn(p[1] - q[1])
    assert res_row[el] == 0
    assert toks[-1] != el and res_row[toks[-1]] > 0
    assert toks[-1] == orc.sample_from_noise(res_row, _fill(0, draw, 1, V))
    # bonus: every draft token accepted, p[g2] has no mass at `el`
    p = _prob_rows(rng, g2 + 1, V)
    for i in range(g2):
        p[i, gen[i]] = q[i, gen[i]] * 2
    p[g2] = _row_without(rng, V, el)
    r, toks, *_ = _verify(p, q, gen, 0, draw - 1)
    assert r[:3] == [g2 + 1, g2, 0]
    assert toks[-1] != el and p[g2, toks[-1]] > 0
    assert toks[-1] == orc.sample_from_noise(p[g2], _fill(0, draw, 1, V))


# ---------------------------------------------------------------------------------------------------------------------
# (c) the loop kernels against the oracle
# ---------------------------------------------------------------------------------------------------------------------
VOCABS = [32000, 32768, 32003]


@pytest.mark.parametrize("V", VOCABS)
def test_loop_draft_sample_matches_oracle(V):
    rng = np.random.Generator(np.random.PCG64(V))
    gamma = 4
    for trial in range(12):
        seed, draw = int(rng.integers(0, 1 << 63)), int(rng.integers(0, 1 << 40))
        n = int(rng.integers(0, gamma))
        dp = _prob_rows(rng, gamma, V, zero_frac=0.3 + 0.05 * trial)
        st = torch.tensor([n, 0, 0, 0, 0, 0, 0, 0], dtype=torch.int32, device=DEV)
        vt = torch.full((gamma + 1,), 100, dtype=torch.int64, device=DEV)
        state = _rng_state(seed, draw)
        ops.loop_draft_sample(_t(dp), st, state, vt)
        assert state.tolist() == [_i64(seed), _i64(draw + 1)]
        want = [100] * (gamma + 1)
        want[n + 1] = orc.sample_from_noise(dp[n], _fill(seed, draw, 1, V))
        assert vt.tolist() == want


@pytest.mark.parametrize("V", VOCABS)
def test_loop_middle_accept_matches_tf_middle_accept(V):
    """The device-loop decision against the step-wise kernel fed the same draws (uniform: element 0 of draw c; sample: draw
    c + 1): state, emitted ids, verify_tokens and proposal rows bit-identical."""
    rng = np.random.Generator(np.random.PCG64(V + 1))
    gamma = 4
    seen = set()
    for trial in range(40):
        seed, draw = int(rng.integers(0, 1 << 63)), int(rng.integers(0, 1 << 40))
        case = trial % 5
        n = gamma - 1 if case == 2 else int(rng.integers(0, gamma))
        k = int(rng.integers(0, 3))
        dp = _prob_rows(rng, gamma, V)
        vp = _prob_rows(rng, gamma + 1, V)
        vt = rng.integers(0, V, gamma + 1).astype(np.int64)
        tok = int(rng.choice(np.flatnonzero(dp[n])))
        vt[n + 1] = tok
        if case == 0:  # certain reject
            vp[n, tok] = 0
        elif case == 1:  # 0 / 0: NaN ratio rejects
            dp[n, tok] = 0
            vp[n, tok] = 0
        elif case == 2:  # accepted at n = gamma - 1: nn = gamma + 1 skips the verify_tokens write
            vp[n, tok] = max(vp[n, tok], dp[n, tok])
        elif case == 3:  # likely accept
            vp[n, tok] = max(vp[n, tok], dp[n, tok] * F32(0.9))
        st0 = [n, k, 0, int(rng.integers(0, 9)), int(rng.integers(0, 9)), 5, 6, 7]
        bufs = []
        for _ in range(2):
            bufs.append(dict(st=torch.tensor(st0, dtype=torch.int32, device=DEV), vt=_t(vt.copy()),
                             ids=torch.full((gamma + 2,), -1, dtype=torch.int64, device=DEV),
                             spec=torch.full((gamma + 2, V), -1.0, dtype=torch.float32, device=DEV)))
        a, b = bufs
        state = _rng_state(seed, draw)
        ops.loop_middle_accept(_t(dp), _t(vp), a["vt"], state, gamma, a["st"], a["ids"], a["spec"])
        assert state.tolist() == [_i64(seed), _i64(draw + 2)]
        u = _t(_fill(seed, draw, 0, 1))
        e = _t(_fill(seed, draw + 1, 1, V))
        ops.middle_accept(_t(dp[n]), _t(vp), b["vt"], u, e, gamma, b["st"], b["ids"], b["spec"])
        for key in ("st", "vt", "ids"):
            assert a[key].tolist() == b[key].tolist(), (trial, key)
        assert torch.equal(a["spec"].view(torch.int32), b["spec"].view(torch.int32)), trial
        accepted = a["st"].tolist()[2] == 1
        seen.add((case, accepted))
        if case in (0, 1):
            assert not accepted
        if case == 2:
            assert accepted and a["vt"].tolist() == vt.tolist()  # nothing written past gamma
    assert {(0, False), (1, False), (2, True), (3, True)} <= seen


def _verify_oracle(p, q, gen, seed, draw, strict_less, eos, st_extra, first, seq_len, pass_len):
    """decoding.py:97-139 as loop_verify computes it: uniforms of draw c (element i for draft token i), one exponential draw
    c + 1 when a token is drawn (after a reject, or after the last draft token was accepted)."""
    g2, V = len(gen), p.shape[-1]
    u = px.uniform(px.words(seed, draw, g2))
    count, rejected, examined, hit = 0, False, 0, False
    for i in range(g2):
        examined += 1
        _, rj = orc.accept_walk([gen[i]], [q[i]], p[i:i + 1], [u[i]], strict_less=strict_less)
        if rj:
            rejected = True
            break
        count += 1
        if gen[i] == eos:
            hit = True
            break
    draws = rejected or count == g2
    toks = [int(t) for t in gen[:count]]
    passed = [first] + [100] * (pass_len - 1)
    passed[1:count + 1] = toks
    if draws:
        e = _fill(seed, draw + 1, 1, V)
        tok = orc.sample_from_noise(orc.max_fn(p[count] - q[count]) if rejected else p[g2], e)
        toks.append(tok)
        passed[count + 1] = tok
        nxt = tok
    else:
        nxt = int(gen[count - 1])
    shift = count + (1 if not rejected and count == g2 else 0)
    res = [len(toks), count, int(rejected), g2, examined, int(hit), st_extra[1], st_extra[0], shift, seq_len + count + 1]
    return res, toks, passed, nxt, seq_len + count + 1, draw + (2 if draws else 1)


@pytest.mark.parametrize("V", VOCABS)
def test_loop_verify_matches_oracle(V):
    rng = np.random.Generator(np.random.PCG64(V + 2))
    seen = set()
    for trial in range(36):
        seed, draw = int(rng.integers(0, 1 << 63)), int(rng.integers(0, 1 << 40))
        case = trial % 6
        g2 = int(rng.integers(2 if case in (1, 3, 4) else 1, 7))
        strict = trial % 12 < 6
        p = _prob_rows(rng, g2 + 1, V)
        q = _prob_rows(rng, g2 + 1, V)
        gen = np.array([int(rng.choice(np.flatnonzero(q[i]))) for i in range(g2)], dtype=np.int64)
        u = px.uniform(px.words(seed, draw, g2))
        eos = -1
        if case == 3:  # an accepted EOS before the last draft token stops the walk without a draw
            j = g2 // 2 - 1
            eos = int(gen[j])
            gen = np.where((gen == eos) & (np.arange(g2) != j), (eos + 1) % V, gen)
        accept_to = {0: 0, 1: g2 // 2, 2: g2, 3: g2, 4: g2 - 1}.get(case, int(rng.integers(0, g2 + 1)))
        for i in range(min(accept_to, g2)):
            p[i, gen[i]] = max(p[i, gen[i]], q[i, gen[i]])  # ratio >= 1: accepted
        if case in (0, 1):  # reject at 0 / mid-way
            p[accept_to, gen[accept_to]] = 0
        elif case == 4:  # ratio == u exactly at the last token: strict_less rejects, `<=` accepts
            j = g2 - 1
            q[j, gen[j]] = F32(0.5)
            p[j, gen[j]] = u[j] * F32(0.5)
        extra = (int(rng.integers(0, 9)), int(rng.integers(0, 9)))
        first, seq_len = int(rng.integers(0, V)), int(rng.integers(100, 100000))
        got = _verify(p, q, gen, seed, draw, strict, eos, extra, first, seq_len, pass_extra=1)
        want = _verify_oracle(p, q, gen, seed, draw, strict, eos, extra, first, seq_len, g2 + 3)
        names = ("res", "tokens", "pass_tokens", "first_token", "seq_len_dev", "philox draw")
        for name, g, w in zip(names, got, want):
            assert g == w, (trial, case, name, g, w)
        res = got[0]
        seen.add((case, strict, res[1], res[2], res[5]))
        if case == 0:
            assert res[1:3] == [0, 1]
        elif case == 2:
            assert res[:3] == [g2 + 1, g2, 0] and res[8] == g2 + 1
        elif case == 3:
            assert res[5] == 1 and res[1] == g2 // 2 and got[5] == draw + 1
        elif case == 4:
            assert res[2] == (1 if strict else 0)
    assert any(s[0] == 1 and 0 < s[2] for s in seen)  # a mid-way reject happened


# ---------------------------------------------------------------------------------------------------------------------
# (d) speculative sampling is lossless
# ---------------------------------------------------------------------------------------------------------------------
Z_1E6 = 4.753424308822899  # standard normal quantile at 1 - 10^-6


def _chi2_threshold(df: int) -> float:
    """Upper 10^-6 quantile of chi-square(df), Wilson-Hilferty."""
    a = 2.0 / (9.0 * df)
    return df * (1.0 - a + Z_1E6 * np.sqrt(a)) ** 3


def _chi2(counts: np.ndarray, probs: np.ndarray):
    """Pearson statistic over the bins with probs > 0, pooled in ascending expected count to >= 5 each; returns (stat, df)."""
    N = counts.sum()
    pos = np.flatnonzero(probs > 0)
    exp = N * probs[pos].astype(np.float64)
    cnt = counts[pos].astype(np.float64)
    order = np.argsort(exp, kind="stable")
    ce, cc = np.cumsum(exp[order]), np.cumsum(cnt[order])
    cut, last = [], 0.0
    for i, v in enumerate(ce):
        if v - last >= 5:
            cut.append(i)
            last = v
    if cut[-1] != len(ce) - 1:
        cut[-1] = len(ce) - 1  # fold an under-filled tail into the last bin
    be = np.diff(np.concatenate([[0.0], ce[cut]]))
    bc = np.diff(np.concatenate([[0.0], cc[cut]]))
    return float(((bc - be) ** 2 / be).sum()), len(be) - 1


def _rows(V: int):
    rng = np.random.Generator(np.random.PCG64(V))
    if V == 1000:
        p = np.exp(2 * rng.standard_normal(V))
        q = np.exp(2 * rng.standard_normal(V))
        p[rng.random(V) < 0.2] = 0
        q[rng.random(V) < 0.2] = 0
    else:  # peaked p; q's support overlaps p's in part only
        p = np.zeros(V)
        q = np.zeros(V)
        sp = rng.permutation(V)[:V // 2]
        sq = np.concatenate([sp[:V // 4], rng.permutation(np.setdiff1d(np.arange(V), sp))[:V // 4]])
        p[sp] = np.exp(3 * rng.standard_normal(sp.size))
        q[sq] = np.exp(2 * rng.standard_normal(sq.size))
    p = (p / p.sum()).astype(np.float32)
    q = (q / q.sum()).astype(np.float32)
    assert ((p > 0) & (q == 0)).any() and ((q > 0) & (p == 0)).any()
    return p, q


def _first_token_counts(p, q, g2, trials, seed=2024, per_graph=100):
    """Counts of the first emitted token over `trials` runs of: g2 draft samples from q (loop_draft_sample), loop_verify
    against p on every row; one CUDA graph holds `per_graph` runs and is replayed on the advancing Philox stream."""
    V = p.size
    P = _t(np.tile(p, (g2 + 1, 1)))
    Q = _t(np.tile(q, (g2 + 1, 1)))
    rng = _rng_state(seed, 0)
    st_draft = [torch.tensor([i, 0, 0, 0, 0, 0, 0, 0], dtype=torch.int32, device=DEV) for i in range(g2)]
    st_ver = torch.tensor([0, g2, 0, 0, 0, 0, 0, 0], dtype=torch.int32, device=DEV)
    vt = torch.zeros(g2 + 1, dtype=torch.int64, device=DEV)
    out_ids = torch.zeros(g2, dtype=torch.int64, device=DEV)
    ft = torch.zeros(1, dtype=torch.int64, device=DEV)
    res = torch.zeros(16, dtype=torch.int32, device=DEV)
    tokens = torch.zeros(g2 + 3, dtype=torch.int64, device=DEV)
    pt = torch.zeros(g2 + 2, dtype=torch.int64, device=DEV)
    sl = torch.zeros(1, dtype=torch.int32, device=DEV)
    counts = torch.zeros(V, dtype=torch.int64, device=DEV)
    one = torch.ones(1, dtype=torch.int64, device=DEV)

    def run():
        for s in st_draft:
            ops.loop_draft_sample(Q, s, rng, vt)
        out_ids.copy_(vt[1:])
        ops.loop_verify(P, Q, out_ids, st_ver, rng, True, -1, ft, res, tokens, pt, sl)
        counts.index_add_(0, tokens[:1], one)

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        run()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(per_graph):
            run()
    counts.zero_()
    sl.zero_()
    rng.copy_(_rng_state(seed, 0))
    for _ in range(trials // per_graph):
        g.replay()
    torch.cuda.synchronize()
    # g2 draft draws, then the verify's uniforms and its exponential (without an EOS every run draws a token)
    assert rng.tolist() == [seed, trials * (g2 + 2)]
    return counts.cpu().numpy()


@pytest.mark.parametrize("V", [1000, 32000])
@pytest.mark.parametrize("g2", [1, 4])
def test_speculative_sampling_is_lossless(V, g2):
    p, q = _rows(V)
    N = 200_000
    counts = _first_token_counts(p, q, g2, N)
    assert counts.sum() == N
    assert counts[p == 0].sum() == 0, np.flatnonzero((p == 0) & (counts > 0))[:10]
    stat, df = _chi2(counts, p)
    thr = _chi2_threshold(df)
    stat_q, df_q = _chi2(counts, q)
    a, b = np.argsort(-p, kind="stable")[:2]
    p2 = p.astype(np.float64)
    p2[a] -= 0.02
    p2[b] += 0.02
    stat_2, df_2 = _chi2(counts, p2)
    print(f"\n[lossless] V {V} g2 {g2}: chi2 vs p {stat:.1f} (df {df}, 1e-6 threshold {thr:.1f}); vs q {stat_q:.1f} "
          f"(threshold {_chi2_threshold(df_q):.1f}); vs p with 2% moved {stat_2:.1f} (threshold {_chi2_threshold(df_2):.1f})")
    assert stat < thr
    assert stat_q > _chi2_threshold(df_q)
    assert stat_2 > _chi2_threshold(df_2)
