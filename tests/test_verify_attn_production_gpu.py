"""tf_verify_attn, the full-KV verify attention, at the shapes the models run it: the cfg2 verify and decode over ~125K
keys, tensor-parallel shards of 4 and 16 heads, the 16-row and 18-row edges of its two row-tile instances, short stores,
the head-sharded retrieval verify, d = 64, a captured graph that follows the device-side length, and a split table.

The kernel lays the (head, 64-key tile) units of all heads on one axis and cuts it into G contiguous ranges, one per CTA
(stream-K), so a CTA routinely ends one head and starts the next.  Every (CTA, head) segment publishes a partial (m, l, O)
to workspace slot CTA + head, and the last CTA to deliver a partial of a head merges that head's partials, in two
independent streams when there are more than 16 of them and R <= 8.  `Plan` restates that split; each test confirms it
against the kernel through the partial slots one launch writes, plants needles (attn_needles) at the first and last key
of every segment and at every fresh key, and compares every head with an fp64 reference.  Each test also checks that its
comparison rejects mutated references: each partial of head 0 and of a head entered by a straddling CTA dropped, a partial
counted twice, the fresh keys dropped, the diagonal moved by one either way, one key too many, and a straddling CTA's
second segment starting on the previous head's K/V.  The negative controls launch no library kernel."""
import math
import os

import numpy as np
import pytest
import torch

from attn_needles import (DEV, Needles, assert_rejected, base_logit, excess, plant_stale, reference,
                          report_time_and_memory, visibility)  # noqa: F401  (report_time_and_memory: autouse fixture)
from oracle import triforce_oracle as orc
from triforce_b200 import ops

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif("TF_ATTN_MIN_TILES" in os.environ, reason="TF_ATTN_MIN_TILES changes the split plan restated here")]
BN = ops.VERIFY_BOX_KEYS        # keys per tile
MAX_ROWS = ops.VERIFY_MAX_ROWS  # rows per partial slot
SPLIT_HDR = 4                   # header words of a split table: {G it was calibrated for, 0, 0, 0}


def cdiv(a: int, b: int) -> int:
    return -(-a // b)


def round_up(x: int, a: int) -> int:
    return cdiv(x, a) * a


def sm_count() -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---------------------------------------------------------------------------------------------------------------------
# the split plan and the workspace layout of verify_attn.cu, restated
# ---------------------------------------------------------------------------------------------------------------------
def grid_size(R: int, H: int, d: int, kv_len_max: int, sms: int) -> int:
    """attn_plan: one wave of resident CTAs (2 per SM; 1 per SM for the 6-stage d = 128, R > 16 instance), but no more
    than the longest input has tiles / min_tiles; head-sharded retrieval-sized stores keep >= 8 tiles per CTA."""
    G = sms if d == 128 and R > 16 else 2 * sms
    min_tiles = 8 if H <= 8 and 2048 <= kv_len_max < 16384 else 1
    return max(1, min(G, H * cdiv(kv_len_max, BN) // min_tiles))


class Plan:
    """The split of one launch.  CTA b streams the units [starts[b], starts[b + 1]) of the H · tph (head, tile) axis, with
    G = min(grid, total) recomputed from the actual kv_len.  The starts are equal (b · total / G), or, when the split
    table's header equals G = grid and total >= 4 G, the table's 32-bit fractions of total."""

    def __init__(self, R, H, d, kv_len, kv_len_max, sms, table=None):
        self.R, self.H, self.d, self.kv_len = R, H, d, kv_len
        self.grid = grid_size(R, H, d, kv_len_max, sms)
        self.tph = cdiv(kv_len, BN)
        self.total = H * self.tph
        self.G = min(self.grid, self.total)
        self.uses_table = (table is not None and self.G == self.grid and self.total >= 4 * self.G
                           and int(table[0]) == self.G)
        if self.uses_table:
            self.starts = [(int(t) * self.total) >> 32 for t in table[SPLIT_HDR:SPLIT_HDR + self.G]] + [self.total]
        else:
            self.starts = [b * self.total // self.G for b in range(self.G + 1)]
        self.segments = []  # (CTA, head, first key, end key), in CTA order
        for b in range(self.G):
            gt, end = self.starts[b], self.starts[b + 1]
            while gt < end:
                h, t0 = divmod(gt, self.tph)
                t1 = min(self.tph, t0 + end - gt)
                self.segments.append((b, h, t0 * BN, min(t1 * BN, kv_len)))
                gt += t1 - t0

    def partials(self, h: int):
        """(CTA, first key, end key) of head h's partials, in merge order."""
        return [(b, lo, hi) for b, hh, lo, hi in self.segments if hh == h]

    def n_partials(self):
        return [len(self.partials(h)) for h in range(self.H)]

    def straddling(self):
        """CTAs that deliver partials of more than one head."""
        per_cta = {}
        for b, _, _, _ in self.segments:
            per_cta[b] = per_cta.get(b, 0) + 1
        return sorted(b for b, n in per_cta.items() if n > 1)

    def entered_heads(self):
        """Heads whose first partial is the second (or later) segment of a CTA that began in an earlier head."""
        return [h for h in range(1, self.H) if self.partials(h)[0][0] == self.partials(h - 1)[-1][0]]

    def cta_of(self, h: int, key: int) -> int:
        return next(b for b, lo, hi in self.partials(h) if lo <= key < hi)

    def dual_stream(self) -> bool:
        """Does some head's merge run two partial streams (d = 128, R <= 8, more than 16 partials)?"""
        return self.d == 128 and self.R <= 8 and max(self.n_partials()) > 16

    def summary(self) -> str:
        P = self.n_partials()
        return (f"G={self.G} (grid {self.grid}, {self.total} tiles), partials per head {min(P)}..{max(P)}"
                f"{' (two-stream merge)' if self.dual_stream() else ''}, {len(self.straddling())} straddling CTAs"
                f"{', split table' if self.uses_table else ''}")


def workspace_layout(H: int, d: int, sms: int) -> dict:
    """Byte offsets in the workspace from its 256-byte-aligned base (attn_workspace): H arrival counters; then m and l
    ([slots][32] fp32) and O ([slots][32][d] fp32) of the partials, slots = 2·SMs + H; then the split tables of the
    2-CTA/SM grid (table 0) and the 1-CTA/SM grid (table 1), each 4 + 2·SMs + 4 words; then 2·SMs per-CTA times."""
    slots_max = 2 * sms
    lay = {"slots": slots_max + H, "m": round_up(4 * H, 256)}
    lay["O"] = lay["m"] + 2 * 4 * lay["slots"] * MAX_ROWS
    lay["table0"] = round_up(lay["O"] + 4 * lay["slots"] * MAX_ROWS * d, 256)
    tab_bytes = 4 * (SPLIT_HDR + slots_max + 4)
    lay["table1"] = lay["table0"] + tab_bytes
    lay["bytes"] = lay["table1"] + tab_bytes + 4 * slots_max + 256  # + the alignment slack of the caller's base
    return lay


def new_workspace(R: int, H: int, d: int, sms: int):
    ws = ops.verify_attn_workspace(R, H, d, DEV)
    lay = workspace_layout(H, d, sms)
    assert ws.numel() == lay["bytes"], "the workspace layout restated here does not match tf_verify_attn_workspace_bytes"
    assert ws.data_ptr() % 256 == 0
    return ws, lay


def ws_words(ws, offset: int, n: int, dtype=torch.float32) -> torch.Tensor:
    return ws[offset:offset + 4 * n].view(dtype)


def partial_m(ws, lay) -> torch.Tensor:
    return ws_words(ws, lay["m"], lay["slots"] * MAX_ROWS).view(lay["slots"], MAX_ROWS)


def split_table(ws, lay, R: int, d: int, sms: int):
    """The split table a launch with these rows reads: table 1 for the 1-CTA/SM grid, table 0 otherwise."""
    off = lay["table1"] if d == 128 and R > 16 else lay["table0"]
    return ws_words(ws, off, SPLIT_HDR + 2 * sms, torch.int32).cpu().numpy().view(np.uint32).tolist()


def assert_partial_slots(ws, lay, plan: Plan, what: str):
    """After one launch on a workspace whose partial m was filled with NaN: exactly the slots CTA + head of the plan's
    segments were written, in rows < R.  (m may be -inf where a row sees no key of a segment; it is never NaN.)"""
    want = torch.zeros((lay["slots"], MAX_ROWS), dtype=torch.bool, device=DEV)
    for b, h, _, _ in plan.segments:
        want[b + h, :plan.R] = True
    bad = torch.nonzero((~partial_m(ws, lay).isnan()) != want)[:, 0].unique().tolist()
    assert not bad, f"{what}: partial slots {bad[:8]} written unlike the plan ({plan.summary()})"


def assert_counters_reset(ws, H: int, what: str):
    assert not ws_words(ws, 0, H, torch.int32).any(), f"{what}: a per-head arrival counter was left non-zero"


# ---------------------------------------------------------------------------------------------------------------------
# needles, comparison and negative controls
# ---------------------------------------------------------------------------------------------------------------------
def plant_case(nd: Needles, K, V, plan: Plan, cap: int):
    """Stale rows from kv_len to cap; in every head, needles at the first and last key of each of its segments and a
    record needle e^3 above them at the last key of its middle partial; needles at the R fresh keys, each with its own V
    row, so a row that sees one fresh key too many or too few moves."""
    kv_len, R = plan.kv_len, plan.R
    L0 = base_logit(kv_len)
    plant_stale(nd, K, V, 0, kv_len, cap)
    for h in range(plan.H):
        parts = plan.partials(h)
        assert len(parts) >= 3, "a middle partial needs partials on both sides"
        record = parts[(len(parts) - 1) // 2][2] - 1
        assert record < kv_len - R
        keys = sorted({k for _, lo, hi in parts for k in (lo, hi - 1)} | {record})
        nd.plant(K, V, 0, keys, [L0 + 3.0 if k == record else L0 for k in keys], head=h)
    nd.plant(K, V, 0, range(kv_len - R, kv_len), [L0] * R)


def head_mutants(plan: Plan, q, K, V, vis, h: int, straddle: bool):
    """Mutated references of head h: each of its partials dropped; with `straddle` (h entered by a straddling CTA), its
    first tile read from head h - 1."""
    qh, Kh, Vh = q[:, h], K[0, h], V[0, h]
    mutants = []
    for p, (b, lo, hi) in enumerate(plan.partials(h)):
        m = vis.clone()
        m[:, lo:hi] = False
        mutants.append((f"head {h} partial {p} (CTA {b}) dropped", reference(qh, Kh, Vh, m)))
    if straddle:
        Km, Vm = Kh.clone(), Vh.clone()
        Km[:BN], Vm[:BN] = K[0, h - 1, :BN], V[0, h - 1, :BN]
        mutants.append((f"head {h}: its first tile read from head {h - 1}", reference(qh, Km, Vm, vis)))
    return mutants


def row_mutants(plan: Plan, q, K, V, vis):
    """Mutated references of head 0 that do not depend on the split."""
    R, kv_len, n = plan.R, plan.kv_len, vis.shape[1]
    qh, Kh, Vh = q[:, 0], K[0, 0], V[0, 0]
    i = torch.arange(R, device=DEV)[:, None]
    j = torch.arange(n, device=DEV)[None, :]
    _, lo, hi = plan.partials(0)[0]
    twice = torch.zeros(n, dtype=torch.float64, device=DEV)
    twice[lo:hi] = math.log(2.0)
    fresh_dropped = vis.clone()
    fresh_dropped[:, kv_len - R:kv_len] = False
    mutants = [("partial 0 counted twice", reference(qh, Kh, Vh, vis, bias=twice)),
               ("fresh keys dropped", reference(qh, Kh, Vh, fresh_dropped)),
               ("diagonal key excluded", reference(qh, Kh, Vh, j < kv_len - R + i)),
               ("kv_len + 1 keys", reference(qh, Kh, Vh, vis | (j == kv_len)))]
    if R > 1:  # (for one row the diagonal moved up is the kv_len + 1 keys mutant)
        mutants.append(("diagonal moved up by one", reference(qh, Kh, Vh, (j <= kv_len - R + i + 1) & (j < kv_len))))
    return mutants


def compare(out, q, K, V, plan: Plan, what: str, mutant_heads=None):
    """Every head against the fp64 reference; the negative controls on head 0 and on `mutant_heads` (default: one head
    entered by a straddling CTA, from the middle of the axis)."""
    entered = plan.entered_heads()
    if mutant_heads is None:
        mutant_heads = [entered[len(entered) // 2]] if entered else []
    vis = visibility(plan.R, plan.kv_len + 1, plan.kv_len, causal=True)
    worst, weakest = (0.0, -1), float("inf")
    for h in range(plan.H):
        want = reference(q[:, h], K[0, h], V[0, h], vis)
        worst = max(worst, (excess(out[:, h], want), h))
        if h == 0 or h in mutant_heads:
            mutants = head_mutants(plan, q, K, V, vis, h, straddle=h in entered)
            if h == 0:
                mutants += row_mutants(plan, q, K, V, vis)
            weakest = min(weakest, assert_rejected(mutants, want, f"{what} head {h}"))
        del want
    print(f"{what}: {plan.summary()}; worst head {worst[1]}, error / tolerance = {worst[0]:.3f}; "
          f"weakest negative control {weakest:.3g}x (heads 0, {mutant_heads})")
    assert worst[0] <= 1.0, f"{what}: head {worst[1]} exceeds the tolerance ({worst[0]:.3g}x)"


def launch(q, maps, plan: Plan, out, ws, kv_len_dev=None):
    """Host length, or the graph form: R on the host + the committed length on the device, grid sized from the store."""
    scale = orc.softmax_scale_fp16(plan.d)
    if kv_len_dev is None:
        ops.verify_attn(q, maps, 0, plan.kv_len, plan.R, plan.H, plan.d, scale, out, ws)
    else:
        ops.verify_attn(q, maps, 0, plan.R, plan.R, plan.H, plan.d, scale, out, ws, kv_len_dev=kv_len_dev)


# ---------------------------------------------------------------------------------------------------------------------
# production shapes
# ---------------------------------------------------------------------------------------------------------------------
CASES = {  # name: R, H, d, kv_len, store capacity, length from the device (grid sized for the capacity)
    "cfg2_full_verify": (8, 32, 128, 124936, 131072, True),
    "cfg2_ar_decode": (1, 32, 128, 124929, 124929 + 64, False),
    "tp8_rows8": (8, 4, 128, 124936, 124936 + 64, False),
    "tp2_rows8": (8, 16, 128, 124936, 124936 + 64, False),
    "tp8_rows9": (9, 4, 128, 124936, 124936 + 64, False),
    "tp2_rows9": (9, 16, 128, 124936, 124936 + 64, False),
    "rows16": (16, 32, 128, 124944, 124944 + 64, False),
    "cfg4_verify": (18, 16, 128, 130066, 130066 + 64, False),
    "short_store": (8, 32, 128, 259, 131072, True),
    "sharded_retrieval": (7, 4, 128, 4103, 4103 + 64, False),
    "d64_rows5": (5, 12, 64, 2005, 2005 + 64, False),
    "d64_rows20": (20, 12, 64, 3990, 3990 + 64, False),
}


def expect_path(name: str, plan: Plan, sms: int):
    """The path each case is meant to reach, for any SM count of an H100 (114 PCIe, 132 SXM)."""
    P, straddling = plan.n_partials(), len(plan.straddling())
    if plan.G % plan.H:  # (when G is a multiple of H, every head starts on a CTA boundary: 4 and 12 heads here)
        assert straddling >= plan.H // 2
    if name in ("cfg2_full_verify", "cfg2_ar_decode", "rows16", "d64_rows5", "d64_rows20"):
        assert plan.G == 2 * sms
    if name in ("cfg2_full_verify", "cfg2_ar_decode", "rows16"):
        assert 3 <= min(P) and max(P) <= 16  # one merge stream
    if name == "cfg2_ar_decode":
        assert plan.kv_len % BN == 1  # the last tile of every head holds one key
    if name.startswith("tp"):
        assert plan.G == 2 * sms
        if plan.H == 4 or plan.G > 16 * plan.H:  # 16 heads have more than 16 partials on >= 129 SMs only
            assert min(P) > 16
        assert plan.dual_stream() == (plan.R == 8 and max(P) > 16)
    if name == "cfg4_verify":
        assert plan.G == sms and min(P) >= 3
    if name == "short_store":
        assert plan.G == plan.total == 160 < plan.grid and straddling == 0
        assert plan.cta_of(0, plan.kv_len - plan.R) != plan.cta_of(0, plan.kv_len - 1)  # fresh keys in two CTAs
    if name == "sharded_retrieval":
        assert plan.grid == plan.G == 32  # 8 tiles per CTA
    if name.startswith("d64"):
        assert min(P) > 16


@pytest.mark.parametrize("name", list(CASES))
def test_verify_attn_production_shape(name):
    R, H, d, kv_len, cap, dev_len = CASES[name]
    sms = sm_count()
    plan = Plan(R, H, d, kv_len, cap if dev_len else kv_len, sms)
    expect_path(name, plan, sms)
    nd = Needles(H, seed=1000 * R + kv_len, d=d)
    K, V = nd.store(1, cap), nd.store(1, cap)
    q = nd.queries(R)
    plant_case(nd, K, V, plan, cap)
    maps = ops.KVTensorMaps(K, V)
    ws, lay = new_workspace(R, H, d, sms)
    kv_len_dev = torch.tensor([kv_len - R], dtype=torch.int32, device=DEV) if dev_len else None
    out, out2 = (torch.empty((R, H, d), dtype=torch.float16, device=DEV) for _ in range(2))
    partial_m(ws, lay).fill_(float("nan"))
    launch(q, maps, plan, out, ws, kv_len_dev)
    torch.cuda.synchronize()
    assert_partial_slots(ws, lay, plan, name)
    launch(q, maps, plan, out2, ws, kv_len_dev)
    torch.cuda.synchronize()
    assert torch.equal(out, out2), "the merge runs in a fixed order: two launches must give the same bits"
    assert_counters_reset(ws, H, name)
    compare(out, q, K, V, plan, name)


# ---------------------------------------------------------------------------------------------------------------------
# a captured graph follows the device-side length
# ---------------------------------------------------------------------------------------------------------------------
def test_verify_attn_graph_replay_follows_device_length():
    """One verify_attn(kv_len_dev=seq_len_dev) launch of the cfg2 verify captured over a 131 072-key store and replayed
    while the committed length grows by 1, 6 and 1 (the fresh rows move inside the last tile), then by 49 (one tile more
    per head, a new split) and then shrinks; the fresh rows and the needles move with it.  Each replay writes the partial
    slots of the plan of its own length, leaves the arrival counters at zero, gives the bits of an eager launch at that
    length and matches the reference."""
    R, H, d, cap = 8, 32, 128, 131072
    sms = sm_count()
    nd = Needles(H, seed=131072, d=d)
    K0, V0 = nd.store(1, cap), nd.store(1, cap)
    K, V = K0.clone(), V0.clone()
    q = nd.queries(R)
    maps = ops.KVTensorMaps(K, V)
    ws, lay = new_workspace(R, H, d, sms)
    seq_len = torch.tensor([124928], dtype=torch.int32, device=DEV)
    out, eager = (torch.empty((R, H, d), dtype=torch.float16, device=DEV) for _ in range(2))
    plan = Plan(R, H, d, 124928 + R, cap, sms)
    launch(q, maps, plan, out, ws, seq_len)  # load the module and set the kernel attributes outside the capture
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        launch(q, maps, plan, out, ws, seq_len)
    seen = set()
    for n in (124928, 124929, 124935, 124936, 124985, 120001):
        kv_len = n + R
        plan = Plan(R, H, d, kv_len, cap, sms)
        seen.add(tuple(plan.starts))
        K.copy_(K0)
        V.copy_(V0)
        plant_case(nd, K, V, plan, cap)
        seq_len.fill_(n)
        partial_m(ws, lay).fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        what = f"graph replay kv_len={kv_len}"
        assert_partial_slots(ws, lay, plan, what)
        assert_counters_reset(ws, H, what)
        launch(q, maps, plan, eager, ws)
        torch.cuda.synchronize()
        assert torch.equal(out, eager), f"{what}: the replay and an eager launch at the same length differ"
        compare(out, q, K, V, plan, what)
    assert len(seen) == 3, "the lengths should give three different splits"


# ---------------------------------------------------------------------------------------------------------------------
# a split table
# ---------------------------------------------------------------------------------------------------------------------
def hand_table(equal: Plan):
    """A split table (header + G 32-bit fractions) that keeps calibrate's invariant, every CTA within [1/2, 2] of the equal
    share, and moves two boundaries of the equal split by less than 0.4 shares:
      * one back onto the last tile of a head hA from just past it: the CTA ahead then streams that one tile of hA and
        enters hA + 1, the fresh keys of hA are cut between two CTAs, and the owners of hA's last tile and of hA + 1's
        first tile are not the ones the equal-split formula gives, so the merge must find them in the table;
      * one forward onto the first tile of a head hB from inside hB - 1: a CTA ends exactly at a head's end.
    Returns (table, hA, hB)."""
    G, total, tph, s = equal.G, equal.total, equal.tph, equal.starts
    share = total / G
    back = [(s[k] - ((h + 1) * tph - 1), k, h) for k in range(1, G) for h in range(1, equal.H - 1)
            if 0 < s[k] - ((h + 1) * tph - 1) <= 0.4 * share]
    _, kA, hA = min(back)
    fwd = [(h * tph - s[k], k, h) for k in range(1, G) for h in range(1, equal.H)
           if 0 < h * tph - s[k] <= 0.4 * share and abs(k - kA) >= 2 and h not in (hA, hA + 1)]
    _, kB, hB = min(fwd)
    starts = list(s)
    starts[kA], starts[kB] = (hA + 1) * tph - 1, hB * tph
    sizes = np.diff(starts)
    assert sizes.min() >= max(1, share / 2) and sizes.max() <= 2 * share
    fracs = [0] + [cdiv(x << 32, total) for x in starts[1:G]]
    assert all((f * total) >> 32 == x and f < 2 ** 32 for f, x in zip(fracs, starts))
    return [G, 0, 0, 0] + fracs, hA, hB


def test_verify_attn_split_table():
    """tf_verify_attn_calibrate installs table 0 where the layout puts it; a hand-made table in that slot (hand_table)
    moves the segments, the merge finds each head's partials by scanning it, and the result matches the reference.  A
    launch with another grid (R = 18 reads table 1; a store too short for the full grid) or with total < 4 G uses the equal
    split and gives the bits of a workspace without a table; so does the full shape after rounds = 0 clears the header."""
    R, H, d = 8, 32, 128
    kv_len = 124928 + 4  # the fresh keys 124 924 .. 124 931 straddle the last tile boundary of every head
    cap = kv_len + 64
    sms = sm_count()
    scale = orc.softmax_scale_fp16(d)
    nd = Needles(H, seed=777, d=d)
    K, V = nd.store(1, cap), nd.store(1, cap)
    q = nd.queries(R)
    maps = ops.KVTensorMaps(K, V)
    ws, lay = new_workspace(R, H, d, sms)
    plain, _ = new_workspace(R, H, d, sms)
    out, out2 = (torch.empty((R, H, d), dtype=torch.float16, device=DEV) for _ in range(2))
    ops.verify_attn_calibrate(q, maps, 0, kv_len, R, H, d, scale, out, ws, rounds=1)
    assert split_table(ws, lay, R, d, sms)[0] == 2 * sms, "the calibrated table is not where the layout puts table 0"
    assert split_table(ws, lay, 18, d, sms)[0] == 0

    equal = Plan(R, H, d, kv_len, kv_len, sms)
    table, hA, hB = hand_table(equal)
    ws_words(ws, lay["table0"], len(table), torch.int32).copy_(
        torch.from_numpy(np.array(table, dtype=np.uint32).view(np.int32)))
    plan = Plan(R, H, d, kv_len, kv_len, sms, table=split_table(ws, lay, R, d, sms))
    assert plan.uses_table and plan.segments != equal.segments
    assert plan.cta_of(hA, kv_len - R) != plan.cta_of(hA, kv_len - 1), "the fresh keys of head hA are cut by the table"
    assert plan.partials(hA + 1)[0][0] == plan.partials(hA)[-1][0] != equal.partials(hA)[-1][0]
    assert plan.partials(hB)[0][1] == 0 and plan.partials(hB)[0][0] != plan.partials(hB - 1)[-1][0]
    print(f"split table: hA = {hA}, hB = {hB}")

    plant_case(nd, K, V, plan, cap)
    partial_m(ws, lay).fill_(float("nan"))
    launch(q, maps, plan, out, ws)
    torch.cuda.synchronize()
    assert_partial_slots(ws, lay, plan, "split table")
    launch(q, maps, plan, out2, ws)
    torch.cuda.synchronize()
    assert torch.equal(out, out2)
    assert_counters_reset(ws, H, "split table")
    compare(out, q, K, V, plan, "split table", mutant_heads=[hA, hA + 1, hB])

    # the equal split whenever the table does not apply: same bits as a workspace without one
    for R2, kv2, dev in [(18, kv_len, False), (8, 300, False), (8, 1500, True)]:
        p = Plan(R2, H, d, kv2, cap if dev else kv2, sms, table=split_table(ws, lay, R2, d, sms))
        assert not p.uses_table
        if dev:
            assert p.grid == table[0] and p.total < 4 * p.G  # the grid matches the header; too few tiles
        q2 = nd.queries(R2)
        dev_len = torch.tensor([kv2 - R2], dtype=torch.int32, device=DEV) if dev else None
        a, b = (torch.empty((R2, H, d), dtype=torch.float16, device=DEV) for _ in range(2))
        launch(q2, maps, p, a, ws, dev_len)
        launch(q2, maps, p, b, plain, dev_len)
        torch.cuda.synchronize()
        assert torch.equal(a, b), f"R={R2} kv_len={kv2}: the split table was not ignored"
    ops.verify_attn_calibrate(q, maps, 0, kv_len, R, H, d, scale, out2, ws, rounds=0)
    assert split_table(ws, lay, R, d, sms)[0] == 0
    launch(q, maps, equal, out, ws)
    launch(q, maps, equal, out2, plain)
    torch.cuda.synchronize()
    assert torch.equal(out, out2)
    assert_counters_reset(ws, H, "split table")
