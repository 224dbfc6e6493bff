"""The wgmma attention (tf_tree_attn_tc) and the retrieval verify attention at the shapes the 7B / 13B models run them:
the 512-node Sequoia tree verify at ~125K and ~50K keys, 128-row prefill chunks in causal mode up to the 124 928-token
prompt, and the gamma+1-row retrieval verify chained behind rope_append under programmatic dependent launch.

Every output is compared with an fp64 evaluation of the same attention on the GPU, one head at a time.  The inputs carry
"needles": the query rows share one direction per head, a few keys lie along it with large, distinctive V rows, so each
needle holds a visible share of the softmax mass and the outputs are O(1).  A key that the kernel drops, double-counts or
wrongly admits then moves the output far outside the tolerance.  Rows past kv_len hold stale needles that would dominate
the softmax if they were read.  Each test also checks that its comparison rejects mutated references (a KV split dropped,
the causal diagonal shifted, a tree-mask bit flipped, one key too many), so the tolerance is known to see those errors;
the negative controls launch no library kernel."""
import os

import numpy as np
import pytest
import torch

from attn_needles import (STALE_V, Needles, assert_rejected, base_logit, excess, plant_stale, reference,
                          report_time_and_memory, visibility)  # noqa: F401  (report_time_and_memory: autouse fixture)
from oracle import triforce_oracle as orc
from triforce_b200 import _C, ops
from triforce_b200.spectree import load_grow_map

pytestmark = pytest.mark.gpu
DEV = "cuda"
D = 128             # head dim (tf_tree_attn_tc supports only 128)
TILE = 128          # keys per tile of tf_tree_attn_tc
BLOCK_ROWS = 128    # query rows per CTA of tf_tree_attn_tc
SCALE = orc.softmax_scale_fp16(D)


# ---------------------------------------------------------------------------------------------------------------------
# split plan
# ---------------------------------------------------------------------------------------------------------------------
def cdiv(a: int, b: int) -> int:
    return -(-a // b)


def tc_splits(R: int, H: int, kv_len: int) -> int:
    """KV splits tf_tree_attn_tc plans for this launch, read off its workspace size: 256 bytes of slack plus, per
    (128-row block, head, split), 128 rows x (128 O + m + l) fp32."""
    blocks = cdiv(R, BLOCK_ROWS)
    per_split = blocks * H * BLOCK_ROWS * (D + 2) * 4
    nbytes = _C.lib().tf_tree_attn_tc_workspace_bytes(R, H, kv_len)
    assert (nbytes - 256) % per_split == 0, nbytes
    return (nbytes - 256) // per_split


def split_key_ranges(R: int, kv_len: int, splits: int, causal: bool):
    """[block][split] -> (first key, end key) streamed by that CTA: the plan of tree_attn_tc.cu written out.  Non-causal:
    every block cuts ceil(tiles / splits) tiles per split.  Causal: block b stops at the tile holding its last row's
    diagonal key kv_len - R + 128 b + 127 and cuts those tiles into `splits` equal parts, so trailing splits of the early
    blocks can be empty (they publish an empty partial).  Empty ranges are (k, k)."""
    tiles_all = cdiv(kv_len, TILE)
    plan = []
    for b in range(cdiv(R, BLOCK_ROWS)):
        last_key = min(kv_len - 1, kv_len - R + BLOCK_ROWS * b + BLOCK_ROWS - 1) if causal else kv_len - 1
        tiles = last_key // TILE + 1 if last_key >= 0 else 0
        per = cdiv(tiles, splits) if causal else cdiv(tiles_all, splits)
        ranges = []
        for sp in range(splits):
            t0, t1 = sp * per, min(tiles, sp * per + per)
            ranges.append((t0 * TILE, min(t1 * TILE, kv_len)) if t1 > t0 else (t0 * TILE, t0 * TILE))
        plan.append(ranges)
    return plan


# ---------------------------------------------------------------------------------------------------------------------
# tree needles and the per-head comparison
# ---------------------------------------------------------------------------------------------------------------------
def tree_needle_column(tree: torch.Tensor):
    """A tree column seen by some rows and not by others, and a row that does not see it."""
    seen = tree.sum(0)
    c = next(c for c in range(1, tree.shape[1]) if 2 <= int(seen[c]) <= tree.shape[0] - 2)
    return c, int(torch.nonzero(~tree[:, c])[0])


def compare_heads(outs, q, K, V, layer: int, vis: torch.Tensor, what: str):
    """Every head of every output in `outs` {name: [R, H, D]} against the fp64 reference; returns head 0's reference."""
    H = q.shape[1]
    worst = {name: (0.0, -1) for name in outs}
    want0 = None
    for h in range(H):
        want = reference(q[:, h], K[layer, h], V[layer, h], vis)
        for name, o in outs.items():
            e = excess(o[:, h], want)
            if e > worst[name][0]:
                worst[name] = (e, h)
        if h == 0:
            want0 = want
        del want
    for name, (e, h) in worst.items():
        print(f"{what} {name}: worst head {h}, error / tolerance = {e:.3f}")
        assert e <= 1.0, f"{what} {name}: head {h} exceeds the tolerance ({e:.3g}x)"
    return want0


# ---------------------------------------------------------------------------------------------------------------------
# Sequoia tree verify: 512 rows against the whole KV
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H,prefix,min_splits", [(32, 124928 + 13, 8), (40, 49152 + 5, 6)], ids=["cfg2_depth", "cfg5"])
def test_tree_verify_production_shape(H, prefix, min_splits):
    """R = T = 512 (the 512-node tree), prefix keys not a multiple of 32 or 128: the tree columns start mid-word and
    mid-tile.  min_splits holds on 114-SM (PCIe) and 132-SM (SXM) H100s."""
    R = T = 512
    kv_len = prefix + T
    cap = kv_len + 64
    splits = tc_splits(R, H, kv_len)
    print(f"tree verify R={R} H={H} kv_len={kv_len}: {splits} KV splits")
    assert splits >= min_splits
    ranges = split_key_ranges(R, kv_len, splits, causal=False)[0]
    assert all(hi > lo for lo, hi in ranges) and ranges[-1][1] == kv_len

    tree = load_grow_map("512")["mask"].bool().to(DEV)  # ancestor-closed: row n sees itself and its ancestors
    c, blind_row = tree_needle_column(tree)
    nd = Needles(H, seed=H * 1000 + prefix)
    K, V = nd.store(1, cap), nd.store(1, cap)
    q = nd.queries(R)
    keys = {0, prefix - 1, prefix + c, kv_len - 1} | {k for lo, hi in ranges for k in (lo, hi - 1)}
    record = ranges[splits // 2][1] - 1  # the last tile of a middle split: higher than every key before it
    L0 = base_logit(kv_len)
    nd.plant(K, V, 0, sorted(keys), [L0 + 3.0 if k == record else L0 for k in sorted(keys)])
    plant_stale(nd, K, V, 0, kv_len, cap)

    maps = ops.KVTensorMaps(K, V)
    mask = torch.from_numpy(orc.pack_tree_mask(tree.cpu().numpy()).view(np.int32)).to(DEV)
    ws = ops.tree_attn_tc_workspace(R, H, kv_len, DEV)
    out = torch.empty((R, H, D), dtype=torch.float16, device=DEV)
    ops.tree_attn_tc(q, maps, 0, kv_len, R, H, D, SCALE, mask, T, out, ws)
    out2 = torch.empty_like(out)
    ops.tree_attn_tc(q, maps, 0, kv_len, R, H, D, SCALE, mask, T, out2, ws)
    # the 32-row blocked path of tf_verify_attn_tree (the model's path with TRIFORCE_TREE_TC=0)
    ws32 = ops.verify_attn_workspace(ops.VERIFY_MAX_ROWS, H, D, DEV)
    out32 = torch.empty_like(out)
    for r0 in range(0, R, ops.VERIFY_MAX_ROWS):
        r1 = r0 + ops.VERIFY_MAX_ROWS
        ops.verify_attn_tree(q[r0:r1], maps, 0, kv_len, r1 - r0, H, D, SCALE, mask[r0:r1], T, out32[r0:r1], ws32)
    torch.cuda.synchronize()
    assert torch.equal(out, out2), "the split merge runs in a fixed order: two launches must give the same bits"

    vis = visibility(R, kv_len + 1, kv_len, tree=tree)
    want = compare_heads({"tree_attn_tc": out, "verify_attn_tree": out32}, q, K, V, 0, vis, f"tree H={H}")
    mutants = []
    for sp, (lo, hi) in enumerate(ranges):
        m = vis.clone()
        m[:, lo:hi] = False
        mutants.append((f"split {sp} dropped", reference(q[:, 0], K[0, 0], V[0, 0], m)))
    m = vis.clone()
    m[blind_row, prefix + c] = True
    mutants.append(("tree bit flipped", reference(q[:, 0], K[0, 0], V[0, 0], m)))
    m = vis.clone()
    m[:, kv_len] = True
    mutants.append(("kv_len + 1 keys", reference(q[:, 0], K[0, 0], V[0, 0], m)))
    assert_rejected(mutants, want, f"tree H={H}")


# ---------------------------------------------------------------------------------------------------------------------
# prefill chunks: 128 rows in causal mode, deep into the prompt
# ---------------------------------------------------------------------------------------------------------------------
def _causal_case(R, H, kv_len, seed, extra_keys=()):
    """Store, queries and needles of a causal launch: the diagonal keys kv_len - R + i of the first block's rows (row i
    sees one that row i-1 does not), the last key of every split of every block, and `extra_keys`."""
    cap = kv_len + 64
    splits = tc_splits(R, H, kv_len)
    plan = split_key_ranges(R, kv_len, splits, causal=True)
    nd = Needles(H, seed)
    K, V = nd.store(1, cap), nd.store(1, cap)
    q = nd.queries(R)
    keys = {kv_len - R + i for i in range(min(R, BLOCK_ROWS))} | {hi - 1 for ranges in plan for lo, hi in ranges if hi > lo}
    keys |= set(extra_keys)
    record = plan[-1][(splits - 1) // 2][1] - 1  # the last tile of a middle split: higher than every key before it
    L0 = base_logit(kv_len)
    nd.plant(K, V, 0, sorted(keys), [L0 + 3.0 if k == record else L0 for k in sorted(keys)])
    plant_stale(nd, K, V, 0, kv_len, cap)
    return splits, plan, q, K, V


def _causal_mutants(q, K, V, R, kv_len, plan, vis, h=0):
    mutants = []
    for b, ranges in enumerate(plan):
        rows = slice(b * BLOCK_ROWS, min(R, b * BLOCK_ROWS + BLOCK_ROWS))
        for sp, (lo, hi) in enumerate(ranges):
            if hi > lo:
                m = vis.clone()
                m[rows, lo:hi] = False
                mutants.append((f"block {b} split {sp} dropped", reference(q[:, h], K[0, h], V[0, h], m)))
    i = torch.arange(R, device=DEV)[:, None]
    j = torch.arange(vis.shape[1], device=DEV)[None, :]
    mutants.append(("diagonal shifted by one", reference(q[:, h], K[0, h], V[0, h], (j <= kv_len - R + i + 1) & (j < kv_len))))
    mutants.append(("kv_len + 1 keys", reference(q[:, h], K[0, h], V[0, h], visibility(R, kv_len + 1, kv_len + 1, causal=True))))
    return mutants


@pytest.mark.parametrize("kv_len,min_splits,max_splits", [(2048, 1, 1), (4096 + 64, 2, 2), (16384, 8, 8), (65536 + 77, 16, 32),
                                                           (124928, 24, 33)])
def test_prefill_chunk_causal_production_depth(kv_len, min_splits, max_splits):
    """A 128-row prompt chunk of a 32-head model at increasing depth: 1, 2, 8, then (SM-count dependent) >= 16 and >= 24
    KV splits; at 124 928 keys (the last chunk of the cfg2 prompt) 33 splits on a 132-SM H100."""
    R, H = 128, 32
    splits, plan, q, K, V = _causal_case(R, H, kv_len, seed=kv_len)
    print(f"prefill chunk R={R} H={H} kv_len={kv_len}: {splits} KV splits")
    assert min_splits <= splits <= max_splits
    maps = ops.KVTensorMaps(K, V)
    ws = ops.tree_attn_tc_workspace(R, H, kv_len, DEV)
    out = torch.empty((R, H, D), dtype=torch.float16, device=DEV)
    ops.tree_attn_tc(q, maps, 0, kv_len, R, H, D, SCALE, None, 0, out, ws, causal=True)
    torch.cuda.synchronize()
    vis = visibility(R, kv_len + 1, kv_len, causal=True)
    want = compare_heads({"tree_attn_tc causal": out}, q, K, V, 0, vis, f"prefill kv_len={kv_len}")
    assert_rejected(_causal_mutants(q, K, V, R, kv_len, plan, vis), want, f"prefill kv_len={kv_len}")


def test_causal_trailing_empty_splits():
    """R = kv_len = 4096, one head: 32 blocks over 32 tiles, 2 splits.  Block b streams tiles 0..b, cut into
    ceil((b+1)/2)-tile splits, so block 0's second split is empty and publishes an empty partial to the merge."""
    R = kv_len = 4096
    H = 1
    splits, plan, q, K, V = _causal_case(R, H, kv_len, seed=4096, extra_keys=(1000, 2222, 3333))
    print(f"causal R={R} H={H} kv_len={kv_len}: {splits} KV splits")
    assert splits == 2
    assert plan[0] == [(0, 128), (128, 128)]               # block 0: one tile, second split empty
    assert plan[2] == [(0, 256), (256, 384)]               # block 2: three tiles, 2 + 1
    assert plan[31] == [(0, 2048), (2048, 4096)]
    assert sum(hi == lo for ranges in plan for lo, hi in ranges) == 1
    maps = ops.KVTensorMaps(K, V)
    ws = ops.tree_attn_tc_workspace(R, H, kv_len, DEV)
    out = torch.empty((R, H, D), dtype=torch.float16, device=DEV)
    ops.tree_attn_tc(q, maps, 0, kv_len, R, H, D, SCALE, None, 0, out, ws, causal=True)
    torch.cuda.synchronize()
    vis = visibility(R, kv_len + 1, kv_len, causal=True)
    want = compare_heads({"tree_attn_tc causal": out}, q, K, V, 0, vis, "causal R=4096")
    assert_rejected(_causal_mutants(q, K, V, R, kv_len, plan, vis), want, "causal R=4096")


def test_causal_block_is_split_on_its_own_keys():
    """The first 128-row block of a 256-row causal launch streams only the tiles up to its own diagonal and splits those
    evenly (16 + 16 of 128 tiles, where the launch-wide cut would be 17 + ...).  The one-block launch of the same rows over
    the keys they see plans the same number of splits, so the two must give the same bits."""
    R, H, kv_len = 256, 32, 16384 + 100
    splits, plan, q, K, V = _causal_case(R, H, kv_len, seed=16484)
    kv0 = kv_len - R + BLOCK_ROWS  # keys visible to block 0
    print(f"causal R={R} H={H} kv_len={kv_len}: {splits} KV splits; block 0 alone: {tc_splits(BLOCK_ROWS, H, kv0)}")
    assert splits == tc_splits(BLOCK_ROWS, H, kv0) == 8
    assert plan[0][0] == (0, 16 * TILE) and cdiv(cdiv(kv_len, TILE), splits) == 17  # per-block cut differs from the launch's
    assert split_key_ranges(BLOCK_ROWS, kv0, splits, causal=True)[0] == [(lo, min(hi, kv0)) for lo, hi in plan[0]]  # same tiles
    maps = ops.KVTensorMaps(K, V)
    out = torch.empty((R, H, D), dtype=torch.float16, device=DEV)
    ops.tree_attn_tc(q, maps, 0, kv_len, R, H, D, SCALE, None, 0, out, ops.tree_attn_tc_workspace(R, H, kv_len, DEV), causal=True)
    out0 = torch.empty((BLOCK_ROWS, H, D), dtype=torch.float16, device=DEV)
    ops.tree_attn_tc(q[:BLOCK_ROWS].contiguous(), maps, 0, kv0, BLOCK_ROWS, H, D, SCALE, None, 0, out0,
                     ops.tree_attn_tc_workspace(BLOCK_ROWS, H, kv0, DEV), causal=True)
    torch.cuda.synchronize()
    assert torch.equal(out[:BLOCK_ROWS], out0)
    vis = visibility(R, kv_len + 1, kv_len, causal=True)
    want = compare_heads({"tree_attn_tc causal": out}, q, K, V, 0, vis, "causal R=256")
    assert_rejected(_causal_mutants(q, K, V, R, kv_len, plan, vis), want, "causal R=256")


# ---------------------------------------------------------------------------------------------------------------------
# layer coordinate of the 4-D tensor maps, bit-exact
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["tree", "causal"])
def test_layer_coordinate_is_exact(mode):
    """The call with layer=l on a 3-layer store gives the bits of the same call on a one-layer store holding layer l."""
    L = 3
    if mode == "tree":
        R, H, kv_len = 512, 4, 8192 + 512 + 13
        tree = load_grow_map("512")["mask"].bool().to(DEV)
        T = 512
        mask = torch.from_numpy(orc.pack_tree_mask(tree.cpu().numpy()).view(np.int32)).to(DEV)
        vis = visibility(R, kv_len + 1, kv_len, tree=tree)
    else:
        R, H, kv_len = 128, 8, 16384
        T, mask = 0, None
        vis = visibility(R, kv_len + 1, kv_len, causal=True)
    cap = kv_len + 64
    splits = tc_splits(R, H, kv_len)
    print(f"layer coordinate ({mode}) R={R} H={H} kv_len={kv_len}: {splits} KV splits")
    assert splits >= 4
    ranges = split_key_ranges(R, kv_len, splits, causal=mode == "causal")[0]
    nd = Needles(H, seed=77 + R)
    K, V = nd.store(L, cap), nd.store(L, cap)
    q = nd.queries(R)
    L0 = base_logit(kv_len)
    for l in range(L):  # different needles (positions, V rows) and stale rows in every layer
        keys = sorted({7 * l, kv_len - 1 - l} | {hi - 1 - 3 * l for lo, hi in ranges})
        nd.plant(K, V, l, keys, [L0] * len(keys))
        plant_stale(nd, K, V, l, kv_len, cap)
    maps = ops.KVTensorMaps(K, V)
    ws = ops.tree_attn_tc_workspace(R, H, kv_len, DEV)
    outs = []
    for l in range(L):
        out = torch.empty((R, H, D), dtype=torch.float16, device=DEV)
        ops.tree_attn_tc(q, maps, l, kv_len, R, H, D, SCALE, mask, T, out, ws, causal=mode == "causal")
        K1, V1 = K[l:l + 1].clone(), V[l:l + 1].clone()
        one = torch.empty_like(out)
        ops.tree_attn_tc(q, ops.KVTensorMaps(K1, V1), 0, kv_len, R, H, D, SCALE, mask, T, one, ws, causal=mode == "causal")
        torch.cuda.synchronize()
        assert torch.equal(out, one), f"layer {l}"
        outs.append(out)
    # the bit comparison can tell the layers apart, and the outputs are right
    assert not torch.equal(outs[0], outs[1]) and not torch.equal(outs[1], outs[2])
    want = compare_heads({"layer 2": outs[2]}, q, K, V, 2, vis, f"layer coordinate ({mode})")
    assert_rejected([(f"layer {l} data", reference(q[:, 0], K[l, 0], V[l, 0], vis)) for l in (0, 1)], want,
                    f"layer coordinate ({mode})")


# ---------------------------------------------------------------------------------------------------------------------
# retrieval verify straight after rope_append, under programmatic dependent launch
# ---------------------------------------------------------------------------------------------------------------------
def test_retrieval_verify_chain_under_pdl():
    """The cfg2 decode step of one layer: rope_append writes the gamma+1 fresh rows behind the 4096-key retrieval budget,
    then verify_attn(clean_keys=4096) runs over budget + gamma + 1 keys.  With programmatic dependent launch its producer
    loads the clean budget tiles before the dependency on rope_append resolves; the fresh slots hold stale needles until
    rope_append overwrites them, so an early read of a fresh row shows.  Eager once, then a captured graph (stale fill,
    append, attention) replayed three times with new inputs."""
    L, H, budget, gamma = 2, 32, 4096, 6
    R = gamma + 1
    kv_len = budget + R
    cap = budget + 64  # the last 64-key tile (fresh rows, then stale rows) lies inside the store
    layer = 1
    g = torch.Generator(device=DEV).manual_seed(4103)
    K = torch.randn((L, H, cap, D), generator=g, device=DEV, dtype=torch.float16)
    V = torch.randn((L, H, cap, D), generator=g, device=DEV, dtype=torch.float16)
    # stale rows: large keys (query·key ~ ±90, logits ~ ±8 against background logits ~ ±1) with large V
    signs = lambda *s: torch.randint(0, 2, s, generator=g, device=DEV).half() * 2 - 1
    stale_k, stale_v = 8 * signs(H, R, D), STALE_V * signs(H, R, D)
    K[:, :, kv_len:] = 8 * signs(L, H, cap - kv_len, D)
    V[:, :, kv_len:] = STALE_V * signs(L, H, cap - kv_len, D)
    pos = np.arange(124928 + 9, 124928 + 9 + R)
    cos_np, sin_np = orc.rope_tables_plain(D, int(pos[-1]) + 1)
    cos, sin = torch.from_numpy(cos_np).to(DEV), torch.from_numpy(sin_np).to(DEV)
    pos32 = torch.from_numpy(pos.astype(np.int32)).to(DEV)
    qkv = torch.empty((R, 3 * H * D), dtype=torch.float16, device=DEV)
    q_out = torch.empty((R, H, D), dtype=torch.float16, device=DEV)
    out = torch.empty((R, H, D), dtype=torch.float16, device=DEV)
    maps = ops.KVTensorMaps(K, V)
    ws = ops.verify_attn_workspace(R, H, D, DEV)
    vis = visibility(R, kv_len + 1, kv_len, causal=True)

    def step():
        K[layer, :, budget:kv_len].copy_(stale_k)
        V[layer, :, budget:kv_len].copy_(stale_v)
        ops.rope_append(qkv, H, D, cos, sin, q_out, K[layer], V[layer], pos_ids=pos32, slot0=budget)
        ops.verify_attn(q_out, maps, layer, kv_len, R, H, D, SCALE, out, ws, clean_keys=budget)

    def check(what):
        torch.cuda.synchronize()
        x = qkv.cpu().numpy().reshape(R, 3, H, D)
        fresh_k = K[layer, :, budget:kv_len].permute(1, 0, 2).cpu().numpy()
        np.testing.assert_array_equal(fresh_k.view(np.uint16), orc.apply_rope(x[:, 1], cos_np, sin_np, pos).view(np.uint16))
        np.testing.assert_array_equal(V[layer, :, budget:kv_len].permute(1, 0, 2).cpu().numpy(), x[:, 2])
        Ks_stale = K[layer].clone()
        Ks_stale[:, budget:kv_len] = stale_k
        Vs_stale = V[layer].clone()
        Vs_stale[:, budget:kv_len] = stale_v
        worst = (0.0, -1)
        rejected = {"stale fresh rows": 0.0, "kv_len + 1 keys": 0.0, "diagonal shifted by one": 0.0}
        i = torch.arange(R, device=DEV)[:, None]
        j = torch.arange(kv_len + 1, device=DEV)[None, :]
        for h in range(H):
            want = reference(q_out[:, h], K[layer, h], V[layer, h], vis)
            e = excess(out[:, h], want)
            worst = max(worst, (e, h))
            for name, m in (("stale fresh rows", reference(q_out[:, h], Ks_stale[h], Vs_stale[h], vis)),
                            ("kv_len + 1 keys", reference(q_out[:, h], K[layer, h], V[layer, h], visibility(R, kv_len + 1, kv_len + 1, causal=True))),
                            ("diagonal shifted by one", reference(q_out[:, h], K[layer, h], V[layer, h], (j <= kv_len - R + i + 1) & (j < kv_len)))):
                rejected[name] = max(rejected[name], excess(m, want))
        print(f"retrieval verify chain ({what}): worst head {worst[1]}, error / tolerance = {worst[0]:.3f}")
        assert worst[0] <= 1.0, f"{what}: head {worst[1]} exceeds the tolerance ({worst[0]:.3g}x)"
        for name, e in rejected.items():
            assert e > 1.0, f"{what}: the comparison does not reject the mutant '{name}' (excess {e:.3g})"

    lib = _C.lib()
    try:
        lib.tf_set_pdl(_C.DEFAULT_PDL_MASK)
        qkv.copy_(torch.randn((R, 3 * H * D), generator=g, device=DEV, dtype=torch.float16))
        step()
        check("eager")
        torch.cuda.synchronize()
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr):
            step()
        for rep in range(3):
            qkv.copy_(torch.randn((R, 3 * H * D), generator=g, device=DEV, dtype=torch.float16))
            gr.replay()
            check(f"graph replay {rep}")
    finally:
        lib.tf_set_pdl(int(os.environ.get("TRIFORCE_PDL", str(_C.DEFAULT_PDL_MASK))))
