"""The target forward at the 7B and 13B widths (head_dim 128, 32 / 40 heads, YaRN factor 32), two layers deep, run through the
engine as bench.py runs cfg2 and cfg5, and compared with an fp64 evaluation of the reference model on the GPU.

cfg2 (7B-wide): a 124 927-token prefill in 128-row chunks (causal tf_tree_attn_tc, last chunk 127 rows), the last prompt
token (retrieval-cache build), a retrieval verify through the captured graph and eagerly, a full-KV verify and a decode
step through the captured full-KV graphs, then the tail update and a second retrieval verify.
cfg5 (13B-wide): a 49 151-token prefill, the last prompt token, the 512-node tree verify over the full KV (one masked
tf_tree_attn_tc pass per layer), the compaction of one accepted root-to-leaf path and a decode step behind it.

The reference computes every op in fp64 and rounds to fp16 where the reference model stores an fp16 tensor
(oracle.LlamaOracle.forward_target): RMSNorm output, q / k / v, each RoPE step, the attention output, both residual adds,
gate, up, SiLU, act, down and the lm_head output.  RoPE tables come from the reference's fp32 recipe (rope.tables_for, tied
to the reference's own tables by test_oracle_golden.py).

Inputs are shaped so that the checks can see what they are meant to see:
  * every RMSNorm weight is 1 + 0.1 N(0, 1) (synthetic weights are all ones), so a swapped or skipped norm shows;
  * in the first half of the heads of each layer k_proj equals q_proj, scaled by TIED: a query scores highest against
    keys of its own token at nearby positions.  Those heads give a row's own fresh key (and a same-token parent in the tree)
    a large share of the softmax, so a missed fresh slot, a short kv_len or a lost ancestor changes the output;
  * in the other half q_proj and k_proj are scaled by PEAKED, so the scores have a spread of ~4 and the softmax is held by
    a few keys: a RoPE position or a key from the wrong layer moves the output by O(1), where random init would give an
    almost uniform average over 125K keys that hides both.  (A larger spread amplifies the legitimate 1-ulp differences
    of q and k into percent-level differences of the output.);
  * lm_head has std 0.01 instead of 0.02, which halves the logits and their absolute error against the fixed atol.
Every check is paired with negative controls built from the reference alone (no library kernel): the same comparison must
reject each of them.
"""
import dataclasses
import time

import pytest
import torch

from triforce_b200.cache import FlashSimpleCache, RetrievalCache, StreamingLLMEvictionCache
from triforce_b200.config import named_config
from triforce_b200.engine import GraphInferenceEngine
from triforce_b200.llama import LlamaModel
from triforce_b200.rope import softmax_scale, tables_for
from triforce_b200.spectree import load_grow_map, pack_mask_bits
from triforce_b200.synth import cuda_state_dict

pytestmark = pytest.mark.gpu
DEV = "cuda"
F16 = torch.float16
LAYERS = 2
TIED = 0.8     # q_proj = k_proj in heads [0, H/2), scaled by this
PEAKED = 1.5   # q_proj and k_proj of heads [H/2, H) scaled by this
LM_HEAD_STD = 0.01
ROWS = 4096    # row chunk of the reference's fp64 GEMMs


@pytest.fixture(autouse=True)
def _report_time_and_memory(request):
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    yield
    torch.cuda.synchronize()
    print(f"\n[{request.node.name}] {time.perf_counter() - t0:.1f} s, peak device memory "
          f"{torch.cuda.max_memory_allocated() / 2**30:.2f} GiB")
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------------
# weights and engine
# ---------------------------------------------------------------------------------------------------------------------
def production_model(name: str, seed: int):
    cfg = dataclasses.replace(named_config(name), num_hidden_layers=LAYERS)
    sd = cuda_state_dict(cfg, seed=seed, lm_head_std=LM_HEAD_STD)
    g = torch.Generator(device=DEV).manual_seed(seed + 1000)
    for key, w in sd.items():
        if w.dim() == 1:  # the RMSNorm weights
            w.copy_(1 + 0.1 * torch.randn(w.shape, generator=g, device=DEV))
    H, d = cfg.num_attention_heads, cfg.head_dim
    for l in range(LAYERS):
        q = sd[f"model.layers.{l}.self_attn.q_proj.weight"].view(H, d, -1)
        k = sd[f"model.layers.{l}.self_attn.k_proj.weight"].view(H, d, -1)
        q[:H // 2].mul_(TIED)
        k[:H // 2].copy_(q[:H // 2])
        q[H // 2:].mul_(PEAKED)
        k[H // 2:].mul_(PEAKED)
    return cfg, sd


def build_engine(cfg, sd, P: int, slots: int, budget=4096, chunk=8, gamma=6):
    """tests/e2e_util.py / test/on_chip.py construction, graphs captured (probs=False: the verify graph returns logits)."""
    target = LlamaModel(cfg, sd, device=DEV)
    ds = named_config("llama-68M")
    draft = LlamaModel(ds, cuda_state_dict(ds, seed=3), device=DEV, is_draft=True)
    cache = FlashSimpleCache(target, slots)
    graph_cache = RetrievalCache(target, max_budget=budget, prefill=P, gamma=gamma, chunk_size=chunk)
    draft_cache = StreamingLLMEvictionCache(draft, start_size=16, recent_size=256 - 16 - gamma, gamma=gamma)
    ge = GraphInferenceEngine(target, cache, graph_cache, draft, draft_cache)
    ge.initialize_cuda_graph(gamma, probs=False)
    return ge


# ---------------------------------------------------------------------------------------------------------------------
# fp64 reference
# ---------------------------------------------------------------------------------------------------------------------
def _f16(x):
    return x.to(F16)


def rmsnorm(h, w, eps):
    x = h.double()
    xn = _f16(x * torch.rsqrt(x.square().mean(-1, keepdim=True) + eps))
    return _f16(w.double() * xn.double())


def linear(x, Wd):
    """fp16 [n, K] times fp64 [N, K]ᵀ, rounded once to fp16."""
    return _f16(x.double() @ Wd.T)


def rope(x, cos, sin, pos):
    """x [n, H, d] fp16 at positions pos [n]: fp16(fp16(x·cos) + fp16(rotate_half(x)·sin)) (products of fp16 are exact)."""
    c, s = cos[pos][:, None].double(), sin[pos][:, None].double()
    xd = x.double()
    h = xd.shape[-1] // 2
    rot = torch.cat([-xd[..., h:], xd[..., :h]], -1)
    return _f16(_f16(xd * c).double() + _f16(rot * s).double())


def attention_ref(q, K, V, limit, scale, tree=None, tree_start=0, heads=4, rows=512):
    """q [R, H, d] fp16; K / V [H, >= limit.max() + 1, d] fp16 (store layout).  Row i sees key j iff j <= limit[i] and, for
    the T columns from `tree_start`, tree[i, j - tree_start].  fp64 scores and softmax, output rounded to fp16.  Blocks of
    `rows` rows stop at the block's last visible key; only the band between the block's first and last limit is masked."""
    R, H, d = q.shape
    out = torch.empty_like(q)
    kmax = int(limit.max()) + 1
    for h0 in range(0, H, heads):
        h1 = min(H, h0 + heads)
        Kd, Vd = K[h0:h1, :kmax].double(), V[h0:h1, :kmax].double()
        for r0 in range(0, R, rows):
            r1 = min(R, r0 + rows)
            lim = limit[r0:r1]
            lo, hi = int(lim.min()) + 1, int(lim.max()) + 1
            s = torch.matmul(q[r0:r1, h0:h1].transpose(0, 1).double(), Kd[:, :hi].transpose(1, 2)).mul_(scale)
            if hi > lo:
                j = torch.arange(lo, hi, device=DEV)
                s[:, :, lo:hi].masked_fill_(j[None, :] > lim[:, None], float("-inf"))
            if tree is not None:
                T = tree.shape[1]
                s[:, :, tree_start:tree_start + T].masked_fill_(~tree[r0:r1], float("-inf"))
            s.sub_(s.amax(-1, keepdim=True)).exp_()
            o = torch.matmul(s, Vd[:, :hi]).div_(s.sum(-1, keepdim=True))
            out[r0:r1, h0:h1] = o.transpose(0, 1).to(F16)
    return out


class Reference:
    """The reference model in fp64 with its own full KV store [L][H, slots, d] (fp16, as the reference caches it)."""

    def __init__(self, cfg, sd, slots):
        self.cfg, self.sd = cfg, sd
        self.H, self.d = cfg.num_attention_heads, cfg.head_dim
        self.eps = cfg.rms_norm_eps
        self.scale = softmax_scale(self.d)
        cos, sin = tables_for(cfg)
        self.cos, self.sin = cos.to(DEV), sin.to(DEV)
        self.K = [torch.zeros((self.H, slots, self.d), dtype=F16, device=DEV) for _ in range(LAYERS)]
        self.V = [torch.zeros_like(k) for k in self.K]
        self.prefill_attention_seconds = None

    def ln(self, l, which):
        return self.sd[f"model.layers.{l}." + ("input_layernorm" if which == 1 else "post_attention_layernorm") + ".weight"]

    def w64(self, l, names):
        full = dict(q="self_attn.q_proj", k="self_attn.k_proj", v="self_attn.v_proj", o="self_attn.o_proj",
                    gate="mlp.gate_proj", up="mlp.up_proj", down="mlp.down_proj")
        return {n: self.sd[f"model.layers.{l}.{full[n]}.weight"].double() for n in names}

    def qkv(self, x, W, pos):
        n = x.shape[0]
        q = rope(linear(x, W["q"]).view(n, self.H, self.d), self.cos, self.sin, pos)
        k = rope(linear(x, W["k"]).view(n, self.H, self.d), self.cos, self.sin, pos)
        return q, k, linear(x, W["v"]).view(n, self.H, self.d)

    def post_attention(self, l, h, a, W, swap_norms=False, swap_gate_up=False):
        """h + o_proj(a), then + down(SiLU(gate) · up) of its RMSNorm."""
        h = _f16(h.double() + linear(a.reshape(h.shape[0], -1), W["o"]).double())
        x = rmsnorm(h, self.ln(l, 1 if swap_norms else 2), self.eps)
        gate, up = (W["up"], W["gate"]) if swap_gate_up else (W["gate"], W["up"])
        g = linear(x, gate).double()
        act = _f16(_f16(g * torch.sigmoid(g)).double() * linear(x, up).double())
        return _f16(h.double() + linear(act, W["down"]).double())

    def logits(self, h):
        x = rmsnorm(h, self.sd["model.norm.weight"], self.eps)
        return linear(x, self.sd["lm_head.weight"].double()).float()

    def forward(self, ids, pos, attend, swap_norms=False, swap_gate_up=False):
        """n rows at positions `pos`; attend(l, q, k, v) stores k / v where that step keeps them and returns the attention."""
        h = self.sd["model.embed_tokens.weight"][ids]
        for l in range(LAYERS):
            W = self.w64(l, ("q", "k", "v", "o", "gate", "up", "down"))
            x = rmsnorm(h, self.ln(l, 2 if swap_norms else 1), self.eps)
            q, k, v = self.qkv(x, W, pos)
            h = self.post_attention(l, h, attend(l, q, k, v), W, swap_norms, swap_gate_up)
            del W
        return self.logits(h)

    def prefill(self, ids):
        """K / V of both layers for prompt rows 0..N-1.  Layer 0 needs the causal attention of every row; layer 1 only its
        K / V.  Row-chunked so that no fp64 copy of a whole [N, hidden] tensor exists."""
        N = ids.numel()
        pos = torch.arange(N, device=DEV)
        h = self.sd["model.embed_tokens.weight"][ids]
        q0 = torch.empty((N, self.H, self.d), dtype=F16, device=DEV)
        W = self.w64(0, ("q", "k", "v"))
        for r0 in range(0, N, ROWS):
            r1 = min(N, r0 + ROWS)
            q0[r0:r1], k, v = self.qkv(rmsnorm(h[r0:r1], self.ln(0, 1), self.eps), W, pos[r0:r1])
            self.K[0][:, r0:r1], self.V[0][:, r0:r1] = k.transpose(0, 1), v.transpose(0, 1)
        del W
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        a0 = attention_ref(q0, self.K[0], self.V[0], pos, self.scale)
        torch.cuda.synchronize()
        self.prefill_attention_seconds = time.perf_counter() - t0
        del q0
        W = self.w64(0, ("o", "gate", "up", "down"))
        for r0 in range(0, N, ROWS):
            r1 = min(N, r0 + ROWS)
            h[r0:r1] = self.post_attention(0, h[r0:r1], a0[r0:r1], W)
        del W, a0
        W = self.w64(1, ("k", "v"))
        for r0 in range(0, N, ROWS):
            r1 = min(N, r0 + ROWS)
            x = rmsnorm(h[r0:r1], self.ln(1, 1), self.eps)
            n = r1 - r0
            k = rope(linear(x, W["k"]).view(n, self.H, self.d), self.cos, self.sin, pos[r0:r1])
            self.K[1][:, r0:r1], self.V[1][:, r0:r1] = k.transpose(0, 1), linear(x, W["v"]).view(n, self.H, self.d).transpose(0, 1)

    def full_kv(self, slot0, limit, kv_of_layer=lambda l: l):
        """attend() of a full-KV step: rows stored at slots slot0.., row i sees keys <= limit[i] of layer kv_of_layer(l)."""
        def attend(l, q, k, v):
            n = q.shape[0]
            self.K[l][:, slot0:slot0 + n], self.V[l][:, slot0:slot0 + n] = k.transpose(0, 1), v.transpose(0, 1)
            src = kv_of_layer(l)
            return attention_ref(q, self.K[src], self.V[src], limit, self.scale)
        return attend


def chunk_scores_ref(K, q, P, chunk):
    """oracle.chunk_mean_keys / chunk_scores on the GPU: fp32 sum of a chunk's rows in row order times fp32(1/chunk),
    rounded to fp16; q·k̄ in fp64 rounded once to fp16.  K [H, >= P, d], q [H, d] → [H, P / chunk] fp16."""
    H, _, d = K.shape
    rows = K[:, :P].float().view(H, P // chunk, chunk, d)
    acc = rows[:, :, 0].clone()
    for j in range(1, chunk):
        acc += rows[:, :, j]
    kbar = (acc * (1.0 / chunk)).half()
    return torch.einsum("hcd,hd->hc", kbar.double(), q.double()).half()


# ---------------------------------------------------------------------------------------------------------------------
# comparisons
# ---------------------------------------------------------------------------------------------------------------------
# Error budget of the engine's logits against the fp64 reference.  Both sides round to fp16 at the same points, so most
# values agree bit for bit; the differences come from values that land on the other side of a rounding point:
#   * fp32 instead of fp64 accumulation inside each op (q/k/v, o, gate/up, down, lm_head; the attention's scores, softmax
#     and P·V; the RMSNorm sum of squares): an fp16 result flips by 1 ulp in a few percent of the elements;
#   * P rounded to fp16 before the P·V product: 2^-11 per weight, averaging out over the keys;
#   * cuBLAS reductions of the 128-row prefill GEMMs (they reach the logits through the stored K / V);
#   * rsqrtf in add_rmsnorm (2 ulp of fp32): a rare flip of the normalised row.
# Each projection over K = 4096..13824 inputs sums the flips of its input into ~0.3-0.5 ulp of noise on its output, which
# then flips about half of the output's roundings; over the ~10 rounding stages of two layers this compounds to ~1.5 fp16
# ulps of the row's scale (2^-10 · 1.5 ≈ 1.5e-3 of its RMS), spread over the whole vocabulary.  Measured on one H100 80GB
# HBM3 at a 700 W power limit: RMS error 1.1e-3..1.4e-3 at a logit RMS of 0.65..0.72 (0.17..0.2 %), maximum 4e-3..9e-3.
# A bound per element with the project's atol of 1e-3 cannot hold for logits near zero, so the bound is per row, on the
# row's norms:
#     rms(got - want) <= LOGIT_ATOL + LOGIT_RTOL · rms(want)    and    max|got - want| <= LOGIT_ATOL + LOGIT_RTOL · max|want|
# with atol 2^-10 and rtol 2^-7 (about 5x the compounded budget; both below the project's 1e-3 / 1e-2).
LOGIT_ATOL = 2.0 ** -10
LOGIT_RTOL = 2.0 ** -7


def logit_excess(got, want):
    """Per row: the larger of the two norm-wise ratios above; <= 1 passes."""
    err = (got.reshape(want.shape).float() - want).abs().nan_to_num(nan=float("inf"))
    rms = err.square().mean(-1).sqrt() / (LOGIT_ATOL + LOGIT_RTOL * want.square().mean(-1).sqrt())
    mx = err.amax(-1) / (LOGIT_ATOL + LOGIT_RTOL * want.abs().amax(-1))
    return torch.maximum(rms, mx)


def check_logits(what, got, want, mutants=()):
    e = logit_excess(got, want)
    err = (got.reshape(want.shape).float() - want).abs()
    print(f"  {what}: max |err| {err.max().item():.2e}, rms err {err.square().mean().sqrt().item():.2e}, rms logit "
          f"{want.square().mean().sqrt().item():.3f}; max excess {e.max().item():.3f} "
          f"(rows: {', '.join(f'{x:.2f}' for x in e[:8].tolist())}{' ...' if e.numel() > 8 else ''})")
    for name, m in mutants:
        me = logit_excess(m, want).max().item()
        print(f"    control '{name}': excess {me:.3g}")
        assert me > 1.0, f"{what}: the comparison does not reject the control '{name}' (excess {me:.3g})"
    assert e.max().item() <= 1.0, f"{what}: logits outside atol {LOGIT_ATOL:.3g} + rtol {LOGIT_RTOL:.3g} of the row's norms"


def ulp16(x):
    """Spacing of fp16 numbers at |x| (2^-24 below the normal range)."""
    _, e = torch.frexp(x.abs().float().clamp_min(2.0 ** -14))
    return torch.ldexp(torch.ones_like(x, dtype=torch.float32), e - 11)


# Stored K / V after the prefill, in fp16 ulps of each element's scale.  An element's scale is its own magnitude (for K
# the norm of the pair j, j + d/2 that RoPE turns together), but at least the RMS of its 128-wide head row: the error of a
# projection is absolute, set by the row it is computed from, and would be many ulps of an element that happens to lie
# near zero.
#   Layer 0: V is one projection of the normalised embedding, rounded once, so it differs from the reference only where
#   cuBLAS's fp32 sum (or an rsqrtf flip of the input) crosses a rounding point: at most 1 ulp.  K is that projection
#   rotated: a 1-ulp input flip moves both rounded products and their sum, at most 3 ulps.
#   Layer 1 inherits the compounded flips of the layer-0 attention, o_proj and MLP (see the logit budget above): about 1
#   ulp of noise, so half of the elements are off by >= 1 ulp; measured at most 11 ulps (H100 80GB HBM3, 700 W).
#   Bound: 16 ulps (1.6 % of the row RMS, where a wrong key, position or layer moves values by O(RMS)) and 3/4 of the
#   elements.
# `frac` bounds the fraction of elements that differ by a whole ulp of their scale or more.
KV_BOUNDS = {0: dict(v_ulps=1, k_ulps=3, frac=2.0 ** -5), 1: dict(v_ulps=16, k_ulps=16, frac=0.75)}


def check_kv_store(kv, ref, n):
    for l in range(LAYERS):
        b = KV_BOUNDS[l]
        for name, got, want, ulps in (("V", kv.value_store[l], ref.V[l], b["v_ulps"]), ("K", kv.key_store[l], ref.K[l], b["k_ulps"])):
            worst, nflip, ndiff = 0.0, 0, 0
            for h in range(ref.H):
                g, w = got[h, :n].float(), want[h, :n].float()
                mag = torch.hypot(w, w.roll(ref.d // 2, -1)) if name == "K" else w.abs()
                floor = w.square().mean(-1, keepdim=True).sqrt()
                ulps_off = (g - w).abs() / ulp16(torch.maximum(mag, floor))
                worst = max(worst, ulps_off.max().item())
                nflip += (ulps_off >= 1).sum().item()
                ndiff += (g != w).sum().item()
            frac = nflip / (ref.H * n * ref.d)
            print(f"  layer {l} {name}[0:{n}]: max {worst:.2f} ulp (bound {ulps}), {frac:.2e} of elements off by >= 1 ulp "
                  f"(bound {b['frac']:.2e}), {ndiff / (ref.H * n * ref.d):.2e} not bit-equal")
            assert worst <= ulps and frac <= b["frac"], f"layer {l} {name} store differs from the reference"


# Chunk scores: fp16(q·k̄) from the engine's K and query against the reference's.  Upstream flips move q and k̄ by
# fractions of an ulp, so a score is off by at most 2 ulps of itself plus 2^-9 of the head's largest |score|
# (the absolute part covers scores near zero, whose error is set by |q|·|k̄|, not by the score).
def check_selection(gc, kv, ref, q_ref, P):
    B, c = gc.max_budget, gc.chunk_size
    sel = B // c
    for l in range(LAYERS):
        want = chunk_scores_ref(ref.K[l], q_ref[l], P, c).float()
        got = gc.chunk_scores[l].float()
        tol = 2 * ulp16(want) + 2.0 ** -9 * want.abs().amax(-1, keepdim=True)
        ex = ((got - want).abs() / tol).max().item()
        print(f"  layer {l} chunk scores: max excess {ex:.3f}")
        assert ex <= 1.0, f"layer {l}: chunk scores differ from the reference"
        idx = gc.topk_idx[l].long()
        assert (idx[:, 0] == 0).all()
        assert ((idx[:, 1:] >= 1) & (idx[:, 1:] < P // c)).all()
        for h in range(ref.H):
            picked = idx[h, 1:]
            assert picked.unique().numel() == sel - 1
            # the engine's set is the top set of its own scores, ties at the cut allowed ...
            mine = got[h, 1:]
            kth = got[h][picked].min()
            assert (mine > kth).sum().item() <= sel - 1 <= (mine >= kth).sum().item()
            # ... and the reference's top set up to chunks whose scores lie within the score error of the cut
            rest = want[h, 1:]
            kth_ref = rest.topk(sel - 1).values[-1]
            window = 2 * (got[h] - want[h]).abs().max()
            inside = torch.zeros(P // c, dtype=torch.bool, device=DEV)
            inside[picked] = True
            assert (want[h][picked] >= kth_ref - window).all(), f"layer {l} head {h}: a chunk below the cut was selected"
            assert not ((rest > kth_ref + window) & ~inside[1:]).any(), f"layer {l} head {h}: a chunk above the cut is missing"
        # the retrieval store is the gather of the engine's own full KV by those indices, bit for bit
        rows = (idx[:, :, None] * c + torch.arange(c, device=DEV)).reshape(ref.H, B)
        for got_store, src in ((gc.key_store, kv.key_store), (gc.value_store, kv.value_store)):
            want_rows = torch.gather(src[l, :, :P], 1, rows[:, :, None].expand(-1, -1, ref.d))
            assert torch.equal(got_store[l, :, :B], want_rows), f"layer {l}: retrieval store is not the gather of the full KV"


def retrieval_store(ref, idx, B, c, gamma):
    """The reference's retrieval cache, gathered from ITS full KV by the engine's chunk indices (a legitimate tie at the
    cut then cannot cascade), with gamma + 1 fresh slots."""
    rows = (idx.long()[:, :, :, None] * c + torch.arange(c, device=DEV)).reshape(LAYERS, ref.H, B)
    K, V = [], []
    for l in range(LAYERS):
        k = torch.zeros((ref.H, B + gamma + 1, ref.d), dtype=F16, device=DEV)
        v = torch.zeros_like(k)
        k[:, :B] = torch.gather(ref.K[l], 1, rows[l][:, :, None].expand(-1, -1, ref.d))
        v[:, :B] = torch.gather(ref.V[l], 1, rows[l][:, :, None].expand(-1, -1, ref.d))
        K.append(k)
        V.append(v)
    return K, V


def retrieval_attend(ref, K, V, B):
    """attend() of a retrieval verify: the rows go to slots B.., row i sees the budget and fresh slots B..B+i."""
    def attend(l, q, k, v):
        n = q.shape[0]
        K[l][:, B:B + n], V[l][:, B:B + n] = k.transpose(0, 1), v.transpose(0, 1)
        return attention_ref(q, K[l], V[l], B + torch.arange(n, device=DEV), ref.scale)
    return attend


def random_ids(n, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(3, 32000, (n,), generator=g).to(DEV)


# ---------------------------------------------------------------------------------------------------------------------
# cfg2: 7B-wide, 124 928-token prompt, retrieval verify / full-KV verify / decode / tail update
# ---------------------------------------------------------------------------------------------------------------------
@torch.inference_mode()
def test_cfg2_width_prefill_retrieval_full_verify_and_tail_update():
    P, B, c, gamma = 124928, 4096, 8, 6
    cfg, sd = production_model("llama-7B-128K", seed=11)
    ge = build_engine(cfg, sd, P, P + 64, B, c, gamma)
    kv, gc = ge.engine.kv_cache, ge.engine.graph_cache
    ref = Reference(cfg, sd, P + 64)
    ids = random_ids(P + 32, seed=12)
    prompt, extra = ids[:P], ids[P:]

    # 1. prefill of P - 1 tokens: 975 chunks of 128 rows and one of 127
    ge.inference(prompt[None, :-1])
    torch.cuda.synchronize()
    assert kv.seq_len == P - 1
    ref.prefill(prompt[:-1])
    print(f"\n  reference prefill: layer-0 causal attention over {P - 1} rows took {ref.prefill_attention_seconds:.1f} s")
    check_kv_store(kv, ref, P - 1)

    # 2. the last prompt token: full-KV attention, then the retrieval build from each layer's query
    logits = ge.inference(prompt[None, -1:])
    q_ref = [None] * LAYERS

    def last_attend(l, q, k, v):
        q_ref[l] = q[0]
        return ref.full_kv(P - 1, torch.tensor([P - 1], device=DEV))(l, q, k, v)

    want = ref.forward(prompt[-1:], torch.tensor([P - 1], device=DEV), last_attend)
    check_logits("last prompt token", logits, want)
    assert kv.seq_len == P
    check_selection(gc, kv, ref, q_ref, P)
    rK, rV = retrieval_store(ref, gc.topk_idx, B, c, gamma)

    # 3. retrieval verify of gamma + 1 rows at P..P+6: captured graph, then eagerly; the two agree bit for bit
    vt = extra[:gamma + 1]
    vpos = torch.arange(P, P + gamma + 1, device=DEV)
    got_graph = ge.graph_verify(vt[None], vpos[None])
    got_eager = ge.engine.model_verify(vt[None], vpos[None])
    assert torch.equal(got_graph, got_eager), "retrieval verify: graph replay and eager forward differ"
    mutants = [
        ("RoPE positions + 1", ref.forward(vt, vpos + 1, retrieval_attend(ref, rK, rV, B))),
        ("ln1 and ln2 swapped", ref.forward(vt, vpos, retrieval_attend(ref, rK, rV, B), swap_norms=True)),
        ("gate and up swapped", ref.forward(vt, vpos, retrieval_attend(ref, rK, rV, B), swap_gate_up=True)),
    ]
    want = ref.forward(vt, vpos, retrieval_attend(ref, rK, rV, B))
    check_logits("retrieval verify", got_graph, want, mutants)

    # 4. full-KV verify of gamma + 2 rows (full_kv_callables[8], kv_len from seq_len_dev), then one decode step
    ft = extra[gamma + 1:2 * gamma + 3]
    fpos = torch.arange(P, P + gamma + 2, device=DEV)
    got = ge.inference(ft[None])
    assert kv.seq_len == P + gamma + 2
    lim = fpos.clone()
    mutants = [
        ("layer 1 attends to layer 0's K/V", ref.forward(ft, fpos, ref.full_kv(P, lim, kv_of_layer=lambda l: 0))),
        ("kv_len short by the row count", ref.forward(ft, fpos, ref.full_kv(P, lim - (gamma + 2)))),
    ]
    want = ref.forward(ft, fpos, ref.full_kv(P, lim))
    check_logits("full-KV verify", got, want, mutants)

    dt = extra[2 * gamma + 3:2 * gamma + 4]
    p1 = P + gamma + 2
    got = ge.decode_step(dt)
    assert kv.seq_len == p1 + 1
    dpos = torch.tensor([p1], device=DEV)
    mutants = [("decode at kv_len - 1", ref.forward(dt, dpos, ref.full_kv(p1, dpos - 1)))]
    want = ref.forward(dt, dpos, ref.full_kv(p1, dpos))
    check_logits("decode step", got, want, mutants)

    # 5. tail update: the committed tokens P..P+8 overwrite the budget tail; verify rows repeating them attend to them
    ge.update_graph_cache()
    n_new = kv.seq_len - P
    stale = [k.clone() for k in rK], [v.clone() for v in rV]
    for l in range(LAYERS):
        rK[l][:, B - n_new:B], rV[l][:, B - n_new:B] = ref.K[l][:, P:P + n_new], ref.V[l][:, P:P + n_new]
        assert torch.equal(gc.key_store[l, :, B - n_new:B], kv.key_store[l, :, P:P + n_new])
        assert torch.equal(gc.value_store[l, :, B - n_new:B], kv.value_store[l, :, P:P + n_new])
    ut = torch.cat([ft, dt])[:gamma + 1]
    upos = torch.arange(kv.seq_len, kv.seq_len + gamma + 1, device=DEV)
    got = ge.graph_verify(ut[None], upos[None])
    mutants = [("retrieval verify without the tail update", ref.forward(ut, upos, retrieval_attend(ref, *stale, B)))]
    want = ref.forward(ut, upos, retrieval_attend(ref, rK, rV, B))
    check_logits("retrieval verify after the tail update", got, want, mutants)


# ---------------------------------------------------------------------------------------------------------------------
# cfg5: 13B-wide, 49 152-token prompt, 512-node tree verify over the full KV, path compaction, decode
# ---------------------------------------------------------------------------------------------------------------------
@torch.inference_mode()
def test_cfg5_width_tree_verify_compaction_and_decode():
    P = 49152
    gm = load_grow_map("512")
    T = gm["size"]
    cfg, sd = production_model("llama-13B-128K", seed=21)
    ge = build_engine(cfg, sd, P, P + T + 64)
    kv = ge.engine.kv_cache
    target = ge.engine.model
    ref = Reference(cfg, sd, P + T + 64)
    prompt = random_ids(P, seed=22)

    ge.inference(prompt[None, :-1])
    ref.prefill(prompt[:-1])
    print(f"\n  reference prefill: layer-0 causal attention over {P - 1} rows took {ref.prefill_attention_seconds:.1f} s")
    check_kv_store(kv, ref, P - 1)
    logits = ge.inference(prompt[None, -1:])
    want = ref.forward(prompt[-1:], torch.tensor([P - 1], device=DEV), ref.full_kv(P - 1, torch.tensor([P - 1], device=DEV)))
    check_logits("last prompt token", logits, want)

    # the tree: positions depth + seq_len, one masked pass over the full KV per layer (tp.py tree_verify_inference)
    seq = kv.seq_len
    mask = gm["mask"].to(DEV).bool()
    depth = gm["depth"].to(DEV)
    bits = pack_mask_bits(gm["mask"]).to(DEV)
    leaf = int(torch.argmax(gm["depth"]))
    parent = {ch: p for p, chs in enumerate(gm["Successors"]) for ch in chs}
    path = [leaf]
    while path[-1] in parent:
        path.append(parent[path[-1]])
    path = path[::-1]
    assert path[0] == 0 and len(path) == int(gm["depth"].max()) + 1
    tokens = random_ids(T, seed=23)
    tokens[parent[leaf]] = tokens[leaf]  # the leaf's tied heads find their own token one position back
    tpos = depth + seq
    got = target.forward_tree_verify(tokens[None], kv, tpos[None], bits)
    assert kv.seq_len == seq + T

    def tree_attend(pos_mask):
        def attend(l, q, k, v):
            ref.K[l][:, seq:seq + T], ref.V[l][:, seq:seq + T] = k.transpose(0, 1), v.transpose(0, 1)
            lim = torch.full((T,), seq + T - 1, device=DEV)
            return attention_ref(q, ref.K[l], ref.V[l], lim, ref.scale, tree=pos_mask, tree_start=seq, heads=4, rows=T)
        return attend

    # The weakest control (excess ~1.4 at the bound): in layer 0 the parent's V equals the leaf's own (same token), so
    # clearing the parent only moves weight from the leaf's token to the rest of the keys.
    cut = mask.clone()
    cut[leaf, parent[leaf]] = False
    mutants = [
        ("one ancestor bit cleared", ref.forward(tokens, tpos, tree_attend(cut))),
        ("rotated at the slot index", ref.forward(tokens, seq + torch.arange(T, device=DEV), tree_attend(mask))),
    ]
    want = ref.forward(tokens, tpos, tree_attend(mask))
    check_logits("tree verify (512 rows)", got, want, mutants)

    # compact the accepted root-to-leaf path (spectree.py verify): the path's rows move to slots seq.., bit for bit; then
    # one decode step behind them reads the compacted rows (its own token repeats the leaf's)
    src = torch.tensor(path, device=DEV) + seq
    n = len(path)
    moved = kv.key_store[:, :, src].clone(), kv.value_store[:, :, src].clone()
    kv.gather_kv_incremental(path, seq)
    assert kv.seq_len == seq + n
    assert torch.equal(kv.key_store[:, :, seq:seq + n], moved[0]) and torch.equal(kv.value_store[:, :, seq:seq + n], moved[1])
    for l in range(LAYERS):
        ref.K[l][:, seq:seq + n], ref.V[l][:, seq:seq + n] = ref.K[l][:, src], ref.V[l][:, src]
    dt = tokens[leaf:leaf + 1]
    dpos = torch.tensor([seq + n], device=DEV)
    got = ge.decode_step(dt)
    want = ref.forward(dt, dpos, ref.full_kv(seq + n, dpos))
    check_logits("decode after the path compaction", got, want)
