"""Shared pieces of the attention tests that compare a kernel with an fp64 evaluation of the same attention, one head at a
time: the visibility rules, the reference, the tolerance and its negative-control check, and the "needle" inputs.

The query rows of a head share one direction; needle keys lie along it with large V rows of random signs, so each needle
holds a visible share of the softmax mass and the outputs are O(1).  A key that a kernel drops, double-counts or wrongly
admits then moves the output far outside the tolerance.  Rows past kv_len hold stale needles that would dominate the
softmax if they were read.  Every helper takes the head dim from its inputs (d = 64 or 128)."""
import math
import time

import pytest
import torch

from oracle import triforce_oracle as orc

# The CPU serves only to rehearse the references and the negative controls without a device; every test that launches a
# kernel is marked gpu.
DEV = "cuda" if torch.cuda.is_available() else "cpu"
Q_ALONG = 8.0       # component of every query row along its head's shared direction
NEEDLE_V = 4.0      # |V| of a needle row (random signs)
STALE_V = 16.0      # |V| of a stale row past kv_len
STALE_CHUNK = 8192  # stale rows planted per call (bounds the fp64 temporaries of a store with a short kv_len)


@pytest.fixture(autouse=True)
def report_time_and_memory(request):
    """Prints the wall time and peak device memory of each test (autouse in every module that imports it)."""
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
# fp64 reference and tolerance
# ---------------------------------------------------------------------------------------------------------------------
def visibility(R: int, n_keys: int, kv_len: int, causal: bool = False, tree: torch.Tensor = None) -> torch.Tensor:
    """bool [R, n_keys]: does query row i see key j?
    causal: row i sees key j iff j <= kv_len - R + i (the R rows are the last R keys);
    tree:   the first kv_len - T keys are seen by every row, key kv_len - T + c by the rows whose tree[i, c] is set;
    no row sees a key >= kv_len."""
    i = torch.arange(R, device=DEV)[:, None]
    j = torch.arange(n_keys, device=DEV)[None, :]
    if causal:
        vis = j <= kv_len - R + i
    else:
        T = 0 if tree is None else tree.shape[1]
        vis = (j < kv_len - T).expand(R, n_keys).clone()
        if T:
            vis[:, kv_len - T:kv_len] = tree
    return vis & (j < kv_len)


def reference(q: torch.Tensor, K: torch.Tensor, V: torch.Tensor, vis: torch.Tensor, bias: torch.Tensor = None) -> torch.Tensor:
    """One head in fp64: q [R, d], K / V [>= n, d] (fp16 store rows), vis [R, n] → softmax(scale · q Kᵀ + bias, masked by
    vis) · V, with the fp16-rounded scale of the head dim; `bias` (fp64, broadcast to [R, n]) shifts logits, e.g. by ln 2
    to count keys twice.  A row that sees no key gets zeros (as the kernels write)."""
    n = vis.shape[1]
    s = (q.double() @ K[:n].double().T) * orc.softmax_scale_fp16(q.shape[-1])
    if bias is not None:
        s += bias
    s.masked_fill_(~vis, float("-inf"))
    return torch.softmax(s, dim=-1).nan_to_num_(0.0) @ V[:n].double()


# Error budget of a kernel output against the fp64 reference, relative to the head's output scale:
#   * output rounded to fp16 ............................ <= 2^-11 |want| (half an ulp)
#   * P rounded to fp16 before the P·V MMA (the softmax denominator sums the unrounded fp32 P)
#                                                     ... <= 2^-11 sum_j p_j |v_j| / l per element, about 2^-11 of the
#                                                         head's output scale here: the needles carry most of the mass
#                                                         and the needle at the row maximum has P = 1 exactly
#   * ex2.approx.ftz (2 ulp of fp32), fp32 scores of exact fp16 products, the fp32 split merge ... below 2^-20
# Sum: about 2^-10 of the output scale.  The tolerance allows twice that: rtol 2^-9 and atol 2^-9 of the head's largest
# output, and never more than assert_attn_close's (rtol 1e-2, atol 2e-3).
RTOL = 2.0 ** -9
ATOL_CAP = 2e-3


def excess(got: torch.Tensor, want: torch.Tensor) -> float:
    """max |got - want| / (atol + RTOL |want|) over one head's [R, d] outputs, atol = min(ATOL_CAP, RTOL max|want|):
    <= 1 passes."""
    atol = min(ATOL_CAP, RTOL * want.abs().max().item())
    err = (got.double() - want).abs().nan_to_num(nan=float("inf"))
    return (err / (atol + RTOL * want.abs())).max().item()


def assert_rejected(mutants, want: torch.Tensor, what: str) -> float:
    """Negative controls: each (name, mutant reference) must fail the comparison against the real reference.  Returns the
    weakest excess."""
    weakest = float("inf")
    for name, m in mutants:
        e = excess(m, want)
        assert e > 1.0, f"{what}: the comparison does not reject the mutant '{name}' (excess {e:.3g})"
        weakest = min(weakest, e)
    return weakest


# ---------------------------------------------------------------------------------------------------------------------
# inputs with needles
# ---------------------------------------------------------------------------------------------------------------------
def base_logit(kv_len: int) -> float:
    """Needle logit (scale · q·k): background scores have a standard deviation of about scale·sqrt(Q_ALONG² + d) (1.2 at
    d = 128, 1.4 at d = 64), so the background weighs at most about kv_len·e^1; a needle at ln(kv_len) + 3 outweighs all
    of it several times."""
    return math.log(kv_len) + 3.0


class Needles:
    """Per-head unit directions u_h; query rows Q_ALONG·u_h plus noise orthogonal to u_h; needle keys b·u_h with
    q·k = Q_ALONG·b set to a chosen logit; needle V rows ±NEEDLE_V with random signs."""

    def __init__(self, H: int, seed: int, d: int = 128):
        self.H, self.d = H, d
        self.scale = orc.softmax_scale_fp16(d)
        self.g = torch.Generator(device=DEV).manual_seed(seed)
        u = torch.randn((H, d), generator=self.g, device=DEV, dtype=torch.float64)
        self.u = u / u.norm(dim=-1, keepdim=True)

    def store(self, L: int, cap: int) -> torch.Tensor:
        return torch.randn((L, self.H, cap, self.d), generator=self.g, device=DEV, dtype=torch.float16)

    def queries(self, R: int) -> torch.Tensor:
        n = torch.randn((R, self.H, self.d), generator=self.g, device=DEV, dtype=torch.float64)
        n -= (n * self.u).sum(-1, keepdim=True) * self.u
        return (Q_ALONG * self.u + n).half().contiguous()

    def plant(self, K, V, layer: int, keys, logits, v_amp: float = NEEDLE_V, head: int = None):
        """Needles at `keys` with the given logits, in every head or only in `head`."""
        keys = torch.as_tensor(list(keys), device=DEV, dtype=torch.long)
        b = torch.as_tensor(list(logits), device=DEV, dtype=torch.float64) / (self.scale * Q_ALONG)
        if head is None:
            K[layer, :, keys] = (b[None, :, None] * self.u[:, None, :]).half()
            signs = torch.randint(0, 2, (self.H, keys.numel(), self.d), generator=self.g, device=DEV).double() * 2 - 1
        else:
            K[layer, head, keys] = (b[:, None] * self.u[head][None, :]).half()
            signs = torch.randint(0, 2, (keys.numel(), self.d), generator=self.g, device=DEV).double() * 2 - 1
        V[layer, head if head is not None else slice(None), keys] = (v_amp * signs).half()


def plant_stale(nd: Needles, K, V, layer: int, kv_len: int, cap: int):
    """Rows kv_len .. cap-1 (left over from a longer sequence, e.g. after kv_compact): keys far above every needle."""
    for k0 in range(kv_len, cap, STALE_CHUNK):
        k1 = min(cap, k0 + STALE_CHUNK)
        nd.plant(K, V, layer, range(k0, k1), [base_logit(kv_len) + 8.0] * (k1 - k0), v_amp=STALE_V)
