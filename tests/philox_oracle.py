"""The device Philox stream of the whole-loop graph, restated on the CPU (csrc/spec_decisions.cuh, used by csrc/loop_graph.cu).

    philox4x32_10       spec_decisions.cuh:71-82    Random123's Philox4x32-10: ten rounds of two 32x32->64 multiplies
                                                    (M0 = 0xD2511F53 on c0, M1 = 0xCD9E8D57 on c2), output
                                                    (hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0), key bumped by
                                                    (0x9E3779B9, 0xBB67AE85) after every round
    element layout      spec_decisions.cuh:90-93    element i of draw `draw` of stream `seed` is lane i % 4 of
                                                    Philox(counter = (i / 4, draw_lo, draw_hi, 0), key = (seed_lo, seed_hi));
                        spec_decisions.cuh:134-141  the sampler's Philox source (ExpoFromPhilox) walks the same layout one
                                                    counter (four elements) at a time
    word -> uniform     philox_to_uniform           u = (float32(x >> 8) + 0.5f) * 2^-24, float32 round-to-nearest-even.  Above
                                                    2^23 the sum is a tie and rounds to even, so x >> 8 == 0xFFFFFF lands on 1.0
                                                    (`uniform_current`).  The kernel maps that single 1.0 to 1 - 2^-24
                                                    (0x3f7fffff), a value the sum never produces (`uniform`); every other word
                                                    keeps its bits
    exponential         philox_exponential          -logf(u) in float32 (CUDA's logf, within 1 ulp); `exponential` gives the
                                                    float64 value the device result is compared with
    one draw            philox_fill_kernel          element i < n of draw `state[1]`; state[1] += 1 per fill
"""
from __future__ import annotations

from typing import Iterable, List, Tuple, Union

import numpy as np

M0, M1 = 0xD2511F53, 0xCD9E8D57
W0, W1 = 0x9E3779B9, 0xBB67AE85
MASK32 = 0xFFFFFFFF
UNIT = 0xFFFFFF  # the 24-bit word whose current uniform is 1.0
ONE_MINUS_ULP = np.uint32(0x3F7FFFFF).view(np.float32)  # 1 - 2^-24, what the fixed map gives UNIT


def philox4x32_10(c0, c1, c2, c3, k0, k1) -> Tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray]:
    """Vectorised Philox4x32-10 over broadcastable counter words and key words; returns four uint32 arrays."""
    m = np.uint64(MASK32)
    c0, c1, c2, c3, k0, k1 = np.broadcast_arrays(*(np.asarray(v, dtype=np.uint64) & m for v in (c0, c1, c2, c3, k0, k1)))
    k0, k1 = k0.copy(), k1.copy()
    for _ in range(10):
        p0 = np.uint64(M0) * c0  # a 32x32 product fits in 64 bits
        p1 = np.uint64(M1) * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & m, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & m
        k0 = (k0 + np.uint64(W0)) & m
        k1 = (k1 + np.uint64(W1)) & m
    return tuple(c.astype(np.uint32) for c in (c0, c1, c2, c3))


def words(seed: int, draws: Union[int, Iterable[int]], n: int) -> np.ndarray:
    """uint32 [len(draws), n] (or [n] for one draw): the Philox word of elements 0 .. n-1 of each draw."""
    scalar = np.ndim(draws) == 0
    d = np.atleast_1d(np.asarray(draws, dtype=np.uint64))[:, None]
    groups = np.arange((n + 3) // 4, dtype=np.uint64)[None, :]
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    r = philox4x32_10(groups, d & np.uint64(MASK32), d >> np.uint64(32), 0, seed & MASK32, seed >> 32)
    w = np.stack(r, axis=-1).reshape(d.shape[0], -1)[:, :n]  # element 4g + lane
    return w[0] if scalar else w


def uniform_current(x: np.ndarray) -> np.ndarray:
    """The word -> uniform map as it stood: 1.0 for x >> 8 == 0xFFFFFF."""
    return ((np.asarray(x, dtype=np.uint32) >> np.uint32(8)).astype(np.float32) + np.float32(0.5)) * np.float32(2.0 ** -24)


def uniform(x: np.ndarray) -> np.ndarray:
    """The kernel's word -> uniform map: strictly inside (0, 1)."""
    u = uniform_current(x)
    return np.where(u < np.float32(1), u, ONE_MINUS_ULP).astype(np.float32)


def exponential(x: np.ndarray) -> np.ndarray:
    """float64 -log(u) of the kernel's uniforms."""
    return -np.log(uniform(x).astype(np.float64))


def unit_draws(seed: int, V: int, draws: Union[int, Iterable[int]]) -> List[Tuple[int, int]]:
    """Every (draw, element < V) whose word has x >> 8 == 0xFFFFFF, in draw then element order; `draws` is a count (draws
    0 .. draws-1) or the draw indices to scan."""
    d_all = np.arange(draws, dtype=np.uint64) if np.ndim(draws) == 0 else np.asarray(list(draws), dtype=np.uint64)
    chunk = max(1, (1 << 21) // max(1, (V + 3) // 4))
    hits = []
    for s in range(0, len(d_all), chunk):
        d = d_all[s:s + chunk]
        rows, cols = np.nonzero((words(seed, d, V) >> np.uint32(8)) == UNIT)
        hits += [(int(d[r]), int(c)) for r, c in zip(rows, cols)]
    return hits
