"""Pearson chi-square against a known distribution, for the tests that check a sampler emits the target's p."""
import numpy as np

Z_1E6 = 4.753424308822899  # standard normal quantile at 1 - 10^-6


def chi2_threshold(df: int) -> float:
    """Upper 10^-6 quantile of chi-square(df), Wilson-Hilferty."""
    a = 2.0 / (9.0 * df)
    return df * (1.0 - a + Z_1E6 * np.sqrt(a)) ** 3


def chi2(counts: np.ndarray, probs: np.ndarray):
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
