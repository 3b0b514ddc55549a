"""Seeded inputs of the dispersion trend + prior launch (`pdq_trend_fit_dev`) whose `TrendOut` records are pinned bit for bit in
tests/golden/trend_prior_ref.npz (written by scripts/make_trend_prior_golden.py, checked by tests/test_gpu_trend_prior.py).

Every case returns (means, genewise, min_disp, max_disp, trigamma_c).  They cover odd and even counts of prior genes, both
kernels (one cluster below 65 536 genes, the cooperative grid kernel from there up), NaN-padded means, flat-tail genes at
min_disp, heavy ties (genes clipped to max_disp with one shared mean, a prior set whose residuals are all equal), and even counts
whose lower median lies in the bins below the upper one, with warps that see no value there.
"""
import numpy as np
from scipy.special import polygamma

MIN_DISP = 1e-8
MAX_DISP = 60.0
TRIGAMMA = float(polygamma(1, (60 - 3) / 2))  # 60 samples, 3 coefficients


def _base(n, seed, sd=0.5):
    rng = np.random.default_rng(seed)
    means = np.exp(rng.normal(4.0, 2.0, n) * np.log(2))
    gw = (4.0 / means + 0.1) * np.exp(rng.normal(0.0, sd, n))
    return rng, means, gw


def plain(n, seed):
    # every gene is finite and far above 100 * min_disp: the prior counts all n genes (odd n -> odd count)
    _, means, gw = _base(n, seed)
    return means, np.clip(gw, 1e-6, MAX_DISP)


def padded(n, seed, pad):
    # a short shard: the last `pad` means are NaN (left out of the fit and of the prior)
    means, gw = plain(n, seed)
    means[n - pad:] = np.nan
    gw[n - pad:] = 0.0
    return means, gw


def flat_tail(n, seed, k):
    # k genes at min_disp: part of the fit, excluded from the prior by the 100 * min_disp rule
    rng, means, gw = _base(n, seed, 0.6)
    gw = np.clip(gw, MIN_DISP, MAX_DISP)
    gw[rng.choice(n, k, replace=False)] = MIN_DISP
    means[rng.choice(n, 50, replace=False)] = np.nan
    return means, gw


def clipped_ties(n, seed, frac):
    # a fraction of the genes above max_disp with one shared mean: after clipping they share one residual, which then holds
    # the median, and their absolute deviations from it (all zero) hold the MAD -- far more equal values than any value bin
    rng, means, gw = _base(n, seed)
    idx = rng.choice(n, int(frac * n), replace=False)
    means[idx] = 0.5
    gw[idx] = 1e3
    return means, gw


def equal_residuals(n, seed, frac):
    # min_disp = 1e-3: most genes shape the fit from below 100 * min_disp (excluded from the prior); the others share one mean
    # and one dispersion, so every residual of the prior is the same value (a histogram range of zero width)
    rng = np.random.default_rng(seed)
    means = np.exp(rng.normal(4.0, 2.0, n) * np.log(2))
    gw = np.clip((1.0 / means + 0.002) * np.exp(rng.normal(0.0, 0.3, n)), 1e-3, 0.099)
    idx = rng.choice(n, int(frac * n), replace=False)
    means[idx] = 5.0
    gw[idx] = 0.25
    return means, gw, 1e-3


def scattered(i):
    # vector i of a seeded family with scattered shapes (300 to 6 000 genes, several blocks per cluster): sparse value bins, where
    # rank k of an even count often opens its bin and the lower median is the largest value of the bins below
    n = int(np.random.default_rng(123).integers(300, 6000, i + 1)[i])
    rng = np.random.default_rng(i)
    means = np.exp(rng.normal(rng.uniform(2, 6), rng.uniform(0.5, 3), n))
    gw = np.clip((rng.uniform(0.5, 8) / means + rng.uniform(0.01, 0.3)) * np.exp(rng.normal(0, rng.uniform(0.2, 1.2), n)), 1e-8, 120.0)
    if i % 3 == 0:
        gw[rng.choice(n, n // 10, replace=False)] = 1e-8
    return means, gw


def gapped(n, seed, empty):
    # residuals in two clusters (about -0.8 and +0.8) with an even count split between them: rank k opens its value bin and the
    # lower median is the largest value of the bins below.  The genes in `empty` sit at min_disp (left out of the prior), so on
    # the grid kernel whole warps see no value at all below that bin
    rng, means, _ = _base(n, seed)
    side = np.where(np.arange(n) % 2 == 0, -0.8, 0.8)
    gw = (4.0 / means + 0.1) * np.exp(side + rng.normal(0.0, 0.05, n))
    for lo, hi in empty:
        gw[lo:hi] = MIN_DISP
    return means, gw


CASES = {
    "plain_1000": lambda: plain(1000, 1),
    "plain_19999": lambda: plain(19999, 2),
    "plain_20000": lambda: plain(20000, 3),
    "plain_65535": lambda: plain(65535, 4),
    "padded_20000": lambda: padded(20000, 5, 37),
    "padded_70000": lambda: padded(70000, 6, 101),
    "flat_tail_20000": lambda: flat_tail(20000, 7, 300),
    "flat_tail_150001": lambda: flat_tail(150001, 8, 2000),
    "clipped_ties_20000": lambda: clipped_ties(20000, 9, 0.6),
    "clipped_ties_150001": lambda: clipped_ties(150001, 10, 0.6),
    "equal_residuals_4000": lambda: equal_residuals(4000, 11, 0.1),
    **{f"scattered_{i}": (lambda i=i: scattered(i)) for i in (5, 22, 50, 72)},
    # 70 000 genes: 35 blocks of 1024 threads on the grid kernel, a stride of 35 840 genes
    "gapped_70000": lambda: gapped(70000, 12, [(0, 4096), (35840, 39936)]),
    "gapped_1000": lambda: gapped(1000, 13, [(0, 64)]),
}


def case(name):
    means, gw, *md = CASES[name]()
    min_disp = md[0] if md else MIN_DISP
    return np.ascontiguousarray(means, np.float64), np.ascontiguousarray(gw, np.float64), min_disp, MAX_DISP, TRIGAMMA
