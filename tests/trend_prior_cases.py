"""Seeded inputs of the dispersion trend + prior launch (`pdq_trend_fit_dev`) whose `TrendOut` records are pinned bit for bit in
tests/golden/trend_prior_ref.npz (written by scripts/make_trend_prior_golden.py, checked by tests/test_gpu_trend_prior.py).

Every case returns (means, genewise, min_disp, max_disp, trigamma_c).  They cover odd and even counts of prior genes, both
kernels (one cluster below 65 536 genes, the cooperative grid kernel from there up), NaN-padded means, flat-tail genes at
min_disp, heavy ties (genes clipped to max_disp with one shared mean, a prior set whose residuals are all equal), and even counts
whose lower median lies in the bins below the upper one, with warps that see no value there.
"""
import functools

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


# ---- cases of the extended-precision checks (tests/trend_checks.py, tests/test_gpu_trend_ref.py) ------------------------------------
# Each returns (means, gw), (means, gw, min_disp), (means, gw, min_disp, trigamma_c) or (means, gw, min_disp, trigamma_c, max_disp).

def spread(n, seed, s):
    # means 10 (1 + s U(-1, 1)), genewise 0.3 exp(N(0, 0.5)): a constant covariate (s = 0), whose minimisers form a line with
    # interior points, and nearly constant ones, whose exact minimiser lies on a bound
    rng = np.random.default_rng(seed)
    means = 10.0 * (1.0 + s * rng.uniform(-1.0, 1.0, n))
    return means, 0.3 * np.exp(rng.normal(0.0, 0.5, n))


def bound_trend(n, seed, which):
    # "flat": genewise falling slightly with 1 / mean, so the minimiser has c1 at its bound; "inverse": a pure 1 / mean trend with a
    # slightly negative intercept, so the minimiser has c0 at its bound.  Both fits fail
    rng, means, _ = _base(n, seed)
    x = 1.0 / means
    base = 0.3 * (1.0 - 0.2 * x / x.max()) if which == "flat" else 4.0 * x - 1e-3 * 4.0 * x.min()
    return means, base * np.exp(rng.normal(0.0, 0.2, n))


def few(k):
    means = np.array([3.0, 40.0, 700.0])[:k]
    return means, (4.0 / means + 0.1) * np.array([1.3, 0.8, 1.1])[:k]


def collapse():
    # each of two means holds one gene at 1 (1.5) among 15 at 1e-9: the first round fits about their mean, so all 32 sit at a
    # ratio of about 16 or below 1e-4 and leave; the gene on the curve is left alone, and the second round has no fit
    means = np.array([10.0] * 16 + [5.0] * 16 + [1 / 0.15])
    gw = np.array([1.0] + [1e-9] * 15 + [1.5] + [1e-9] * 15 + [0.0833])
    return means, gw, 1e-10


def clipped_high(n, seed):
    # max_disp 1: a third of the prior genes are clipped, and clipping moves them from above the median residual to below it
    means, gw = plain(n, seed)
    return means, gw, MIN_DISP, TRIGAMMA, 1.0


def planted(n, seed, later=True):
    """A seeded vector with genes at every threshold of the launch: ratios to the first round's fit of 15 (1 +- 1e-6) and
    1e-4 (1 +- 1e-6), and (`later`) of 15 (1 +- 1e-6) to the second round's fit, after a few genes far above the curve have left
    (placed by fixed-point iteration in long double: the planted genes move the fit), genewise exactly
    100 min_disp and one ulp below, genes clipped at min_disp and max_disp, NaN means (all-zero genes, genewise 0), and zero
    means (an infinite covariate, genewise at min_disp)."""
    import trend_checks as tk

    rng, means, gw = _base(n, seed)
    gw = np.clip(gw, 1e-6, 10.0)
    gw[:6] = [100 * MIN_DISP, np.nextafter(100 * MIN_DISP, 0.0), 1e-10, 1e3, 1e-10, 200.0]
    means[6:9], gw[6:9] = np.nan, 0.0
    means[9:11], gw[9:11] = 0.0, MIN_DISP
    k = np.array([15 * (1 + 1e-6), 15 * (1 - 1e-6), 1e-4 * (1 + 1e-6), 1e-4 * (1 - 1e-6)])
    j = np.arange(11, 15)
    k2 = np.array([15 * (1 + 1e-6), 15 * (1 - 1e-6)])[:2 if later else 0]
    j2 = np.arange(15, 17) if later else np.arange(0)
    means[j2] = 50.0  # mid-range means, where the round-1 fit lies above the round-2 fit: their first ratio stays below 15
    far = np.arange(17, 23) if later else np.arange(0)  # far above the curve: they leave after the first round, lifting its fit
    means[far] = 50.0
    def fit(c, g):
        return c[0] + c[1] * tk.LD(1) / np.asarray(means[g], dtype=tk.LD)

    for _ in range(60):
        x, t = tk.prepare(means, gw, MIN_DISP, MAX_DISP)
        c1, c2 = tk.outer(x, t)["rounds"][:2]
        if (np.allclose(np.asarray(gw[j], dtype=tk.LD) / fit(c1, j), k, rtol=1e-9, atol=0)
                and np.allclose(np.asarray(gw[j2], dtype=tk.LD) / fit(c2, j2), k2, rtol=1e-9, atol=0)):
            break
        gw[j] = np.float64(tk.LD(k) * fit(c1, j))
        gw[j2] = np.float64(tk.LD(k2) * fit(c2, j2))
        gw[far] = np.float64(np.minimum(tk.LD(40) * fit(c1, far), tk.LD(50)))
    else:
        raise AssertionError(f"the planted genes did not settle: {np.asarray(gw[j], dtype=tk.LD) / fit(c1, j) / k - 1}, "
                             f"{np.asarray(gw[j2], dtype=tk.LD) / fit(c2, j2) / k2 - 1}")
    assert (np.asarray(gw[j2], dtype=tk.LD) / fit(c1, j2) < 15).all()  # the second-round genes survive the first round
    return means, gw


def prior_floor(n, seed, side):
    # trigamma chosen so that squared_logres - trigamma = 0.25 (1 + side 1e-6) at the reference's fit
    import trend_checks as tk

    means, gw = plain(n, seed)
    ref = tk.reference((means, gw, MIN_DISP, MAX_DISP, TRIGAMMA))
    return means, gw, MIN_DISP, float(ref["sq"] - tk.LD(0.25) * (1 + tk.LD(side) * tk.LD(1e-6)))


def dof(n, seed, k):
    # k residual degrees of freedom: trigamma(k / 2) is large, and the prior variance sits on its floor
    means, gw = plain(n, seed)
    return means, gw, MIN_DISP, float(polygamma(1, k / 2))


def no_prior(n, seed):
    # every clipped genewise below 100 min_disp: the prior has no gene, and squared_logres and prior_var are NaN
    rng, means, _ = _base(n, seed)
    return means, np.clip((0.4 / means + 0.01) * np.exp(rng.normal(0.0, 0.3, n)), 1e-3, 0.099), 1e-3


REF_CASES = {
    # thread count 256 / 512 / 1024 and cluster size 1, 2, 4, 8, 16 of the one-cluster kernel, the switch to the grid kernel, and
    # the gathered vector of 10^6 genes
    **{f"plain_{n}": (lambda n=n: plain(n, 20 + n % 97)) for n in (900, 2000, 4000, 8000, 16000, 24576, 24577, 49152, 49153, 65536)},
    "plain_1000000": lambda: plain(1000000, 21),
    **{f"spread_{s}": (lambda s=s: spread(500, 1, s)) for s in (0.0, 1e-9, 1e-6, 1e-3, 1e-2)},
    "spread_0_20000": lambda: spread(20000, 2, 0.0),
    "flat_trend": lambda: bound_trend(3000, 22, "flat"),
    "inverse_trend": lambda: bound_trend(3000, 23, "inverse"),
    **{f"few_{k}": (lambda k=k: few(k)) for k in (1, 2, 3)},
    "collapse": collapse,
    "clipped_high": lambda: clipped_high(3000, 29),
    "planted_3001": lambda: planted(3001, 24, later=False),
    "planted_70000": lambda: planted(70000, 25),
    "prior_floor_above": lambda: prior_floor(3000, 26, 1.0),
    "prior_floor_below": lambda: prior_floor(3000, 26, -1.0),
    **{f"dof_{k}": (lambda k=k: dof(2001, 27, k)) for k in (1, 2, 3)},
    "no_prior": lambda: no_prior(2000, 28),
}
# seeded cases whose exemption count must be zero; the degenerate and planted ones may hold exemptions only at their planted genes
PLANTED = {"planted_3001", "planted_70000"}


def case(name):
    return tuple(v.copy() if isinstance(v, np.ndarray) else v for v in _case(name))


@functools.lru_cache(maxsize=None)
def _case(name):
    out = (CASES.get(name) or REF_CASES[name])()
    means, gw = out[0], out[1]
    min_disp = out[2] if len(out) > 2 else MIN_DISP
    trig = out[3] if len(out) > 3 else TRIGAMMA
    max_disp = out[4] if len(out) > 4 else MAX_DISP
    return np.ascontiguousarray(means, np.float64), np.ascontiguousarray(gw, np.float64), min_disp, max_disp, trig
