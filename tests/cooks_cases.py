"""Seeded inputs of Cook's distances (cooks_checks.py), generated at test time: counts, size factors, a design, mu and hat
diagonals, and the F cutoff of the call (dds.py:1073).

Every case holds, in its first columns, the genes the decisions turn on (SPECIAL): an all-zero gene, two samples with
equal maximal distances and counts on either side of the rest (first-occurrence argmax), an outlier with exactly 2 and one with
exactly 3 larger counts elsewhere, and outliers planted 1e-6 (relative) above and below the cutoff.  The other genes are
negative binomial, a fifth of them zero-inflated so that ties of zeros straddle the trim cut, with mu near the truth and hat
diagonals of about p / N, one percent of them pushed towards 1 (up to 1 - 1e-6)."""
import numpy as np
from scipy.stats import f as f_dist

import cooks_checks as cc
from edge_cases import _design
from team_checks import paired_design

SPECIAL = ("all_zero", "tied_argmax", "two_larger", "three_larger", "above_cutoff", "below_cutoff")
PLANT_REL = 1e-6


def levels(sizes, rng):
    """Intercept and L - 1 indicators of an L-level factor whose levels hold `sizes` samples, in shuffled sample order."""
    lv = rng.permutation(np.repeat(np.arange(len(sizes)), sizes))
    X = np.zeros((lv.size, len(sizes)))
    X[:, 0] = 1.0
    for k in range(1, len(sizes)):
        X[lv == k, k] = 1.0
    return X


def continuous(N, rng):
    return np.stack([np.ones(N), rng.normal(size=N)], axis=1)


# name -> (tier, design builder(rng), G); N follows from the design
def _cases():
    c = {}
    for p in (1, 2, 3, 5, 8, 12, 16):
        c[f"width_p{p}"] = ("narrow", lambda rng, p=p: _design(rng, 8 * p + 40, p), 40)
    c["width_p17_paired"] = ("wide", lambda rng: paired_design(17, rng), 24)
    c["width_p21_levels"] = ("wide", lambda rng: levels([4] * 21, rng), 24)
    c["width_p33"] = ("wide", lambda rng: _design(rng, 200, 33), 24)
    c["width_p64_levels"] = ("wide", lambda rng: levels([3] * 64, rng), 24)
    c["width_p65_paired"] = ("large", lambda rng: paired_design(65, rng), 16)
    c["width_p70_levels"] = ("large", lambda rng: levels([3, 4] * 35, rng), 16)
    c["width_p101"] = ("large", lambda rng: _design(rng, 420, 101), 16)
    c["width_p128_levels"] = ("large", lambda rng: levels([3, 4, 5, 3] * 32, rng), 16)
    c["cells_3_to_200"] = ("narrow", lambda rng: levels([3, 4, 7, 8, 23, 24, 25, 31, 32, 33, 200], rng), 40)
    c["cells_mixed_singletons"] = ("narrow", lambda rng: levels([5, 1, 2, 9, 1, 26, 2, 3], rng), 40)
    for N in (3, 7, 8, 15, 16, 17):
        c[f"nocell_n{N}"] = ("narrow", lambda rng, N=N: continuous(N, rng), 40)
    c["nocell_paired_p5"] = ("narrow", lambda rng: paired_design(5, rng), 40)
    return c


CASES = _cases()
NARROW = [k for k, v in CASES.items() if v[0] == "narrow"]
WIDE = [k for k, v in CASES.items() if v[0] != "narrow"]

# GPU only.  Default lanes: T = 8 from G ~ 17 k genes, 16 from ~8.5 k on a 132-SM H100 (pdq_api.cu pick_lgT), whose per-gene
# staging of 2 * 8 * N bytes then exceeds 96 KB per block and widens the lane groups.  The references are computed on
# CHECK_GENES genes of those (the special genes and a seeded sample).
WIDENED = {
    "widened_n400": ("narrow", lambda rng: levels([200, 200], rng), 17000),
    "widened_n500": ("narrow", lambda rng: levels([100] * 5, rng), 17000),
    "widened_n1000": ("narrow", lambda rng: levels([250] * 4, rng), 8500),
    "widened_n3000": ("narrow", lambda rng: levels([1000] * 3, rng), 8500),
}
CHECK_GENES = 400
# above the shared-memory ceiling of the staging (about 3 400 samples in cells for k_cooks, 14 500 for k_wide_cooks)
CEILING = {
    "ceiling_n4000_p2": ("narrow", lambda rng: levels([2000, 2000], rng), 48),
    "ceiling_n8000_p2": ("narrow", lambda rng: levels([4000, 4000], rng), 48),
    "ceiling_n4000_p5_nocell": ("narrow", lambda rng: _design(rng, 4000, 5), 48),
    "ceiling_n8000_p5": ("narrow", lambda rng: levels([1600] * 5, rng), 48),
    "ceiling_n16000_p17": ("wide", lambda rng: levels([941] * 16 + [944], rng), 24),
}
ALL = {**CASES, **WIDENED, **CEILING}


def _seed(name):
    return [sum(name.encode()), len(name)]


def make(name):
    """The inputs of case `name` (a key of ALL)."""
    tier, build, G = ALL[name]
    rng = np.random.default_rng(_seed(name))
    X = np.ascontiguousarray(build(rng), dtype=np.float64)
    N, p = X.shape
    sf = np.exp(rng.normal(0.0, 0.25, N))
    base = np.exp(rng.normal(3.0, 1.5, G))
    eff = rng.normal(0.0, 0.3, (p, G))
    eff[0] = 0.0
    mu_true = sf[:, None] * base[None, :] * np.exp(np.clip(X @ eff, -4, 4))
    alpha = 0.05 + 2.0 / base
    r = 1.0 / alpha
    counts = rng.negative_binomial(r[None, :], r[None, :] / (r[None, :] + mu_true)).astype(np.int64)
    zi = rng.random(G) < 0.2
    counts[:, zi] *= rng.random((N, int(zi.sum()))) >= 0.6
    mu = mu_true * np.exp(rng.normal(0.0, 0.05, (N, G)))
    hat = np.clip(rng.uniform(0.5, 1.5, (N, G)) * p / N, 1e-4, 0.95)
    high = rng.random((N, G)) < 0.01
    hat[high] = 1.0 - 10.0 ** -rng.uniform(1, 6, int(high.sum()))
    hat[0, -1] = 1.0 - 1e-6
    case = {"name": name, "tier": tier, "X": X, "sf": sf, "counts": counts, "mu": mu, "hat": hat,
            "cutoff": float(f_dist.ppf(0.99, p, N - p))}
    _plant(case, rng)
    for k in ("counts", "mu", "hat"):
        case[k] = np.ascontiguousarray(case[k])
    return case


def _plant(case, rng):
    """The special genes (SPECIAL, columns 0..5).  Their other samples have y = mu = 10 + a small integer, so a distance of 0."""
    X, counts, mu, hat = case["X"], case["counts"], case["mu"], case["hat"]
    N = X.shape[0]
    cells, global_mode = cc.cells_of(X)
    big = max(cells, key=len)          # the two deciding samples sit in the largest cell (any sample in the no-cell mode)
    a, b = int(big.min()), int(big.max())
    rest = np.setdiff1d(np.arange(N), [a, b])
    for g in range(len(SPECIAL)):
        y = 10 + rng.integers(0, 3, N)
        counts[:, g] = y
        mu[:, g] = y
        hat[:, g] = np.clip(rng.uniform(0.5, 1.5, N) * X.shape[1] / N, 1e-4, 0.95)
    counts[:, 0] = 0
    mu[:, 0] = 0.5
    # equal distances at a < b: (16 - 10)^2 = (4 - 10)^2 with equal mu and hat; only the first has fewer than 3 larger counts
    counts[a, 1], counts[b, 1] = 16, 4
    mu[[a, b], 1] = 10.0
    hat[[a, b], 1] = 0.99
    # an outlier of 50 counts with exactly 2 / 3 samples of 60 (at their mean) elsewhere
    for g, k in ((2, 2), (3, 3)):
        counts[a, g], mu[a, g], hat[a, g] = 50, 10.0, 0.99
        others = rest[:k] if len(rest) >= k else rest
        counts[others, g] = 60
        mu[others, g] = 60.0
    # 30 counts at mu = 10, the hat diagonal solved for a distance of cutoff * (1 +- PLANT_REL)
    for g, s in ((4, 1.0), (5, -1.0)):
        counts[a, g], mu[a, g] = 30, 10.0
        ref = cc.reference(case, genes=[g])
        alpha = float(ref["disp"][0])
        V = 10.0 + alpha * 100.0
        t = case["cutoff"] * (1.0 + s * PLANT_REL) * X.shape[1] * V / 400.0  # h / (1 - h)^2
        hat[a, g] = ((2 * t + 1) - np.sqrt(4 * t + 1)) / (2 * t)
