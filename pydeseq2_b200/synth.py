"""Synthetic negative-binomial count generator (SURVEY.md §8(d), BASELINE.md §3).

Modelled on DESeq2's ``makeExampleDESeqDataSet`` (which the reference's shipped
``datasets/synthetic`` also derives from, ``datasets/README.md:6-8``):
per gene ``beta0/ln2 ~ N(4, 2)``, other coefficients ``/ln2 ~ N(0, 0.5)``,
``alpha_g = 4/exp(beta0) + 0.1``, ``sf_i = exp(N(0, 0.2))``, ``y ~ NB(mean=sf_i*exp(x_i.beta_g),
size=1/alpha_g)`` as int64 in the reference's native layout: (N samples, G genes), C-contiguous,
gene index fastest-varying (``dds.py:245-249``).
"""
from __future__ import annotations

import numpy as np

LN2 = np.log(2.0)

DESIGNS = ("two_level", "factorial", "continuous", "intercept", "five", "eight")


def design_matrix(N: int, kind: str, seed: int = 0) -> np.ndarray:
    """The three design shapes BASELINE.json's configs name."""
    i = np.arange(N)
    cond = (i >= N // 2).astype(float)
    if kind == "two_level":  # C2 / C5: p=2, lin_reg_mu branch of dds.py:747-756
        cols = [np.ones(N), cond]
    elif kind == "factorial":  # C3: p=3, four unique rows -> IRLS-initialised mu_hat (dds.py:757-765)
        cols = [np.ones(N), cond, (i % 2).astype(float)]
    elif kind == "continuous":  # C4: p=3 with a continuous covariate
        z = np.random.default_rng(seed + 7919).normal(0.0, 1.0, N)
        cols = [np.ones(N), cond, z]
    elif kind == "intercept":  # p=1 (the reference fits this for VST / iterative size factors, dds.py:425-430)
        cols = [np.ones(N)]
    elif kind == "five":  # p=5: two binary factors, a 3-level factor (two dummies), no continuous term
        cols = [np.ones(N), cond, (i % 2).astype(float), (i % 3 == 1).astype(float), (i % 3 == 2).astype(float)]
    elif kind == "eight":  # p=8 (the largest supported): three factors (one with 3 levels) and three continuous covariates
        z = np.random.default_rng(seed + 7919).normal(0.0, 1.0, (3, N))
        cols = [np.ones(N), cond, (i % 2).astype(float), (i % 3 == 1).astype(float), (i % 3 == 2).astype(float), z[0], z[1], z[2]]
    else:
        raise ValueError(f"unknown design kind {kind!r}; expected one of {DESIGNS}")
    return np.ascontiguousarray(np.stack(cols, axis=1))


def make_counts(N: int, G: int, kind: str = "two_level", seed: int = 0, chunk: int = 1 << 16, mean_log2: float = 4.0,
                sample_seed: int | None = None):
    """Return ``(counts int64 (N, G), X float64 (N, p), truth dict)``.  ``mean_log2`` shifts the expression level
    (4 = the reference-like default; 18 gives counts of 1e5-1e7 like the reference's ``large_counts`` test).
    ``sample_seed``: draw the per-SAMPLE quantities (design matrix, true size factors) from this seed and only the per-gene
    ones from ``seed`` -- gene shards of one cohort (same samples, different genes) are ``sample_seed`` fixed, ``seed`` = rank."""
    rng = np.random.default_rng(seed)
    X = design_matrix(N, kind, seed if sample_seed is None else sample_seed)
    p = X.shape[1]
    if sample_seed is None:
        sf = np.exp(rng.normal(0.0, 0.2, N))
    else:
        sf = np.exp(np.random.default_rng(sample_seed + 1000003).normal(0.0, 0.2, N))
    beta = np.empty((G, p))
    beta[:, 0] = rng.normal(mean_log2, 2.0, G) * LN2
    beta[:, 1:] = rng.normal(0.0, 0.5, (G, p - 1)) * LN2
    alpha = 4.0 / np.exp(beta[:, 0]) + 0.1
    counts = np.empty((N, G), dtype=np.int64)
    for g0 in range(0, G, chunk):  # bounded temporaries for the 10^6-gene config
        g1 = min(G, g0 + chunk)
        mu = sf[:, None] * np.exp(X @ beta[g0:g1].T)
        size = 1.0 / alpha[g0:g1]
        counts[:, g0:g1] = rng.negative_binomial(size[None, :], size[None, :] / (size[None, :] + mu))
    return counts, X, {"beta": beta, "alpha": alpha, "sf": sf}
