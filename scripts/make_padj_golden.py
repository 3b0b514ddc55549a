"""Generate tests/golden/padj_*.npz from the REAL reference: ``DeseqStats._independent_filtering`` / ``_p_value_adjustment``
(ds.py:486-542) called on a stand-in ``self`` that holds only what those two methods read (``base_mean``, ``p_values``, ``alpha``,
``dds.var_names``).  TEST INFRASTRUCTURE: writes only the ``padj_*`` fixtures, every other golden stays untouched.

    PYDESEQ2_SRC=<PyDESeq2 0.5.3 checkout> python scripts/make_padj_golden.py

The reference is imported through the shims of ``oracle/make_golden.py``.  Each file holds ``base_mean``, ``pvalues``, ``alpha``,
``independent_filter`` and the reference's ``padj``; with the filter also its ``theta``, ``cutoffs``, ``num_rej`` (the counts of
ds.py:509-514, restated with the same calls) and ``j``, the column whose BH values the reference kept -- checked here against its
``padj``.
"""
from __future__ import annotations

import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import make_golden as mg  # noqa: E402  (sets up the reference's import path; exits without PYDESEQ2_SRC)
import numpy as np  # noqa: E402
import pandas as pd  # noqa: E402


def reference_padj(base_mean, pvalues, alpha, independent_filter):
    from pydeseq2.ds import DeseqStats

    names = pd.Index([f"g{i}" for i in range(len(base_mean))])
    me = types.SimpleNamespace(base_mean=pd.Series(base_mean, index=names), p_values=pd.Series(pvalues, index=names), alpha=alpha,
                               dds=types.SimpleNamespace(var_names=names))
    (DeseqStats._independent_filtering if independent_filter else DeseqStats._p_value_adjustment)(me)
    return me.padj.to_numpy(dtype=float)


def filter_tables(base_mean, pvalues, alpha):
    """theta, cutoffs, num_rej and j of ds.py:495-525, with the reference's own lowess and scipy's BH."""
    from pydeseq2.utils import lowess
    from scipy.stats import false_discovery_control

    lower = np.mean(base_mean == 0)
    theta = np.linspace(lower, 0.95 if lower < 0.95 else 1, 50)
    cutoffs = np.quantile(base_mean, theta)
    cols = np.full((len(base_mean), 50), np.nan)
    for i, c in enumerate(cutoffs):
        use = (base_mean >= c) & ~np.isnan(pvalues)
        if use.any():
            cols[use, i] = false_discovery_control(pvalues[use], method="bh")
    num_rej = (cols < alpha).sum(0).astype(int)
    fit = lowess(theta, num_rej, frac=1 / 5)
    j = 0
    if num_rej.max() > 10:
        res = num_rej[num_rej > 0] - fit[num_rej > 0]
        above = np.where(num_rej > fit.max() - np.sqrt(np.mean(res**2)))[0]
        j = int(above[0]) if above.size else 0
    return theta, cutoffs, num_rej, j, cols[:, j]


def gen(name, base_mean, pvalues, alpha=0.05, independent_filter=True, expect_j=None):
    base_mean, pvalues = np.asarray(base_mean, dtype=float), np.asarray(pvalues, dtype=float)
    padj = reference_padj(base_mean, pvalues, alpha, independent_filter)
    out = dict(base_mean=base_mean, pvalues=pvalues, alpha=alpha, independent_filter=independent_filter, padj=padj)
    if independent_filter:
        theta, cutoffs, num_rej, j, col = filter_tables(base_mean, pvalues, alpha)
        assert np.array_equal(col, padj, equal_nan=True), f"padj_{name}: the restated column {j} is not the reference's padj"
        assert expect_j is None or expect_j(j), f"padj_{name}: j = {j}"
        out.update(theta=theta, cutoffs=cutoffs, num_rej=num_rej, j=j)
    np.savez_compressed(os.path.join(mg.OUT, f"padj_{name}.npz"), **out)
    print(f"padj_{name}: G={len(base_mean)}" + (f" j={out['j']} max num_rej={out['num_rej'].max()}" if independent_filter else ""))


def typical(G, rng, zero=0.02, nan=0.05):
    """Log-normal base means (a share of exact zeros) and p-values that carry signal only in the better expressed genes, so that
    filtering out the low ones pays: the filter keeps a cutoff above the first."""
    bm = np.exp(rng.normal(3.0, 2.0, G))
    bm[rng.random(G) < zero] = 0.0
    signal = (rng.random(G) < 0.3) & (bm > np.quantile(bm, 0.4))
    p = np.where(signal, rng.beta(0.1, 8.0, G), rng.random(G))
    p[rng.random(G) < nan] = np.nan
    return bm, p


def main():
    rng = np.random.default_rng(20261017)
    gen("typical", *typical(20000, rng), expect_j=lambda j: j > 0)
    bm, p = typical(3000, rng, zero=0.96)
    gen("mostly_zero", bm, p)
    gen("few_rejections", np.exp(rng.normal(2.0, 1.5, 800)), rng.uniform(0.2, 1.0, 800), expect_j=lambda j: j == 0)
    # ties everywhere: base means from six values, p-values from a handful, exact 0 and 1 included
    G = 4000
    bm = rng.choice([0.0, 0.5, 1.0, 3.0, 10.0, 100.0], G)
    p = rng.choice([0.0, 1e-6, 1e-4, 0.003, 0.02, 0.04, 0.3, 1.0], G, p=[0.05, 0.1, 0.1, 0.15, 0.15, 0.1, 0.25, 0.1])
    p[rng.random(G) < 0.03] = np.nan
    gen("ties", bm, p)
    gen("ties_alpha_0_1", bm, p, alpha=0.1)
    gen("g1", [5.0], [0.01])
    gen("g2", [0.0, 4.0], [0.03, 0.2])
    gen("g3", [1.0, 2.0, 3.0], [0.001, np.nan, 0.04])
    # one tested gene above the upper cutoffs: one-member subsets (scipy returns the lone p-value unclipped)
    bm = np.r_[np.zeros(30), np.linspace(1, 2, 9), 1000.0]
    p = np.r_[rng.random(30), rng.random(9) * 0.02, 0.004]
    gen("one_member", bm, p)
    gen("no_filter", *typical(5000, rng), independent_filter=False)


if __name__ == "__main__":
    main()
