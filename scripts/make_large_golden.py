"""Generate tests/golden/large_*.npz from the REAL reference orchestrator: designs of 65..128 columns (paired designs
``~subject + condition`` of 64, 100 and 127 subjects, a factor with 70 levels).  TEST INFRASTRUCTURE: writes only the ``large_*``
fixtures, every other golden stays untouched.

    PYDESEQ2_SRC=<PyDESeq2 0.5.3 checkout> python scripts/make_large_golden.py [case ...]

Built on scripts/make_wide_golden.py (``paired_design``, ``_written``) and the existing generators, so the layouts are those of
the ``wide_*`` fixtures:

* ``large_<case>``     -- ``deseq2()`` + ``summary()``, as ``sf_e2e_*``;
* ``large_ct_<case>``  -- several ``DeseqStats(dds, contrast=c)`` on one fit, as ``ct_*``;
* ``large_vst_<case>`` -- ``vst(use_design=True)``, as ``vst_*``.
"""
from __future__ import annotations

import itertools
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_wide_golden as mwg  # noqa: E402  (the reference's import path, the generators and their helpers)
import numpy as np  # noqa: E402

mcg, sfg, vg = mwg.mcg, mwg.sfg, mwg.vg
G = 300


def e2e(name, counts, X, contrast):
    mwg._written(sfg.gen_e2e, "large_", name, counts, X, np.asarray(contrast, dtype=float), dict(size_factors_fit_type="ratio"))


def paired(subjects, seed):
    X = mwg.paired_design(subjects)
    return X, mcg.counts_for(X, G, seed)


def levels_p70():
    """70 levels x 7 replicates (N = 490): the lin_reg_mu branch; planted outliers are replaced and refitted, and gene 1, whose
    only counts are an outlier, becomes all-zero after the replacement."""
    X, _ = mcg.factor_design(70, 7)
    c = mcg.counts_for(X, G, 72)
    rng = np.random.default_rng(73)
    for g in rng.choice(np.arange(2, G), 12, replace=False):
        c[rng.integers(X.shape[0]), g] = int(c[:, g].max() * 400 + 5000)  # Cook's distance scales with 1 / p
    c[:, 0] = 0
    c[:, 1] = 0
    c[9, 1] = 90000
    return X, c


def main(which):
    if "paired_p65" in which:
        X, c = paired(64, 81)
        e2e("paired_p65", c, X, np.eye(65)[64])
    if "paired_p101" in which or "vst" in which:
        X, c = paired(100, 82)
        if "paired_p101" in which:
            e2e("paired_p101", c, X, np.eye(101)[100])
        if "vst" in which:
            mwg._written(vg.gen, "large_vst_", "paired_p101_design", c, X, use_design=True)
    if "paired_p128" in which:
        X, c = paired(127, 83)
        e2e("paired_p128", c, X, np.eye(128)[127])
    if "levels_p70_outliers" in which or "ct" in which:
        X, c = levels_p70()
        if "levels_p70_outliers" in which:
            e2e("levels_p70_outliers", c, X, np.eye(70)[3])
        if "ct" in which:
            pairs = []
            for i, j in list(itertools.combinations(range(70), 2))[::121]:
                v = np.zeros(70)
                v[j] += 1.0
                if i:
                    v[i] -= 1.0
                pairs.append(dict(contrast=v))
            mwg._written(mcg.gen, "large_", "ct_levels_p70", c, X, pairs,
                         expect=lambda r: r["final_refitted"].sum() > 0 and r["final_new_all_zero"].sum() == 1)


if __name__ == "__main__":
    main(set(sys.argv[1:]) or {"paired_p65", "paired_p101", "paired_p128", "levels_p70_outliers", "ct", "vst"})
