"""Generate tests/golden/wide_*.npz from the REAL reference orchestrator: designs of 17..64 columns (paired designs
``~subject + condition``, a factor with 17 levels, a continuous covariate).  TEST INFRASTRUCTURE: writes only the ``wide_*`` fixtures,
every other golden stays untouched.

    PYDESEQ2_SRC=<PyDESeq2 0.5.3 checkout> python scripts/make_wide_golden.py

The reference is imported through the shims of ``oracle/make_golden.py``, and the files are written by the generators of the
existing fixtures, so they have those fixtures' layouts:

* ``wide_<case>``     -- ``deseq2()`` + ``summary()``: counts, design, contrast, the ``results_df`` columns and the final state (size
  factors, genewise / fitted / MAP dispersions, LFC, replaced / refitted / ``cooks_outlier()``), as ``sf_e2e_*``
  (scripts/make_size_factor_golden.py ``gen_e2e``);
* ``wide_ct_<case>``  -- several ``DeseqStats(dds, contrast=c)`` on one fit, as ``ct_*`` (scripts/make_contrast_golden.py);
* ``wide_vst_<case>`` -- ``vst(use_design=True)``, as ``vst_*`` (scripts/make_vst_golden.py).
"""
from __future__ import annotations

import itertools
import os
import shutil
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_contrast_golden as mcg  # noqa: E402  (sets up the reference's import path through oracle/make_golden.py)
import make_size_factor_golden as sfg  # noqa: E402
import make_vst_golden as vg  # noqa: E402
import numpy as np  # noqa: E402

mg = sfg.mg


def paired_design(subjects, covariate=False, seed=0):
    """~subject + condition (+ a continuous covariate): intercept, subject dummies 2..S, condition (last column, or the one before
    the covariate)."""
    subj = np.repeat(np.arange(subjects), 2)
    cols = [np.ones(2 * subjects)] + [(subj == s).astype(float) for s in range(1, subjects)] + [np.tile([0.0, 1.0], subjects)]
    if covariate:
        cols.append(np.random.default_rng(seed).normal(0.0, 1.0, 2 * subjects))
    return np.stack(cols, axis=1)


def _written(gen, prefix, name, *args, **kwargs):
    """Run one of the existing generators into a scratch directory and move its file to tests/golden/wide_<...>.npz."""
    tmp = tempfile.mkdtemp()
    saved = (mg.OUT, sfg.OUT, vg.OUT)
    mg.OUT = sfg.OUT = vg.OUT = tmp
    try:
        gen(name, *args, **kwargs)
    finally:
        mg.OUT, sfg.OUT, vg.OUT = saved
    (produced,) = os.listdir(tmp)
    target = os.path.join(mg.OUT, f"{prefix}{name}.npz")
    shutil.move(os.path.join(tmp, produced), target)
    shutil.rmtree(tmp)
    print(f"  -> {os.path.relpath(target)}")


def e2e(name, counts, X, contrast):
    _written(sfg.gen_e2e, "wide_", name, counts, X, np.asarray(contrast, dtype=float), dict(size_factors_fit_type="ratio"))


def main():
    G = 300
    # 20 subjects x 2 conditions: p = 21, N = 40.  Every design row is its own cell, so the reference starts the genewise search from
    # an IRLS fit (not lin_reg_mu) and no count can be replaced
    X21 = paired_design(20)
    c21 = mcg.counts_for(X21, G, 61)
    e2e("paired_p21", c21, X21, np.eye(21)[20])
    _written(vg.gen, "wide_vst_", "paired_p21_design", c21, X21, use_design=True)

    # a 17-level factor, 7 replicates each (N = 119): the lin_reg_mu branch, outliers replaced and refitted (cells of >= 7)
    X17, _ = mcg.factor_design(17, 7)
    c17 = mcg.counts_for(X17, G, 62)
    rng = np.random.default_rng(63)
    for g in rng.choice(np.arange(2, G), 12, replace=False):
        c17[rng.integers(X17.shape[0]), g] = int(c17[:, g].max() * 40 + 500)
    c17[:, 0] = 0
    c17[:, 1] = 0
    c17[9, 1] = 900  # its only counts are an outlier: all zero after the replacement
    e2e("levels_p17_outliers", c17, X17, np.eye(17)[3])
    pairs = []
    for i, j in list(itertools.combinations(range(17), 2))[::9]:
        v = np.zeros(17)
        v[j] += 1.0
        if i:
            v[i] -= 1.0
        pairs.append(dict(contrast=v))
    _written(mcg.gen, "wide_", "ct_levels_p17", c17, X17, pairs,
             expect=lambda r: r["final_refitted"].sum() > 0 and r["final_new_all_zero"].sum() == 1)

    # 31 subjects x 2 + a per-sample continuous covariate: p = 33, N = 62
    X33 = paired_design(31, covariate=True, seed=64)
    e2e("paired_covariate_p33", mcg.counts_for(X33, G, 70), X33, np.eye(33)[31])

    # 63 subjects x 2: p = 64, N = 126, the limit
    X64 = paired_design(63)
    e2e("paired_p64", mcg.counts_for(X64, G, 66), X64, np.eye(64)[63])


if __name__ == "__main__":
    main()
