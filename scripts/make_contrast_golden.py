"""Generate tests/golden/ct_*.npz from the REAL reference orchestrator: one ``DeseqDataSet.deseq2()`` followed by several
``DeseqStats(dds, contrast=...)`` on the same dataset (ds.py:303-360 once per contrast).  TEST INFRASTRUCTURE: writes only the
``ct_*`` fixtures, every other golden stays untouched.

    PYDESEQ2_SRC=<PyDESeq2 0.5.3 checkout> python scripts/make_contrast_golden.py

The reference is imported through the shims of ``oracle/make_golden.py``.  Contrasts are numeric vectors (the shim has no formula
contrasts).  Each file holds the counts and design; the dataset's final LFC, dispersions, size factors, ``_normed_means``,
replaced / refitted / new-all-zero genes and ``cooks_outlier()``; and per contrast ``k``: ``c{k}_contrast``, ``c{k}_lfc_null``,
``c{k}_alt`` ("" for None), ``c{k}_cooks_filter`` / ``c{k}_independent_filter`` / ``c{k}_alpha`` / ``c{k}_prior_lfc_var`` (NaN for
None), the five ``results_df`` columns after ``baseMean`` (that one once, ``final_baseMean``) and the unfiltered ``statistics`` / ``SE`` / ``p_values`` of ``run_wald_test``.
"""
from __future__ import annotations

import itertools
import os
import sys
import warnings

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_size_factor_golden as sfg  # noqa: E402  (sets up the reference's import path through oracle/make_golden.py)
import numpy as np  # noqa: E402

mg = sfg.mg


def factor_design(levels, reps, batch=False):
    """Expanded treatment coding of a factor with `levels` levels, `reps` samples each (+ a two-level batch column)."""
    lv = np.repeat(np.arange(levels), reps)
    X = np.zeros((len(lv), levels))
    X[:, 0] = 1.0
    for j in range(1, levels):
        X[:, j] = lv == j
    if batch:
        X = np.c_[X, (np.arange(len(lv)) % 2).astype(float)]
    return X, lv


def counts_for(X, G, seed):
    """Negative-binomial counts whose dispersions follow DESeq2's parametric trend a0 + a1 / mean (the trend fit converges)."""
    rng = np.random.default_rng(seed)
    beta = np.c_[rng.normal(5.0, 1.5, G), rng.normal(0.0, 1.0, (G, X.shape[1] - 1)) * (rng.random((G, 1)) < 0.4)]
    sf = np.exp(rng.normal(0.0, 0.2, X.shape[0]))
    mu = sf[:, None] * np.exp(X @ beta.T)
    d = (0.05 + 2.0 / np.exp(beta[:, 0])) * np.exp(rng.normal(0, 0.3, G))
    return rng.negative_binomial(1 / d, 1 / (1 + mu * d)).astype(np.int64)


def gen(name, counts, X, tests, dds_kwargs=None, expect=None):
    from pydeseq2.ds import DeseqStats

    N, G = counts.shape
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        dds = sfg._dataset(counts, X, **(dds_kwargs or {}))
        dds.deseq2()
    assert dds.var["fitted_dispersions"].nunique() > 1, f"ct_{name}: the parametric trend did not converge"
    replaced = np.asarray(dds.var["replaced"], dtype=bool) if "replaced" in dds.var else np.zeros(G, bool)
    refitted = np.asarray(dds.var["refitted"], dtype=bool) if "refitted" in dds.var else np.zeros(G, bool)
    new_zero = np.isin(dds.var_names, np.asarray(getattr(dds, "new_all_zeroes_genes", []), dtype=str))
    out = dict(counts=counts, design=X, final_LFC=dds.varm["LFC"].values, final_dispersions=dds.var["dispersions"].values,
               final_size_factors=dds.obs["size_factors"].values, final_normed_means=dds.var["_normed_means"].values,
               final_replaced=replaced.astype(float), final_refitted=refitted.astype(float), final_new_all_zero=new_zero.astype(float),
               final_cooks_outlier=np.asarray(dds.cooks_outlier(), dtype=float), n_contrasts=np.int64(len(tests)))
    for k, t in enumerate(tests):
        kw = dict(cooks_filter=t.get("cooks_filter", True), independent_filter=t.get("independent_filter", True),
                  alpha=t.get("alpha", 0.05), prior_LFC_var=t.get("prior_lfc_var"), lfc_null=t.get("lfc_null", 0.0),
                  alt_hypothesis=t.get("alt"))
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            ds = DeseqStats(dds, contrast=np.asarray(t["contrast"], dtype=float), inference=mg.ref_inference(), quiet=True, **kw)
            ds.run_wald_test()
            unf = dict(statistics=ds.statistics.values.copy(), SE=ds.SE.values.copy(), p_values=ds.p_values.values.copy())
            ds.summary()
        res = ds.results_df
        out["final_baseMean"] = res["baseMean"].values
        c = f"c{k:02d}_"
        out.update({c + "contrast": np.asarray(t["contrast"], dtype=float), c + "lfc_null": np.float64(kw["lfc_null"]),
                    c + "alt": np.array(kw["alt_hypothesis"] or ""), c + "cooks_filter": np.float64(kw["cooks_filter"]),
                    c + "independent_filter": np.float64(kw["independent_filter"]), c + "alpha": np.float64(kw["alpha"]),
                    c + "prior_lfc_var": np.asarray(kw["prior_LFC_var"] if kw["prior_LFC_var"] is not None else np.nan, dtype=float),
                    c + "log2FoldChange": res["log2FoldChange"].values,
                    c + "lfcSE": res["lfcSE"].values, c + "stat": res["stat"].values, c + "pvalue": res["pvalue"].values,
                    c + "padj": res["padj"].values, c + "statistics": unf["statistics"], c + "SE": unf["SE"], c + "p_values": unf["p_values"]})
    if expect is not None:
        assert expect(out), f"ct_{name}: the case does not hold what it is meant to"
    np.savez_compressed(os.path.join(mg.OUT, f"ct_{name}.npz"), **out)
    print(f"ct_{name}: N={N} G={G} p={X.shape[1]} K={len(tests)} replaced={int(replaced.sum())} refitted={int(refitted.sum())} "
          f"new_all_zero={int(new_zero.sum())} cooks_outlier={int(out['final_cooks_outlier'].sum())}")


def main():
    # a 3-level factor (A, B, C) with a batch column: B vs A, C vs A, C vs B and a weighted average of B and C against A
    X, _ = factor_design(3, 8, batch=True)
    c = counts_for(X, 200, 51)
    three = [dict(contrast=[0, 1, 0, 0]), dict(contrast=[0, 0, 1, 0]), dict(contrast=[0, -1, 1, 0]), dict(contrast=[0, 0.25, 0.75, 0])]
    gen("three_level_batch", c, X, three)

    # the same fit under every alternative, lfc_null = +-0.5 (negative only where the reference accepts it), no filtering, a prior
    prior = np.array([2.0, 1.5, 1.0, 3.0])
    alts = [dict(contrast=[0, 1, 0, 0], alt=a, lfc_null=t, cooks_filter=False, independent_filter=False, prior_lfc_var=prior)
            for a, t in (("greaterAbs", 0.5), ("lessAbs", 0.5), ("greater", 0.5), ("less", 0.5), ("greater", -0.5), ("less", -0.5),
                         (None, 0.5), (None, -0.5))]
    alts.append(dict(contrast=[0, -1, 1, 0], alt="lessAbs", lfc_null=0.5, alpha=0.1))
    gen("alternatives", c, X, alts)

    # injected outliers: genes replaced and refitted, one whose only counts are the outlier (all zero after the replacement), and
    # an all-zero gene.  No batch column here: outliers are replaced only in cells of at least 7 samples (dds.py:1301-1358)
    X3, _ = factor_design(3, 8)
    o = counts_for(X3, 200, 54)
    rng = np.random.default_rng(52)
    for g in rng.choice(np.arange(3, 200), 8, replace=False):
        o[rng.integers(24), g] = int(o[:, g].max() * 40 + 500)
    o[:, 0] = 0
    o[5, 0] = 900
    o[:, 1] = 0
    gen("outliers", o, X3, [dict(contrast=[0, 1, 0]), dict(contrast=[0, 0, 1]), dict(contrast=[0, -1, 1])], expect=lambda r: r["final_refitted"].sum() > 0 and r["final_new_all_zero"][0] == 1
        and r["final_new_all_zero"].sum() == 1 and np.isnan(r["final_LFC"][1]).all())

    # a 10-level factor (p = 10, a wide unit) with all 45 pairwise contrasts
    X10, _ = factor_design(10, 4)
    c10 = counts_for(X10, 200, 53)
    pairs = []
    for i, j in itertools.combinations(range(10), 2):
        v = np.zeros(10)
        v[j] += 1.0
        if i:
            v[i] -= 1.0
        pairs.append(dict(contrast=v))
    gen("ten_levels", c10, X10, pairs)


if __name__ == "__main__":
    main()
