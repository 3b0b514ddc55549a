"""Generate tests/golden/sf_*.npz from the REAL reference orchestrator (``DeseqDataSet.fit_size_factors`` with
``size_factors_fit_type="poscounts"`` and ``control_genes``, dds.py:584-711).  TEST INFRASTRUCTURE: writes only the ``sf_*`` fixtures,
every other golden stays untouched.

    PYDESEQ2_SRC=<PyDESeq2 0.5.3 checkout> python scripts/make_size_factor_golden.py

The reference is imported through the shims of ``oracle/make_golden.py`` (same setup as every other fixture).  Three kinds of file:

* ``sf_<case>``      -- counts, fit type, the control genes as given (mask, positions or names) and resolved to a mask, and what
  ``fit_size_factors`` left behind: ``obs["size_factors"]``, ``logmeans``, ``filtered_genes``, ``var["_normed_means"]``;
* ``sf_e2e_<case>``  -- the final tables of ``deseq2()`` + ``summary()`` (the ``e2e_*`` layout of oracle/make_golden.py);
* ``sf_vst_<case>``  -- ``vst_fit()`` + ``vst_transform()`` on training samples and the transform of held-out samples.
"""
from __future__ import annotations

import os
import sys
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import make_golden as mg  # noqa: E402  (sets up the reference's import path; exits without PYDESEQ2_SRC)
import numpy as np  # noqa: E402
import pandas as pd  # noqa: E402

OUT = mg.OUT


def _normalize_indices(self, index):
    """AnnData's resolution of an ``(obs, var)`` index to positions -- slices, boolean masks, integer positions or names -- which
    ``fit_size_factors`` uses for control genes (dds.py:645).  The anndata shim of oracle/refshim_orch has no such method; it is
    added to the shim's class here, for this script only."""
    def one(ix, names):
        if isinstance(ix, slice):
            return np.arange(len(names))[ix]
        if isinstance(ix, (str, int, np.integer)):
            ix = [ix]
        a = np.asarray(ix.values if isinstance(ix, pd.Series) else ix)
        if a.dtype.kind in "OUS":
            pos = names.get_indexer(a)
            if (pos < 0).any():
                raise KeyError(f"Values {list(a[pos < 0])} are not valid obs/ var names or indices.")
            return pos
        if a.dtype == bool:
            if len(a) != len(names):
                raise IndexError(f"Boolean index of shape {a.shape} does not match the AnnData index of shape ({len(names)},).")
            return np.flatnonzero(a)
        return a.astype(int)

    rows, cols = index
    return one(rows, self.obs.index), one(cols, self.var.index)


def _with_normalize_indices():
    import anndata

    if not hasattr(anndata.AnnData, "_normalize_indices"):
        anndata.AnnData._normalize_indices = _normalize_indices


def _dataset(counts, X, **kw):
    from pydeseq2.dds import DeseqDataSet

    N, G = counts.shape
    idx = [f"s{i}" for i in range(N)]
    counts_df = pd.DataFrame(counts, index=idx, columns=[f"g{i}" for i in range(G)])
    design_df = pd.DataFrame(X, index=idx, columns=[f"x{j}" for j in range(X.shape[1])])
    meta = pd.DataFrame({"dummy": np.arange(N)}, index=idx)
    return DeseqDataSet(counts=counts_df, metadata=meta, design=design_df, inference=mg.ref_inference(), quiet=True, **kw)


def _mask(control, G):
    m = np.zeros(G, dtype=bool)
    if control is not None:
        c = np.asarray(control)
        m[c if c.dtype == bool else (np.array([int(s[1:]) for s in c]) if c.dtype.kind in "OUS" else c)] = True
    return m


def gen_sf(name, counts, fit_type, control=None, expect=None):
    """fit_size_factors(fit_type, control_genes) as the reference runs it; `expect` asserts what makes the case worth having."""
    N, G = counts.shape
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        dds = _dataset(counts, np.ones((N, 1)))
        dds.fit_size_factors(fit_type=fit_type, control_genes=control)
    sf = dds.obs["size_factors"].values
    out = dict(counts=np.asarray(counts, dtype=np.int64), fit_type=np.array(fit_type), control=_mask(control, G),
               has_control=np.float64(control is not None),
               control_given=np.asarray(control if control is not None else [], dtype=object if control is not None and
                                        np.asarray(control).dtype.kind in "OUS" else None),
               size_factors=sf, logmeans=np.asarray(dds.logmeans, dtype=float), filtered_genes=np.asarray(dds.filtered_genes, dtype=bool),
               normed_means=dds.var["_normed_means"].values,
               warned=np.float64(any("Switching to iterative" in str(w.message) for w in caught)))
    if out["control_given"].dtype == object:
        out["control_given"] = out["control_given"].astype(str)
    if expect is not None:
        assert expect(out), f"sf_{name}: the case does not hold what it is meant to"
    np.savez_compressed(os.path.join(OUT, f"sf_{name}.npz"), **out)
    print(f"sf_{name}: N={N} G={G} {fit_type} control={control is not None} NaN={int(np.isnan(sf).sum())} "
          f"filtered={int(out['filtered_genes'].sum())}")


def gen_e2e(name, counts, X, contrast, dds_kwargs):
    from pydeseq2.ds import DeseqStats

    N, G = counts.shape
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        dds = _dataset(counts, X, **dds_kwargs)
        dds.deseq2()
        ds = DeseqStats(dds, contrast=contrast, inference=mg.ref_inference(), quiet=True)
        ds.summary()
    assert not any("did not converge" in str(w.message) for w in caught), f"sf_e2e_{name}: the parametric trend did not converge"
    res = ds.results_df
    ctl = dds_kwargs.get("control_genes")
    out = dict(counts=counts, design=X, contrast=contrast, size_factors_fit_type=np.array(dds_kwargs["size_factors_fit_type"]),
               control=_mask(ctl, G), has_control=np.float64(ctl is not None),
               final_baseMean=res["baseMean"].values, final_log2FoldChange=res["log2FoldChange"].values, final_lfcSE=res["lfcSE"].values,
               final_stat=res["stat"].values, final_pvalue=res["pvalue"].values, final_padj=res["padj"].values,
               final_LFC=dds.varm["LFC"].values, final_dispersions=dds.var["dispersions"].values,
               final_genewise=dds.var["genewise_dispersions"].values, final_fitted=dds.var["fitted_dispersions"].values,
               final_size_factors=dds.obs["size_factors"].values,
               final_replaced=np.asarray(dds.var["replaced"], dtype=float) if "replaced" in dds.var else np.zeros(G),
               final_refitted=np.asarray(dds.var["refitted"], dtype=float) if "refitted" in dds.var else np.zeros(G),
               final_cooks_outlier=np.asarray(dds.cooks_outlier(), dtype=float))
    np.savez_compressed(os.path.join(OUT, f"sf_e2e_{name}.npz"), **out)
    print(f"sf_e2e_{name}: N={N} G={G} replaced={int(out['final_replaced'].sum())} refitted={int(out['final_refitted'].sum())} "
          f"cooks_outlier={int(out['final_cooks_outlier'].sum())} padj<alpha={int((res['padj'] < 0.05).sum())}")


def gen_vst(name, counts, X, n_train, dds_kwargs):
    train, held = counts[:n_train], counts[n_train:]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        dds = _dataset(train, X[:n_train], **dds_kwargs)
        dds.vst(use_design=False, fit_type="parametric")
        heldout_vst = dds.vst_transform(np.asarray(held, dtype=np.int64))
    assert dds.vst_fit_type == "parametric"
    ctl = dds_kwargs.get("control_genes")
    out = dict(counts=np.asarray(train, dtype=np.int64), design=X[:n_train], size_factors_fit_type=np.array(dds_kwargs["size_factors_fit_type"]),
               control=_mask(ctl, train.shape[1]), has_control=np.float64(ctl is not None),
               vst_counts=np.asarray(dds.layers["vst_counts"], dtype=float), vst_trend_coeffs=np.asarray(dds.uns["vst_trend_coeffs"], dtype=float),
               vst_genewise_dispersions=dds.var["vst_genewise_dispersions"].values, size_factors=dds.obs["size_factors"].values,
               logmeans=np.asarray(dds.logmeans, dtype=float), filtered_genes=np.asarray(dds.filtered_genes, dtype=bool),
               heldout_counts=np.asarray(held, dtype=np.int64), heldout_vst=np.asarray(heldout_vst, dtype=float))
    np.savez_compressed(os.path.join(OUT, f"sf_vst_{name}.npz"), **out)
    print(f"sf_vst_{name}: N={train.shape[0]} G={train.shape[1]} held-out {held.shape[0]}")


def sparse_counts(N, G, seed, zero_frac):
    """Seeded two-level counts in which EVERY gene holds at least one zero (pseudobulk-like): median of ratios cannot run on them."""
    counts, X, _ = mg.synth(N, G, "two_level", seed=seed)
    rng = np.random.default_rng(seed + 1)
    counts[rng.random((N, G)) < zero_frac] = 0
    counts[rng.integers(0, N, G), np.arange(G)] = 0
    return counts, X


def main():
    _with_normalize_indices()
    G_odd = 301
    c, X = sparse_counts(24, G_odd, 41, 0.2)
    assert (c == 0).any(0).all()
    usable_per_sample = lambda o: ((o["counts"] > 0) & o["filtered_genes"][None, :]).sum(1)  # noqa: E731
    gen_sf("poscounts_every_gene_zero", c, "poscounts",
           expect=lambda o: np.isfinite(o["size_factors"]).all() and len(set(usable_per_sample(o) % 2)) == 2)  # odd and even counts

    # genes whose positive counts are all 1 (log mean 0: left out), all-zero genes and a gene with a single 1
    c1 = c.copy()
    c1[:, :12] = (c1[:, :12] > 0).astype(np.int64)
    c1[:, 12:15] = 0
    c1[:, 15] = 0
    c1[3, 15] = 1
    gen_sf("poscounts_ones", c1, "poscounts", expect=lambda o: not o["filtered_genes"][:16].any() and np.isfinite(o["size_factors"]).all())

    # a sample with no positive count among the usable genes: its median is NaN, and the geometric mean spreads it to every sample
    c2 = c.copy()
    c2[:, :3] = (c2[:, :3] > 0).astype(np.int64)  # positive counts all 1: not usable
    c2[5, :] = 0
    c2[5, :3] = 1
    gen_sf("poscounts_sample_without_usable_gene", c2, "poscounts", expect=lambda o: np.isnan(o["size_factors"]).all())

    # median of ratios over control genes, given three ways; the ratio table needs genes without zeros
    d, X2, _ = mg.synth(20, 200, "two_level", seed=42)
    d[0, ::3] = 0
    names = [f"g{i}" for i in range(0, 200, 7)]
    pos = list(range(0, 200, 7))
    mask = np.zeros(200, dtype=bool)
    mask[pos] = True
    finite = lambda o: np.isfinite(o["size_factors"]).all()  # noqa: E731
    gen_sf("ratio_control_mask", d, "ratio", mask, expect=finite)
    gen_sf("ratio_control_positions", d, "ratio", pos, expect=finite)
    gen_sf("ratio_control_names", d, "ratio", names, expect=finite)
    # every control gene holds a zero: no finite log mean among them, NaN size factors and no error
    gen_sf("ratio_control_no_finite_gene", d, "ratio", list(range(0, 200, 3)), expect=lambda o: np.isnan(o["size_factors"]).all())
    gen_sf("poscounts_control", c, "poscounts", list(range(1, G_odd, 4)), expect=finite)
    gen_sf("poscounts_control_even", c, "poscounts", list(range(2, 202)), expect=finite)

    # deseq2() + summary() with poscounts on a table in which every gene holds a zero
    e, X3 = sparse_counts(40, 600, 43, 0.1)
    rng = np.random.default_rng(44)
    for g in rng.choice(600, 8, replace=False):  # outliers, as in the e2e_* fixtures
        e[rng.integers(40), g] = int(e[:, g].max() * 40 + 500)
    contrast = np.array([0.0, 1.0])
    gen_e2e("poscounts", e, X3, contrast, {"size_factors_fit_type": "poscounts"})
    gen_e2e("poscounts_control", e, X3, contrast, {"size_factors_fit_type": "poscounts", "control_genes": list(range(0, 600, 5))})

    # vst() with poscounts, then the held-out transform against the fit's log means and filtered genes
    v, X4 = sparse_counts(30, 400, 45, 0.15)
    gen_vst("poscounts", v, X4, 24, {"size_factors_fit_type": "poscounts"})


if __name__ == "__main__":
    main()
