"""Generate tests/golden/wide_shrink_*.npz from the REAL reference: apeGLM shrinkage (``lfc_shrink_nbinom_glm``) of designs of 17..64
columns.  TEST INFRASTRUCTURE: writes only the ``wide_shrink_*`` fixtures, every other golden stays untouched.  ``gen_calls`` and
``gen_tape`` take the output prefix, so scripts/make_large_shrink_golden.py writes the ``large_shrink*`` fixtures with them.

    PYDESEQ2_SRC=<PyDESeq2 0.5.3 checkout> python scripts/make_wide_shrink_golden.py

The reference is imported through the shims of ``oracle/make_golden.py``.  Two kinds of fixture:

* ``wide_shrink_<case>`` -- one call of the real ``DefaultInference.lfc_shrink_nbinom_glm`` on the reference's own final state of an
  existing ``wide_*`` fixture (scripts/make_wide_golden.py): its size factors, MAP dispersions, the MLE LFCs and Wald SEs of the
  shrunk coefficient (``mle_lfc`` / ``mle_se``, that column only), with the adapted prior scale from the reference's ``DeseqStats._fit_prior_var``.  The inputs are the
  reference's, so these fixtures do not depend on how closely the backend's own fit reproduces the reference's.  Layout of
  ``shrink_*`` (oracle/make_golden.py ``gen_shrink_calls``), except that the inverse Hessians are stored as column
  ``shrink_index`` for all genes (``inv_hessian_col``) and in full only for the first genes (``inv_hessians_head``: at most 40, and
  at most ``HEAD_BYTES`` of raw data -- 40 genes at p = 17 and 21, 15 at p = 33, 4 at p = 64), which keeps every file under
  600 KB.  ``nit`` / ``nfev``: scipy's iteration and evaluation counts per gene.
* ``wide_shrinktape_paired_p21`` -- ``deseq2()``, ``summary()`` and ``lfc_shrink(coeff=condition)`` through the real orchestrator on
  the paired p = 21 design.  ``final_log2FoldChange`` / ``final_lfcSE`` are what ds.py:414-431 writes into LFC / SE, taken from
  the call's outputs: under pandas 3 (copy-on-write) the reference's own in-place update misses ``results_df``, which keeps the MLE
  (stored as ``results_*``, as ``oracle/make_golden.py`` ``gen_shrink_tape`` does).  Also the prior scale and the flags.
"""
from __future__ import annotations

import os
import sys
import warnings

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_size_factor_golden as sfg  # noqa: E402  (sets up the reference's import path through oracle/make_golden.py)
import numpy as np  # noqa: E402

mg = sfg.mg
HEAD, HEAD_BYTES = 40, 1 << 17


def _counted_minimize():
    """Record scipy's nit / nfev of every minimize call nbinomGLM makes (the reference imports `minimize` into pydeseq2.utils)."""
    import pydeseq2.utils as ut

    inner, seen = ut.minimize, []

    def wrapped(*a, **k):
        res = inner(*a, **k)
        seen.append((int(res.nit), int(res.nfev)))
        return res

    ut.minimize = wrapped
    return seen, lambda: setattr(ut, "minimize", inner)


def gen_calls(name, source, shrink_index, adapt=True, prefix="wide_"):
    z = np.load(os.path.join(mg.OUT, f"{source}.npz"))
    counts, X = np.asarray(z["counts"], dtype=np.int64), np.asarray(z["design"], dtype=float)
    assert z["contrast"][shrink_index] == 1.0 and np.count_nonzero(z["contrast"]) == 1, "the stored SEs must be those of shrink_index"
    keep = ~(counts == 0).all(0) & np.isfinite(z["final_dispersions"])
    counts = np.ascontiguousarray(counts[:, keep])
    mle_lfc = np.asarray(z["final_LFC"], dtype=float)[keep, shrink_index]
    mle_se = np.asarray(z["final_lfcSE"], dtype=float)[keep] * np.log(2)
    prior_var = mg.real_fit_prior_var(mle_lfc, mle_se) if adapt else np.nan
    prior_scale = float(np.minimum(np.sqrt(prior_var), 1)) if adapt else 1.0
    size, offset = 1.0 / np.asarray(z["final_dispersions"], dtype=float)[keep], np.log(np.asarray(z["final_size_factors"], dtype=float))
    seen, restore = _counted_minimize()
    try:
        lfcs, ih, conv = mg.ref_inference().lfc_shrink_nbinom_glm(design_matrix=X, counts=counts, size=size, offset=offset,
                                                                 prior_no_shrink_scale=15, prior_scale=prior_scale, optimizer="L-BFGS-B",
                                                                 shrink_index=shrink_index)
    finally:
        restore()
    G, p = counts.shape[1], X.shape[1]
    head = min(HEAD, HEAD_BYTES // (8 * p * p))
    assert len(seen) == G, (len(seen), G)
    nit, nfev = np.array(seen, dtype=np.int64).T
    np.savez_compressed(os.path.join(mg.OUT, f"{prefix}shrink_{name}.npz"), counts=counts, X=X, size=size, offset=offset, mle_lfc=mle_lfc,
                        mle_se=mle_se, prior_var=np.float64(prior_var), prior_scale=np.float64(prior_scale),
                        prior_no_shrink_scale=np.float64(15.0), shrink_index=np.int64(shrink_index), lfcs=lfcs,
                        inv_hessians_head=np.ascontiguousarray(ih[:head]), inv_hessian_col=np.ascontiguousarray(ih[:, :, shrink_index]),
                        converged=np.asarray(conv, dtype=float), nit=nit, nfev=nfev)
    print(f"{prefix}shrink_{name}: G={G} p={X.shape[1]} idx={shrink_index} prior_scale={prior_scale:.4g} "
          f"converged={np.mean(conv):.3f} nfev median {int(np.median(nfev))} max {int(nfev.max())}")


def gen_tape(name, source, coeff_idx, prefix="wide_"):
    """deseq2() + summary() + lfc_shrink(coeff) through the real orchestrator on the counts and design of a wide_* / large_*
    fixture."""
    from pydeseq2.ds import DeseqStats

    z = np.load(os.path.join(mg.OUT, f"{source}.npz"))
    counts, X, contrast = np.asarray(z["counts"], dtype=np.int64), np.asarray(z["design"], dtype=float), np.asarray(z["contrast"], dtype=float)
    calls = []

    class Rec(type(mg.ref_inference())):
        def lfc_shrink_nbinom_glm(self, **k):
            res = super().lfc_shrink_nbinom_glm(**k)
            res = (res[0], res[1], np.asarray(res[2], dtype=float))  # pandas-3: float flags
            calls.append((k, res))
            return res

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        dds = sfg._dataset(counts, X, size_factors_fit_type="ratio")
        dds.inference = Rec(n_cpus=1)
        dds.deseq2()
        ds = DeseqStats(dds, contrast=contrast, inference=Rec(n_cpus=1), quiet=True)
        ds.summary()
        mle_log2 = ds.results_df["log2FoldChange"].values.copy()
        coeff = ds.LFC.columns[coeff_idx]
        prior_var = ds._fit_prior_var(coeff_idx=coeff_idx)
        ds.lfc_shrink(coeff=coeff, adapt=True)
    (k, (lfcs, ih, conv)), = calls
    res = ds.results_df
    nz = ~(counts == 0).all(0)
    assert len(lfcs) == nz.sum()
    shr_log2 = np.full(counts.shape[1], np.nan)
    shr_se = np.full(counts.shape[1], np.nan)
    shr_log2[nz] = lfcs[:, coeff_idx] / np.log(2)
    shr_se[nz] = np.sqrt(np.abs(ih[:, coeff_idx, coeff_idx])) / np.log(2)
    out = dict(counts=counts, design=X, contrast=contrast, shrink_index=np.int64(coeff_idx), prior_scale=np.float64(k["prior_scale"]),
               prior_var=np.float64(prior_var), final_log2FoldChange=shr_log2, final_lfcSE=shr_se, converged=np.asarray(conv, dtype=float),
               mle_log2FoldChange=mle_log2, results_log2FoldChange=res["log2FoldChange"].values, results_lfcSE=res["lfcSE"].values,
               results_pvalue=res["pvalue"].values, results_padj=res["padj"].values, results_baseMean=res["baseMean"].values)
    np.savez_compressed(os.path.join(mg.OUT, f"{prefix}shrinktape_{name}.npz"), **out)
    same = np.allclose(out["results_log2FoldChange"], shr_log2, equal_nan=True, rtol=0, atol=0)
    print(f"{prefix}shrinktape_{name}: G={counts.shape[1]} p={X.shape[1]} idx={coeff_idx} prior_scale={float(k['prior_scale']):.4g} "
          f"results_df holds the shrunk column: {same}")


def main():
    gen_calls("paired_p21", "wide_paired_p21", 20)
    gen_calls("paired_p21_noadapt", "wide_paired_p21", 20, adapt=False)
    gen_calls("levels_p17_outliers", "wide_levels_p17_outliers", 3)
    gen_calls("paired_covariate_p33", "wide_paired_covariate_p33", 31)
    gen_calls("paired_p64", "wide_paired_p64", 63)
    gen_tape("paired_p21", "wide_paired_p21", 20)


if __name__ == "__main__":
    main()
