"""The wide_* fixtures of scripts/make_wide_golden.py (designs of 17..64 columns) and their end-to-end check, shared by the CPU
suite (oracle) and the GPU suite (opt-in backend)."""
import numpy as np

from conftest import load_golden
from parity import rel_err, report

WIDE_E2E = ["wide_paired_p21", "wide_levels_p17_outliers", "wide_paired_covariate_p33", "wide_paired_p64"]
RTOL = 1e-4  # the e2e_* tolerance (tests/test_gpu_chain.py); p-values and padj at 10x, as parity.check_e2e

# Genes allowed outside RTOL per fixture, and how far they may be (relative).  N - p is 19 (p = 21), 29 (p = 33) and 62 (p = 64):
# there the dispersion likelihoods are flat, L-BFGS-B stops within ~1e-5 of a flat optimum, and a gene close to the reference's
# "genewise far above the trend" rule (dds.py:918-932) can take the other side of it, which moves its final dispersion by a few
# percent and its LFC by ~1e-2.  The bounds are the worst errors measured against the real reference's tables, the oracle's and
# the H100's together (DESIGN.md §8).
BUDGET = {"wide_paired_p21": (1, 0.06), "wide_levels_p17_outliers": (0, RTOL), "wide_paired_covariate_p33": (2, 0.01),
          "wide_paired_p64": (1, 0.03)}


def check_wide_e2e(inf, name, resident=False):
    from pydeseq2_b200.workflow import deseq2_results

    g = load_golden(name)
    counts, X = np.ascontiguousarray(g["counts"], dtype=np.int64), g["design"]
    if resident:
        from pydeseq2_b200.pipeline import ResidentFit
        from pydeseq2_b200.workflow import deseq2_results_resident

        nz = ~(counts == 0).all(0)
        rf = ResidentFit(inf._ops.ctx, X, None)
        rf.upload(np.ascontiguousarray(counts[:, nz]))
        try:
            r = deseq2_results_resident(rf, g["contrast"], non_zero=nz)
        finally:
            rf.close()
    else:
        r = deseq2_results(counts, X, inf, g["contrast"])
    # decisions and NaN patterns must agree exactly
    np.testing.assert_array_equal(r.replaced, g["final_replaced"] == 1, err_msg="replaced genes")
    np.testing.assert_array_equal(r.refitted, g["final_refitted"] == 1, err_msg="refitted genes")
    np.testing.assert_array_equal(r.cooks_outlier, g["final_cooks_outlier"] == 1, err_msg="Cook's outlier genes")
    np.testing.assert_array_equal(np.isnan(r.pvalue), np.isnan(g["final_pvalue"]), err_msg="masked p-values")
    np.testing.assert_array_equal(np.isnan(r.padj), np.isnan(g["final_padj"]), err_msg="independent-filtering threshold")
    np.testing.assert_allclose(r.size_factors, g["final_size_factors"], rtol=1e-12)
    np.testing.assert_allclose(r.base_mean, g["final_baseMean"], rtol=1e-12)
    genes, bound = BUDGET[name]
    big = g["final_pvalue"] >= 1e-20
    rec, fails = {}, []
    for key, got, want, rtol, atol in (
            ("lfc", r.lfc, g["final_LFC"], RTOL, 1e-8), ("dispersions", r.dispersions, g["final_dispersions"], RTOL, 0.0),
            ("genewise", r.genewise_dispersions, g["final_genewise"], RTOL, 0.0),
            ("fitted", r.fitted_dispersions, g["final_fitted"], RTOL, 0.0),
            ("log2FoldChange", r.log2_fold_change, g["final_log2FoldChange"], RTOL, 1e-8),
            ("lfcSE", r.lfc_se, g["final_lfcSE"], RTOL, 0.0), ("stat", r.stat, g["final_stat"], RTOL, 1e-8),
            ("pvalue", r.pvalue, g["final_pvalue"], 10 * RTOL, 0.0), ("padj", r.padj, g["final_padj"], 10 * RTOL, 0.0)):
        got, want = np.asarray(got, dtype=float), np.asarray(want, dtype=float)
        bad = ~np.isclose(got, want, rtol=rtol, atol=atol, equal_nan=True)
        if key in ("pvalue", "padj"):
            bad &= big
        rows = bad if bad.ndim == 1 else bad.any(1)
        worst = float(np.nanmax(rel_err(got, want)[bad])) if bad.any() else 0.0  # over the entries outside rtol only
        rec[key + "_genes"], rec[key + "_worst"] = int(rows.sum()), worst
        # BH couples the genes (padj is a running minimum over the sorted p-values): one p-value moves several padj, so padj is
        # held to the bound, not to the gene count
        if (rows.sum() > genes and key != "padj") or (rows.any() and worst > max(bound, rtol)):
            fails.append(f"{key}: {int(rows.sum())} genes outside rtol={rtol}, worst {worst:.3g} (budget {genes} genes, {bound:g})")
    report("wide_e2e", name + (" [resident]" if resident else ""), **rec)
    assert not fails, "; ".join(fails)
