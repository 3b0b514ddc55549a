"""Shared parity checks: the same assertions run against the host emulator (CPU suite) and against the
CUDA library through the C ABI (`-m gpu`).  Tolerances follow BASELINE.json's north star: LFCs, dispersions
and Wald statistics within 1e-4 relative of the reference CPU backend (the per-call checks below are much
tighter where the arithmetic allows it)."""
import numpy as np

from conftest import tape_calls

ALTS = ((None, 0.0), ("greater", 0.3), ("less", 0.3), ("greaterAbs", 0.3), ("lessAbs", 0.3))

# per-call isolation tolerances (identical inputs into reference and device code)
TOL_BETA = 1e-6     # same start, same update, same stopping rule -> differences are rounding only
TOL_MU = 1e-6
TOL_HAT = 1e-6
TOL_ALPHA = 2e-5    # L-BFGS-B itself stops within ~3e-6 of the optimum (SURVEY.md App. B); bar is 1e-4
TOL_WALD = 1e-9


def report(kind, name, **fields):
    """Append one JSON line per parity case (measured mismatch fractions / worst errors) to the file named by the environment
    variable PDQ_PARITY_REPORT, when it is set.  Never fails a test."""
    import json
    import os

    path = os.environ.get("PDQ_PARITY_REPORT")
    if not path:
        return
    try:
        with open(path, "a") as f:
            f.write(json.dumps({"kind": kind, "case": name, **fields}) + "\n")
    except OSError:
        pass


def mismatch(got, want, rtol, atol=0.0, mask=None):
    """(fraction of entries off by more than rtol, worst relative error) over `mask`ed rows."""
    got, want = np.asarray(got, dtype=float), np.asarray(want, dtype=float)
    bad = ~np.isclose(got, want, rtol=rtol, atol=atol, equal_nan=True)
    err = rel_err(got, want)
    if mask is not None:
        bad, err = bad[mask], err[mask]
    if bad.size == 0:
        return 0.0, 0.0
    return float(bad.mean()), float(np.nanmax(err))


def rel_err(got, want, floor=1e-12):
    got, want = np.asarray(got, dtype=float), np.asarray(want, dtype=float)
    both_nan = np.isnan(got) & np.isnan(want)
    err = np.abs(got - want) / np.maximum(np.abs(want), floor)
    err[both_nan] = 0.0
    return err


def assert_close(got, want, rtol, what, atol=0.0, mask=None):
    got, want = np.asarray(got, dtype=float), np.asarray(want, dtype=float)
    assert got.shape == want.shape, f"{what}: shape {got.shape} vs {want.shape}"
    bad = ~(np.isclose(got, want, rtol=rtol, atol=atol, equal_nan=True))
    if mask is not None:
        bad &= mask
    assert not bad.any(), (
        f"{what}: {bad.sum()} / {bad.size} entries off by more than rtol={rtol}; worst rel err "
        f"{np.nanmax(rel_err(got, want)[bad]):.3e} at {np.argwhere(bad)[:5].tolist()}"
    )


def check_calls(inf, g, tol_alpha=TOL_ALPHA):
    """`g` is a calls_*.npz golden (outputs of the REAL reference); `inf` a B200Inference."""
    c, X, sf, N = g["counts"], g["X"], g["sf"], g["counts"].shape[0]
    max_disp = max(10.0, N)
    assert_close(inf.fit_rough_dispersions(g["normed"], X), g["rough"], 1e-8, "rough", atol=1e-12)
    assert_close(inf.fit_moments_dispersions(g["normed"], sf), g["moments"], 1e-9, "moments", atol=1e-12)
    assert_close(inf.lin_reg_mu(c, sf, X, 0.5), g["lin_mu"], 1e-9, "lin_reg_mu")

    for tag, disp in (("irls0", g["mom"]), ("lfc", g["disp"])):
        b, m, h, cv = inf.irls(c, sf, X, disp, 0.5, 1e-8)
        # genes the reference itself flags as not converged (IRLS hit maxiter, then L-BFGS-B gave up on the kinked
        # clamped objective, utils.py:374-403) carry an optimiser-path-dependent value: flags must agree, values need not
        ok = g[f"{tag}_conv"] == 1.0
        assert_close(b[ok], g[f"{tag}_beta"][ok], TOL_BETA, f"{tag} beta", atol=1e-9)
        assert_close(m[:, ok], g[f"{tag}_mu"][:, ok], TOL_MU, f"{tag} mu", atol=1e-12)
        assert_close(h[:, ok], g[f"{tag}_hat"][:, ok], TOL_HAT, f"{tag} hat", atol=1e-12)
        np.testing.assert_array_equal(cv, g[f"{tag}_conv"])
        assert np.isfinite(b).all()
        assert cv.dtype == np.float64

    lo, hi = 1e-8, max_disp
    for tag, kw, ahat in (("gw", {}, g["mom"]),
                          ("map", dict(prior_disp_var=float(g["prior_var"]), cr_reg=True, prior_reg=True), g["trend"])):
        a, cv = inf.alpha_mle(c, X, g["mu_hat"], ahat, lo, hi, **kw)
        want = g[f"{tag}_alpha"]
        ok = g[f"{tag}_conv"] == 1.0
        # at tiny dispersions the reference's own gradient is rounding noise (1/alpha^2 cancellation): compare
        # those genes after the caller's clip only (dds.py:792-794)
        interior = ok & (want > 1e-5) & (want < hi * (1 - 1e-9))
        assert_close(a[interior], want[interior], tol_alpha, f"{tag} alpha (interior optimum)")
        edge = ok & ~interior
        assert np.all(np.clip(a[edge], lo, hi) < 1e-4) or not edge.any() or np.allclose(
            np.clip(a[edge], lo, hi), np.clip(want[edge], lo, hi), rtol=1e-3), f"{tag} alpha (bound cases)"
        assert (cv[ok] == 1.0).all()

    for alt, null in ALTS:
        tag = alt or "two_sided"
        pv, st, se = inf.wald_test(X, g["disp"], g["lfc_beta"], g["lfc_mu"], g["ridge"], g["contrast"], null, alt)
        assert_close(se, g[f"wald_{tag}_se"], TOL_WALD, f"wald {tag} se")
        assert_close(st, g[f"wald_{tag}_stat"], TOL_WALD, f"wald {tag} stat", atol=1e-14)
        assert_close(pv, g[f"wald_{tag}_p"], 1e-8, f"wald {tag} p", atol=1e-300)


def check_tape(inf, t, name):
    """Replay every Inference call the reference orchestrator made (tape_*.npz)."""
    for meth, args, kw, outs in tape_calls(t):
        res = getattr(inf, meth)(*args, **kw)
        res = res if isinstance(res, tuple) else (res,)
        for k, (got, want) in enumerate(zip(res, outs)):
            got = np.asarray(got, dtype=float)
            if got.ndim == 0:
                got, want = got.reshape(1), np.ravel(want)
            if meth == "alpha_mle" and k == 0:
                conv = outs[1] == 1.0
                assert_close(got[conv], want[conv], 1e-4, f"{name}:{meth} alpha")
            elif meth == "alpha_mle":
                assert (got[outs[1] == 1.0] == 1.0).all()
            elif meth == "dispersion_trend_gamma_glm":
                # the device fit converges to the minimiser; scipy's L-BFGS-B (the reference) stops within ~1e-5 of it
                assert_close(got, want, 1e-4, f"{name}:{meth}[{k}]")
            elif meth == "wald_test" and k == 0:
                assert_close(got, want, 1e-7, f"{name}:{meth} p", atol=1e-300)
            else:
                assert_close(got, want, 1e-6, f"{name}:{meth}[{k}]", atol=1e-10)


SHRINK = ["shrink_two_level_n24", "shrink_factorial_n30", "shrink_factorial_n30_idx1", "shrink_continuous_n40",
          "shrink_two_level_n200", "shrink_two_level_n200_noadapt", "shrink_large_counts_n12", "shrink_five_columns_n36",
          "shrink_few_samples_n4", "shrinktape_single_factor", "shrinktape_single_factor_noadapt", "shrinktape_multi_factor",
          "shrinktape_continuous", "shrinktape_large_counts"]
# apeGLM: the backend walks the reference's optimiser path, so it lands on the reference's (loosely converged) iterate:
# measured <= 5e-10 on every fixture; the tolerance leaves room for a different summation order on the device
TOL_SHRINK = 1e-7


def check_shrink(inf, g, tol=TOL_SHRINK):
    """`lfc_shrink_nbinom_glm` against the real reference's outputs (oracle/make_golden.py `gen_shrink_*`)."""
    k = int(g["shrink_index"])
    lfcs, ih, conv = inf.lfc_shrink_nbinom_glm(g["X"], g["counts"], g["size"], g["offset"], float(g["prior_no_shrink_scale"]),
                                               float(g["prior_scale"]), "L-BFGS-B", k)
    assert lfcs.shape == g["lfcs"].shape and ih.shape == g["inv_hessians"].shape
    np.testing.assert_array_equal(conv, g["converged"])
    assert_close(lfcs, g["lfcs"], tol, "shrunk coefficients", atol=1e-10)
    assert_close(ih, g["inv_hessians"], tol, "inverse Hessians", atol=1e-14)
    if "r_log2FoldChange" in g:  # the reference's own test: within 2 % of R's apeglm (tests/test_pydeseq2.py:256-296 ...)
        got = lfcs[:, k] / np.log(2)
        assert np.nanmax(np.abs(g["r_log2FoldChange"] - got) / np.abs(g["r_log2FoldChange"])) < 0.02
        se = np.sqrt(np.abs(ih[:, k, k])) / np.log(2)
        np.testing.assert_allclose(se, g["final_lfcSE"], rtol=tol)


E2E = ["e2e_two_level_n24", "e2e_factorial_n20", "e2e_two_level_n16_bh", "e2e_continuous_n30",
       # the reference's orchestrator-level edge cases (its tests/test_edge_cases.py:323-465)
       "e2e_edge_few_samples", "e2e_edge_few_samples_and_outlier", "e2e_edge_new_all_zero_gene",
       # its alternative-hypothesis test (tests/test_pydeseq2.py:180-225), R tables alongside
       "e2e_alt_lessAbs", "e2e_alt_greaterAbs", "e2e_alt_less", "e2e_alt_greater",
       # mean-type trend (:121-145) and outliers without the Cook's refit (:228-253)
       "e2e_mean_fit", "e2e_no_refit_outliers"]
TAPES_E2E = ["tape_single_factor", "tape_multi_factor", "tape_continuous", "tape_wide", "tape_multi_factor_outliers"]


def assert_mostly_close(got, want, rtol, what, atol=0.0, max_frac=0.0, slack=100.0):
    """All entries within `rtol`, except at most `max_frac` of them, which must still be within `slack * rtol`.

    The budget exists for the path-dependent fits: IRLS stops on a relative deviance change of 1e-8 and, on a flat likelihood
    (an outlier gene with dispersion ~3), two runs whose dispersions differ by 1e-6 can stop one iteration apart, i.e. ~1e-3
    apart in beta -- the reference would do the same to itself (SURVEY.md App. B)."""
    got, want = np.asarray(got, dtype=float), np.asarray(want, dtype=float)
    bad = ~np.isclose(got, want, rtol=rtol, atol=atol, equal_nan=True)
    if bad.mean() > max_frac:
        assert_close(got, want, rtol, what, atol=atol)
    assert_close(got, want, slack * rtol, what + " (outside the mismatch budget)", atol=slack * atol)


def check_e2e(inf, g, rtol, name="", max_frac=0.0, resident=False):
    """`workflow.deseq2_results` (deseq2() + summary(): refit of Cook's outliers, Cook's / independent filtering, BH) against the
    final tables of the real orchestrator (oracle/make_golden.py `gen_e2e`, `gen_tape`)."""
    from pydeseq2_b200.workflow import deseq2_results

    kw = {}
    if "independent_filter" in g:
        kw = dict(independent_filter=bool(g["independent_filter"]), cooks_filter=bool(g["cooks_filter"]), alpha=float(g["alpha"]))
    if "alt_hypothesis" in g:
        kw.update(alt_hypothesis=str(g["alt_hypothesis"]) or None, lfc_null=float(g["lfc_null"]))
    if "fit_type" in g:
        kw.update(fit_type=str(g["fit_type"]), refit_cooks=bool(g["refit_cooks"]))
    if resident:  # counts in HBM, one resident pass + resident refit of the replaced genes (workflow.deseq2_results_resident)
        from pydeseq2_b200.pipeline import ResidentFit
        from pydeseq2_b200.workflow import deseq2_results_resident

        counts = np.ascontiguousarray(g["counts"], dtype=np.int64)
        nz = ~(counts == 0).all(0)
        rf = ResidentFit(inf._ops.ctx, g["design"], None)  # size factors by median of ratios on the device
        rf.upload(np.ascontiguousarray(counts[:, nz]))
        try:
            r = deseq2_results_resident(rf, g["contrast"], non_zero=nz, **kw)
        finally:
            rf.close()
        name = name + " [resident]"
    else:
        r = deseq2_results(g["counts"], g["design"], inf, g["contrast"], **kw)
    # decisions first: they are discrete, so they must agree exactly
    np.testing.assert_array_equal(r.replaced, g["final_replaced"] == 1, err_msg="replaced genes")
    if "final_refitted" in g:
        np.testing.assert_array_equal(r.refitted, g["final_refitted"] == 1, err_msg="refitted genes")
    np.testing.assert_array_equal(r.cooks_outlier, g["final_cooks_outlier"] == 1, err_msg="Cook's outlier genes")
    pv_ref = g["final_pvalue"] if "final_pvalue" in g else g["final_pvalues"]
    np.testing.assert_array_equal(np.isnan(r.pvalue), np.isnan(pv_ref), err_msg="masked p-values")
    np.testing.assert_array_equal(np.isnan(r.padj), np.isnan(g["final_padj"]), err_msg="independent-filtering threshold")
    np.testing.assert_allclose(r.size_factors, g["final_size_factors"], rtol=1e-12)
    rec = {}
    for key, a, b, at in (("lfc", r.lfc, g["final_LFC"], 1e-8), ("dispersions", r.dispersions, g["final_dispersions"], 0.0),
                          ("genewise", r.genewise_dispersions, g["final_genewise"], 0.0), ("pvalue", r.pvalue, pv_ref, 0.0),
                          ("padj", r.padj, g["final_padj"], 0.0)):
        f, w = mismatch(a, b, rtol if key not in ("pvalue", "padj") else 10 * rtol, at,
                        (pv_ref >= 1e-20) if key in ("pvalue", "padj") else None)
        rec[key + "_frac"], rec[key + "_worst"] = f, w
    report("e2e", name, rtol=rtol, genes=int(np.asarray(pv_ref).size), **rec)
    assert_mostly_close(r.lfc, g["final_LFC"], rtol, "LFC", 1e-8, max_frac)
    assert_close(r.dispersions, g["final_dispersions"], rtol, "dispersions")
    assert_close(r.genewise_dispersions, g["final_genewise"], rtol, "genewise dispersions")
    if "final_stat" in g:
        assert_mostly_close(r.stat, g["final_stat"], rtol, "Wald statistic", 1e-8, max_frac)
    big = pv_ref >= 1e-20
    assert_mostly_close(r.pvalue[big], pv_ref[big], 10 * rtol, "p-values", 0.0, max_frac)
    ok = ~np.isnan(g["final_padj"])
    assert_mostly_close(r.padj[ok & big], g["final_padj"][ok & big], 10 * rtol, "adjusted p-values", 0.0, max_frac)
    if "final_baseMean" in g:
        assert_close(r.base_mean, g["final_baseMean"], 1e-12, "baseMean")
        assert_mostly_close(r.log2_fold_change, g["final_log2FoldChange"], rtol, "log2FoldChange", 1e-8, max_frac)
        assert_mostly_close(r.lfc_se, g["final_lfcSE"], rtol, "lfcSE", 0.0, max_frac)
        assert_close(r.fitted_dispersions, g["final_fitted"], rtol, "fitted dispersions")
    if "r_stat" in g and "r_padj" in g:  # the reference's own criteria against R DESeq2 (2 %; |stat| for lessAbs; p-values where stat != 0)
        assert np.array_equal(np.isnan(r.pvalue), np.isnan(g["r_pvalue"])) and np.array_equal(np.isnan(r.padj), np.isnan(g["r_padj"]))
        assert np.max(np.abs(g["r_log2FoldChange"] - r.log2_fold_change) / np.abs(g["r_log2FoldChange"])) < 0.02
        st = np.abs(r.stat) if kw.get("alt_hypothesis") == "lessAbs" else r.stat
        with np.errstate(invalid="ignore", divide="ignore"):  # 0/0 where both statistics are exactly 0 (pandas' max skips NaN)
            assert np.nanmax(np.abs(g["r_stat"] - st) / np.abs(g["r_stat"])) < 0.02
        nzs = g["r_stat"] != 0
        assert np.max(np.abs(g["r_pvalue"][nzs] - r.pvalue[nzs]) / g["r_pvalue"][nzs]) < 0.02
    return r
