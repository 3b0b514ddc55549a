"""Shared pieces of the contrast tests (tests/test_contrasts.py on the host emulator, tests/test_gpu_contrasts.py on the device): the
ct_* goldens of scripts/make_contrast_golden.py and seeded designs checked against the oracle's restatement of utils.wald_test."""
import numpy as np

from conftest import load_golden

CT = ["ct_three_level_batch", "ct_alternatives", "ct_outliers", "ct_ten_levels"]
ALTS = [None, "greaterAbs", "lessAbs", "greater", "less"]


def contrasts_of(g):
    """[(contrast, lfc_null (log2), alt, cooks_filter, independent_filter, alpha, prior_lfc_var or None, k)] of a golden."""
    out = []
    for k in range(int(g["n_contrasts"])):
        c = f"c{k:02d}_"
        prior = g[c + "prior_lfc_var"]
        out.append((g[c + "contrast"], float(g[c + "lfc_null"]), str(g[c + "alt"]) or None, bool(g[c + "cooks_filter"]),
                    bool(g[c + "independent_filter"]), float(g[c + "alpha"]), None if np.isnan(prior).all() else prior, k))
    return out


def p_tol(stat, rtol):
    """Relative tolerance of a p-value from the relative tolerance of its statistic z: d log sf(z) / d log z ~ z^2 in the tail."""
    return rtol * np.maximum(1.0, np.nan_to_num(np.asarray(stat)) ** 2)


def stat_atol(cs, lfc, lfc_null, se, rtol):
    """(K, G) absolute tolerance of the statistic c'(b - t) / se where the dot product cancels: rtol * sum_j |c_j| (|b_j| + |t|) / se."""
    t = np.abs(np.broadcast_to(np.asarray(lfc_null, dtype=float), (len(cs),)))[:, None]
    return rtol * (np.abs(cs) @ np.abs(lfc).T + np.abs(cs).sum(1)[:, None] * t) / np.asarray(se)


def assert_tests_close(got, want, rtol, what="", atol_stat=1e-300):
    """(pvalue, stat, se) against (pvalue, stat, se): identical NaN patterns; stat / se within rtol (the statistic also within
    `atol_stat`, see stat_atol), p-values within p_tol."""
    gp, gs, ge = (np.asarray(a, dtype=float) for a in got)
    wp, ws, we = (np.asarray(a, dtype=float) for a in want)
    for a, b, name in ((gp, wp, "pvalue"), (gs, ws, "stat"), (ge, we, "se")):
        np.testing.assert_array_equal(np.isnan(a), np.isnan(b), err_msg=f"{what} {name}: NaN pattern")
    ok = ~np.isnan(ws)
    bad = ok & (np.abs(gs - ws) > rtol * np.abs(ws) + np.broadcast_to(atol_stat, ws.shape))
    assert not bad.any(), f"{what} stat: {bad.sum()} entries off, e.g. {gs[bad][:3]} vs {ws[bad][:3]}"
    np.testing.assert_allclose(ge, we, rtol=rtol, atol=1e-300, err_msg=f"{what} se")
    ok = ~np.isnan(wp)
    tol = p_tol(ws, rtol)[ok]
    err = np.abs(gp[ok] - wp[ok]) / np.maximum(np.abs(wp[ok]), 1e-300)
    assert (err <= tol).all(), f"{what} pvalue: worst {err.max():.3g} relative"


def golden_wald_tests(inf, name):
    """`wald_tests` on the golden's stored dataset state, every contrast in one call; returns (g, pv, stat, se) with (K, G)."""
    g = load_golden(name)
    cases = contrasts_of(g)
    # one call per ridge: the alternatives golden gives some contrasts a prior
    out = [None] * len(cases)
    for prior in {None if c[6] is None else tuple(c[6]) for c in cases}:
        sel = [c for c in cases if (None if c[6] is None else tuple(c[6])) == prior]
        ridge = None if prior is None else np.diag(1 / np.asarray(prior) ** 2)
        pv, st, se = inf.wald_tests(g["design"], g["final_size_factors"], g["final_dispersions"], g["final_LFC"],
                                    np.array([c[0] for c in sel]), ridge, np.log(2) * np.array([c[1] for c in sel]),
                                    [c[2] for c in sel])
        for i, c in enumerate(sel):
            out[c[7]] = (pv[i], st[i], se[i])
    return g, [o[0] for o in out], [o[1] for o in out], [o[2] for o in out]


def check_golden_wald(inf, name, rtol=1e-9):
    """Against the unfiltered statistics / SE / p-values of the reference's run_wald_test, genes made all-zero by the outlier
    replacement excluded (the override of ds.py:355-360 is the caller's)."""
    g, pv, st, se = golden_wald_tests(inf, name)
    keep = g["final_new_all_zero"] == 0
    for k in range(len(pv)):
        c = f"c{k:02d}_"
        assert_tests_close((pv[k][keep], st[k][keep], se[k][keep]), (g[c + "p_values"][keep], g[c + "statistics"][keep], g[c + "SE"][keep]),
                           rtol, f"{name} contrast {k}")


def seeded_case(p, N, G, K, seed):
    """A design with a factor and continuous columns, fitted-looking coefficients and dispersions, K random contrasts."""
    rng = np.random.default_rng(seed)
    X = np.ones((N, p))
    if p > 1:
        lv = rng.integers(0, min(p, 4), N)
        for j in range(1, p):
            X[:, j] = (lv == j) if j < min(p, 4) else rng.normal(0, 0.5, N)
    sf = np.exp(rng.normal(0, 0.3, N))
    lfc = rng.normal(0, 0.7, (G, p))
    lfc[:, 0] += rng.uniform(1, 7, G)
    disp = np.exp(rng.normal(-2, 1, G))
    cs = rng.normal(0, 1, (K, p))
    return X, sf, disp, lfc, cs


def oracle_wald_tests(X, sf, disp, lfc, cs, ridge, lfc_null, alts):
    """The oracle's restatement of utils.wald_test, one call per contrast, on the host mu the reference builds (ds.py:320-324)."""
    from oracle.nbglm import OracleInference

    ref = OracleInference(n_cpus=1)
    mu = np.exp(X @ lfc.T) * sf[:, None]
    outs = [ref.wald_test(X, disp, lfc, mu, ridge, c, t, a) for c, t, a in zip(cs, lfc_null, alts)]
    return tuple(np.array([o[i] for o in outs]) for i in range(3))


def stats_groups(g):
    """The golden's contrasts grouped by the DeseqStats options they share (one deseq2_stats call per group)."""
    groups = {}
    for c in contrasts_of(g):
        key = (c[3], c[4], c[5], None if c[6] is None else tuple(c[6]))
        groups.setdefault(key, []).append(c)
    return groups


def check_stats_e2e(inf, name, rtol, max_frac=0.005, resident=False):
    """`workflow.deseq2_stats` on the fit of `deseq2_results` (or `deseq2_results_resident`) against the reference's results_df of
    every contrast, at the e2e tolerances of parity.check_e2e."""
    from parity import assert_mostly_close
    from pydeseq2_b200.workflow import deseq2_results, deseq2_results_resident, deseq2_stats

    g = load_golden(name)
    counts, X = np.ascontiguousarray(g["counts"], dtype=np.int64), g["design"]
    first = contrasts_of(g)[0][0]
    if resident:
        from pydeseq2_b200.pipeline import ResidentFit

        nz = ~(counts == 0).all(0)
        rf = ResidentFit(inf._ops.ctx, X, None)
        rf.upload(np.ascontiguousarray(counts[:, nz]))
        try:
            res = deseq2_results_resident(rf, first, non_zero=nz)
        finally:
            rf.close()
    else:
        res = deseq2_results(counts, X, inf, first)
    np.testing.assert_array_equal(res.replaced, g["final_replaced"] == 1, err_msg="replaced genes")
    np.testing.assert_array_equal(res.refitted, g["final_refitted"] == 1, err_msg="refitted genes")
    np.testing.assert_array_equal(res.replaced & ~res.refitted, g["final_new_all_zero"] == 1, err_msg="new all-zero genes")
    np.testing.assert_array_equal(res.cooks_outlier, g["final_cooks_outlier"] == 1, err_msg="Cook's outlier genes")
    for (cf, inf_, alpha, prior), cases in stats_groups(g).items():
        out = deseq2_stats(res, X, inf, np.array([c[0] for c in cases]), lfc_null=np.array([c[1] for c in cases]),
                           alt_hypothesis=[c[2] for c in cases], cooks_filter=cf, independent_filter=inf_, alpha=alpha,
                           prior_lfc_var=None if prior is None else np.array(prior))
        assert len(out) == len(cases)
        for r, c in zip(out, cases):
            p = f"c{c[7]:02d}_"
            what = f"{name} contrast {c[7]}"
            for key, got in (("pvalue", r.pvalue), ("padj", r.padj)):
                np.testing.assert_array_equal(np.isnan(got), np.isnan(g[p + key]), err_msg=f"{what}: NaN pattern of {key}")
            np.testing.assert_allclose(r.base_mean, g["final_baseMean"], rtol=1e-12)
            assert_mostly_close(r.log2_fold_change, g[p + "log2FoldChange"], rtol, what + " log2FoldChange", 1e-8, max_frac)
            assert_mostly_close(r.lfc_se, g[p + "lfcSE"], rtol, what + " lfcSE", 0.0, max_frac)
            assert_mostly_close(r.stat, g[p + "stat"], rtol, what + " stat", 1e-8, max_frac)
            big = ~np.isnan(g[p + "pvalue"]) & (np.nan_to_num(g[p + "pvalue"]) >= 1e-20)
            assert_mostly_close(r.pvalue[big], g[p + "pvalue"][big], 10 * rtol, what + " pvalue", 0.0, max_frac)
            ok = big & ~np.isnan(g[p + "padj"])
            assert_mostly_close(r.padj[ok], g[p + "padj"][ok], 10 * rtol, what + " padj", 0.0, max_frac)
    return res
