"""GPU suite: designs of 17..64 columns on a backend that opted in (B200Inference(wide_designs=True)), against the oracle."""
import dataclasses

import numpy as np
import pytest

from edge_cases import _counts, _design
from oracle import nbglm
from pydeseq2_b200._lib import B200Error
from pydeseq2_b200.pipeline import median_of_ratios
from wide_cases import WIDE_E2E, check_wide_e2e

pytestmark = pytest.mark.gpu

FORCE_IRLS_OPTIMIZER, FORCE_ALPHA_GRID = 1, 2


@pytest.fixture(scope="module")
def wide():
    from pydeseq2_b200.inference import B200Inference

    return B200Inference(device=0, wide_designs=True)


@pytest.fixture(scope="module")
def ora():
    return nbglm.OracleInference(n_cpus=4)


def _set_debug(inf, flags):
    inf._ops.ctx.check(inf._ops.lib.pdq_set_debug_flags(inf._ops.ctx.h, flags))


def _problem(p, N):
    rng = np.random.default_rng(100 + p)
    X = _design(rng, N, p)
    c = _counts(rng, X, 48)
    sf = c.sum(1) / np.exp(np.log(c.sum(1)).mean())  # the widest designs leave a zero in every gene: no median of ratios
    return rng, X, c, np.ascontiguousarray(c / sf[:, None]), sf


def _penalised_nll(c, sf, X, disp, b, min_mu=0.5):
    """The optimiser branch's objective (utils.py:374-403): the mu-dependent part of nb_nll + 0.5e-6 |b|^2, per gene."""
    mu = np.maximum(sf[:, None] * np.exp(X @ b.T), min_mu)
    r = 1 / disp
    return ((c + r) * np.log(r + mu) - c * np.log(mu)).sum(0) + 0.5e-6 * (b * b).sum(1)


@pytest.mark.parametrize("p,N", [(17, 171), (21, 211), (24, 241), (32, 321), (48, 481), (64, 641)])
def test_every_plugin_method_against_the_oracle(wide, ora, p, N):
    """tests/edge_cases.check_design_width for the wide widths, without apeGLM shrinkage (refused for p > 16)."""
    rng, X, c, normed, sf = _problem(p, N)
    G = c.shape[1]
    max_disp = float(max(10, N))
    np.testing.assert_allclose(wide.fit_rough_dispersions(normed, X), ora.fit_rough_dispersions(normed, X), rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(wide.fit_moments_dispersions(normed, sf), ora.fit_moments_dispersions(normed, sf), rtol=1e-10)
    mom = np.clip(np.minimum(ora.fit_rough_dispersions(normed, X), ora.fit_moments_dispersions(normed, sf)), 1e-8, max_disp)
    np.testing.assert_allclose(wide.lin_reg_mu(c, sf, X, 0.5), ora.lin_reg_mu(c, sf, X, 0.5), rtol=1e-9)
    b, m, h, cv = wide.irls(c, sf, X, mom, 0.5, 1e-8)
    rb, rm, rh, rcv = ora.irls(c, sf, X, mom, 0.5, 1e-8)
    # at these shapes the reference itself leaves up to ~10 % of the genes unconverged (p = 64: 43 of 48 converge)
    both = (rcv == 1) & (cv == 1)
    assert both.mean() > 0.85
    close = np.isclose(b, rb, rtol=1e-6, atol=1e-9).all(axis=1)
    ok = both & close
    assert ok.sum() >= 0.9 * both.sum()
    # genes that left IRLS for the optimiser branch on either side: both minimise the same objective, the reference with
    # L-BFGS-B to its loose tolerance and from another path; the kernel's end point must be at least as low
    opt = both & ~close
    f, rf = _penalised_nll(c[:, opt], sf, X, mom[opt], b[opt]), _penalised_nll(c[:, opt], sf, X, mom[opt], rb[opt])
    assert np.all(f <= rf + 1e-7 * np.abs(rf)), (f - rf)
    np.testing.assert_allclose(b[ok], rb[ok], rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(m[:, ok], rm[:, ok], rtol=1e-6)
    np.testing.assert_allclose(h[:, ok], rh[:, ok], rtol=1e-6, atol=1e-12)
    mu_hat = np.ascontiguousarray(rm)
    a, ac = wide.alpha_mle(c, X, mu_hat, mom, 1e-8, max_disp)
    ra, rac = ora.alpha_mle(c, X, mu_hat, mom, 1e-8, max_disp)
    interior = (rac == 1) & (ac == 1) & (ra > 1e-5) & (ra < 0.99 * max_disp)
    assert interior.mean() > 0.5
    assert np.mean(np.isclose(a[interior], ra[interior], rtol=1e-4)) >= 0.97
    trend = np.clip(ra, 1e-8, max_disp) * np.exp(rng.normal(0, 0.3, G))
    a2, ac2 = wide.alpha_mle(c, X, mu_hat, trend, 1e-8, max_disp, prior_disp_var=0.5, cr_reg=True, prior_reg=True)
    ra2, rac2 = ora.alpha_mle(c, X, mu_hat, trend, 1e-8, max_disp, prior_disp_var=0.5, cr_reg=True, prior_reg=True)
    both = (rac2 == 1) & (ac2 == 1)
    np.testing.assert_allclose(a2[both], ra2[both], rtol=1e-4)
    disp = np.clip(ra2, 1e-8, max_disp)
    contrast = np.zeros(p)
    contrast[-1] = 1.0
    ridge = np.diag(np.repeat(1e-6, p))
    for alt, null in ((None, 0.0), ("greaterAbs", 0.2), ("lessAbs", 0.2), ("greater", 0.1), ("less", 0.1)):
        pv, st, se = wide.wald_test(X, disp, rb, mu_hat, ridge, contrast, null, alt)
        rp, rs, rse = ora.wald_test(X, disp, rb, mu_hat, ridge, contrast, null, alt)
        np.testing.assert_allclose(se, rse, rtol=1e-9)
        np.testing.assert_allclose(st, rs, rtol=1e-9, atol=1e-12)
        np.testing.assert_allclose(pv, rp, rtol=1e-8, atol=1e-300)
    with pytest.raises(B200Error, match="not implemented"):
        wide.lfc_shrink_nbinom_glm(X, c, 1.0 / disp, np.log(sf), 15, 0.4, "L-BFGS-B", p - 1)


def test_many_contrasts_against_the_oracle(wide, ora):
    """wald_tests (K contrasts of one fit, mu rebuilt from the coefficients) against the oracle's wald_test per contrast."""
    p, N = 21, 211
    rng, X, c, normed, sf = _problem(p, N)
    mom = np.clip(np.minimum(ora.fit_rough_dispersions(normed, X), ora.fit_moments_dispersions(normed, sf)), 1e-8, N)
    b, _, _, _ = ora.irls(c, sf, X, mom, 0.5, 1e-8)
    cs = np.eye(p)[[1, 5, p - 1]] - np.eye(p)[[2, 6, 3]]
    pv, st, se = wide.wald_tests(X, sf, mom, b, cs, ridge_factor=np.diag(np.repeat(1e-6, p)))
    mu = np.ascontiguousarray(np.exp(X @ b.T) * sf[:, None])
    for k, ck in enumerate(cs):
        rp, rs, rse = ora.wald_test(X, mom, b, mu, np.diag(np.repeat(1e-6, p)), ck, 0.0, None)
        np.testing.assert_allclose(se[k], rse, rtol=1e-9)
        np.testing.assert_allclose(st[k], rs, rtol=1e-9, atol=1e-12)
        np.testing.assert_allclose(pv[k], rp, rtol=1e-8, atol=1e-300)


def test_forced_optimizer_branch_and_alpha_grid(wide, ora):
    p, N = 21, 211
    _, X, c, normed, sf = _problem(p, N)
    max_disp = float(max(10, N))
    mom = np.clip(np.minimum(ora.fit_rough_dispersions(normed, X), ora.fit_moments_dispersions(normed, sf)), 1e-8, max_disp)
    rm = ora.irls(c, sf, X, mom, 0.5, 1e-8)[1]
    plain = wide.irls(c, sf, X, mom, 0.5, 1e-8)
    _set_debug(wide, FORCE_IRLS_OPTIMIZER)
    try:
        b, m, h, cv = wide.irls(c, sf, X, mom, 0.5, 1e-8)
    finally:
        _set_debug(wide, 0)
    assert wide.last_irls_fallbacks == c.shape[1]
    # as edge_cases.check_irls_bounded_optimizer: where the min_mu clamp is inactive the objective is smooth and the projected
    # Newton iteration reports success; IRLS stops on its deviance test short of the optimum, so they agree to that level
    ok = (plain[1] >= 0.5).all(0) & (cv == 1)
    assert ok.sum() >= 0.5 * c.shape[1]  # 27 of these 48 genes on an H100
    np.testing.assert_allclose(b[ok], plain[0][ok], rtol=5e-3, atol=1e-4)
    # ... and against the reference's OWN optimiser branch (maxiter=1 forces it, utils.py:374), as check_irls_bounded_optimizer:
    # the penalised objective at least as low, the coefficients close where scipy reports success
    f, rf = [], []
    for i in np.flatnonzero(ok)[:12]:
        rb_i, _, _, rc_i = nbglm.irls_gene(c[:, i], sf, X, mom[i], 0.5, 1e-8, maxiter=1)
        f_i, rf_i = _penalised_nll(c[:, i:i + 1], sf, X, mom[i:i + 1], b[i:i + 1])[0], _penalised_nll(c[:, i:i + 1], sf, X, mom[i:i + 1], rb_i[None])[0]
        assert f_i <= rf_i + 1e-9 * abs(rf_i), i
        if rc_i:  # scipy stops at factr 1e7 on a 21-dimensional objective: up to 3.0e-4 apart measured, with ours no higher
            np.testing.assert_allclose(b[i], rb_i, rtol=2e-3, atol=5e-4)
    mu_hat = np.ascontiguousarray(rm)
    _set_debug(wide, FORCE_ALPHA_GRID)
    try:
        a, ac = wide.alpha_mle(c, X, mu_hat, mom, 1e-8, max_disp)
    finally:
        _set_debug(wide, 0)
    assert (ac == 0).all()
    want = np.array([np.exp(nbglm.grid_fit_alpha(c[:, i], X, mu_hat[:, i], mom[i], 1e-8, max_disp)) for i in range(c.shape[1])])
    close = np.isclose(a, want, rtol=1e-9)
    assert close.mean() >= 0.9
    assert np.all(np.abs(np.log(a) - np.log(want)) <= 2 * (np.log(max_disp) - np.log(1e-8)) / 99 * 2 / 99 + 1e-12)


def test_limit_with_the_opt_in(wide):
    """Above 64 columns: the Python check and, behind it, the C ABI (design packs and pdq_wald_contrasts) refuse with the limit."""
    import ctypes as C

    from pydeseq2_b200._lib import as_f64p

    X = np.ones((80, 65))
    with pytest.raises(B200Error, match="p <= 64"):
        wide.lin_reg_mu(np.ones((80, 3), dtype=np.int64), np.ones(80), X, 0.5)
    ctx, lib = wide._ops.ctx, wide._ops.lib
    G, K, p = 3, 2, 65
    out = [np.zeros((K, G)) for _ in range(3)]
    alt = np.zeros(K, np.int32)
    rc = lib.pdq_wald_contrasts(ctx.h, as_f64p(X), as_f64p(np.ones(80)), 80, p, as_f64p(np.ones(G)), as_f64p(np.zeros((G, p))), G,
                                as_f64p(np.eye(p)), K, as_f64p(np.ones((K, p))), as_f64p(np.zeros(K)), alt.ctypes.data_as(C.POINTER(C.c_int)),
                                *(as_f64p(o) for o in out), G)
    assert rc == -3 and b"p <= 64" in lib.pdq_last_error(ctx.h)
    rc = lib.pdq_lin_reg_mu(ctx.h, np.ones((80, G), dtype=np.int64).ctypes.data_as(C.POINTER(C.c_int64)), G, 80, G, as_f64p(np.ones(80)),
                            as_f64p(X), p, 0.5, as_f64p(np.zeros((80, G))))
    assert rc == -3 and b"wide designs support p <= 64" in lib.pdq_last_error(ctx.h)


def test_opt_in_off_refuses_a_cached_wide_design():
    """Turning the opt-in off refuses a wide design again, also one whose pack the context still holds."""
    from pydeseq2_b200.inference import B200Inference

    inf = B200Inference(device=0, wide_designs=True)
    _, X, c, _, sf = _problem(17, 60)
    inf.lin_reg_mu(c, sf, X, 0.5)  # the pack is now cached
    inf._ops.ctx.set_wide_designs(False)
    with pytest.raises(B200Error, match="p <= 16"):
        inf.lin_reg_mu(c, sf, X, 0.5)
    ctx, lib = inf._ops.ctx, inf._ops.lib
    from pydeseq2_b200._lib import as_f64p, as_i64p

    N, G = c.shape
    c = np.ascontiguousarray(c)
    rc = lib.pdq_lin_reg_mu(ctx.h, as_i64p(c), G, N, G, as_f64p(sf), as_f64p(np.ascontiguousarray(X)), 17, 0.5, as_f64p(np.zeros((N, G))))
    assert rc == -3 and b"p <= 16" in lib.pdq_last_error(ctx.h)


MULTIMODAL = pytest.mark.xfail(strict=True, reason=(
    "known deviation: 3 of 300 genes have a genewise dispersion objective with two local minima (one at the lower bound 1e-8); "
    "the reference's L-BFGS-B ends at the bound, the kernel's root search at the interior minimum, and the global trend then "
    "moves every MAP dispersion by up to ~1 % (DESIGN.md §8)"))


@pytest.mark.parametrize("resident", [False, True])
@pytest.mark.parametrize("name", [n if n in ("wide_paired_p21", "wide_levels_p17_outliers") else pytest.param(n, marks=MULTIMODAL)
                                  for n in WIDE_E2E])
def test_end_to_end_tables_match_the_real_orchestrator(wide, name, resident):
    """deseq2() + summary() through both drivers against the final tables the real reference wrote (scripts/make_wide_golden.py):
    replaced / refitted / Cook's-outlier sets and NaN patterns identical, values within the e2e tolerance except the measured
    per-fixture budget of tests/wide_cases.py (flat likelihoods at small N - p).  The 17-level case runs the lin_reg_mu start, the
    Cook's replacement and the refit of both drivers."""
    check_wide_e2e(wide, name, resident=resident)


def test_contrasts_of_the_17_level_fit_against_the_reference(wide):
    """wald_tests on the reference's stored fit, 16 pairwise contrasts: <= 1e-9 from its run_wald_test."""
    from contrast_cases import check_golden_wald

    check_golden_wald(wide, "wide_ct_levels_p17", 1e-9)


@pytest.mark.parametrize("resident", [False, True])
def test_deseq2_stats_of_the_17_level_fit(wide, resident):
    """workflow.deseq2_stats on both drivers against every contrast's results_df, as for the ct_* fixtures."""
    from contrast_cases import check_stats_e2e

    check_stats_e2e(wide, "wide_ct_levels_p17", 2e-4, max_frac=0.02, resident=resident)


def test_vst_with_the_design_against_the_reference(wide):
    """vst(use_design=True) on the paired p = 21 design: trend and transformed counts within 1e-4 (as the vst_* fixtures)."""
    from conftest import load_golden
    from pydeseq2_b200.workflow import vst

    z = load_golden("wide_vst_paired_p21_design")
    fit = vst(z["counts"], z["design"], wide, fit_type=str(z["fit_type"]), use_design=True)
    assert fit.kind == str(z["vst_fit_type"]) == "parametric"
    np.testing.assert_allclose(fit.size_factors, z["size_factors"], rtol=1e-10)
    np.testing.assert_allclose(fit.coeffs, z["vst_trend_coeffs"], rtol=1e-4)
    got, want = fit.vst_counts, z["vst_counts"]
    np.testing.assert_array_equal(np.isfinite(got), np.isfinite(want))
    ok = np.isfinite(want)
    assert np.all(np.abs(got[ok] - want[ok]) <= 1e-4 * np.maximum(np.abs(want[ok]), 1.0))


def test_opt_in_leaves_narrow_designs_byte_identical():
    """The opt-in changes nothing for p <= 16: a plugin-path fit and a C2-shaped resident pass (20 000 genes x 200 samples) are
    byte-equal with it on and off."""
    from pydeseq2_b200.inference import B200Inference
    from pydeseq2_b200.pipeline import ResidentFit, fit_host
    from pydeseq2_b200.synth import make_counts

    counts, X, _ = make_counts(200, 20000, "two_level", seed=7)
    counts = np.ascontiguousarray(counts[:, ~(counts == 0).all(0)])
    _, sf = median_of_ratios(counts)
    small = np.ascontiguousarray(counts[:, :2000])
    outs = []
    for on in (False, True):
        inf = B200Inference(device=0, wide_designs=on)
        a = fit_host(small, X, inf, size_factors=sf)
        rf = ResidentFit(inf._ops.ctx, X, sf, with_cooks=True)
        rf.upload(counts)
        r = rf.run()
        outs.append((a, r))
    (a0, r0), (a1, r1) = outs
    for name in ("lfc", "dispersions", "pvalue", "stat", "se", "mu_lfc", "hat"):
        np.testing.assert_array_equal(np.asarray(getattr(a0, name)), np.asarray(getattr(a1, name)), err_msg=name)
    items = ([(f.name, getattr(r0, f.name), getattr(r1, f.name)) for f in dataclasses.fields(r0)] if dataclasses.is_dataclass(r0)
             else list(zip(r0.keys(), r0.values(), r1.values())) if isinstance(r0, dict) else [(str(i), u, v) for i, (u, v) in enumerate(zip(r0, r1))])
    assert items
    for name, v0, v1 in items:
        if isinstance(v0, np.ndarray):
            np.testing.assert_array_equal(v0, v1, err_msg=name)
