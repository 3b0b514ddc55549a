"""GPU suite: designs of 65..128 columns on a backend that opted in (B200Inference(wide_designs=True, large_designs=True)),
against the oracle, and the opt-in contract of pdq_set_large_designs."""
import ctypes as C

import numpy as np
import pytest

from edge_cases import _counts, _design
from large_cases import LARGE_E2E, MULTIMODAL_REASON, check_large_e2e
from oracle import nbglm
from pydeseq2_b200._lib import B200Error, as_f64p, as_i64p
from test_large_designs import paired

pytestmark = pytest.mark.gpu

FORCE_IRLS_OPTIMIZER, FORCE_ALPHA_GRID, FAIL_IRLS_OPTIMIZER = 1, 2, 8


@pytest.fixture(scope="module")
def large():
    from pydeseq2_b200.inference import B200Inference

    return B200Inference(device=0, wide_designs=True, large_designs=True)


@pytest.fixture(scope="module")
def ora():
    return nbglm.OracleInference(n_cpus=4)


def _set_debug(inf, flags):
    inf._ops.ctx.check(inf._ops.lib.pdq_set_debug_flags(inf._ops.ctx.h, flags))


def _problem(p, N, G=48):
    rng = np.random.default_rng(100 + p)
    X = _design(rng, N, p)
    c = _counts(rng, X, G)
    sf = c.sum(1) / np.exp(np.log(c.sum(1)).mean())
    return rng, X, c, np.ascontiguousarray(c / sf[:, None]), sf


def _penalised_nll(c, sf, X, disp, b, min_mu=0.5):
    """The optimiser branch's objective (utils.py:374-403): the mu-dependent part of nb_nll + 0.5e-6 |b|^2, per gene."""
    mu = np.maximum(sf[:, None] * np.exp(X @ b.T), min_mu)
    r = 1 / disp
    return ((c + r) * np.log(r + mu) - c * np.log(mu)).sum(0) + 0.5e-6 * (b * b).sum(1)


def _mom(ora, normed, X, sf, max_disp):
    return np.clip(np.minimum(ora.fit_rough_dispersions(normed, X), ora.fit_moments_dispersions(normed, sf)), 1e-8, max_disp)


@pytest.mark.parametrize("p", [65, 80, 101, 128])
def test_every_plugin_method_against_the_oracle(large, ora, p):
    """tests/edge_cases.check_design_width's tolerances for the large widths, as the wide suite does for 17..64."""
    N = 10 * p + 1  # as the wide suite: at N = 5 p the reference itself leaves up to 40 % of the genes unconverged at p = 128
    rng, X, c, normed, sf = _problem(p, N)
    G = c.shape[1]
    max_disp = float(max(10, N))
    np.testing.assert_allclose(large.fit_rough_dispersions(normed, X), ora.fit_rough_dispersions(normed, X), rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(large.fit_moments_dispersions(normed, sf), ora.fit_moments_dispersions(normed, sf), rtol=1e-10)
    mom = _mom(ora, normed, X, sf, max_disp)
    np.testing.assert_allclose(large.lin_reg_mu(c, sf, X, 0.5), ora.lin_reg_mu(c, sf, X, 0.5), rtol=1e-9)
    b, m, h, cv = large.irls(c, sf, X, mom, 0.5, 1e-8)
    rb, rm, rh, rcv = ora.irls(c, sf, X, mom, 0.5, 1e-8)
    both = (rcv == 1) & (cv == 1)
    # as in the wide suite, the optimiser branch reports convergence more strictly than scipy: at p = 128, 39 of 48 on an H100
    assert both.mean() > (0.85 if p < 128 else 0.75)
    close = np.isclose(b, rb, rtol=1e-6, atol=1e-9).all(axis=1)
    ok = both & close
    assert ok.sum() >= 0.9 * both.sum()
    opt = both & ~close  # the optimiser branch on either side: the kernel's end point at least as low
    f, rf = _penalised_nll(c[:, opt], sf, X, mom[opt], b[opt]), _penalised_nll(c[:, opt], sf, X, mom[opt], rb[opt])
    assert np.all(f <= rf + 1e-7 * np.abs(rf)), (f - rf)
    np.testing.assert_allclose(b[ok], rb[ok], rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(m[:, ok], rm[:, ok], rtol=1e-6)
    np.testing.assert_allclose(h[:, ok], rh[:, ok], rtol=1e-6, atol=1e-12)
    mu_hat = np.ascontiguousarray(rm)
    a, ac = large.alpha_mle(c, X, mu_hat, mom, 1e-8, max_disp)
    ra, rac = ora.alpha_mle(c, X, mu_hat, mom, 1e-8, max_disp)
    interior = (rac == 1) & (ac == 1) & (ra > 1e-5) & (ra < 0.99 * max_disp)
    assert interior.mean() > 0.5
    assert np.mean(np.isclose(a[interior], ra[interior], rtol=1e-4)) >= 0.97
    trend = np.clip(ra, 1e-8, max_disp) * np.exp(rng.normal(0, 0.3, G))
    a2, ac2 = large.alpha_mle(c, X, mu_hat, trend, 1e-8, max_disp, prior_disp_var=0.5, cr_reg=True, prior_reg=True)
    ra2, rac2 = ora.alpha_mle(c, X, mu_hat, trend, 1e-8, max_disp, prior_disp_var=0.5, cr_reg=True, prior_reg=True)
    both = (rac2 == 1) & (ac2 == 1)
    np.testing.assert_allclose(a2[both], ra2[both], rtol=1e-4)
    disp = np.clip(ra2, 1e-8, max_disp)
    contrast = np.zeros(p)
    contrast[-1] = 1.0
    ridge = np.diag(np.repeat(1e-6, p))
    for alt, null in ((None, 0.0), ("greaterAbs", 0.2), ("lessAbs", 0.2), ("greater", 0.1), ("less", 0.1)):
        pv, st, se = large.wald_test(X, disp, rb, mu_hat, ridge, contrast, null, alt)
        rp, rs, rse = ora.wald_test(X, disp, rb, mu_hat, ridge, contrast, null, alt)
        np.testing.assert_allclose(se, rse, rtol=1e-9)
        np.testing.assert_allclose(st, rs, rtol=1e-9, atol=1e-12)
        np.testing.assert_allclose(pv, rp, rtol=1e-8, atol=1e-300)
    with pytest.raises(B200Error, match="not implemented"):
        large.lfc_shrink_nbinom_glm(X, c, 1.0 / disp, np.log(sf), 15, 0.4, "L-BFGS-B", p - 1)


def test_many_contrasts_against_the_oracle(large, ora):
    """wald_tests (K contrasts of one fit, ridge from device memory) against the oracle's wald_test per contrast."""
    p, N = 101, 505
    _, X, c, normed, sf = _problem(p, N)
    mom = _mom(ora, normed, X, sf, N)
    b, _, _, _ = ora.irls(c, sf, X, mom, 0.5, 1e-8)
    cs = np.eye(p)[[1, 5, p - 1]] - np.eye(p)[[2, 6, 3]]
    pv, st, se = large.wald_tests(X, sf, mom, b, cs, ridge_factor=np.diag(np.repeat(1e-6, p)))
    mu = np.ascontiguousarray(np.exp(X @ b.T) * sf[:, None])
    for k, ck in enumerate(cs):
        rp, rs, rse = ora.wald_test(X, mom, b, mu, np.diag(np.repeat(1e-6, p)), ck, 0.0, None)
        np.testing.assert_allclose(se[k], rse, rtol=1e-9)
        np.testing.assert_allclose(st[k], rs, rtol=1e-9, atol=1e-12)
        np.testing.assert_allclose(pv[k], rp, rtol=1e-8, atol=1e-300)


def test_forced_optimizer_branch_and_alpha_grid(large, ora):
    p, N = 80, 401
    _, X, c, normed, sf = _problem(p, N)
    max_disp = float(max(10, N))
    mom = _mom(ora, normed, X, sf, max_disp)
    rm = ora.irls(c, sf, X, mom, 0.5, 1e-8)[1]
    plain = large.irls(c, sf, X, mom, 0.5, 1e-8)
    _set_debug(large, FORCE_IRLS_OPTIMIZER)
    try:
        b, m, h, cv = large.irls(c, sf, X, mom, 0.5, 1e-8)
    finally:
        _set_debug(large, 0)
    assert large.last_irls_fallbacks == c.shape[1]
    # where the min_mu clamp is inactive the objective is smooth: where the projected Newton iteration reports success there, its
    # end point is at least as low as IRLS's deviance-test stop and agrees with it to that level (with N = 5 p most genes have a
    # sample on the clamp; there the iteration may stop on a kink, as at 17..64 columns)
    ok = (plain[1] >= 0.5).all(0) & (cv == 1)
    assert ok.any()
    f, fp = _penalised_nll(c[:, ok], sf, X, mom[ok], b[ok]), _penalised_nll(c[:, ok], sf, X, mom[ok], plain[0][ok])
    assert np.all(f <= fp + 1e-9 * np.abs(fp))
    # IRLS stops on its deviance test; along the flat directions of 80 columns that leaves coefficients up to 1.7e-3 apart (H100)
    np.testing.assert_allclose(b[ok], plain[0][ok], rtol=5e-3, atol=5e-3)
    # a failed minimiser (grid_fit_beta is for two columns only): same coefficients, every gene reported unconverged
    _set_debug(large, FORCE_IRLS_OPTIMIZER | FAIL_IRLS_OPTIMIZER)
    try:
        b2, _, _, cv2 = large.irls(c, sf, X, mom, 0.5, 1e-8)
    finally:
        _set_debug(large, 0)
    assert (cv2 == 0).all()
    np.testing.assert_array_equal(b2, b)
    mu_hat = np.ascontiguousarray(rm)
    _set_debug(large, FORCE_ALPHA_GRID)
    try:
        a, ac = large.alpha_mle(c, X, mu_hat, mom, 1e-8, max_disp)
    finally:
        _set_debug(large, 0)
    assert (ac == 0).all()
    want = np.array([np.exp(nbglm.grid_fit_alpha(c[:, i], X, mu_hat[:, i], mom[i], 1e-8, max_disp)) for i in range(c.shape[1])])
    close = np.isclose(a, want, rtol=1e-9)
    assert close.mean() >= 0.9
    assert np.all(np.abs(np.log(a) - np.log(want)) <= 2 * (np.log(max_disp) - np.log(1e-8)) / 99 * 2 / 99 + 1e-12)


@pytest.mark.parametrize("subjects", [64, 100])
def test_resident_pass_matches_the_plugin_path(large, subjects):
    """A paired design through ResidentFit (three tail launches, device trend) and through the plugin calls (fit_host): the same
    kernels, so the same decisions and values to the e2e tolerance."""
    from pydeseq2_b200.pipeline import ResidentFit, fit_host, median_of_ratios

    X = paired(subjects)
    rng = np.random.default_rng(subjects)
    G = 1500
    beta = np.c_[rng.normal(5.0, 1.5, G), rng.normal(0.0, 0.5, (G, X.shape[1] - 1)) * (rng.random((G, 1)) < 0.4)]
    mu = np.exp(rng.normal(0.0, 0.2, X.shape[0]))[:, None] * np.exp(X @ beta.T)
    d = (0.05 + 2.0 / np.exp(beta[:, 0])) * np.exp(rng.normal(0, 0.3, G))
    c = rng.negative_binomial(1 / d, 1 / (1 + mu * d)).astype(np.int64)
    c = np.ascontiguousarray(c[:, ~(c == 0).all(0)])
    sf = median_of_ratios(c)[1]
    a = fit_host(c, X, large, size_factors=sf)
    rf = ResidentFit(large._ops.ctx, X, sf)
    rf.upload(c)
    r = rf.run()
    rf.close()
    for name in ("dispersions", "pvalue"):
        got, want = np.asarray(r[name]), np.asarray(getattr(a, name))
        np.testing.assert_array_equal(np.isnan(got), np.isnan(want), err_msg=name)
        ok = ~np.isnan(want)
        assert np.mean(np.isclose(got[ok], want[ok], rtol=1e-4, atol=1e-12)) >= 0.99, name
    lfc, want = np.asarray(r["lfc"]).reshape(-1, X.shape[1])[:, -1], np.asarray(a.lfc)[:, -1]
    assert np.mean(np.isclose(lfc, want, rtol=1e-4, atol=1e-6)) >= 0.99


def test_opt_in_contract():
    """pdq_set_large_designs, message by message: its limit, the wide tier's limit without it, the narrow limit without
    wide designs, a cached pack refused once it is off, and apeGLM shrinkage refused with or without wide shrinkage."""
    from pydeseq2_b200.inference import B200Inference

    inf = B200Inference(device=0, wide_designs=True, large_designs=True)
    ctx, lib = inf._ops.ctx, inf._ops.lib
    G = 3

    def lin(X):
        N, p = X.shape
        y = np.ones((N, G), dtype=np.int64)
        return lib.pdq_lin_reg_mu(ctx.h, as_i64p(y), G, N, G, as_f64p(np.ones(N)), as_f64p(np.ascontiguousarray(X)), p, 0.5,
                                  as_f64p(np.zeros((N, G))))

    def contrasts(X):
        N, p = X.shape
        K = 2
        out = [np.zeros((K, G)) for _ in range(3)]
        alt = np.zeros(K, np.int32)
        return lib.pdq_wald_contrasts(ctx.h, as_f64p(np.ascontiguousarray(X)), as_f64p(np.ones(N)), N, p, as_f64p(np.ones(G)),
                                      as_f64p(np.zeros((G, p))), G, as_f64p(np.eye(p)), K, as_f64p(np.ones((K, p))),
                                      as_f64p(np.zeros(K)), alt.ctypes.data_as(C.POINTER(C.c_int)), *(as_f64p(o) for o in out), G)

    X129 = np.ones((300, 129))
    with pytest.raises(B200Error, match="p <= 128"):
        inf.lin_reg_mu(np.ones((300, G), dtype=np.int64), np.ones(300), X129, 0.5)
    assert lin(X129) == -3 and b"wide designs support p <= 128" in lib.pdq_last_error(ctx.h)
    assert contrasts(X129) == -3 and b"pdq_wald_contrasts: design has 129 columns; wide designs support p <= 128" in lib.pdq_last_error(ctx.h)
    # p = 128 is accepted, p = 65 packs are cached
    X65 = paired(64)
    c = np.ascontiguousarray(np.random.default_rng(0).poisson(20, (X65.shape[0], G)).astype(np.int64))
    assert lin(paired(127)) == 0
    inf.lin_reg_mu(c, np.ones(X65.shape[0]), X65, 0.5)
    # apeGLM shrinkage above 64 columns: not implemented, with and without wide shrinkage
    for ws in (False, True):
        ctx.set_wide_shrink(ws)
        with pytest.raises(B200Error, match="not implemented"):
            inf.lfc_shrink_nbinom_glm(X65, c, np.ones(G), np.zeros(X65.shape[0]), 15, 0.4, "L-BFGS-B", 64)
    ctx.set_wide_shrink(False)
    # large designs off again: the cached p = 65 pack is refused with the wide tier's limit and message
    ctx.set_large_designs(False)
    with pytest.raises(B200Error, match="p <= 64"):
        inf.lin_reg_mu(c, np.ones(X65.shape[0]), X65, 0.5)
    assert lin(X65) == -3 and b"wide designs support p <= 64" in lib.pdq_last_error(ctx.h)
    assert contrasts(X65) == -3 and b"wide designs support p <= 64" in lib.pdq_last_error(ctx.h)
    # large designs without wide designs: the narrow limit
    ctx.set_large_designs(True)
    ctx.set_wide_designs(False)
    with pytest.raises(B200Error, match="p <= 16"):
        inf.lin_reg_mu(c, np.ones(X65.shape[0]), X65, 0.5)
    assert lin(paired(16)) == -3 and b"this build supports p <= 16" in lib.pdq_last_error(ctx.h)


@pytest.mark.parametrize("p", [17, 33, 64])
def test_large_opt_in_leaves_wide_designs_byte_identical(p):
    """Designs of 64 columns or fewer run the same kernels with large designs on and off: a plugin-path fit is byte-equal."""
    from pydeseq2_b200.inference import B200Inference
    from pydeseq2_b200.pipeline import fit_host

    _, X, c, _, sf = _problem(p, 10 * p + 1)
    outs = [fit_host(c, X, B200Inference(device=0, wide_designs=True, large_designs=on), size_factors=sf) for on in (False, True)]
    for name in ("lfc", "dispersions", "genewise", "map", "pvalue", "stat", "se", "mu_lfc", "hat"):
        np.testing.assert_array_equal(np.asarray(getattr(outs[0], name)), np.asarray(getattr(outs[1], name)), err_msg=name)


def test_large_opt_in_leaves_a_resident_pass_byte_identical():
    """A C2-shaped resident pass (20 000 genes x 200 samples, two-level design) is byte-equal with large designs on and off."""
    from pydeseq2_b200.inference import B200Inference
    from pydeseq2_b200.pipeline import ResidentFit, median_of_ratios
    from pydeseq2_b200.synth import make_counts

    counts, X, _ = make_counts(200, 20000, "two_level", seed=7)
    counts = np.ascontiguousarray(counts[:, ~(counts == 0).all(0)])
    _, sf = median_of_ratios(counts)
    outs = []
    for on in (False, True):
        inf = B200Inference(device=0, wide_designs=True, large_designs=on)
        rf = ResidentFit(inf._ops.ctx, X, sf, with_cooks=True)
        rf.upload(counts)
        outs.append(rf.run())
        rf.close()
    r0, r1 = outs
    assert r0.keys() == r1.keys()
    for name in r0:
        v0, v1 = r0[name], r1[name]
        if isinstance(v0, np.ndarray):
            np.testing.assert_array_equal(v0, v1, err_msg=name)


@pytest.mark.parametrize("subjects", [20, 100], ids=["p21", "p101"])
def test_pipelined_wald_tests_are_byte_identical(monkeypatch, subjects):
    """wald_tests (K = 4) and wald_test through the gene-block pipeline and without it: byte-equal.  The pipeline uploads the
    Wald ridge and contrast into the design's device buffer once per gene block, on that block's stream, so an upload may
    overwrite the buffer while the previous block's kernel reads it; every upload of one call writes the same bytes.
    pipe_begin splits a call when G >= 4096, staging is on and every large host buffer is page-locked: here the (K, G) outputs
    of wald_tests (K G = 65 536 elements, from which the backend hands out page-locked outputs) and the (N, G) mu of wald_test.
    G = 16 384 gives four blocks of 4 096 genes, so the pipelined context counts four times the launches of the other."""
    from pydeseq2_b200.inference import B200Inference

    X = paired(subjects)
    N, p = X.shape
    G, K = 16384, 4
    rng = np.random.default_rng(subjects)
    lfc = np.c_[rng.normal(5.0, 1.0, G), rng.normal(0.0, 0.3, (G, p - 1))]
    disp = np.exp(rng.uniform(np.log(0.05), np.log(0.5), G))
    sf = np.exp(rng.normal(0.0, 0.2, N))
    cs = np.eye(p)[[p - 1, 1, 2, p - 1]] - np.eye(p)[[0, 2, 3, 1]]
    alts = [None, "greaterAbs", "greater", "lessAbs"]
    monkeypatch.delenv("PDQ_PIPELINE", raising=False)
    infs = [B200Inference(device=0, wide_designs=True, large_designs=True)]
    monkeypatch.setenv("PDQ_PIPELINE", "0")  # read when the context is created
    infs.append(B200Inference(device=0, wide_designs=True, large_designs=True))
    outs, launches = [], []
    for inf in infs:
        ctx = inf._ops.ctx
        mu = ctx.pinned_empty((N, G))
        mu[:] = sf[:, None] * np.exp(X @ lfc.T)
        n0 = ctx.launches()
        many = inf.wald_tests(X, sf, disp, lfc, cs, lfc_null=0.1, alt_hypothesis=alts)
        n1 = ctx.launches()
        one = inf.wald_test(X, disp, lfc, mu, np.diag(np.repeat(1e-6, p)), cs[0], 0.1, "greaterAbs")
        launches.append((n1 - n0, ctx.launches() - n1))
        outs.append(list(many) + list(one))
    assert launches[0] == (4 * launches[1][0], 4 * launches[1][1])
    assert np.isfinite(outs[1][0]).mean() > 0.99
    for name, a, b in zip(["pvalue", "stat", "se"] * 2, *outs):
        np.testing.assert_array_equal(a.view(np.uint64), b.view(np.uint64), err_msg=name)


@pytest.mark.parametrize("resident", [False, True])
@pytest.mark.parametrize("name", [n if n in ("large_paired_p101", "large_levels_p70_outliers") else
                                  pytest.param(n, marks=pytest.mark.xfail(strict=True, reason=MULTIMODAL_REASON)) for n in LARGE_E2E])
def test_end_to_end_tables_match_the_real_orchestrator(large, name, resident):
    """deseq2() + summary() through both drivers against the final tables the real reference wrote (scripts/make_large_golden.py):
    replaced / refitted / Cook's-outlier sets and NaN patterns identical, values within the e2e tolerance except the measured
    per-fixture budget of tests/large_cases.py.  The 70-level case runs the lin_reg_mu start, Cook's replacement and the refit of
    both drivers."""
    check_large_e2e(large, name, resident=resident)


def test_contrasts_of_the_70_level_fit_against_the_reference(large):
    """wald_tests on the reference's stored fit, 20 pairwise contrasts: <= 1e-9 from its run_wald_test."""
    from contrast_cases import check_golden_wald

    check_golden_wald(large, "large_ct_levels_p70", 1e-9)


@pytest.mark.parametrize("resident", [False, True])
def test_deseq2_stats_of_the_70_level_fit(large, resident):
    """workflow.deseq2_stats on both drivers against every contrast's results_df, at the tolerances of the wide suite."""
    from contrast_cases import check_stats_e2e

    check_stats_e2e(large, "large_ct_levels_p70", 2e-4, max_frac=0.02, resident=resident)


def test_vst_with_the_design_against_the_reference(large):
    """vst(use_design=True) on the paired p = 101 design: trend and transformed counts within 1e-4 (as the vst_* fixtures)."""
    from conftest import load_golden
    from pydeseq2_b200.workflow import vst

    z = load_golden("large_vst_paired_p101_design")
    fit = vst(z["counts"], z["design"], large, fit_type=str(z["fit_type"]), use_design=True)
    assert fit.kind == str(z["vst_fit_type"]) == "parametric"
    np.testing.assert_allclose(fit.size_factors, z["size_factors"], rtol=1e-10)
    np.testing.assert_allclose(fit.coeffs, z["vst_trend_coeffs"], rtol=1e-4)
    got, want = fit.vst_counts, z["vst_counts"]
    np.testing.assert_array_equal(np.isfinite(got), np.isfinite(want))
    ok = np.isfinite(want)
    assert np.all(np.abs(got[ok] - want[ok]) <= 1e-4 * np.maximum(np.abs(want[ok]), 1.0))
