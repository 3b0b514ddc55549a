"""GPU suite: apeGLM shrinkage of designs of 17..64 columns on a backend that opted in to wide designs and wide shrinkage
(B200Inference(wide_designs=True, wide_shrink=True)), against the real reference's calls (scripts/make_wide_shrink_golden.py), the
oracle, and the real orchestrator's shrunk results table."""
import numpy as np
import pytest

from conftest import load_golden
from edge_cases import _counts, _design
from oracle import nbglm
from parity import SHRINK, TOL_SHRINK, report
from pydeseq2_b200._lib import B200Error
from wide_cases import RTOL

pytestmark = pytest.mark.gpu

NOT_IMPLEMENTED = b"lfc_shrink: apeGLM shrinkage of designs with more than 16 columns is not implemented"

# Per fixture: genes whose end point is not within TOL_SHRINK of scipy's, and how much higher (relative) the kernel's scaled
# objective may be there.  The kernel walks scipy's L-BFGS-B iteration, but its sums run in another order; an iterate that differs in
# the last bits can take another line-search step, and from there the paths separate, each ending where the ftol = 1e-8 rule stops
# it.  In the 17-level case the adapted prior scale is 0.001 (the prior variance at its lower bound): the shrunk coefficient sits
# in the Cauchy prior's spike, and 36 of 299 paths separate; the kernel's objective is lower at 19 of them (by up to 1.3e-5) and
# higher at 17, by at most 6.7e-10.  Measured on an H100 (DESIGN.md §8).
BUDGET_CALLS = {"wide_shrink_paired_p21": (0, 1e-10), "wide_shrink_paired_p21_noadapt": (0, 1e-10),
                "wide_shrink_levels_p17_outliers": (36, 1e-9), "wide_shrink_paired_covariate_p33": (10, 1e-10),
                "wide_shrink_paired_p64": (6, 1e-10)}
# shrunk log2FoldChange / lfcSE of the end-to-end p = 21 case: genes outside the e2e tolerance and their worst relative error.  The
# shrinkage runs on the fit's own dispersions, so the genes of the unshrunk table's budget (tests/wide_cases.py) carry over.
# Measured on an H100 for both drivers: 2 genes, 1.3e-3.
BUDGET_E2E = (2, 2e-3)


@pytest.fixture(scope="module")
def both():
    from pydeseq2_b200.inference import B200Inference

    return B200Inference(device=0, wide_designs=True, wide_shrink=True)


@pytest.fixture(scope="module")
def ora():
    return nbglm.OracleInference(n_cpus=4)


def scaled_objective(X, y, size, offset, prior_no_shrink_scale, prior_scale, k, b):
    """The reference's objective (nbinomFn, utils.py:1148-1207) at the rows of `b`, divided by max(f(0), 1) as nbinomGLM does."""
    def f(b):
        xb = b @ X.T
        nll = (y * xb - (y + size[:, None]) * np.logaddexp(xb + offset, np.log(size)[:, None])).sum(1)
        others = np.delete(b, k, axis=1)
        prior = (others ** 2).sum(1) / (2 * prior_no_shrink_scale ** 2) + np.log1p((b[:, k] / prior_scale) ** 2)
        return prior - nll

    return f(b) / np.maximum(f(np.zeros_like(b)), 1.0)


def check_against(inf, X, counts, size, offset, scale, k, lfcs_ref, ih_col_ref, conv_ref, ih_head_ref, name, budget, slack=1e-10):
    """Converged flags equal; LFCs and column k of the inverse Hessians within TOL_SHRINK except at most `budget` genes, where the
    kernel's end point must have a scaled objective no higher than the reference's plus `slack` relative."""
    lfcs, ih, conv = inf.lfc_shrink_nbinom_glm(X, counts, size, offset, 15, scale, "L-BFGS-B", k)
    G, p = lfcs.shape
    assert ih.shape == (G, p, p)
    np.testing.assert_array_equal(conv, conv_ref)
    same = (np.isclose(lfcs, lfcs_ref, rtol=TOL_SHRINK, atol=1e-10).all(1)
            & np.isclose(ih[:, :, k], ih_col_ref, rtol=TOL_SHRINK, atol=1e-14).all(1))
    if ih_head_ref is not None:
        h = len(ih_head_ref)
        same[:h] &= np.isclose(ih[:h], ih_head_ref, rtol=TOL_SHRINK, atol=1e-14).all((1, 2))
    div = ~same
    y = np.asarray(counts, dtype=float).T
    f, fr = (scaled_objective(X, y[div], size[div], offset, 15.0, scale, k, b[div]) for b in (lfcs, lfcs_ref))
    report("wide_shrink", name, genes=int(G), divergent=int(div.sum()),
           worst_lfc=float(np.max(np.abs(lfcs - lfcs_ref) / np.maximum(np.abs(lfcs_ref), 1e-10))) if G else 0.0,
           worst_objective_gap=float(np.max((f - fr) / np.abs(fr))) if div.any() else 0.0)
    assert div.sum() <= budget, (name, int(div.sum()), np.flatnonzero(div)[:10])
    assert np.all(f <= fr + slack * np.abs(fr)), (name, (f - fr) / np.abs(fr))
    return lfcs, ih, conv


@pytest.mark.parametrize("name", list(BUDGET_CALLS))
def test_calls_match_the_reference(both, name):
    g = load_golden(name)
    check_against(both, g["X"], g["counts"], g["size"], g["offset"], float(g["prior_scale"]), int(g["shrink_index"]), g["lfcs"],
                  g["inv_hessian_col"], g["converged"], g["inv_hessians_head"], name, *BUDGET_CALLS[name])


def _problem(p, N):
    rng = np.random.default_rng(100 + p)
    X = _design(rng, N, p)
    c = _counts(rng, X, 48)
    sf = c.sum(1) / np.exp(np.log(c.sum(1)).mean())
    disp = 4 / np.maximum(c.mean(0), 1.0) + 0.1
    return X, c, sf, disp


@pytest.mark.parametrize("p,N", [(17, 171), (24, 241), (32, 321), (48, 481), (64, 641)])
def test_against_the_oracle(both, ora, p, N):
    """Last column and a middle column, adapted-looking and unit prior scales.  Measured on an H100: every gene within TOL_SHRINK
    of the oracle; scipy's sums come from the host's BLAS, so two genes may still take another path."""
    X, c, sf, disp = _problem(p, N)
    size, offset = 1.0 / disp, np.log(sf)
    for k, scale in ((p - 1, 0.4), (p // 2, 1.0)):
        rl, rih, rc = ora.lfc_shrink_nbinom_glm(X, c, size, offset, 15, scale, "L-BFGS-B", k)
        check_against(both, X, c, size, offset, scale, k, rl, rih[:, :, k], rc, rih, f"oracle_p{p}_k{k}", 2)


@pytest.mark.parametrize("resident", [False, True])
def test_end_to_end_shrinkage_matches_the_real_orchestrator(both, resident):
    """deseq2() + summary() + lfc_shrink(coeff=condition) through both drivers against the real orchestrator on the paired p = 21
    design: the shrunk log2FoldChange / lfcSE within the e2e tolerance except BUDGET_E2E."""
    from pydeseq2_b200.workflow import deseq2_results, deseq2_results_resident

    g = load_golden("wide_shrinktape_paired_p21")
    counts, X, k = np.ascontiguousarray(g["counts"], dtype=np.int64), g["design"], int(g["shrink_index"])
    if resident:
        from pydeseq2_b200.pipeline import ResidentFit

        nz = ~(counts == 0).all(0)
        rf = ResidentFit(both._ops.ctx, X, None)
        rf.upload(np.ascontiguousarray(counts[:, nz]))
        try:
            r = deseq2_results_resident(rf, g["contrast"], non_zero=nz, shrink_coeff=k)
        finally:
            rf.close()
    else:
        r = deseq2_results(counts, X, both, g["contrast"], shrink_coeff=k)
    assert r.shrink_prior_scale == pytest.approx(float(g["prior_scale"]), rel=RTOL)
    genes, bound = BUDGET_E2E
    rec, fails = {}, []
    for key, got, want in (("log2FoldChange", r.log2_fold_change, g["final_log2FoldChange"]), ("lfcSE", r.lfc_se, g["final_lfcSE"])):
        got = np.asarray(got, dtype=float)
        np.testing.assert_array_equal(np.isnan(got), np.isnan(want), err_msg=key)
        bad = ~np.isclose(got, want, rtol=RTOL, atol=1e-8, equal_nan=True)
        worst = float(np.nanmax(np.abs(got - want)[bad] / np.abs(want[bad]))) if bad.any() else 0.0
        rec[key + "_genes"], rec[key + "_worst"] = int(bad.sum()), worst
        if bad.sum() > genes or worst > bound:
            fails.append((key, int(bad.sum()), worst))
    report("wide_shrink_e2e", "paired_p21" + (" [resident]" if resident else ""), **rec)
    assert not fails, fails
    # p-values are not touched by the shrinkage
    np.testing.assert_array_equal(np.isnan(r.pvalue), np.isnan(g["results_pvalue"]))


def test_resident_shrink_equals_the_plugin_call(both):
    """ResidentFit.lfc_shrink (resident counts, strided download of column k and the [k, k] entries) against lfc_shrink_host on the
    same run's dispersions and tables."""
    from pydeseq2_b200.pipeline import FitResult, ResidentFit, lfc_shrink_host

    g = load_golden("wide_shrinktape_paired_p21")
    counts, X, k = np.ascontiguousarray(g["counts"], dtype=np.int64), g["design"], int(g["shrink_index"])
    counts = np.ascontiguousarray(counts[:, ~(counts == 0).all(0)])
    G = counts.shape[1]
    rf = ResidentFit(both._ops.ctx, X, None)
    try:
        rf.upload(counts)
        r = rf.run(contrast=np.eye(X.shape[1])[k])
        sh_dev = rf.lfc_shrink(r, k)
        fit = FitResult(*([None] * len(FitResult.__dataclass_fields__)))
        fit.size_factors, fit.non_zero, fit.dispersions = rf.sf, np.ones(G, bool), np.asarray(r["dispersions"])
        fit.lfc, fit.se = np.asarray(r["lfc"]), np.asarray(r["se"])
        sh_host = lfc_shrink_host(fit, counts, X, both, k)
    finally:
        rf.close()
    assert sh_dev.prior_scale == sh_host.prior_scale
    np.testing.assert_allclose(sh_dev.lfc, sh_host.lfc, rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(sh_dev.se, sh_host.se, rtol=1e-9)
    np.testing.assert_array_equal(sh_dev.converged, sh_host.converged)


def test_opt_in_contract():
    """Wide shrinkage is its own opt-in on top of wide designs."""
    import ctypes as C

    from pydeseq2_b200._lib import as_f64p, as_i64p
    from pydeseq2_b200.inference import B200Inference

    with pytest.raises(ValueError, match="wide_designs"):
        B200Inference(device=0, wide_shrink=True)
    X, c, sf, disp = _problem(17, 60)
    args = (X, c, 1.0 / disp, np.log(sf), 15, 0.4, "L-BFGS-B", 16)
    inf = B200Inference(device=0, wide_designs=True)
    ctx, lib = inf._ops.ctx, inf._ops.lib
    # wide designs on, wide shrinkage off: the error code and message of the parent
    with pytest.raises(B200Error, match="not implemented"):
        inf.lfc_shrink_nbinom_glm(*args)
    assert lib.pdq_last_error(ctx.h) == NOT_IMPLEMENTED
    ctx.set_wide_shrink(True)
    lfcs, ih, conv = inf.lfc_shrink_nbinom_glm(*args)
    assert np.isfinite(lfcs).all() and np.isfinite(ih).all() and set(np.unique(conv)) <= {0.0, 1.0}
    # off again: refused, also with the design pack cached
    ctx.set_wide_shrink(False)
    with pytest.raises(B200Error, match="not implemented"):
        inf.lfc_shrink_nbinom_glm(*args)
    assert lib.pdq_last_error(ctx.h) == NOT_IMPLEMENTED
    # wide shrinkage on, wide designs off: refused as any design of more than 16 columns, by the Python check and the C ABI
    ctx.set_wide_shrink(True)
    ctx.set_wide_designs(False)
    with pytest.raises(B200Error, match="p <= 16"):
        inf.lfc_shrink_nbinom_glm(*args)
    N, G = c.shape
    out = [np.zeros((G, 17)), np.zeros((G, 17, 17)), np.zeros(G)]
    n_grid = C.c_int(0)
    rc = lib.pdq_lfc_shrink_nbinom_glm(ctx.h, as_f64p(np.ascontiguousarray(X)), as_i64p(c), G, N, G, 17, as_f64p(1.0 / disp),
                                       as_f64p(np.log(sf)), 15.0, 0.4, 16, *(as_f64p(o) for o in out), C.byref(n_grid))
    assert rc == -3 and b"p <= 16" in lib.pdq_last_error(ctx.h)


def test_wide_shrink_leaves_narrow_designs_byte_identical():
    """Every narrow shrink_* / shrinktape_* fixture gives byte-equal outputs with wide shrinkage on and off."""
    from pydeseq2_b200.inference import B200Inference

    off, on = B200Inference(device=0, wide_designs=True), B200Inference(device=0, wide_designs=True, wide_shrink=True)
    for name in SHRINK:
        g = load_golden(name)
        args = (g["X"], g["counts"], g["size"], g["offset"], float(g["prior_no_shrink_scale"]), float(g["prior_scale"]), "L-BFGS-B",
                int(g["shrink_index"]))
        for a, b in zip(off.lfc_shrink_nbinom_glm(*args), on.lfc_shrink_nbinom_glm(*args)):
            np.testing.assert_array_equal(a, b, err_msg=name)
