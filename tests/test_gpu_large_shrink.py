"""GPU suite: apeGLM shrinkage of designs of 65..128 columns on a backend that opted in to wide designs, wide shrinkage, large
designs and large shrinkage (B200Inference(wide_designs=True, wide_shrink=True, large_designs=True, large_shrink=True)), against the
real reference's calls (scripts/make_large_shrink_golden.py), the oracle, and the real orchestrator's shrunk results table."""
import ctypes as C

import numpy as np
import pytest

from conftest import load_golden
from oracle import nbglm
from parity import TOL_SHRINK
from pydeseq2_b200._lib import B200Error, as_f64p, as_i64p
from test_gpu_wide_shrink import BUDGET_CALLS as WIDE_BUDGET_CALLS
from test_gpu_wide_shrink import _problem, check_against
from test_large_designs import paired
from wide_cases import RTOL

pytestmark = pytest.mark.gpu

NOT_IMPLEMENTED_16 = b"lfc_shrink: apeGLM shrinkage of designs with more than 16 columns is not implemented"
NOT_IMPLEMENTED_64 = b"lfc_shrink: apeGLM shrinkage of designs with more than 64 columns is not implemented"

# Per fixture: genes whose end point is not within TOL_SHRINK of scipy's, and how much higher (relative) the kernel's scaled
# objective may be there (see tests/test_gpu_wide_shrink.py: sums in another order can make a line search take another step, and
# from there the paths separate until the ftol = 1e-8 rule stops each; the more columns, the more genes separate).  Measured on an
# H100 (DESIGN.md §8): 3, 16, 15, 23 and 47 genes, worst gaps 9.3e-14, 7.6e-11, 2.0e-10, 4.0e-8 and 3.2e-6.  In the 70-level case
# the adapted prior scale is 0.001, which puts the shrunk coefficient in the Cauchy prior's spike, as in the 17-level wide case.
BUDGET_CALLS = {"large_shrink_paired_p65": (3, 1e-10), "large_shrink_paired_p101": (16, 1e-10),
                "large_shrink_paired_p101_noadapt": (15, 3e-10), "large_shrink_paired_p128": (23, 5e-8),
                "large_shrink_levels_p70_outliers": (47, 4e-6)}
# against the oracle (48 genes): genes off scipy's path per width, over both shrunk columns and every W; the kernel's objective is
# within 1e-13 of the oracle's at every one of them (measured on an H100)
BUDGET_ORACLE = {65: 2, 80: 2, 101: 10, 128: 16}
# shrunk log2FoldChange / lfcSE of the end-to-end p = 101 case: genes outside the e2e tolerance and their worst relative error.  The
# shrinkage starts from the fit's own dispersions (within RTOL of the reference's, tests/large_cases.py), and at 101 columns the
# shrunk fit moves with them: measured on an H100 for both drivers, 45 genes, 1.2e-2 (log2FoldChange) and 11 genes, 3.2e-4 (lfcSE).
BUDGET_E2E = (45, 1.2e-2)


def _backend(**kw):
    from pydeseq2_b200.inference import B200Inference

    return B200Inference(device=0, wide_designs=True, wide_shrink=True, large_designs=True, **kw)


@pytest.fixture(scope="module")
def all4():
    return _backend(large_shrink=True)


@pytest.fixture(scope="module")
def ora():
    return nbglm.OracleInference(n_cpus=4)


@pytest.mark.parametrize("name", list(BUDGET_CALLS))
def test_calls_match_the_reference(all4, name):
    g = load_golden(name)
    check_against(all4, g["X"], g["counts"], g["size"], g["offset"], float(g["prior_scale"]), int(g["shrink_index"]), g["lfcs"],
                  g["inv_hessian_col"], g["converged"], g["inv_hessians_head"], name, *BUDGET_CALLS[name])


def _check_oracle(inf, ora, p, tag):
    X, c, sf, disp = _problem(p, 10 * p + 1)
    size, offset = 1.0 / disp, np.log(sf)
    for k, scale in ((p - 1, 0.4), (p // 2, 1.0)):
        rl, rih, rc = ora.lfc_shrink_nbinom_glm(X, c, size, offset, 15, scale, "L-BFGS-B", k)
        check_against(inf, X, c, size, offset, scale, k, rl, rih[:, :, k], rc, rih, f"oracle_p{p}_k{k}{tag}", BUDGET_ORACLE[p])


@pytest.mark.parametrize("p", [65, 80, 101, 128])
def test_against_the_oracle(all4, ora, p):
    """Last column (scale 0.4) and a middle column (scale 1), 48 genes, N = 10 p + 1."""
    _check_oracle(all4, ora, p, "")


@pytest.mark.parametrize("warps", [2, 4, 8])
def test_every_team_width_agrees_with_the_oracle(ora, monkeypatch, warps):
    """The same problem at p = 101 with 2, 4 and 8 warps per gene (PDQ_LARGE_WARPS, read when a design pack is made), so every
    width runs whatever large_warps picks."""
    monkeypatch.setenv("PDQ_LARGE_WARPS", str(warps))
    _check_oracle(_backend(large_shrink=True), ora, 101, f"_w{warps}")


@pytest.mark.parametrize("resident", [False, True])
def test_end_to_end_shrinkage_matches_the_real_orchestrator(all4, resident):
    """deseq2() + summary() + lfc_shrink(coeff=condition) through both drivers against the real orchestrator on the paired p = 101
    design: the prior scale within RTOL, the shrunk log2FoldChange / lfcSE within the e2e tolerance except BUDGET_E2E, and the
    p-values untouched."""
    from parity import report
    from pydeseq2_b200.workflow import deseq2_results, deseq2_results_resident

    g = load_golden("large_shrinktape_paired_p101")
    counts, X, k = np.ascontiguousarray(g["counts"], dtype=np.int64), g["design"], int(g["shrink_index"])
    if resident:
        from pydeseq2_b200.pipeline import ResidentFit

        nz = ~(counts == 0).all(0)
        rf = ResidentFit(all4._ops.ctx, X, None)
        rf.upload(np.ascontiguousarray(counts[:, nz]))
        try:
            r = deseq2_results_resident(rf, g["contrast"], non_zero=nz, shrink_coeff=k)
            u = deseq2_results_resident(rf, g["contrast"], non_zero=nz)
        finally:
            rf.close()
    else:
        r = deseq2_results(counts, X, all4, g["contrast"], shrink_coeff=k)
        u = deseq2_results(counts, X, all4, g["contrast"])
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
    report("large_shrink_e2e", "paired_p101" + (" [resident]" if resident else ""), **rec)
    assert not fails, fails
    # p-values are not touched by the shrinkage: the same as the unshrunk run's, NaN where the reference's are
    np.testing.assert_array_equal(np.asarray(r.pvalue), np.asarray(u.pvalue))
    np.testing.assert_array_equal(np.isnan(r.pvalue), np.isnan(g["results_pvalue"]))


def test_resident_shrink_equals_the_plugin_call(all4):
    """ResidentFit.lfc_shrink (resident counts, strided download of column k and the [k, k] entries) against lfc_shrink_host on the
    same run's dispersions and tables, at p = 101.  The two calls reach the kernel through different buffers and set-up, and at 101
    columns their end points differ by up to 4e-9 (measured on an H100), so they are held to TOL_SHRINK."""
    from pydeseq2_b200.pipeline import FitResult, ResidentFit, lfc_shrink_host

    g = load_golden("large_shrinktape_paired_p101")
    counts, X, k = np.ascontiguousarray(g["counts"], dtype=np.int64), g["design"], int(g["shrink_index"])
    counts = np.ascontiguousarray(counts[:, ~(counts == 0).all(0)])
    G = counts.shape[1]
    rf = ResidentFit(all4._ops.ctx, X, None)
    try:
        rf.upload(counts)
        r = rf.run(contrast=np.eye(X.shape[1])[k])
        sh_dev = rf.lfc_shrink(r, k)
        fit = FitResult(*([None] * len(FitResult.__dataclass_fields__)))
        fit.size_factors, fit.non_zero, fit.dispersions = rf.sf, np.ones(G, bool), np.asarray(r["dispersions"])
        fit.lfc, fit.se = np.asarray(r["lfc"]), np.asarray(r["se"])
        sh_host = lfc_shrink_host(fit, counts, X, all4, k)
    finally:
        rf.close()
    assert sh_dev.prior_scale == sh_host.prior_scale
    np.testing.assert_allclose(sh_dev.lfc, sh_host.lfc, rtol=TOL_SHRINK, atol=1e-12)
    np.testing.assert_allclose(sh_dev.se, sh_host.se, rtol=TOL_SHRINK)
    np.testing.assert_array_equal(sh_dev.converged, sh_host.converged)


def test_opt_in_contract():
    """pdq_set_large_shrink, message by message and by C ABI code: wide shrinkage off, large designs off (cached pack), large
    shrinkage off, all on, and large shrinkage off again."""
    inf = _backend()
    ctx, lib = inf._ops.ctx, inf._ops.lib
    G = 3
    X = paired(64)
    N = X.shape[0]
    c = np.ascontiguousarray(np.random.default_rng(0).poisson(20, (N, G)).astype(np.int64))
    size, offset = np.ones(G), np.zeros(N)
    args = (X, c, size, offset, 15, 0.4, "L-BFGS-B", 64)

    def abi():
        out = [np.zeros((G, 65)), np.zeros((G, 65, 65)), np.zeros(G)]
        n_grid = C.c_int(0)
        return lib.pdq_lfc_shrink_nbinom_glm(ctx.h, as_f64p(np.ascontiguousarray(X)), as_i64p(c), G, N, G, 65, as_f64p(size),
                                             as_f64p(offset), 15.0, 0.4, 64, *(as_f64p(o) for o in out), C.byref(n_grid))

    def refused(match, msg):
        with pytest.raises(B200Error, match=match):
            inf.lfc_shrink_nbinom_glm(*args)
        assert lib.pdq_last_error(ctx.h) == msg
        assert abi() == -3 and lib.pdq_last_error(ctx.h) == msg

    # wide shrinkage off: the narrow message, whatever the other opt-ins
    ctx.set_wide_shrink(False)
    ctx.set_large_shrink(True)
    refused("not implemented", NOT_IMPLEMENTED_16)
    # all four on: runs (the p = 65 pack is cached from here on)
    ctx.set_wide_shrink(True)
    lfcs, ih, conv = inf.lfc_shrink_nbinom_glm(*args)
    assert lfcs.shape == (G, 65) and ih.shape == (G, 65, 65) and np.isfinite(lfcs).all() and np.isfinite(ih).all()
    assert set(np.unique(conv)) <= {0.0, 1.0}
    assert abi() == 0
    # large designs off: the wide tier's limit, also for the cached pack
    ctx.set_large_designs(False)
    with pytest.raises(B200Error, match="p <= 64"):
        inf.lfc_shrink_nbinom_glm(*args)
    assert abi() == -3 and b"wide designs support p <= 64" in lib.pdq_last_error(ctx.h)
    # large shrinkage off (large designs on again): not implemented above 64 columns, as before the opt-in existed
    ctx.set_large_designs(True)
    ctx.set_large_shrink(False)
    refused("not implemented", NOT_IMPLEMENTED_64)
    # on, then off again
    ctx.set_large_shrink(True)
    assert abi() == 0
    ctx.set_large_shrink(False)
    refused("not implemented", NOT_IMPLEMENTED_64)


def test_large_shrink_leaves_wide_designs_byte_identical():
    """Every wide_shrink_* fixture (17..64 columns) gives byte-equal outputs with large shrinkage on and off."""
    off, on = _backend(), _backend(large_shrink=True)
    for name in WIDE_BUDGET_CALLS:
        g = load_golden(name)
        args = (g["X"], g["counts"], g["size"], g["offset"], float(g["prior_no_shrink_scale"]), float(g["prior_scale"]), "L-BFGS-B",
                int(g["shrink_index"]))
        for a, b in zip(off.lfc_shrink_nbinom_glm(*args), on.lfc_shrink_nbinom_glm(*args)):
            np.testing.assert_array_equal(a, b, err_msg=name)
