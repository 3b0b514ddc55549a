"""CPU suite: the large_shrink* fixtures (scripts/make_large_shrink_golden.py, apeGLM shrinkage of designs of 65..128 columns)
against the oracle's lfc_shrink_nbinom_glm, which runs scipy's L-BFGS-B as the reference does, and the checks of
B200Inference(large_shrink=True) that run before any device work.  tests/test_gpu_large_shrink.py holds the GPU kernel to the
fixtures."""
import numpy as np
import pytest

from conftest import load_golden
from oracle import nbglm
from pydeseq2_b200.inference import B200Inference

LARGE_SHRINK = ["large_shrink_paired_p65", "large_shrink_paired_p101", "large_shrink_paired_p101_noadapt", "large_shrink_paired_p128",
                "large_shrink_levels_p70_outliers"]


@pytest.fixture(scope="module")
def ora():
    return nbglm.OracleInference(n_cpus=4)


@pytest.mark.parametrize("name", LARGE_SHRINK)
def test_oracle_reproduces_the_reference(ora, name):
    g = load_golden(name)
    k, (N, G), p = int(g["shrink_index"]), g["counts"].shape, g["X"].shape[1]
    assert 65 <= p <= 128 and g["lfcs"].shape == (G, p) and g["inv_hessian_col"].shape == (G, p)
    assert g["inv_hessians_head"].shape == (min(G, 40, (1 << 17) // (8 * p * p)), p, p) and g["nit"].shape == g["nfev"].shape == (G,)
    assert g["offset"].shape == (N,) and g["size"].shape == (G,) and g["mle_lfc"].shape == g["mle_se"].shape == (G,)
    if "noadapt" in name:
        assert float(g["prior_scale"]) == 1.0
    else:  # the prior scale the reference derived from the MLE LFCs and their SEs (ds.py:551-585)
        assert nbglm.fit_shrink_prior_var(g["mle_lfc"], g["mle_se"]) == pytest.approx(float(g["prior_var"]), rel=1e-9)
        assert float(g["prior_scale"]) == min(np.sqrt(float(g["prior_var"])), 1.0)
    lfcs, ih, conv = ora.lfc_shrink_nbinom_glm(g["X"], g["counts"], g["size"], g["offset"], float(g["prior_no_shrink_scale"]),
                                               float(g["prior_scale"]), "L-BFGS-B", k)
    np.testing.assert_array_equal(conv, g["converged"])
    np.testing.assert_allclose(lfcs, g["lfcs"], rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(ih[:, :, k], g["inv_hessian_col"], rtol=1e-9, atol=1e-14)
    np.testing.assert_allclose(ih[:len(g["inv_hessians_head"])], g["inv_hessians_head"], rtol=1e-9, atol=1e-14)


def test_end_to_end_fixture_layout():
    g = load_golden("large_shrinktape_paired_p101")
    N, G = g["counts"].shape
    k = int(g["shrink_index"])
    assert g["design"].shape == (N, 101) and k == 100 and g["contrast"][k] == 1.0
    assert 0.0 < float(g["prior_scale"]) <= 1.0
    for key in ("final_log2FoldChange", "final_lfcSE", "mle_log2FoldChange", "results_pvalue", "results_padj"):
        assert g[key].shape == (G,), key
    # the shrunk column differs from the MLE one, and shrinks it towards zero on most genes (85 %: with a prior scale of 0.63 the
    # refit of the 100 other coefficients moves some small LFCs outwards by up to 0.004)
    ok = np.isfinite(g["final_log2FoldChange"]) & np.isfinite(g["mle_log2FoldChange"])
    assert (np.abs(g["final_log2FoldChange"][ok]) <= np.abs(g["mle_log2FoldChange"][ok]) + 1e-12).mean() > 0.8
    assert not np.array_equal(g["final_log2FoldChange"], g["mle_log2FoldChange"])


@pytest.mark.parametrize("kw", [dict(wide_designs=True, wide_shrink=True), dict(wide_designs=True, large_designs=True),
                                dict(large_designs=True, wide_shrink=True), dict()])
def test_large_shrink_needs_the_other_three_opt_ins(kw):
    # raised before any context is created, so no device is needed (without wide_designs, by the check of wide_shrink or
    # large_designs first)
    with pytest.raises(ValueError, match="=True needs"):
        B200Inference(device=0, large_shrink=True, **kw)
