"""GPU suite (`-m gpu`): poscounts and control-gene size factors through the real kernels (k_log_means, k_size_factor_median,
k_size_factor_geomean) against the sf_* goldens of the real orchestrator and the reference's numpy expressions (sf_cases.py), and
the drivers that use them: workflow.deseq2_results / deseq2_results_resident, vst_resident."""
import ctypes as C
import warnings

import numpy as np
import pytest

from conftest import load_golden
from parity import check_e2e
from sf_cases import SF_CASES, SF_E2E, SF_VST, assert_logmeans, assert_size_factors, case_args, check_sf_e2e, fit_size_factors
from test_vst import assert_vst_close

pytestmark = pytest.mark.gpu

RTOL = 1e-4  # the e2e tolerance of tests/test_gpu_chain.py


@pytest.fixture(scope="module")
def inf():
    from pydeseq2_b200.inference import B200Inference

    return B200Inference(device=0)


def ex_host(inf, counts, kind, control):
    """pdq_size_factors_ex on host buffers: (rc, sf, logmeans)."""
    ctx = inf._ops.ctx
    counts = np.ascontiguousarray(counts, dtype=np.int64)
    N, G = counts.shape
    sf, lm = np.empty(N), np.empty(G)
    ctl = None if control is None else np.ascontiguousarray(control, dtype=np.uint8)
    rc = ctx.lib.pdq_size_factors_ex(ctx.h, counts.ctypes.data_as(C.POINTER(C.c_int64)), G, N, G, kind,
                                     None if ctl is None else ctl.ctypes.data, sf.ctypes.data_as(C.POINTER(C.c_double)),
                                     lm.ctypes.data_as(C.POINTER(C.c_double)))
    return rc, sf, lm


def ex_dev(inf, counts, kind, control):
    """pdq_size_factors_ex_dev on device buffers: (sf, logmeans)."""
    ctx = inf._ops.ctx
    counts = np.ascontiguousarray(counts, dtype=np.int64)
    N, G = counts.shape
    ptrs = [ctx.malloc(n) for n in (N * G * 8, N * 8, G * 8, G)]
    try:
        ctx.h2d(ptrs[0], counts)
        if control is not None:
            ctx.h2d(ptrs[3], np.ascontiguousarray(control, dtype=np.uint8))
        ctx.check(ctx.lib.pdq_size_factors_ex_dev(ctx.h, ptrs[0], G, N, G, kind, ptrs[3] if control is not None else None, ptrs[1],
                                                  ptrs[2]))
        sf, lm = np.empty(N), np.empty(G)
        ctx.d2h(sf, ptrs[1])
        ctx.d2h(lm, ptrs[2])
        ctx.sync()
    finally:
        for p in ptrs:
            ctx.free(p)
    return sf, lm


@pytest.mark.parametrize("name", SF_CASES)
def test_device_matches_reference(inf, name):
    z = load_golden(name)
    kind, control = case_args(z)
    normed, sf, lm = inf.size_factors(z["counts"], return_logmeans=True, fit_type=kind, control_genes=control)
    assert_size_factors(sf, z["size_factors"])
    assert_logmeans(lm, z["logmeans"])
    ctl = z["control"] if z["has_control"] else None
    rc, sf_h, lm_h = ex_host(inf, z["counts"], 1 if kind == "poscounts" else 0, ctl)
    sf_d, lm_d = ex_dev(inf, z["counts"], 1 if kind == "poscounts" else 0, ctl)
    assert rc == 0
    np.testing.assert_array_equal(sf_h, sf_d)  # host and device flavours: the same launches
    np.testing.assert_array_equal(lm_h, lm_d)
    np.testing.assert_array_equal(sf_h, sf)


def seeded(N, G, zero_frac, seed):
    rng = np.random.default_rng(seed)
    mu = np.exp(rng.normal(3.0, 1.5, G))
    counts = rng.negative_binomial(4, 4 / (4 + mu[None, :] * rng.uniform(0.5, 2.0, (N, 1))))
    counts[rng.random((N, G)) < zero_frac] = 0
    return counts.astype(np.int64)


@pytest.mark.parametrize("N,G,zero_frac", [(200, 20000, 0.0), (200, 20000, 0.7), (500, 60000, 0.0), (500, 60000, 0.7),
                                           (2000, 7500, 0.7), (31, 4001, 0.3)])
@pytest.mark.parametrize("kind,with_control", [("ratio", True), ("poscounts", False), ("poscounts", True)])
def test_device_matches_numpy_on_seeded_tables(inf, N, G, zero_frac, kind, with_control):
    counts = seeded(N, G, zero_frac, seed=N + G)
    ctl = None
    if with_control:
        ctl = np.zeros(G, dtype=bool)
        ctl[np.random.default_rng(G).choice(G, G // 10, replace=False)] = True
    want_sf, want_lm, _ = fit_size_factors(counts, kind, ctl)
    if kind == "ratio" and np.isinf(want_lm).all():
        with pytest.raises(ValueError, match="Every gene contains at least one zero"):
            inf.size_factors(counts, fit_type=kind, control_genes=ctl)
        return
    _, sf, lm = inf.size_factors(counts, return_logmeans=True, fit_type=kind, control_genes=ctl)
    assert_size_factors(sf, want_sf)
    assert_logmeans(lm, want_lm)
    sf_d, lm_d = ex_dev(inf, counts, 1 if kind == "poscounts" else 0, ctl)
    np.testing.assert_array_equal(sf_d, sf)
    np.testing.assert_array_equal(lm_d, lm)


@pytest.mark.parametrize("N,G", [(200, 20000), (24, 301), (9, 1)])
def test_ratio_over_every_gene_equals_the_old_entry_byte_for_byte(inf, N, G):
    counts = seeded(N, G, 0.0, seed=7) + 1
    counts[0, : G // 3] = 0
    ctx = inf._ops.ctx
    sf_old, lm_old = np.empty(N), np.empty(G)
    ctx.check(ctx.lib.pdq_size_factors(ctx.h, counts.ctypes.data_as(C.POINTER(C.c_int64)), G, N, G,
                                       sf_old.ctypes.data_as(C.POINTER(C.c_double)), lm_old.ctypes.data_as(C.POINTER(C.c_double))))
    rc, sf, lm = ex_host(inf, counts, 0, None)
    assert rc == 0
    assert sf.tobytes() == sf_old.tobytes() and lm.tobytes() == lm_old.tobytes()


def test_unknown_kind_is_invalid(inf):
    counts = np.ones((3, 4), dtype=np.int64)
    for kind in (-1, 2, 7):
        rc, _, _ = ex_host(inf, counts, kind, None)
        assert rc == -2  # PDQ_ERR_INVALID


@pytest.mark.parametrize("name", SF_E2E)
def test_deseq2_results_poscounts(monkeypatch, inf, name):
    check_sf_e2e(monkeypatch, check_e2e, inf, load_golden(name), RTOL, name, max_frac=0.005)


@pytest.mark.parametrize("name", SF_E2E)
def test_deseq2_results_resident_poscounts(monkeypatch, inf, name):
    check_sf_e2e(monkeypatch, check_e2e, inf, load_golden(name), RTOL, name, max_frac=0.005, resident=True)


@pytest.mark.parametrize("name", SF_E2E)
def test_resident_sorted_gene_order_equals_unsorted(inf, name):
    from pydeseq2_b200.pipeline import ResidentFit

    g = load_golden(name)
    counts = np.ascontiguousarray(g["counts"], dtype=np.int64)
    nz = ~(counts == 0).all(0)
    assert nz.sum() >= 256
    ctl = g["control"][nz] if g["has_control"] else None
    sfs = []
    for sort in (True, False):
        rf = ResidentFit(inf._ops.ctx, g["design"], None, sort_genes=sort, size_factors_fit_type=str(g["size_factors_fit_type"]),
                         control_genes=ctl)
        try:
            rf.upload(np.ascontiguousarray(counts[:, nz]))
            assert (rf._perm is not None) is sort
            sfs.append(rf.sf.copy())
        finally:
            rf.close()
    np.testing.assert_array_equal(sfs[0], sfs[1])
    assert_size_factors(sfs[0], g["final_size_factors"])


def test_resident_names_samples_without_usable_gene(inf):
    from pydeseq2_b200.pipeline import ResidentFit

    z = load_golden("sf_poscounts_sample_without_usable_gene")
    counts = np.ascontiguousarray(z["counts"][:, ~(z["counts"] == 0).all(0)])
    rf = ResidentFit(inf._ops.ctx, np.ones((counts.shape[0], 1)), None, size_factors_fit_type="poscounts")
    try:
        with pytest.raises(ValueError, match=r"sample\(s\) \[5\] have no usable gene"):
            rf.upload(counts)
    finally:
        rf.close()


@pytest.mark.parametrize("name", SF_VST)
def test_vst_resident_poscounts(inf, name):
    from pydeseq2_b200.workflow import vst_resident

    z = load_golden(name)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        fit = vst_resident(inf, z["counts"], z["design"], size_factors_fit_type=str(z["size_factors_fit_type"]),
                           control_genes=z["control"] if z["has_control"] else None)
    assert fit.kind == "parametric"
    assert_size_factors(fit.size_factors, z["size_factors"])
    assert_logmeans(fit.logmeans, z["logmeans"])
    np.testing.assert_array_equal(fit.filtered_genes, z["filtered_genes"])
    np.testing.assert_allclose(fit.coeffs, z["vst_trend_coeffs"], rtol=1e-4)
    assert_vst_close(np.asarray(fit.vst_counts), z["vst_counts"])
    assert_vst_close(fit.transform(z["heldout_counts"]), z["heldout_vst"])
