"""GPU suite (`-m gpu`): the variance-stabilising transform through the real kernels (k_vst_transform, the held-out
k_size_factor_median) against the reference's numpy expressions and the vst_* goldens of the real orchestrator."""
import numpy as np
import pytest

from test_vst import VST_CASES, assert_same_pattern, assert_vst_close, heldout_case, norm_transform_numpy, run_case, vst_numpy

pytestmark = pytest.mark.gpu

KINDS = [("parametric", (0.05, 2.3)), ("parametric", (1e-3, 40.0)), ("mean", (0.2,)), ("mean", (1e-6,))]


@pytest.fixture(scope="module")
def inf():
    from pydeseq2_b200.inference import B200Inference

    return B200Inference(device=0)


def close_to_closed_form(got, counts, sf, kind, coeffs, rel=1e-13):
    want = vst_numpy(counts / sf[:, None], kind, coeffs)
    assert_same_pattern(got, want)
    ok = np.isfinite(want)
    err = np.abs(got[ok] - want[ok]) / np.maximum(np.abs(want[ok]), 1.0)
    assert err.max() <= rel, err.max()


@pytest.mark.parametrize("kind,coeffs", KINDS)
def test_gpu_element_function_wide_range(inf, kind, coeffs):
    rng = np.random.default_rng(5)
    y = np.concatenate([np.arange(0, 200), np.round(2.0 ** rng.uniform(0, 40, 1000)).astype(np.int64), [2**40, 2**40 - 1]])
    counts = y[:1200].reshape(4, 300).astype(np.int64)
    sf = np.array([0.37, 2.9, 1.0, 0.011])
    close_to_closed_form(inf.vst_transform(counts, sf, kind, coeffs), counts, sf, kind, coeffs)


@pytest.mark.parametrize("kind,coeffs", KINDS)
@pytest.mark.parametrize("G,pad", [(1001, 0), (1000, 0), (999, 3), (1000, 6)])
def test_gpu_transform_8000_samples_ragged_and_padded(inf, kind, coeffs, G, pad):
    # host entry point: a padded host view is repacked to pitch G on the device, so G decides the kernel path (odd G: scalar
    # kernel path; even G: paired loads); padded DEVICE pitches are covered by test_gpu_dev_entry_point_paths
    rng = np.random.default_rng(G + pad)
    big = rng.negative_binomial(3, 0.02, size=(8000, G + pad)).astype(np.int64)
    counts = big[:, :G]
    sf = rng.uniform(0.3, 3.0, 8000)
    close_to_closed_form(inf.vst_transform(counts, sf, kind, coeffs), counts, sf, kind, coeffs)


@pytest.mark.parametrize("G,ld,ldo", [
    (999, 1002, 1004),   # paired loads on an even padded input pitch with the odd last gene of every row on the scalar tail
    (1000, 1002, 1000),  # paired loads, padded input, dense output
    (257, 257, 260),     # odd input pitch: scalar path, padded output
    (256, 258, 259),     # odd output pitch: scalar path
])
@pytest.mark.parametrize("kind,coeffs", [KINDS[0], KINDS[2]])
def test_gpu_dev_entry_point_paths(inf, G, ld, ldo, kind, coeffs):
    from pydeseq2_b200 import _lib

    ctx = inf._ops.ctx
    c_d = _lib.c_dptr
    N = 37
    rng = np.random.default_rng(G + ld + ldo)
    table = rng.integers(0, 10**6, size=(N, ld)).astype(np.int64)
    table[:, G:] = -1  # padding the kernel must not read into the output
    sf = rng.uniform(0.5, 2.0, N)
    dc, ds, do = ctx.malloc(table.nbytes), ctx.malloc(sf.nbytes), ctx.malloc(N * ldo * 8)
    try:
        ctx.h2d(dc, table)
        ctx.h2d(ds, sf)
        pad = np.full((N, ldo), 7.0)
        ctx.h2d(do, pad)
        c0, c1 = coeffs[0], (coeffs[1] if len(coeffs) > 1 else 0.0)
        k = 0 if kind == "parametric" else 1
        ctx.check(ctx.lib.pdq_vst_transform_dev(ctx.h, c_d(dc), ld, N, G, c_d(ds), k, c0, c1, c_d(do), ldo))
        out = np.empty((N, ldo))
        ctx.d2h(out, do)
        ctx.sync()
        close_to_closed_form(out[:, :G], table[:, :G], sf, kind, coeffs)
        assert (out[:, G:] == 7.0).all()  # nothing written past G
        assert ctx.lib.pdq_vst_transform_dev(ctx.h, c_d(dc), ld, N, G, c_d(ds), 2, 0.3, 0.0, c_d(do), ldo) == -2
        assert ctx.lib.pdq_vst_transform_dev(ctx.h, c_d(dc), ld, N, G, c_d(ds), 0, 0.0, 1.0, c_d(do), ldo) == -2
        assert ctx.lib.pdq_vst_transform_dev(ctx.h, c_d(dc), G - 1, N, G, c_d(ds), 1, 0.3, 0.0, c_d(do), ldo) == -2
    finally:
        for p in (dc, ds, do):
            ctx.free(p)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_gpu_heldout_size_factors(inf, seed):
    test, lm = heldout_case(seed)
    filtered = ~np.isinf(lm)
    _, sf = inf.size_factors(test, logmeans=np.where(filtered, lm, -np.inf))
    _, want = norm_transform_numpy(test, lm, filtered)
    assert_same_pattern(sf, want)
    np.testing.assert_array_equal(sf == 0, want == 0)
    ok = np.isfinite(want) & (want != 0)
    np.testing.assert_allclose(sf[ok], want[ok], rtol=1e-12)


@pytest.mark.parametrize("name", VST_CASES)
def test_gpu_workflow_vst_matches_orchestrator(inf, name):
    z, fit, caught = run_case(name, inf)
    assert fit.kind == str(z["vst_fit_type"])
    assert any("did not converge" in str(w.message) for w in caught) == bool(z["fell_back"])
    if fit.kind == "parametric":
        np.testing.assert_allclose(fit.coeffs, z["vst_trend_coeffs"], rtol=1e-4)
    else:
        np.testing.assert_allclose(fit.coeffs[0], z["mean_disp"], rtol=1e-4)
    assert_vst_close(fit.vst_counts, z["vst_counts"])
    if "heldout_counts" in z:
        assert_vst_close(fit.transform(z["heldout_counts"]), z["heldout_vst"])


def _resident_vs_host(inf, counts, X, **kw):
    import warnings

    from pydeseq2_b200.workflow import vst, vst_resident

    with warnings.catch_warnings(record=True) as wh:
        warnings.simplefilter("always")
        host = vst(counts, X, inf, **kw)
    with warnings.catch_warnings(record=True) as wr:
        warnings.simplefilter("always")
        res = vst_resident(inf, counts, X, **kw)
    assert res.kind == host.kind
    assert sorted(str(w.message) for w in wr) == sorted(str(w.message) for w in wh)
    np.testing.assert_allclose(res.size_factors, host.size_factors, rtol=1e-12)
    np.testing.assert_array_equal(res.non_zero, host.non_zero)
    if host.logmeans is not None:
        np.testing.assert_array_equal(np.isinf(res.logmeans), np.isinf(host.logmeans))
    np.testing.assert_allclose(res.genewise, host.genewise, rtol=1e-9)
    np.testing.assert_allclose(res.coeffs, host.coeffs, rtol=1e-8)
    assert_vst_close(res.vst_counts, host.vst_counts, rel=1e-7)
    return host, res


@pytest.mark.parametrize("name", ["vst_two_level_n24", "vst_two_level_n24_design", "vst_factorial_n20_design", "vst_continuous_n30_mean",
                                  "vst_fallback_to_mean", "vst_single_factor_parametric", "vst_train_test"])
def test_gpu_vst_resident_equals_plugin_call_driver(inf, name):
    from conftest import load_golden

    z = load_golden(name)
    _, res = _resident_vs_host(inf, z["counts"], z["design"], fit_type=str(z["fit_type"]), use_design=bool(z["use_design"]))
    assert_vst_close(res.vst_counts, z["vst_counts"])  # and the real orchestrator's
    if "heldout_counts" in z:
        assert_vst_close(res.transform(z["heldout_counts"]), z["heldout_vst"])


@pytest.mark.parametrize("N,G,kind", [(200, 20000, "two_level"), (60, 3001, "factorial")])
def test_gpu_vst_resident_larger_tables(inf, N, G, kind):
    from pydeseq2_b200.synth import make_counts

    counts, X, _ = make_counts(N, G, kind, seed=9)
    counts[:, [0, 17, G - 1]] = 0  # all-zero genes: transformed like every other gene, no dispersion
    host, res = _resident_vs_host(inf, counts, X)
    assert np.isnan(res.genewise[[0, 17, G - 1]]).all()
    _resident_vs_host(inf, counts, X, fit_type="mean", use_design=True, size_factors=host.size_factors)


def test_gpu_c2_size_against_closed_form(inf):
    from pydeseq2_b200.synth import make_counts

    counts, _, _ = make_counts(200, 20000, "two_level", seed=21)
    with np.errstate(divide="ignore"):
        lm = np.log(counts).mean(0)
    _, sf = norm_transform_numpy(counts, lm, ~np.isinf(lm))
    _, sf_gpu = inf.size_factors(counts)
    np.testing.assert_allclose(sf_gpu, sf, rtol=1e-12)
    for kind, coeffs in KINDS[:1] + KINDS[2:3]:
        close_to_closed_form(inf.vst_transform(counts, sf_gpu, kind, coeffs), counts, sf_gpu, kind, coeffs)
