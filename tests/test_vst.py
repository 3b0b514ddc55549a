"""CPU suite: the variance-stabilising transform (DeseqDataSet.vst / vst_fit / vst_transform, dds.py:349-514).

The kernels' per-element function and the held-out median selection run through the host emulator (tests/emu/vst_emu.cpp, the
same source as k_vst_transform / k_size_factor_median) and are compared with the reference's numpy expressions; `workflow.vst`
and the `vst_transform` override of `integration.b200_dataset_class()` are compared with what the real orchestrator stored in
the vst_* goldens (scripts/make_vst_golden.py)."""
import glob
import os
import sys
import types
import warnings

import numpy as np
import pandas as pd
import pytest
from scipy.stats import trim_mean

from conftest import GOLDEN, load_golden

VST_CASES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN, "vst_*.npz")))


# ---------------------------------------------------------------------------------------------- numpy restatements of the reference
def vst_numpy(normed, kind, coeffs):
    """dds.py:488-510 on normalised counts."""
    with np.errstate(divide="ignore", invalid="ignore"):
        if kind == "parametric":
            a0, a1 = coeffs
            return np.log2((1 + a1 + 2 * a0 * normed + 2 * np.sqrt(a0 * normed * (1 + a1 + a0 * normed))) / (4 * a0))
        d = float(np.ravel(coeffs)[0])
        return (2 * np.arcsinh(np.sqrt(d * normed)) - np.log(d) - np.log(4)) / np.log(2)


def norm_transform_numpy(counts, logmeans, filtered):
    """preprocessing.deseq2_norm_transform (preprocessing.py:59-102)."""
    with np.errstate(divide="ignore", invalid="ignore"):
        lr = np.log(counts)[:, filtered] - logmeans[filtered]
        sf = np.exp(np.median(lr, axis=1))
        return counts / sf[:, None], sf


def assert_same_pattern(got, want):
    for f in (np.isnan, np.isposinf, np.isneginf):
        np.testing.assert_array_equal(f(got), f(want))


def assert_vst_close(got, want, rel=1e-4):
    assert got.shape == want.shape
    assert_same_pattern(got, want)
    ok = np.isfinite(want)
    assert np.all(np.abs(got[ok] - want[ok]) <= rel * np.maximum(np.abs(want[ok]), 1.0))


@pytest.fixture(scope="module")
def ops():
    from emu.vst_ops import VstEmuOps

    return VstEmuOps()


@pytest.fixture(scope="module")
def backend(ops):
    from pydeseq2_b200.inference import B200Inference

    return B200Inference(_ops=ops)


# ---------------------------------------------------------------------------------------------- per-element function
@pytest.mark.parametrize("kind,coeffs", [("parametric", (0.05, 2.3)), ("parametric", (1e-3, 40.0)), ("parametric", (3.0, 1e-6)),
                                         ("mean", (0.2,)), ("mean", (1e-6,)), ("mean", (25.0,))])
def test_element_function_matches_closed_form(backend, kind, coeffs):
    rng = np.random.default_rng(5)
    y = np.concatenate([np.arange(0, 200), np.unique(np.round(2.0 ** rng.uniform(0, 40, 600))).astype(np.int64),
                        [2**40, 2**40 - 1, 2**33 + 7]]).astype(np.int64)
    G = len(y) // 2
    counts = y[: 2 * G].reshape(2, G)
    sf = np.array([0.37, 2.9])
    got = backend.vst_transform(counts, sf, kind, coeffs)
    want = vst_numpy(counts / sf[:, None], kind, coeffs)
    assert np.all(np.abs(got - want) <= 1e-13 * np.maximum(np.abs(want), 1.0))


def test_zero_size_factor_gives_numpy_inf_nan(backend):
    counts = np.array([[0, 3, 7], [4, 0, 1]], dtype=np.int64)
    sf = np.array([0.0, 1.5])
    for kind, coeffs in (("parametric", (0.1, 2.0)), ("mean", (0.3,))):
        got = backend.vst_transform(counts, sf, kind, coeffs)
        with np.errstate(divide="ignore", invalid="ignore"):
            want = vst_numpy(counts / sf[:, None], kind, coeffs)
        assert_same_pattern(got, want)
        assert np.isnan(got[0, 0]) and np.isposinf(got[0, 1])


def test_transform_rejects_bad_parameters(backend):
    counts = np.ones((2, 3), dtype=np.int64)
    sf = np.ones(2)
    with pytest.raises(NotImplementedError):
        backend.vst_transform(counts, sf, "local", (0.1, 1.0))
    with pytest.raises(ValueError):
        backend.vst_transform(counts, sf, "parametric", (0.0, 1.0))
    with pytest.raises(ValueError):
        backend.vst_transform(counts, sf, "mean", (-1.0,))
    with pytest.raises(ValueError):
        backend.vst_transform(counts, np.ones(3), "mean", (0.1,))


def test_padded_input_pitch(backend):
    rng = np.random.default_rng(2)
    big = rng.integers(0, 500, size=(5, 41)).astype(np.int64)
    view = big[:, :37]  # row pitch 41 elements, 37 genes
    sf = rng.uniform(0.5, 2.0, 5)
    got = backend.vst_transform(view, sf, "parametric", (0.02, 1.7))
    np.testing.assert_array_equal(got, backend.vst_transform(np.ascontiguousarray(view), sf, "parametric", (0.02, 1.7)))


# ---------------------------------------------------------------------------------------------- held-out size factors
def heldout_case(seed, N=9, G=120):
    rng = np.random.default_rng(seed)
    train = rng.negative_binomial(5, 0.05, size=(20, G)).astype(np.int64)
    train[3, :7] = 0  # genes left out of the median (log mean -inf)
    with np.errstate(divide="ignore"):
        lm = np.log(train).mean(0)
    kept = np.flatnonzero(np.isfinite(lm))
    if len(kept) % 2:
        lm[kept[-1]] = -np.inf
        kept = kept[:-1]
    test = rng.negative_binomial(5, 0.05, size=(N, G)).astype(np.int64)
    test[0, :] = 0                       # every kept gene zero: size factor 0
    test[1, : G // 2 + 5] = 0            # more than half zero: size factor 0
    test[2, kept[: len(kept) // 2]] = 0  # exactly half of an even number of kept genes zero: the lower middle value is -inf
    test[3, 10:20] = 0                   # a few zeros: finite
    return test, lm


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_heldout_size_factors_match_norm_transform(backend, seed):
    test, lm = heldout_case(seed)
    filtered = ~np.isinf(lm)
    normed, sf = backend.size_factors(test, logmeans=np.where(filtered, lm, -np.inf))
    want_normed, want_sf = norm_transform_numpy(test, lm, filtered)
    assert_same_pattern(sf, want_sf)
    np.testing.assert_array_equal(sf == 0, want_sf == 0)
    ok = np.isfinite(want_sf) & (want_sf != 0)
    np.testing.assert_allclose(sf[ok], want_sf[ok], rtol=1e-12)
    assert sf[0] == 0 and sf[1] == 0 and sf[2] == 0 and sf[3] > 0
    assert_same_pattern(normed, want_normed)


def test_heldout_size_factors_without_kept_genes_are_nan(backend):
    test = np.ones((2, 4), dtype=np.int64)
    _, sf = backend.size_factors(test, logmeans=np.full(4, -np.inf))
    assert np.isnan(sf).all()


def test_size_factors_without_logmeans_unchanged(backend):
    t = load_golden("tape_single_factor")
    _, sf = backend.size_factors(t["counts"].astype(np.int64))
    np.testing.assert_allclose(sf, t["final_size_factors"], rtol=1e-12)


# ---------------------------------------------------------------------------------------------- workflow.vst against the orchestrator
def run_case(name, backend):
    from pydeseq2_b200.workflow import vst

    z = load_golden(name)
    kw = {}
    if "after_deseq2" in name:  # the dataset's size factors and log means are reused
        kw = dict(size_factors=z["size_factors"], logmeans=z["logmeans"])
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        fit = vst(z["counts"], z["design"], backend, fit_type=str(z["fit_type"]), use_design=bool(z["use_design"]), **kw)
    return z, fit, caught


@pytest.mark.parametrize("name", VST_CASES)
def test_workflow_vst_matches_orchestrator(backend, name):
    z, fit, caught = run_case(name, backend)
    assert fit.kind == str(z["vst_fit_type"])
    fell_back = any("did not converge" in str(w.message) for w in caught)
    assert fell_back == bool(z["fell_back"])
    np.testing.assert_allclose(fit.size_factors, z["size_factors"], rtol=1e-10)
    np.testing.assert_allclose(fit.logmeans, z["logmeans"], rtol=1e-12)
    gd = z["vst_genewise_dispersions"]
    np.testing.assert_array_equal(np.isnan(fit.genewise), np.isnan(gd))
    if fit.kind == "parametric":
        np.testing.assert_allclose(fit.coeffs, z["vst_trend_coeffs"], rtol=1e-4)
    else:
        np.testing.assert_allclose(fit.coeffs[0], z["mean_disp"], rtol=1e-4)
    assert_vst_close(fit.vst_counts, z["vst_counts"])
    if "heldout_counts" in z:
        assert_vst_close(fit.transform(z["heldout_counts"]), z["heldout_vst"])
        assert not np.isfinite(z["heldout_vst"][-1]).all()  # the held-out sample with size factor 0


def test_single_factor_close_to_r(backend):
    for name in ("vst_single_factor_parametric", "vst_single_factor_parametric_design", "vst_single_factor_mean"):
        z, fit, _ = run_case(name, backend)
        np.testing.assert_allclose(fit.vst_counts, z["r_vst"], rtol=1e-4)


def test_use_design_with_mean_warns(backend):
    _, _, caught = run_case("vst_single_factor_mean_design", backend)
    assert any("use_design=True is only useful" in str(w.message) for w in caught)


def test_transform_without_logmeans_refits_with_leak_warning(backend):
    from pydeseq2_b200.workflow import vst

    z = load_golden("vst_two_level_n24")
    fit = vst(z["counts"], z["design"], backend, size_factors=z["size_factors"])
    assert fit.logmeans is None
    new = z["counts"][:6]
    with pytest.warns(UserWarning, match="leak"):
        got = fit.transform(new)
    with np.errstate(divide="ignore"):
        lm = np.log(new).mean(0)
    normed, _ = norm_transform_numpy(new, lm, ~np.isinf(lm))
    assert_vst_close(got, vst_numpy(normed, fit.kind, fit.coeffs), rel=1e-12)


# ---------------------------------------------------------------------------------------------- the DeseqDataSet override
class StandInDataSet:
    """The parts of DeseqDataSet (dds.py) that vst_transform reads; records every call that falls through to the base class."""

    def __init__(self, counts, inference):
        N, G = counts.shape
        self.X, self.inference, self.min_disp = counts, inference, 1e-8
        self.obs, self.var, self.uns, self.layers = pd.DataFrame(index=range(N)), pd.DataFrame(index=range(G)), {}, {}
        self.logmeans = self.filtered_genes = None
        self.base_calls = []

    def vst_transform(self, counts=None):
        self.base_calls.append(("vst_transform", None if counts is None else counts.shape))
        return "base"


@pytest.fixture
def dataset_class(monkeypatch):
    pkg, dds = types.ModuleType("pydeseq2"), types.ModuleType("pydeseq2.dds")
    dds.DeseqDataSet = StandInDataSet
    pkg.dds = dds
    monkeypatch.setitem(sys.modules, "pydeseq2", pkg)
    monkeypatch.setitem(sys.modules, "pydeseq2.dds", dds)
    from pydeseq2_b200.integration import b200_dataset_class

    return b200_dataset_class()


def fitted_dataset(cls, z, backend):
    d = cls(z["counts"], backend)
    d.obs["size_factors"] = z["size_factors"]
    d.logmeans, d.filtered_genes = z["logmeans"], ~np.isinf(z["logmeans"])
    d.vst_fit_type = str(z["vst_fit_type"])
    d.var["vst_genewise_dispersions"] = z["vst_genewise_dispersions"]
    if "vst_trend_coeffs" in z:
        d.uns["vst_trend_coeffs"] = pd.Series(z["vst_trend_coeffs"], index=["a0", "a1"])
    return d


@pytest.mark.parametrize("name", ["vst_train_test", "vst_train_test_mean", "vst_fallback_to_mean"])
def test_override_goes_to_backend(dataset_class, backend, name):
    z = load_golden(name)
    d = fitted_dataset(dataset_class, z, backend)
    assert_vst_close(d.vst_transform(), z["vst_counts"], rel=1e-12)
    if "heldout_counts" in z:
        assert_vst_close(d.vst_transform(z["heldout_counts"]), z["heldout_vst"], rel=1e-12)
    assert d.base_calls == []


def test_override_falls_back_to_reference(dataset_class, backend):
    z = load_golden("vst_train_test")
    held = z["heldout_counts"]
    d = dataset_class(z["counts"], backend)  # no fit at all: the reference raises its RuntimeError
    assert d.vst_transform() == "base"
    d = fitted_dataset(dataset_class, z, backend)
    del d.uns["vst_trend_coeffs"]            # parametric without coefficients: the reference's RuntimeError
    assert d.vst_transform() == "base"
    d = fitted_dataset(dataset_class, z, backend)
    d.logmeans = None                        # iteratively fitted size factors: the reference warns and re-fits
    assert d.vst_transform(held) == "base"
    d = fitted_dataset(dataset_class, z, backend)
    assert d.vst_transform(held.astype(float)) == "base"  # not an integer table
    d = fitted_dataset(dataset_class, z, backend)
    d.vst_fit_type = "local"                 # unknown fit type: the reference's NotImplementedError
    assert d.vst_transform() == "base"
    d = fitted_dataset(dataset_class, z, object())  # a backend without vst_transform
    assert d.vst_transform(held) == "base"
    assert all(c[0] == "vst_transform" for c in d.base_calls)
