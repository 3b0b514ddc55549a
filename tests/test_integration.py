"""CPU suite: `integration.b200_dataset_class()` -- the DeseqDataSet subclass that sends size factors and Cook's distances to the
backend -- on a stand-in for `pydeseq2.dds.DeseqDataSet` (the reference's own class is not part of this repository).  The stand-in
holds the attributes the overrides read and write and records every call that falls through to the base class; the device
algorithms run through the host emulator and are compared with what the real orchestrator stored in the tape goldens."""
import sys
import types

import numpy as np
import pandas as pd
import pytest

from conftest import load_golden


class StandInDataSet:
    """The parts of DeseqDataSet (dds.py) that the overrides touch."""

    def __init__(self, counts, design, inference, size_factors_fit_type="ratio", low_memory=False):
        N, G = counts.shape
        self.X, self.inference, self.size_factors_fit_type, self.low_memory = counts, inference, size_factors_fit_type, low_memory
        self.n_obs, self.n_vars = N, G
        self.layers, self.obsm = {}, {"design_matrix": pd.DataFrame(design)}
        self.obs, self.var = pd.DataFrame(index=range(N)), pd.DataFrame(index=range(G))
        self.base_calls = []

    def fit_size_factors(self, fit_type=None, control_genes=None):
        self.base_calls.append(("fit_size_factors", fit_type, control_genes))

    def calculate_cooks(self):
        self.base_calls.append(("calculate_cooks",))

    def fit_MAP_dispersions(self):
        self.base_calls.append(("fit_MAP_dispersions",))
        self.var["dispersions"] = 0.1


@pytest.fixture
def dataset_class(monkeypatch):
    pkg, dds = types.ModuleType("pydeseq2"), types.ModuleType("pydeseq2.dds")
    dds.DeseqDataSet = StandInDataSet
    pkg.dds = dds
    monkeypatch.setitem(sys.modules, "pydeseq2", pkg)
    monkeypatch.setitem(sys.modules, "pydeseq2.dds", dds)
    from pydeseq2_b200.integration import b200_dataset_class

    cls = b200_dataset_class()
    assert issubclass(cls, StandInDataSet)
    return cls


@pytest.fixture(scope="module")
def backend():
    from emu.emu_ops import EmuOps
    from pydeseq2_b200.inference import B200Inference

    return B200Inference(_ops=EmuOps())


def test_size_factors_come_from_the_backend(dataset_class, backend):
    t = load_golden("tape_single_factor")
    d = dataset_class(t["counts"].astype(np.int64), t["design"], backend)
    assert d.fit_size_factors() is None and d.base_calls == []
    np.testing.assert_allclose(d.obs["size_factors"].values, t["final_size_factors"], rtol=1e-12)
    normed = t["counts"] / t["final_size_factors"][:, None]
    np.testing.assert_allclose(d.layers["normed_counts"], normed, rtol=1e-12)
    np.testing.assert_allclose(d.var["_normed_means"].values, normed.mean(0), rtol=1e-12)
    with np.errstate(divide="ignore"):
        want_logmeans = np.log(t["counts"]).mean(0)
    np.testing.assert_allclose(d.logmeans, want_logmeans, rtol=1e-12)  # kept for vst_transform, like deseq2_norm_fit
    np.testing.assert_array_equal(d.filtered_genes, ~np.isinf(want_logmeans))


def test_size_factors_fall_back_to_the_reference(dataset_class, backend):
    t = load_golden("tape_single_factor")
    counts = t["counts"].astype(np.int64)
    with_zero = counts.copy()
    with_zero[0] = 0  # every gene holds a zero: the backend raises, the reference's iterative estimator takes over
    d = dataset_class(with_zero, t["design"], backend)
    d.fit_size_factors()
    assert d.base_calls == [("fit_size_factors", None, None)] and "size_factors" not in d.obs
    d = dataset_class(counts, t["design"], backend, size_factors_fit_type="poscounts")
    d.fit_size_factors()
    assert d.base_calls == [("fit_size_factors", None, None)]
    d = dataset_class(counts, t["design"], backend)
    d.fit_size_factors(control_genes=[0, 1])
    assert d.base_calls == [("fit_size_factors", None, [0, 1])]
    d = dataset_class(counts, t["design"], object())  # a backend without size_factors
    d.fit_size_factors(fit_type="ratio")
    assert d.base_calls == [("fit_size_factors", "ratio", None)]


@pytest.mark.parametrize("low_memory", [False, True])
def test_cooks_come_from_the_backend(dataset_class, backend, low_memory):
    t = load_golden("tape_single_factor")
    nz = t["final_non_zero"] == 1
    d = dataset_class(t["counts"].astype(np.int64), t["design"], backend, low_memory=low_memory)
    d.obs["size_factors"] = t["final_size_factors"]
    d.var["non_zero"] = nz
    d.var["dispersions"] = 0.1
    d.obsm["_mu_LFC"], d.obsm["_hat_diagonals"] = t["final_mu_LFC"], t["final_hat"]
    assert d.calculate_cooks() is None and d.base_calls == []
    np.testing.assert_allclose(d.layers["cooks"][:, nz], t["final_cooks"][:, nz], rtol=1e-9)
    assert np.isnan(d.layers["cooks"][:, ~nz]).all()
    assert ("_mu_LFC" in d.obsm) is (not low_memory) and ("_hat_diagonals" in d.obsm) is (not low_memory)


def test_cooks_fit_missing_dispersions_first_and_fall_back_without_backend(dataset_class, backend):
    t = load_golden("tape_single_factor")
    nz = t["final_non_zero"] == 1
    d = dataset_class(t["counts"].astype(np.int64), t["design"], backend)
    d.obs["size_factors"] = t["final_size_factors"]
    d.var["non_zero"] = nz
    d.obsm["_mu_LFC"], d.obsm["_hat_diagonals"] = t["final_mu_LFC"], t["final_hat"]
    d.calculate_cooks()
    assert d.base_calls == [("fit_MAP_dispersions",)] and "cooks" in d.layers
    d = dataset_class(t["counts"].astype(np.int64), t["design"], object())
    d.calculate_cooks()
    assert d.base_calls == [("calculate_cooks",)] and "cooks" not in d.layers
