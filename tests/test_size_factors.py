"""CPU suite: poscounts and control-gene size factors (DeseqDataSet.fit_size_factors, dds.py:584-711).

A numpy restatement of the reference (sf_cases.fit_size_factors) is pinned to the sf_* goldens of the real orchestrator
(scripts/make_size_factor_golden.py); the device's per-entry functions and selection code run through the host emulator
(tests/emu/sf_emu.cpp, the same source as
k_log_means / k_size_factor_median / k_size_factor_geomean) and are compared with the same goldens, through `B200Inference`,
`workflow.deseq2_results` / `vst` and the drop-in `DeseqDataSet` subclass."""
import sys
import types
import warnings

import numpy as np
import pandas as pd
import pytest

from conftest import load_golden
from oracle import nbglm
from parity import check_e2e
from sf_cases import SF_CASES, SF_E2E, SF_VST, assert_logmeans, assert_size_factors, case_args, check_sf_e2e, fit_size_factors
from test_vst import assert_vst_close


@pytest.fixture(scope="module")
def ops():
    from emu.sf_ops import SfEmuOps

    return SfEmuOps()


@pytest.fixture(scope="module")
def backend(ops):
    from pydeseq2_b200.inference import B200Inference

    return B200Inference(_ops=ops)


def test_every_kind_of_case_is_covered():
    assert {"sf_poscounts_every_gene_zero", "sf_poscounts_ones", "sf_poscounts_sample_without_usable_gene", "sf_ratio_control_mask",
            "sf_ratio_control_positions", "sf_ratio_control_names", "sf_ratio_control_no_finite_gene",
            "sf_poscounts_control"} <= set(SF_CASES)
    assert SF_E2E == ["sf_e2e_poscounts", "sf_e2e_poscounts_control"] and SF_VST == ["sf_vst_poscounts"]


# ---------------------------------------------------------------------------------------------- numpy restatements
@pytest.mark.parametrize("name", SF_CASES)
def test_numpy_restatement_matches_reference_bit_for_bit(name):
    z = load_golden(name)
    sf, lm, filtered = fit_size_factors(z["counts"], str(z["fit_type"]), z["control"] if z["has_control"] else None)
    np.testing.assert_array_equal(sf, z["size_factors"])
    np.testing.assert_array_equal(lm, z["logmeans"])
    np.testing.assert_array_equal(filtered, z["filtered_genes"])


@pytest.mark.parametrize("name", SF_CASES)
def test_workflow_numpy_restatement_matches_reference(name):
    from pydeseq2_b200.pipeline import filtered_genes, size_factors_numpy

    z = load_golden(name)
    kind = str(z["fit_type"])
    normed, sf, lm = size_factors_numpy(z["counts"], kind, z["control"] if z["has_control"] else None)
    assert_size_factors(sf, z["size_factors"], rtol=1e-14)  # sums in row-major order: the log means may differ in the last bit
    assert_logmeans(lm, z["logmeans"], atol=1e-14)
    np.testing.assert_array_equal(filtered_genes(lm, kind), z["filtered_genes"])


# ---------------------------------------------------------------------------------------------- device algorithm (emulator)
@pytest.mark.parametrize("name", SF_CASES)
def test_emulator_matches_reference(backend, name):
    z = load_golden(name)
    kind, control = case_args(z)
    normed, sf, lm = backend.size_factors(z["counts"], return_logmeans=True, fit_type=kind, control_genes=control)
    assert_size_factors(sf, z["size_factors"])
    assert_logmeans(lm, z["logmeans"])
    if np.isfinite(z["size_factors"]).all():
        np.testing.assert_allclose(normed.mean(0), z["normed_means"], rtol=1e-12)


def test_ratio_over_every_gene_through_the_new_entry_equals_the_old_one(ops):
    t = load_golden("tape_single_factor")
    counts = np.ascontiguousarray(t["counts"], dtype=np.int64)
    N, G = counts.shape
    old, new, lm = np.empty(N), np.empty(N), np.empty(G)
    ops.size_factors(counts, G, N, G, old)
    ops.size_factors_ex(counts, G, N, G, 0, None, new, lm)
    np.testing.assert_array_equal(old, new)


def test_unknown_kind_is_invalid(ops):
    counts = np.ones((2, 3), dtype=np.int64)
    sf, lm = np.empty(2), np.empty(3)
    for kind in (-1, 2):
        assert ops.size_factors_ex_rc(counts, 3, 2, 3, kind, None, sf, lm) == -2  # PDQ_ERR_INVALID


def test_bad_arguments_raise(backend):
    counts = np.ones((3, 4), dtype=np.int64)
    with pytest.raises(ValueError):
        backend.size_factors(counts, fit_type="iterative")
    with pytest.raises(ValueError):
        backend.size_factors(counts, fit_type="poscounts", control_genes=np.ones(5, dtype=bool))
    with pytest.raises(ValueError):
        backend.size_factors(counts, control_genes=[0, 7])
    with pytest.raises(ValueError):
        backend.size_factors(counts, control_genes=np.array([0.5, 1.0]))
    with pytest.raises(ValueError):
        backend.size_factors(counts, logmeans=np.zeros(4), fit_type="poscounts")
    with pytest.raises(ValueError):
        backend.size_factors(counts, logmeans=np.zeros(4), control_genes=[0])


def test_ratio_with_control_genes_still_raises_when_every_gene_holds_a_zero(backend):
    counts = np.arange(1, 13, dtype=np.int64).reshape(3, 4)
    counts[0] = 0
    with pytest.raises(ValueError, match="Every gene contains at least one zero"):
        backend.size_factors(counts, control_genes=[0, 1])


# ---------------------------------------------------------------------------------------------- workflow
class OracleBackend(nbglm.OracleInference):
    """The oracle plus Cook's distances: a backend without `size_factors` (the workflow then restates them in numpy)."""

    def calculate_cooks(self, counts, size_factors, design_matrix, mu, hat, return_matrix=True):
        return nbglm.calculate_cooks(counts, counts / size_factors[:, None], design_matrix, mu, hat)


@pytest.mark.parametrize("name", SF_E2E)
def test_deseq2_results_poscounts_with_oracle_backend(monkeypatch, name):
    check_sf_e2e(monkeypatch, check_e2e, OracleBackend(n_cpus=4), load_golden(name), 1e-8, name)


@pytest.mark.parametrize("name", SF_E2E)
def test_deseq2_results_poscounts_with_device_algorithms(monkeypatch, backend, name):
    check_sf_e2e(monkeypatch, check_e2e, backend, load_golden(name), 1e-4, name, max_frac=0.005)


def test_workflow_rejects_iterative_and_names_samples_without_usable_gene(backend):
    from pydeseq2_b200 import workflow as wf

    z = load_golden("sf_poscounts_sample_without_usable_gene")
    X = np.ones((z["counts"].shape[0], 1))
    with pytest.raises(NotImplementedError):
        wf.deseq2_results(z["counts"], X, backend, size_factors_fit_type="iterative")
    with pytest.raises(NotImplementedError):
        wf.vst(z["counts"], X, backend, size_factors_fit_type="iterative")
    with pytest.raises(ValueError, match=r"sample\(s\) \[5\] have no usable gene"):
        wf.vst(z["counts"], X, backend, size_factors_fit_type="poscounts")
    with pytest.raises(ValueError, match=r"sample\(s\) \[5\] have no usable gene"):
        wf.deseq2_results(z["counts"], X, OracleBackend(n_cpus=1), size_factors_fit_type="poscounts")


@pytest.mark.parametrize("name", SF_VST)
def test_workflow_vst_poscounts_matches_reference(backend, name):
    from pydeseq2_b200.workflow import vst

    z = load_golden(name)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        fit = vst(z["counts"], z["design"], backend, size_factors_fit_type=str(z["size_factors_fit_type"]),
                  control_genes=z["control"] if z["has_control"] else None)
    assert fit.kind == "parametric"
    assert_size_factors(fit.size_factors, z["size_factors"])
    assert_logmeans(fit.logmeans, z["logmeans"])
    np.testing.assert_array_equal(fit.filtered_genes, z["filtered_genes"])
    np.testing.assert_allclose(fit.coeffs, z["vst_trend_coeffs"], rtol=1e-4)
    assert_vst_close(fit.vst_counts, z["vst_counts"])
    assert_vst_close(fit.transform(z["heldout_counts"]), z["heldout_vst"])


# ---------------------------------------------------------------------------------------------- the DeseqDataSet override
class StandInDataSet:
    """The parts of DeseqDataSet (dds.py) that fit_size_factors reads and writes, with the reference's `control_genes` attribute
    (None by default, dds.py:319) and AnnData's `_normalize_indices`; records every call that falls through to the base class."""

    def __init__(self, counts, inference, size_factors_fit_type="ratio", control_genes=None):
        N, G = counts.shape
        self.X, self.inference = counts, inference
        self.size_factors_fit_type, self.control_genes = size_factors_fit_type, control_genes
        self.layers, self.obs = {}, pd.DataFrame(index=range(N))
        self.var = pd.DataFrame(index=[f"g{i}" for i in range(G)])
        self.logmeans = self.filtered_genes = None
        self.base_calls = []

    def _normalize_indices(self, index):
        cols = np.asarray(index[1])
        if cols.dtype.kind in "US":
            cols = self.var.index.get_indexer(cols)
        return slice(None), (np.flatnonzero(cols) if cols.dtype == bool else cols)

    def fit_size_factors(self, fit_type=None, control_genes=None):
        self.base_calls.append(("fit_size_factors", fit_type, control_genes))


def stand_in_class(monkeypatch, **kw):
    pkg, dds = types.ModuleType("pydeseq2"), types.ModuleType("pydeseq2.dds")
    dds.DeseqDataSet = StandInDataSet
    pkg.dds = dds
    monkeypatch.setitem(sys.modules, "pydeseq2", pkg)
    monkeypatch.setitem(sys.modules, "pydeseq2.dds", dds)
    from pydeseq2_b200.integration import b200_dataset_class

    return b200_dataset_class(**kw)


def test_ratio_reaches_the_backend_with_the_reference_control_genes_attribute(monkeypatch, backend):
    cls = stand_in_class(monkeypatch)
    t = load_golden("tape_single_factor")
    d = cls(t["counts"].astype(np.int64), backend)  # control_genes=None, as DeseqDataSet.__init__ always sets it
    assert d.fit_size_factors() is None and d.base_calls == []
    np.testing.assert_allclose(d.obs["size_factors"].values, t["final_size_factors"], rtol=1e-12)


@pytest.mark.parametrize("name", SF_CASES)
def test_all_size_factors_go_to_the_backend(monkeypatch, backend, name):
    z = load_golden(name)
    if str(z["fit_type"]) == "ratio" and not z["has_control"]:
        pytest.skip("plain ratio")
    cls = stand_in_class(monkeypatch, all_size_factors=True)
    given = z["control_given"] if z["has_control"] else None
    # half of the cases give the control genes at init, the other half to fit_size_factors (which overrides the attribute)
    at_init = given is None or SF_CASES.index(name) % 2 == 0
    d = cls(z["counts"], backend, size_factors_fit_type=str(z["fit_type"]), control_genes=given if at_init else [0])
    assert d.fit_size_factors(**({} if at_init else {"control_genes": given})) is None and d.base_calls == []
    assert_size_factors(d.obs["size_factors"].values, z["size_factors"])
    assert_logmeans(d.logmeans, z["logmeans"])
    np.testing.assert_array_equal(d.filtered_genes, z["filtered_genes"])
    if np.isfinite(z["size_factors"]).all():
        np.testing.assert_allclose(d.var["_normed_means"].values, z["normed_means"], rtol=1e-12)
        np.testing.assert_allclose(d.layers["normed_counts"], z["counts"] / z["size_factors"][:, None], rtol=1e-12)


def test_all_size_factors_still_falls_back_to_the_reference(monkeypatch, backend):
    cls = stand_in_class(monkeypatch, all_size_factors=True)
    t = load_golden("tape_single_factor")
    counts = t["counts"].astype(np.int64)
    d = cls(counts, backend, size_factors_fit_type="iterative")
    d.fit_size_factors()
    assert d.base_calls == [("fit_size_factors", None, None)]
    with_zero = counts.copy()
    with_zero[0] = 0  # every gene holds a zero: ratio goes to the reference's iterative fallback, with or without control genes
    for ctl in (None, [0, 1]):
        d = cls(with_zero, backend)
        d.fit_size_factors(control_genes=ctl)
        assert d.base_calls == [("fit_size_factors", None, ctl)] and "size_factors" not in d.obs
    d = cls(counts, object(), size_factors_fit_type="poscounts")  # a backend without size_factors
    d.fit_size_factors()
    assert d.base_calls == [("fit_size_factors", None, None)]
