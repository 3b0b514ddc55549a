"""CPU suite: Wald tests of K contrasts on one fit (`B200Inference.wald_tests` -> pdq_wald_contrasts, `workflow.deseq2_stats`,
`integration.b200_stats_class`) through the host emulator of k_wald_contrasts, against the ct_* goldens of the real orchestrator
(scripts/make_contrast_golden.py) and the oracle's restatement of utils.wald_test."""
import sys
import types

import numpy as np
import pandas as pd
import pytest

from contrast_cases import ALTS, CT, assert_tests_close, check_golden_wald, check_stats_e2e, contrasts_of, oracle_wald_tests, seeded_case
from conftest import load_golden


@pytest.fixture(scope="module")
def emu():
    from emu.emu_ops import EmuOps
    from pydeseq2_b200.inference import B200Inference

    return B200Inference(_ops=EmuOps())


@pytest.fixture(scope="module")
def emu8():
    from emu.emu_ops import EmuOps
    from pydeseq2_b200.inference import B200Inference

    return B200Inference(_ops=EmuOps(lanes=8))


@pytest.mark.parametrize("name", CT)
def test_wald_tests_against_golden_dataset_state(emu, emu8, name):
    check_golden_wald(emu, name)
    check_golden_wald(emu8, name)  # lane-cooperative sums and the contrasts shared out over the lanes


@pytest.mark.parametrize("K", [1, 45])
@pytest.mark.parametrize("p", range(1, 17))
def test_wald_tests_against_oracle(emu, emu8, p, K):
    X, sf, disp, lfc, cs = seeded_case(p, 3 * p + 10, 12, K, seed=100 * p + K)
    alts = [ALTS[k % 5] for k in range(K)]
    nulls = np.where(np.arange(K) % 2, 0.3, -0.2)
    nulls[np.isin(alts, ["greaterAbs", "lessAbs"])] = 0.4
    ridge = np.diag(np.repeat(1e-6, p))
    want = oracle_wald_tests(X, sf, disp, lfc, cs, ridge, nulls, alts)
    for inf in (emu, emu8):
        assert_tests_close(inf.wald_tests(X, sf, disp, lfc, cs, ridge, nulls, alts), want, 1e-12, f"p={p} K={K}")


def test_one_contrast_gives_vectors_and_non_finite_genes_nan(emu):
    X, sf, disp, lfc, cs = seeded_case(3, 20, 10, 1, seed=7)
    lfc[2, 1], disp[5] = np.nan, np.inf
    pv, st, se = emu.wald_tests(X, sf, disp, lfc, cs[0])
    assert pv.shape == st.shape == se.shape == (10,)
    bad = np.zeros(10, bool)
    bad[[2, 5]] = True
    assert np.isnan(pv[bad]).all() and np.isnan(st[bad]).all() and np.isnan(se[bad]).all() and np.isfinite(pv[~bad]).all()
    want = oracle_wald_tests(X, sf, disp[~bad], lfc[~bad], cs, np.diag(np.repeat(1e-6, 3)), [0.0], [None])
    assert_tests_close((pv[~bad], st[~bad], se[~bad]), tuple(w[0] for w in want), 1e-12)


def test_wald_tests_argument_errors(emu):
    X, sf, disp, lfc, cs = seeded_case(3, 20, 10, 4, seed=8)
    with pytest.raises(KeyError):
        emu.wald_tests(X, sf, disp, lfc, cs, alt_hypothesis="two-sided")
    with pytest.raises(KeyError):
        emu.wald_tests(X, sf, disp, lfc, cs, alt_hypothesis=[None, "less", "bigger", None])
    with pytest.raises(ValueError):
        emu.wald_tests(X, sf, disp, lfc, cs[:, :2])                      # contrast width
    with pytest.raises(ValueError):
        emu.wald_tests(X, sf, disp, lfc, np.zeros((0, 3)))               # no contrast
    with pytest.raises(ValueError):
        emu.wald_tests(X, sf, disp[:-1], lfc, cs)                        # genes disagree
    with pytest.raises(ValueError):
        emu.wald_tests(X, sf[:-1], disp, lfc, cs)                        # samples disagree
    with pytest.raises(ValueError):
        emu.wald_tests(X, sf, disp, lfc, cs, lfc_null=[0.0, 0.1])        # one lfc_null per contrast
    with pytest.raises(ValueError):
        emu.wald_tests(X, sf, disp, lfc, cs, ridge_factor=np.eye(2))


def test_emulator_entry_rejects_bad_tables():
    from emu.emu_ops import EmuOps

    ops = EmuOps()
    X, sf, disp, lfc, cs = seeded_case(3, 20, 10, 2, seed=9)
    out = [np.empty((2, 10)) for _ in range(3)]
    args = (X, sf, 20, 3, disp, lfc, 10, np.eye(3) * 1e-6)
    ok = np.zeros(2, np.int32)
    assert ops.wald_contrasts_rc(*args, 2, cs, np.zeros(2), np.array([0, 5], np.int32), *out, 10) == -2
    assert ops.wald_contrasts_rc(*args, 0, cs, np.zeros(2), ok, *out, 10) == -2
    assert ops.wald_contrasts_rc(*args, 2, cs, np.zeros(2), ok, *out, 9) == -2
    assert ops.wald_contrasts_rc(*args, 2, cs, np.zeros(2), ok, *out, 10) == 0


@pytest.mark.parametrize("name", CT)
def test_deseq2_stats_against_golden(emu, name):
    # twice the e2e tolerance of tests/test_workflow.py, with a budget of four of these 200 genes; the fit itself (not the Wald
    # test, checked at 1e-9 above) puts a few p-values of ct_outliers 1.1e-3 from the reference, and the p = 10 fit of ct_ten_levels
    # (4 samples per level) one SE 1.1e-2 away, which moves the BH-adjusted p-values of its neighbours by up to 2e-2
    check_stats_e2e(emu, name, 2e-3 if name == "ct_ten_levels" else 2e-4, max_frac=0.02)


def test_deseq2_stats_with_one_contrast_equals_deseq2_results(emu):
    from pydeseq2_b200.workflow import deseq2_results, deseq2_stats

    g = load_golden("ct_outliers")
    counts, X = np.ascontiguousarray(g["counts"], dtype=np.int64), g["design"]
    zero = (counts == 0).all(0)
    for c, t, alt in (([0, 0, 1.0], 0.0, None), ([0, -1, 1.0], 0.5, "greater")):
        a = deseq2_results(counts, X, emu, np.array(c), lfc_null=t, alt_hypothesis=alt)
        b = deseq2_stats(deseq2_results(counts, X, emu, np.array([0, 1.0, 0])), X, emu, np.array(c), lfc_null=t, alt_hypothesis=alt)[0]
        for f in ("stat", "lfc_se", "pvalue", "padj", "log2_fold_change"):
            np.testing.assert_allclose(getattr(b, f)[~zero], getattr(a, f)[~zero], rtol=1e-10, atol=1e-300, err_msg=f)
        # all-zero genes: NaN statistics, as the reference's run_wald_test gives them (deseq2_results reports 0 there)
        assert np.isnan(b.stat[zero]).all() and np.isnan(b.lfc_se[zero]).all() and np.isnan(g["c00_statistics"][zero]).all()


def test_deseq2_stats_argument_errors(emu):
    from pydeseq2_b200.workflow import deseq2_results, deseq2_stats

    g = load_golden("ct_three_level_batch")
    X = g["design"]
    res = deseq2_results(np.ascontiguousarray(g["counts"], dtype=np.int64), X, emu, np.array([0, 1.0, 0, 0]))
    with pytest.raises(ValueError):
        deseq2_stats(res, X, emu, np.ones(3))
    with pytest.raises(ValueError):
        deseq2_stats(res, X, emu, np.eye(4), lfc_null=[0.0, 0.1])
    for alt in ("greaterAbs", "lessAbs"):
        with pytest.raises(ValueError):
            deseq2_stats(res, X, emu, np.eye(4)[1:], lfc_null=-0.5, alt_hypothesis=alt)
    with pytest.raises(KeyError):
        deseq2_stats(res, X, emu, np.eye(4)[1:], alt_hypothesis="two-sided")
    import dataclasses

    with pytest.raises(ValueError):
        deseq2_stats(dataclasses.replace(res, shrink_prior_scale=1.0), X, emu, np.eye(4)[1:])


def test_deseq2_stats_numpy_fallback_for_backends_without_wald_tests(emu):
    from pydeseq2_b200.workflow import deseq2_results, deseq2_stats

    class NoWaldTests:
        pass

    g = load_golden("ct_outliers")
    X = g["design"]
    res = deseq2_results(np.ascontiguousarray(g["counts"], dtype=np.int64), X, emu, np.array([0, 1.0, 0]))
    cs = np.array([c[0] for c in contrasts_of(g)])
    for alt in ALTS:
        t = 0.3 if alt else -0.3
        dev = deseq2_stats(res, X, emu, cs, lfc_null=t, alt_hypothesis=alt)
        ref = deseq2_stats(res, X, NoWaldTests(), cs, lfc_null=t, alt_hypothesis=alt)
        for a, b in zip(dev, ref):
            assert_tests_close((a.pvalue, a.stat, a.lfc_se), (b.pvalue, b.stat, b.lfc_se), 1e-11, str(alt))


# ---- integration.b200_stats_class on a stand-in for pydeseq2.ds.DeseqStats
class StandInDataSet:
    def __init__(self, g, refit_cooks=True):
        G = g["final_LFC"].shape[0]
        self.var_names = pd.Index([f"g{i}" for i in range(G)])
        self.obs = pd.DataFrame({"size_factors": g["final_size_factors"]})
        self.var = pd.DataFrame({"dispersions": g["final_dispersions"], "replaced": g["final_replaced"] == 1}, index=self.var_names)
        self.refit_cooks = refit_cooks
        self.new_all_zeroes_genes = self.var_names[g["final_new_all_zero"] == 1]


class StandInStats:
    """The parts of DeseqStats (ds.py) that run_wald_test reads and writes."""

    def __init__(self, dds, g, k, inference):
        c = contrasts_of(g)[k]
        self.dds, self.inference, self.quiet, self.shrunk_LFCs = dds, inference, True, False
        self.design_matrix = pd.DataFrame(g["design"])
        self.LFC = pd.DataFrame(g["final_LFC"], index=dds.var_names)
        self.contrast_vector, self.lfc_null, self.alt_hypothesis, self.prior_LFC_var = c[0], c[1], c[2], c[6]
        self.base_calls = []

    def run_wald_test(self):
        self.base_calls.append("run_wald_test")


@pytest.fixture
def stats_class(monkeypatch):
    pkg, ds = types.ModuleType("pydeseq2"), types.ModuleType("pydeseq2.ds")
    ds.DeseqStats = StandInStats
    pkg.ds = ds
    monkeypatch.setitem(sys.modules, "pydeseq2", pkg)
    monkeypatch.setitem(sys.modules, "pydeseq2.ds", ds)
    from pydeseq2_b200.integration import b200_stats_class

    cls = b200_stats_class()
    assert issubclass(cls, StandInStats)
    return cls


@pytest.mark.parametrize("name", ["ct_alternatives", "ct_outliers"])
def test_stats_class_runs_the_wald_test_on_the_backend(stats_class, emu, name):
    g = load_golden(name)
    dds = StandInDataSet(g)
    new_zero = g["final_new_all_zero"] == 1
    for k in range(int(g["n_contrasts"])):
        ds = stats_class(dds, g, k, emu)
        assert ds.run_wald_test() is None and ds.base_calls == []
        c = f"c{k:02d}_"
        assert list(ds.p_values.index) == list(dds.var_names)
        assert_tests_close((ds.p_values.values, ds.statistics.values, ds.SE.values), (g[c + "p_values"], g[c + "statistics"], g[c + "SE"]),
                           1e-9, f"{name} contrast {k}")
        if new_zero.any():  # the override of ds.py:355-360
            assert (ds.SE.values[new_zero] == 0).all() and (ds.statistics.values[new_zero] == 0).all()
            assert (ds.p_values.values[new_zero] == 1).all()


def test_stats_class_falls_back_to_the_reference(stats_class, emu):
    g = load_golden("ct_three_level_batch")
    ds = stats_class(StandInDataSet(g), g, 0, object())  # a backend without wald_tests
    ds.run_wald_test()
    assert ds.base_calls == ["run_wald_test"] and not hasattr(ds, "p_values")
    dds = StandInDataSet(g)
    dds.obs = dds.obs.drop(columns="size_factors")
    ds = stats_class(dds, g, 0, emu)
    ds.run_wald_test()
    assert ds.base_calls == ["run_wald_test"] and not hasattr(ds, "p_values")
