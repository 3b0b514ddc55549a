"""CPU suite: adjusted p-values (`B200Inference.adjust_pvalues` -> pdq_padj_rejections / pdq_padj_bh, `workflow.filter_threshold`,
`integration.b200_stats_class`) through the host emulator of pdq_padj.cuh, bit for bit against numpy's quantiles, scipy's
Benjamini-Hochberg, the padj_* goldens of the real DeseqStats (scripts/make_padj_golden.py) and the padj columns of every e2e_* and
ct_* golden."""
import glob
import os
import sys
import types

import numpy as np
import pandas as pd
import pytest

from conftest import GOLDEN, load_golden
from padj_cases import PADJ, rejections, same, scipy_bh, vectors
from pydeseq2_b200 import workflow

E2E = sorted(os.path.basename(f)[:-4] for f in glob.glob(os.path.join(GOLDEN, "e2e_*.npz")))
CT = sorted(os.path.basename(f)[:-4] for f in glob.glob(os.path.join(GOLDEN, "ct_*.npz")))


@pytest.fixture(scope="module")
def ops():
    from emu.padj_emu import PadjEmuOps

    return PadjEmuOps()


@pytest.fixture(scope="module")
def emu(ops):
    from pydeseq2_b200.inference import B200Inference

    return B200Inference(_ops=ops)


@pytest.mark.parametrize("G,seed,ties", [(1, 0, False), (2, 1, False), (2, 2, True), (3, 3, True), (17, 4, False), (1000, 5, True),
                                         (5001, 6, False)])
def test_cutoffs_are_numpy_quantiles(ops, G, seed, ties):
    bm = vectors(G, seed, ties)[0]
    for theta in (workflow.filter_theta(bm), np.linspace(0.0, 1.0, 50), np.linspace(0.3, 1.0, 64), np.array([1.0])):
        for x in (bm, np.zeros(G)):
            cut, _ = rejections(ops, x, np.full(G, 0.5), theta, 0.05)
            assert same(cut, np.quantile(x, theta)), (G, seed, theta[0])


def test_nan_base_mean_makes_every_cutoff_nan(ops):
    bm, p = vectors(100, 7)
    bm[17] = np.nan
    theta = workflow.filter_theta(bm)
    cut, num = rejections(ops, bm, p, theta, 0.05)
    assert np.isnan(cut).all() and np.isnan(np.quantile(bm, theta)).all() and (num == 0).all()


@pytest.mark.parametrize("G,seed,ties", [(1, 10, False), (2, 11, True), (3, 12, False), (64, 13, True), (400, 14, False),
                                         (3000, 15, True)])
def test_bh_is_scipy(ops, G, seed, ties):
    bm, p = vectors(G, seed, ties)
    cuts = np.array([-np.inf, 0.0, np.median(bm), bm.max(), np.inf])
    K = len(cuts)
    pv = np.tile(p, (K, 1))
    out = np.full((K, G + 3), 7.0)
    ops.padj_bh(bm, G, pv, G, K, cuts, out, G + 3)
    for k, c in enumerate(cuts):
        assert same(out[k, :G], scipy_bh(bm, p, c)), (k, c)
    assert (out[:, G:] == 7.0).all()  # ld_out > G: the pitch is left alone


@pytest.mark.parametrize("seed", range(6))
def test_rejection_counts_are_scipy(ops, seed):
    G = [5, 40, 333, 2000, 2000, 800][seed]
    bm, p = vectors(G, 100 + seed, ties=seed % 2 == 1)
    rng = np.random.default_rng(seed)
    if seed >= 4:  # values whose BH value lands on alpha: the exact comparison decides
        r = rng.integers(1, G + 1, G)
        p = np.where(rng.random(G) < 0.5, 0.05 * r / G, p)
    pv = np.stack([p, rng.permutation(p), np.where(rng.random(G) < 0.5, p, np.nan)])
    theta = workflow.filter_theta(bm)
    for alpha in (0.05, 0.1, 1.0, 1.5, 0.0):
        cut, num = rejections(ops, bm, pv, theta, alpha)
        for k in range(3):
            want = [(scipy_bh(bm, pv[k], c) < alpha).sum() for c in cut]
            assert list(num[k]) == want, (seed, alpha, k)


@pytest.mark.parametrize("name", PADJ)
def test_padj_goldens(emu, ops, name):
    g = load_golden(name)
    bm, p, alpha, filt = g["base_mean"], g["pvalues"], float(g["alpha"]), bool(g["independent_filter"])
    assert same(emu.adjust_pvalues(bm, p, alpha, filt), g["padj"])
    if filt:
        theta = workflow.filter_theta(bm)
        assert same(theta, g["theta"])
        cut, num = rejections(ops, bm, p, theta, alpha)
        assert same(cut, g["cutoffs"]) and list(num[0]) == list(g["num_rej"])
        assert workflow.filter_threshold(theta, num[0].astype(int)) == int(g["j"])


def test_padj_goldens_as_rows_of_one_call(emu):
    """Rows of one call are independent: the goldens of equal length stacked into one (K, G) call."""
    g = load_golden("padj_ties"), load_golden("padj_ties_alpha_0_1")
    for filt in (True, False):
        out = emu.adjust_pvalues(g[0]["base_mean"], np.stack([g[0]["pvalues"], g[1]["pvalues"][::-1]]), 0.05, filt)
        for k, pk in enumerate((g[0]["pvalues"], g[1]["pvalues"][::-1])):
            assert same(out[k], emu.adjust_pvalues(g[0]["base_mean"], pk, 0.05, filt))
    assert same(out[0], scipy_bh(g[0]["base_mean"], g[0]["pvalues"], -np.inf))


@pytest.mark.parametrize("name", E2E)
def test_e2e_golden_padj(emu, name):
    g = load_golden(name)
    filt = bool(g["independent_filter"]) if "independent_filter" in g else True
    alpha = float(g["alpha"]) if "alpha" in g else 0.05
    assert same(emu.adjust_pvalues(g["final_baseMean"], g["final_pvalue"], alpha, filt), g["final_padj"])


@pytest.mark.parametrize("name", CT)
def test_contrast_golden_padj(emu, name):
    g = load_golden(name)
    for k in range(int(g["n_contrasts"])):
        c = f"c{k:02d}_"
        out = emu.adjust_pvalues(g["final_baseMean"], g[c + "pvalue"], float(g[c + "alpha"]), bool(g[c + "independent_filter"]))
        assert same(out, g[c + "padj"]), (name, k)


def test_argument_errors(ops, emu):
    bm, p = vectors(50, 3)
    pv = np.ascontiguousarray(np.tile(p, (2, 1)))
    cut, num, out, theta = np.empty(50), np.empty((2, 50), dtype=np.int32), np.empty((2, 50)), workflow.filter_theta(bm)
    assert ops.padj_rejections_rc(bm, 50, pv, 50, 0, theta, 50, 0.05, cut, num) == -2   # K <= 0
    assert ops.padj_rejections_rc(bm, 50, pv, 49, 2, theta, 50, 0.05, cut, num) == -2   # ld < G
    assert ops.padj_rejections_rc(bm, 50, pv, 50, 2, theta, 65, 0.05, cut, num) == -2   # more than 64 thresholds
    assert ops.padj_bh_rc(bm, 50, pv, 50, 2, np.zeros(2), out, 49) == -2               # ld_out < G
    bad = pv.copy()
    bad[1, 3] = 1.5
    assert ops.padj_rejections_rc(bm, 50, bad, 50, 2, theta, 50, 0.05, cut, num) == -2
    assert ops.padj_bh_rc(bm, 50, bad, 50, 2, np.zeros(2), out, 50) == -2
    with pytest.raises(ValueError, match="between 0. and 1."):
        emu.adjust_pvalues(bm, bad)
    with pytest.raises(ValueError, match="pvalues must be"):
        emu.adjust_pvalues(bm, p[:-1])


def test_drivers_use_the_backend(emu):
    """workflow._adjust and deseq2_stats go through adjust_pvalues on a backend that has it, the host restatement otherwise."""
    g = load_golden("padj_typical")
    bm, p = g["base_mean"], g["pvalues"]
    assert same(workflow._adjust(bm, p, True, 0.05, None, emu), g["padj"])
    host = workflow._adjust(bm, p, True, 0.05, None, object())
    assert np.array_equal(np.isnan(host), np.isnan(g["padj"]))
    np.testing.assert_allclose(host, g["padj"], rtol=1e-15, atol=0)
    from pydeseq2_b200.inference import B200Inference

    without = B200Inference(_ops=types.SimpleNamespace())  # ops without the two entry points: None, and the host restatement
    assert without.adjust_pvalues(bm, p) is None
    assert same(workflow._adjust(bm, p, True, 0.05, None, without), host)


# ---- integration.b200_stats_class on a stand-in for pydeseq2.ds.DeseqStats
class StandInStats:
    """The parts of DeseqStats (ds.py) that _independent_filtering / _p_value_adjustment read and write."""

    def __init__(self, g, inference):
        names = pd.Index([f"g{i}" for i in range(len(g["base_mean"]))])
        self.dds = types.SimpleNamespace(var_names=names)
        self.base_mean, self.p_values = pd.Series(g["base_mean"], index=names), pd.Series(g["pvalues"], index=names)
        self.alpha, self.inference, self.base_calls = float(g["alpha"]), inference, []

    def _independent_filtering(self):
        self.base_calls.append("_independent_filtering")

    def _p_value_adjustment(self):
        self.base_calls.append("_p_value_adjustment")


@pytest.fixture
def stats_class(monkeypatch):
    pkg, ds, utils = types.ModuleType("pydeseq2"), types.ModuleType("pydeseq2.ds"), types.ModuleType("pydeseq2.utils")
    ds.DeseqStats = StandInStats
    calls = []

    def lowess(*a, **k):  # the reference's smoother, as far as these goldens go
        calls.append(1)
        return workflow.lowess(*a, **k)

    utils.lowess = lowess
    pkg.ds, pkg.utils = ds, utils
    monkeypatch.setitem(sys.modules, "pydeseq2", pkg)
    monkeypatch.setitem(sys.modules, "pydeseq2.ds", ds)
    monkeypatch.setitem(sys.modules, "pydeseq2.utils", utils)
    from pydeseq2_b200.integration import b200_stats_class

    cls = b200_stats_class()
    cls.lowess_calls = calls
    return cls


@pytest.mark.parametrize("name", ["padj_typical", "padj_no_filter"])
def test_stats_class_adjusts_on_the_backend(stats_class, emu, name):
    g = load_golden(name)
    ds = stats_class(g, emu)
    if bool(g["independent_filter"]):
        assert ds._independent_filtering() is None and stats_class.lowess_calls
    else:
        assert ds._p_value_adjustment() is None
    assert ds.base_calls == [] and list(ds.padj.index) == list(ds.dds.var_names)
    assert same(ds.padj.to_numpy(), g["padj"])


def test_stats_class_falls_back_to_the_reference(stats_class):
    from pydeseq2_b200.inference import B200Inference

    # a backend without adjust_pvalues, and one whose ops cannot run it
    for backend in (object(), B200Inference(_ops=types.SimpleNamespace())):
        ds = stats_class(load_golden("padj_g3"), backend)
        ds._independent_filtering()
        ds._p_value_adjustment()
        assert ds.base_calls == ["_independent_filtering", "_p_value_adjustment"] and not hasattr(ds, "padj")
