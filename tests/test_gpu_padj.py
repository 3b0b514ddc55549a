"""GPU suite: pdq_padj_rejections / pdq_padj_bh (pdq_padj.cu) on an H100 -- bit for bit against the host emulator of
pdq_padj.cuh, the padj_* goldens of the real DeseqStats, numpy's quantiles and scipy's Benjamini-Hochberg (G = 10^6 with K = 45,
odd G, ld > G), the C ABI's argument checks, and the padj of `deseq2_results`, `deseq2_results_resident` and `deseq2_stats`
against scipy on their own p-values."""
import ctypes as C

import numpy as np
import pytest

from conftest import load_golden
from padj_cases import PADJ, rejections, same, scipy_bh, vectors
from pydeseq2_b200 import workflow

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def inf():
    from pydeseq2_b200.inference import B200Inference

    return B200Inference(device=0)


@pytest.fixture(scope="module")
def emu():
    from emu.padj_emu import PadjEmuOps
    from pydeseq2_b200.inference import B200Inference

    return B200Inference(_ops=PadjEmuOps())


def reference_padj(bm, pv, alpha, independent_filter):
    """numpy / scipy on each row: np.quantile, false_discovery_control per cutoff, the project's lowess and threshold rule."""
    out = np.empty(pv.shape)
    for k, p in enumerate(pv):
        if not independent_filter:
            out[k] = scipy_bh(bm, p, -np.inf)
            continue
        theta = workflow.filter_theta(bm)
        cols = [scipy_bh(bm, p, c) for c in np.quantile(bm, theta)]
        num_rej = np.array([(c < alpha).sum() for c in cols])
        out[k] = cols[workflow.filter_threshold(theta, num_rej)]
    return out


@pytest.mark.parametrize("name", PADJ)
def test_goldens_on_the_device(inf, emu, name):
    g = load_golden(name)
    bm, p, alpha, filt = g["base_mean"], g["pvalues"], float(g["alpha"]), bool(g["independent_filter"])
    got = inf.adjust_pvalues(bm, p, alpha, filt)
    assert same(got, g["padj"]) and same(got, emu.adjust_pvalues(bm, p, alpha, filt))
    if filt:
        theta = workflow.filter_theta(bm)
        cut, num = rejections(inf._ops, bm, p, theta, alpha)
        assert same(cut, g["cutoffs"]) and list(num[0]) == list(g["num_rej"])


@pytest.mark.parametrize("G,K,seed,ties", [(1, 3, 1, False), (2, 2, 2, True), (3, 5, 3, False), (1023, 4, 4, True), (1025, 7, 5, False),
                                           (20001, 45, 6, False), (60000, 6, 7, True)])
def test_device_against_emulator(inf, emu, G, K, seed, ties):
    bm, p = vectors(G, seed, ties)
    rng = np.random.default_rng(seed)
    pv = np.stack([rng.permutation(p) for _ in range(K)])
    theta = workflow.filter_theta(bm)
    for alpha in (0.05, 0.1):
        c_dev, n_dev = rejections(inf._ops, bm, pv, theta, alpha)
        c_emu, n_emu = rejections(emu._ops, bm, pv, theta, alpha)
        assert same(c_dev, c_emu) and np.array_equal(n_dev, n_emu)
    for filt in (True, False):
        assert same(inf.adjust_pvalues(bm, pv, 0.05, filt), emu.adjust_pvalues(bm, pv, 0.05, filt))


def test_million_genes_45_rows_against_scipy(inf):
    """G = 10^6, K = 45: every cutoff, every count and every adjusted p-value of a handful of rows against numpy / scipy; the
    whole (K, G) table against the emulator-free restatement row by row would take minutes, so rows 0, 22 and 44 are checked."""
    G, K = 1_000_000, 45
    bm, p = vectors(G, 42)
    rng = np.random.default_rng(43)
    pv = np.stack([np.where(rng.random(G) < 0.02, np.nan, rng.permutation(p)) for _ in range(K)])
    theta = workflow.filter_theta(bm)
    cut, num = rejections(inf._ops, bm, pv, theta, 0.05)
    assert same(cut, np.quantile(bm, theta))
    got = inf.adjust_pvalues(bm, pv, 0.05, True)
    for k in (0, 22, 44):
        cols = [scipy_bh(bm, pv[k], c) for c in cut]
        assert list(num[k]) == [(c < 0.05).sum() for c in cols], k
        assert same(got[k], cols[workflow.filter_threshold(theta, num[k].astype(int))]), k


def test_pitches(inf):
    """ld > G on the way in and ld_out > G on the way out, odd G."""
    G, K = 4097, 3
    bm, p = vectors(G, 9)
    wide = np.full((K, G + 5), 0.25)
    wide[:, :G] = np.stack([p, p[::-1], p])
    cut = np.array([-np.inf, np.median(bm), 0.0])
    out = np.full((K, G + 7), 3.0)
    inf._ops.padj_bh(bm, G, wide, G + 5, K, cut, out, G + 7)
    for k in range(K):
        assert same(out[k, :G], scipy_bh(bm, wide[k, :G], cut[k])), k
    assert (out[:, G:] == 3.0).all()
    theta = workflow.filter_theta(bm)
    cutoffs, num = np.empty(50), np.empty((K, 50), dtype=np.int32)
    inf._ops.padj_rejections(bm, G, wide, G + 5, K, theta, 50, 0.05, cutoffs, num)
    assert np.array_equal(num, rejections(inf._ops, bm, np.ascontiguousarray(wide[:, :G]), theta, 0.05)[1])


def test_argument_errors(inf):
    from pydeseq2_b200._lib import B200Error

    L, h = inf._ops.lib, inf._ops.ctx.h
    f64p = C.POINTER(C.c_double)
    bm, p = vectors(64, 3)
    pv = np.ascontiguousarray(np.tile(p, (2, 1)))
    theta, cut, num, out = workflow.filter_theta(bm), np.empty(64), np.empty((2, 64), dtype=np.int32), np.empty((2, 64))
    ptr = lambda a: a.ctypes.data_as(f64p)  # noqa: E731
    ip = num.ctypes.data_as(C.POINTER(C.c_int))
    assert L.pdq_padj_rejections(h, ptr(bm), 64, ptr(pv), 64, 0, ptr(theta), 50, 0.05, ptr(cut), ip) == -2
    assert L.pdq_padj_rejections(h, ptr(bm), 64, ptr(pv), 63, 2, ptr(theta), 50, 0.05, ptr(cut), ip) == -2
    assert L.pdq_padj_rejections(h, ptr(bm), 64, ptr(pv), 64, 2, ptr(theta), 65, 0.05, ptr(cut), ip) == -2
    assert L.pdq_padj_rejections(h, ptr(bm), 0, ptr(pv), 64, 2, ptr(theta), 50, 0.05, ptr(cut), ip) == -2
    assert L.pdq_padj_bh(h, ptr(bm), 64, ptr(pv), 64, 2, ptr(cut), ptr(out), 63) == -2
    assert L.pdq_padj_bh(h, ptr(bm), 64, None, 64, 2, ptr(cut), ptr(out), 64) == -2
    bad = pv.copy()
    bad[1, 5] = -0.5
    with pytest.raises(B200Error, match="outside"):
        inf._ops.padj_bh(bm, 64, bad, 64, 2, np.zeros(2), out, 64)
    with pytest.raises(ValueError, match="between 0. and 1."):
        inf.adjust_pvalues(bm, bad)
    assert same(inf.adjust_pvalues(bm, p), reference_padj(bm, p[None, :], 0.05, True)[0])  # the context is still usable
    assert same(inf.adjust_pvalues(bm, p, independent_filter=False), scipy_bh(bm, p, -np.inf))


@pytest.mark.parametrize("name", ["e2e_two_level_n24", "e2e_two_level_n16_bh", "ct_outliers"])
def test_drivers_padj_is_scipy_on_their_own_pvalues(inf, name):
    from pydeseq2_b200.pipeline import ResidentFit
    from pydeseq2_b200.workflow import deseq2_results, deseq2_results_resident, deseq2_stats

    g = load_golden(name)
    counts, X = np.ascontiguousarray(g["counts"], dtype=np.int64), g["design"]
    filt = bool(g["independent_filter"]) if "independent_filter" in g else True
    res = deseq2_results(counts, X, inf, independent_filter=filt)
    assert same(res.padj, reference_padj(res.base_mean, res.pvalue[None, :], 0.05, filt)[0])
    nz = ~(counts == 0).all(0)
    rf = ResidentFit(inf._ops.ctx, X, None)
    rf.upload(np.ascontiguousarray(counts[:, nz]))
    try:
        rr = deseq2_results_resident(rf, non_zero=nz, independent_filter=filt)
    finally:
        rf.close()
    assert same(rr.padj, reference_padj(rr.base_mean, rr.pvalue[None, :], 0.05, filt)[0])
    p = X.shape[1]
    cs = np.eye(p)[1:] if p > 1 else np.eye(1)
    for alpha in (0.05, 0.1):
        out = deseq2_stats(res, X, inf, cs, independent_filter=filt, alpha=alpha)
        want = reference_padj(res.base_mean, np.stack([r.pvalue for r in out]), alpha, filt)
        for r, w in zip(out, want):
            assert same(r.padj, w)
