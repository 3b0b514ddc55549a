"""GPU suite (`-m gpu`): Cook's distances, the trimmed-moments dispersions and the outlier / replaced decisions of k_cooks
(designs of up to 16 columns) and k_wide_cooks (17..128) against the extended-precision reference of cooks_checks.py, on the
seeded cases of cooks_cases.py: every width tier, cell layouts at the trim-class and ntrim edges, lanes per gene 1..32 and the
default choice, the sizes that widen the lane groups, and sample counts above the shared-memory ceiling of the per-gene staging
(staged in a global workspace instead).  Both entry points: the host-buffer call and pdq_cooks_dev on padded pitches, with and
without the distance matrix.  End to end: ResidentFit's Cook's stage, and both deseq2 drivers on 8 000 samples.

Set PDQ_COOKS_REPORT to a file path to have the worst error / bound per tier, lane width and quantity written there as JSON."""
import ctypes as C
import functools
import json
import os

import numpy as np
import pytest

import cooks_cases as cs
import cooks_checks as cc
from pydeseq2_b200._lib import as_f64p

pytestmark = pytest.mark.gpu

LANES = [0, 1, 2, 4, 8, 16, 32]  # 0: the default choice
REPORT = {}


@pytest.fixture(scope="module")
def infs():
    from pydeseq2_b200.inference import B200Inference

    yield {T: B200Inference(device=0, lanes_per_gene=T, wide_designs=True, large_designs=True) for T in LANES}
    path = os.environ.get("PDQ_COOKS_REPORT")
    if path:
        with open(path, "w") as f:
            json.dump(REPORT, f, indent=1, sort_keys=True)


def _record(key, worst):
    for q in ("disp", "cooks"):
        REPORT[f"{key}/{q}"] = max(REPORT.get(f"{key}/{q}", 0.0), worst[q])
    assert worst["exempt"] == 0, f"{key}: {worst['exempt']} genes exempted at the cutoff or an argmax tie"


@functools.lru_cache(maxsize=2)
def _case(name):
    return cs.make(name)


@functools.lru_cache(maxsize=2)
def _ref(name, genes=None):
    return cc.reference(_case(name), genes=None if genes is None else list(genes))


def _host(inf, c, matrix=True):
    return inf.calculate_cooks(c["counts"], c["sf"], c["X"], c["mu"], c["hat"], return_matrix=matrix)


def _dev(inf, c, matrix):
    """pdq_cooks_dev on pitches ld = G + 3, ld2 = G + 5, ld_out = G + 7 (NaN padding, which must stay untouched), or with
    cooks_out = NULL."""
    ctx, lib = inf._ops.ctx, inf._ops.lib
    X, sf = c["X"], c["sf"]
    N, G = c["counts"].shape
    ld, ld2, ld_out = G + 3, G + 5, G + 7

    def padded(a, width, fill):
        out = np.full((N, width), fill, dtype=a.dtype)
        out[:, :G] = a
        return out

    bufs = []

    def up(a):
        ptr = ctx.malloc(a.nbytes)
        bufs.append(ptr)
        ctx.h2d(ptr, a)
        return ptr

    d_c, d_mu, d_h = up(padded(c["counts"], ld, -7)), up(padded(c["mu"], ld2, np.nan)), up(padded(c["hat"], ld2, np.nan))
    d_ck = up(np.full((N, ld_out), np.nan)) if matrix else None
    d_out = up(np.full(3 * G, np.nan))
    d = C.c_void_p()
    ctx.check(lib.pdq_design_create(ctx.h, as_f64p(X), as_f64p(sf), N, X.shape[1], C.byref(d)))
    try:
        ctx.check(lib.pdq_cooks_dev(ctx.h, d, d_c, ld, G, d_mu, d_h, ld2, c["cutoff"], d_ck, ld_out if matrix else 0, d_out,
                                    d_out + 8 * G, d_out + 16 * G))
        ctx.sync()
        out = np.empty(3 * G)
        ctx.d2h(out, d_out)
        ck = None
        if matrix:
            m = np.empty((N, ld_out))
            ctx.d2h(m, d_ck)
            assert np.isnan(m[:, G:]).all(), "pdq_cooks_dev wrote past G columns"
            ck = np.ascontiguousarray(m[:, :G])
    finally:
        lib.pdq_design_destroy(ctx.h, d)
        for ptr in bufs:
            ctx.free(ptr)
    return ck, out[:G], out[G:2 * G] == 1.0, out[2 * G:] == 1.0


def _same_bits(a, b, what):
    for k, (u, v) in enumerate(zip(a[1:], b[1:])):
        np.testing.assert_array_equal(np.asarray(u, dtype=np.float64).view(np.int64), np.asarray(v, dtype=np.float64).view(np.int64),
                                      err_msg=f"{what}: output {k + 1}")


def _tier_key(c, T):
    return f"{c['tier']}/T={'default' if T == 0 else T}"


@pytest.mark.parametrize("name", list(cs.CASES))
def test_cases_at_every_lane_width(infs, name):
    """The host-buffer call at lanes per gene 1..32 and the default (the wide kernels always run 32): within the bounds,
    decisions exact, the same per-gene bits without the distance matrix."""
    c, ref = _case(name), _ref(name)
    for T in (LANES if c["tier"] == "narrow" else [0]):
        got = _host(infs[T], c)
        _record(_tier_key(c, T), cc.check(got, ref, f"{name}, T = {T}"))
        _same_bits(got, _host(infs[T], c, matrix=False), f"{name}, T = {T}, no matrix")


@pytest.mark.parametrize("name", list(cs.CASES) + list(cs.CEILING))
def test_device_form_on_padded_pitches(infs, name):
    """pdq_cooks_dev with ld, ld2, ld_out > G, with and without the matrix: the same bits as each other and as the host-buffer
    call, within the bounds.  Above the staging ceiling (CEILING: 4 000..16 000 samples) this is the global-workspace path."""
    inf = infs[0]
    c, ref = _case(name), _ref(name)
    got = _dev(inf, c, True)
    _record(_tier_key(c, 0) + "/device form", cc.check(got, ref, f"{name}, pdq_cooks_dev"))
    _same_bits(got, _dev(inf, c, False), f"{name}, pdq_cooks_dev without the matrix")
    host = _host(inf, c)
    _same_bits(got, host, f"{name}, device form vs host form")
    np.testing.assert_array_equal(got[0].view(np.int64), host[0].view(np.int64))


@pytest.mark.parametrize("name", list(cs.CEILING))
def test_above_the_staging_ceiling(infs, name):
    """Sample counts whose staging exceeds the shared memory of a block even at 32 lanes: the host-buffer call at the default
    lanes and at T = 1 (widened to 32 either way) -- these were refused as unsupported before the global workspace."""
    c, ref = _case(name), _ref(name)
    for T in (0, 1) if c["tier"] == "narrow" else (0,):
        got = _host(infs[T], c)
        _record(f"{c['tier']}/ceiling/T={'default' if T == 0 else T}", cc.check(got, ref, f"{name}, T = {T}"))


@pytest.mark.parametrize("name", list(cs.WIDENED))
def test_widened_lane_groups(infs, name):
    """G large enough for the default 8 / 16 lanes per gene, N large enough that a block's staging passes 96 KB there: the
    launcher widens the lane groups.  The reference covers CHECK_GENES genes (the special ones and a seeded sample)."""
    c = _case(name)
    G = c["counts"].shape[1]
    genes = tuple(sorted(set(range(len(cs.SPECIAL))) | set(np.random.default_rng(7).choice(G, cs.CHECK_GENES, replace=False).tolist())))
    ref = _ref(name, genes)
    idx = np.array(genes)
    for T in (0, 1):
        ck, disp, outl, repl = _host(infs[T], c)
        _record(f"narrow/widened/T={'default' if T == 0 else T}",
                cc.check((ck[:, idx], disp[idx], outl[idx], repl[idx]), ref, f"{name}, T = {T}"))


def test_resident_fit_cooks_stage(infs):
    """ResidentFit(with_cooks=True): robust dispersions and flags bit-equal to the plugin call on the resident mu and hat."""
    from pydeseq2_b200.pipeline import ResidentFit, median_of_ratios
    from pydeseq2_b200.synth import make_counts

    inf = infs[0]
    counts, X, _ = make_counts(48, 3000, "factorial", seed=5)
    counts = np.ascontiguousarray(counts[:, ~(counts == 0).all(0)])
    rng = np.random.default_rng(5)
    hit = rng.choice(counts.shape[1], 60, replace=False)
    counts[rng.integers(0, 48, 60), hit] *= 30
    _, sf = median_of_ratios(counts)
    N, G = counts.shape
    rf = ResidentFit(inf._ops.ctx, X, sf, with_cooks=True, sort_genes=False)
    rf.upload(counts)
    r = rf.run()
    mu, hat = np.empty((N, G)), np.empty((N, G))
    inf._ops.ctx.d2h(mu, rf._main.mu)
    inf._ops.ctx.d2h(hat, rf._main.hat)
    ck, rd, outl, repl = inf.calculate_cooks(counts, sf, X, mu, hat)
    np.testing.assert_array_equal(np.asarray(r["robust_dispersions"]).view(np.int64), rd.view(np.int64))
    np.testing.assert_array_equal(np.asarray(r["cooks_outlier"]), outl)
    np.testing.assert_array_equal(np.asarray(r["cooks_replaced"]), repl)
    assert outl.sum() >= 1 and repl.sum() >= 1
    from scipy.stats import f as f_dist

    case = {"X": X, "sf": sf, "counts": counts, "mu": mu, "hat": hat, "cutoff": float(f_dist.ppf(0.99, X.shape[1], N - X.shape[1]))}
    _record("resident", cc.check((ck, rd, outl, repl), cc.reference(case), "ResidentFit"))


def test_deseq2_drivers_on_8000_samples(infs):
    """deseq2_results and deseq2_results_resident on a two-level design of 8 000 samples run to completion (the Cook's step
    used to refuse the design: its staging exceeded shared memory), and the Cook's layer passes the checks."""
    from scipy.stats import f as f_dist

    from pydeseq2_b200.pipeline import ResidentFit
    from pydeseq2_b200.synth import make_counts
    from pydeseq2_b200.workflow import deseq2_results, deseq2_results_resident

    inf = infs[0]
    counts, X, _ = make_counts(8000, 1000, "two_level", seed=8)
    counts = np.ascontiguousarray(counts[:, ~(counts == 0).all(0)])
    N, G = counts.shape
    res = deseq2_results(counts, X, inf, keep_cooks=True)
    fit = res.fit
    nz = res.non_zero
    c_nz = np.ascontiguousarray(counts[:, nz])
    got = inf.calculate_cooks(c_nz, res.size_factors, X, fit.mu_lfc, fit.hat)
    np.testing.assert_array_equal(res.cooks[:, nz].view(np.int64), got[0].view(np.int64))
    case = {"X": X, "sf": res.size_factors, "counts": c_nz, "mu": np.ascontiguousarray(fit.mu_lfc),
            "hat": np.ascontiguousarray(fit.hat), "cutoff": float(f_dist.ppf(0.99, X.shape[1], N - X.shape[1]))}
    _record("deseq2_results n=8000", cc.check(got, cc.reference(case), "deseq2_results, N = 8000"))
    rf = ResidentFit(inf._ops.ctx, X, res.size_factors)
    rf.upload(c_nz)
    rr = deseq2_results_resident(rf)
    assert rr.pvalue.shape == (int(nz.sum()),) and np.isfinite(rr.pvalue).mean() > 0.9
    both = np.isfinite(rr.pvalue) & np.isfinite(res.pvalue[nz])
    assert np.isclose(rr.pvalue[both], res.pvalue[nz][both], rtol=1e-4, atol=1e-12).mean() > 0.99
