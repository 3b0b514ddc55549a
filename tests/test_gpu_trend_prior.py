"""The dispersion trend + prior launch (`pdq_trend_fit_dev`) against `TrendOut` records pinned in tests/golden/trend_prior_ref.npz
(scripts/make_trend_prior_golden.py, tests/trend_prior_cases.py).

The prior's medians are exact order statistics, so however the kernel finds them the record must not move.  The one-cluster
kernel adds its partial sums in a fixed order: its record is compared bit for bit.  The grid kernel adds its per-block partial sums
with global atomics, in arrival order, so its coefficients may move in the last bits between runs (they did when the fixture was
recorded), and so may the loss; its medians are compared bit for bit whenever the coefficients come out bit-identical, and to
1e-10 otherwise, and its counts always bit for bit.
"""
import os

import numpy as np
import pytest

import trend_prior_cases as tc
from conftest import load_golden

V_BINS, CAND_CAP = 2048, 1024  # kVBins, kCandCap of pdq_trend.cuh
EXACT_FIELDS = [2, 3, 4, 5, 7, 10, 11, 12, 13, 14, 15]  # status, rounds, used, iterations, converged, n_above, pad


def bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


@pytest.fixture(scope="module")
def ref():
    return load_golden("trend_prior_ref")


@pytest.fixture(scope="module")
def ctx():
    from pydeseq2_b200 import _lib

    c = _lib.Context(0)
    yield c
    c.close()


def trend_record(ctx, means, gw, min_disp, max_disp, trigamma_c):
    from pydeseq2_b200 import _lib

    n = len(means)
    dm, dg, dout = ctx.malloc(n * 8), ctx.malloc(n * 8), ctx.malloc(128)
    try:
        ctx.h2d(dm, means)
        ctx.h2d(dg, gw)
        ctx.check(ctx.lib.pdq_trend_fit_dev(ctx.h, _lib.c_dptr(dm), _lib.c_dptr(dg), n, min_disp, max_disp, trigamma_c,
                                            _lib.c_dptr(dout), _lib.c_dptr(0)))
        out = np.zeros(16)
        ctx.d2h(out, dout)
        ctx.sync()
        return out
    finally:
        for p in (dm, dg, dout):
            ctx.free(p)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["0", "1"])
@pytest.mark.parametrize("name", list(tc.CASES))
def test_gpu_trend_record_matches_fixture(ctx, ref, name, mode):
    os.environ["PDQ_TREND_GRID"] = mode
    try:
        got = trend_record(ctx, *tc.case(name))
    finally:
        del os.environ["PDQ_TREND_GRID"]
    want = ref[f"{name}__grid{mode}"]
    assert want[2] == 0.0 and np.isfinite(want[8])  # every case fits, so the prior is computed
    if mode == "0":
        np.testing.assert_array_equal(bits(got), bits(want))
        return
    np.testing.assert_array_equal(bits(got[EXACT_FIELDS]), bits(want[EXACT_FIELDS]))
    np.testing.assert_allclose(got[6], want[6], rtol=1e-12)  # the loss is a sum in arrival order
    if np.array_equal(bits(got[:2]), bits(want[:2])):  # same coefficients -> same residuals -> the same exact medians
        np.testing.assert_array_equal(bits(got[[8, 9]]), bits(want[[8, 9]]))
    else:
        np.testing.assert_allclose(got[[0, 1, 8, 9]], want[[0, 1, 8, 9]], rtol=1e-10)


@pytest.mark.gpu
def test_gpu_trend_record_is_reproducible_on_one_cluster(ctx):
    args = tc.case("plain_20000")
    os.environ["PDQ_TREND_GRID"] = "0"
    try:
        a, b = trend_record(ctx, *args), trend_record(ctx, *args)
    finally:
        del os.environ["PDQ_TREND_GRID"]
    np.testing.assert_array_equal(bits(a), bits(b))


def _bin_of_rank(v, k, lo, hi):
    # the bin function of median_bins: clamp(floor((v - lo) * scale)), scale = kVBins / (hi - lo)
    scale = V_BINS / (hi - lo)
    b = np.clip(np.floor((v - lo) * scale), 0, V_BINS - 1).astype(np.int64)
    counts = np.bincount(b, minlength=V_BINS)
    kb = int(np.searchsorted(np.cumsum(counts), k, side="right"))
    return counts[kb]


def _residuals(name, rec):
    means, gw, min_disp, max_disp, _ = tc.case(name)
    t = np.clip(gw, min_disp, max_disp)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.log(t) - np.log(rec[0] + rec[1] / means)
    return r[(t >= 100 * min_disp) & ~np.isnan(means)]


@pytest.mark.parametrize("name", ["clipped_ties_20000", "clipped_ties_150001"])
def test_tie_cases_overflow_the_candidate_buffer(ref, name):
    """These cases take the exact fallback of both medians: the value bin that holds the median, and the one that holds the
    median absolute deviation, each contain more values than the candidate buffer."""
    r = _residuals(name, ref[f"{name}__grid0"])
    k = len(r) // 2
    med = np.median(r)
    assert _bin_of_rank(r, k, r.min(), r.max()) > CAND_CAP
    d = np.abs(r - med)
    assert _bin_of_rank(d, k, 0.0, d.max()) > CAND_CAP
    assert ref[f"{name}__grid0"][8] == 0.0  # more than half the residuals are equal: the MAD is zero


def test_equal_residual_case_has_a_range_of_zero_width(ref):
    r = _residuals("equal_residuals_4000", ref["equal_residuals_4000__grid0"])
    assert len(r) == 400 and r.min() == r.max()


def test_plain_cases_stay_within_the_candidate_buffer(ref):
    # the fast path itself is what the other cases exercise
    for name in ("plain_1000", "plain_19999", "plain_20000", "plain_65535", "padded_70000", "flat_tail_150001"):
        r = _residuals(name, ref[f"{name}__grid0"])
        k = len(r) // 2
        assert _bin_of_rank(r, k, r.min(), r.max()) <= CAND_CAP
        d = np.abs(r - np.median(r))
        assert _bin_of_rank(d, k, 0.0, d.max()) <= CAND_CAP


@pytest.mark.parametrize("name,threads", [("gapped_70000", 35 * 1024), ("gapped_1000", 1024)])
def test_gapped_cases_leave_grid_warps_without_a_value_below_the_bin(ref, name, threads):
    """The even-count path where rank k opens its value bin, so the lower median is the largest value of the bins below, with
    whole warps of the grid kernel (thread t takes genes t, t + threads, ...) that see no value below that bin: their share of
    the maximum is the empty key."""
    means, gw, min_disp, max_disp, _ = tc.case(name)
    rec = ref[f"{name}__grid1"]
    t = np.clip(gw, min_disp, max_disp)
    r = np.log(t) - np.log(rec[0] + rec[1] / means)
    r[(t < 100 * min_disp) | np.isnan(means)] = np.nan
    v = r[~np.isnan(r)]
    k = len(v) // 2
    assert len(v) % 2 == 0
    scale = V_BINS / (v.max() - v.min())
    bins = np.where(np.isnan(r), V_BINS, np.clip(np.floor((r - v.min()) * scale), 0, V_BINS - 1))
    counts = np.bincount(bins[~np.isnan(r)].astype(np.int64), minlength=V_BINS)
    b = int(np.searchsorted(np.cumsum(counts), k, side="right"))
    assert counts[:b].sum() == k  # rank k is the first value of bin b
    thread_has_below = np.zeros(threads, bool)
    np.logical_or.at(thread_has_below, np.arange(len(r)) % threads, bins < b)
    assert (~thread_has_below.reshape(-1, 32).any(axis=1)).any()
