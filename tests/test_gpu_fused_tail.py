"""GPU suite: the fused tail of the resident pass (MAP dispersion search -> final dispersions -> LFC fit + Wald test as a pair of
kernels with per-tile hand-off, ``pdq_map_irls_wald_dev``) against the same three stages as separate launches.
No per-gene arithmetic differs between the two, so every result must agree bit for bit."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

KEYS = ("mom", "genewise", "genewise_converged", "map", "map_converged", "dispersions", "lfc", "lfc_converged", "pvalue", "stat", "se",
        "normed_means", "fitted", "outlier", "prior_var", "squared_logres")
COOKS_KEYS = ("robust_dispersions", "cooks_outlier", "cooks_replaced")


@pytest.fixture(scope="module")
def inf():
    from pydeseq2_b200.inference import B200Inference

    return B200Inference(device=0)


@pytest.fixture
def force(inf):
    ctx = inf._ops.ctx

    def f(flags):
        ctx.check(ctx.lib.pdq_set_debug_flags(ctx.h, flags))

    yield f
    f(0)


def _data(N, G, kind, seed, X=None):
    from pydeseq2_b200.pipeline import median_of_ratios
    from pydeseq2_b200.synth import make_counts

    counts, Xs, _ = make_counts(N, G, kind, seed)
    counts = np.ascontiguousarray(counts[:, ~(counts == 0).all(0)])
    return counts, (Xs if X is None else X), median_of_ratios(counts)[1]


def _tail_status(ctx):
    st = C.c_uint64(1)
    ctx.check(ctx.lib.pdq_map_irls_status(ctx.h, C.byref(st)))
    return st.value


def _fit(inf, counts, X, sf, fused, passes=3, **kw):
    """`passes` runs of one ResidentFit (eager, captured, replays); every pass' results, and the wait's error word after each."""
    from pydeseq2_b200.pipeline import ResidentFit

    ctx = inf._ops.ctx
    rf = ResidentFit(ctx, X, sf, **kw)
    rf.fuse_tail = fused
    rf.upload(counts)
    out = []
    try:
        for _ in range(passes):
            out.append(rf.run())
            assert _tail_status(ctx) == 0
    finally:
        rf.close()
    return out


def _assert_same(a, b, keys=KEYS):
    for k in keys:
        np.testing.assert_array_equal(np.asarray(a[k]), np.asarray(b[k]), err_msg=k)


def _compare(inf, counts, X, sf, passes=3, keys=KEYS, **kw):
    sep = _fit(inf, counts, X, sf, False, passes=2, **kw)[-1]
    fused = _fit(inf, counts, X, sf, True, passes=passes, **kw)
    for r in fused:  # the eager pass, the captured pass and every replay
        _assert_same(r, sep, keys)
    return sep


@pytest.mark.parametrize("N,G,kind,seed", [(200, 6000, "two_level", 0), (60, 3000, "factorial", 1), (48, 3000, "continuous", 2)])
def test_fused_equals_separate(inf, N, G, kind, seed):
    sep = _compare(inf, *_data(N, G, kind, seed))
    assert np.isfinite(sep["dispersions"]).all() and np.isfinite(sep["lfc"]).all()


@pytest.mark.parametrize("G", [37, 1001, 5003])
def test_fused_gene_counts_off_the_tile_grid(inf, G):
    """G not a multiple of the tile size; fewer tiles than one wave of warps (and, below 256 genes, the unsorted gene order)."""
    counts, X, sf = _data(24, G, "two_level", 3)
    _compare(inf, counts, X, sf)


def test_fused_wide_design(inf):
    """p = 9: the translation unit of the wide designs."""
    rng = np.random.default_rng(9)
    N = 91
    X = np.column_stack([np.ones(N), (np.arange(N) % 2).astype(float), rng.normal(size=(N, 7)) * 0.3])
    _compare(inf, *_data(N, 1200, "two_level", 4, X=X))


@pytest.mark.parametrize("flags", [2, 1, 3], ids=["alpha_grid", "irls_optimizer", "both"])
def test_fused_forced_fallbacks(inf, force, flags):
    """PDQ_DEBUG_FORCE_ALPHA_GRID defers every tile to k_alpha_grid + k_irls_deferred; PDQ_DEBUG_FORCE_IRLS_OPTIMIZER sends every
    gene through the optimiser branch behind the pair."""
    counts, X, sf = _data(40, 700, "factorial", 5)
    plain = _fit(inf, counts, X, sf, True, passes=1)[0]
    force(flags)
    forced = _compare(inf, counts, X, sf)
    if flags & 2:
        assert (forced["map_converged"] == 0).all()
        assert not np.array_equal(forced["map"], plain["map"])
    force(0)
    _assert_same(_fit(inf, counts, X, sf, True, passes=1)[0], plain)  # the control words carry nothing over from the forced passes


def test_fused_replays(inf):
    """Eager pass, captured pass and ten graph replays in a row: the pass number, the ticket counter and the flagged-gene counts
    are maintained by the launch itself."""
    counts, X, sf = _data(100, 4000, "two_level", 6)
    _compare(inf, counts, X, sf, passes=12)


def test_fused_with_cooks(inf):
    counts, X, sf = _data(30, 2000, "two_level", 7)
    _compare(inf, counts, X, sf, keys=KEYS + COOKS_KEYS, with_cooks=True)


def test_profile_keeps_the_stage_names(inf):
    """Stage timings come from the separate launches, under their names, whatever fuse_tail says."""
    from pydeseq2_b200.pipeline import ResidentFit

    counts, X, sf = _data(24, 1500, "two_level", 8)
    rf = ResidentFit(inf._ops.ctx, X, sf)
    assert rf.fuse_tail
    rf.upload(counts)
    try:
        a = rf.run()
        b = rf.run(profile=True)
        assert {"alpha_mle_map", "select_dispersions", "irls_lfc_wald"} <= set(rf.stage_ms)
        _assert_same(a, b)
    finally:
        rf.close()
