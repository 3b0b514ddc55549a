"""GPU suite: the glue of the resident pass -- the start values folded into the genewise dispersion search (``fold_moments``,
``pdq_mom_alpha_mle_dev``), one caller-order launch per half of the result slab (``pdq_scatter_segments_dev``), the genewise half
copied to the host on a branch of the stream and the tail half written into the page-locked host block by its reorder launch --
against the sequence it replaces: the start values as a launch of their own, one scatter of the whole slab at the end of the pass
(two row scatters and a copy of the trend record) and one copy of the whole slab.  No per-gene arithmetic differs between the two,
so every result must agree bit for bit."""
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


def _old_glue_fit():
    """ResidentFit with the pass' old glue: separate start-value launch, the whole slab scattered at the end, one copy."""
    from pydeseq2_b200.pipeline import ResidentFit

    class OldGlue(ResidentFit):
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            self.fold_moments = False

        def _to_caller_order(self, seg, host=False):  # the tail half's output step: the old reorder and one copy
            if seg is self._seg_gw:
                return
            if self._perm is not None:
                L, h, c_d = self.lib, self.ctx.h, self._lib_mod.c_dptr
                self.ctx.check(L.pdq_scatter_rows_dev(h, c_d(self.d_slab), c_d(self.d_slab_out), c_d(self.d_perm), self.G, 15, self.Gs, 1))
                self.ctx.check(L.pdq_scatter_rows_dev(h, c_d(self.d_slab + self._off_beta * 8),
                                                      c_d(self.d_slab_out + self._off_beta * 8), c_d(self.d_perm), self.G, 1, self.Gs,
                                                      self.p))
                self.ctx.check(L.pdq_memcpy_d2d(h, c_d(self.d_slab_out + self._off_t16 * 8), c_d(self.d_t16), 16 * 8))
            self.ctx.d2h(self._h_slab, self.d_slab_out)

        def _copy_out(self, ranges, side=False):  # single-GPU passes copy the genewise half only, on the side branch
            pass

    return OldGlue


def _fit(inf, counts, X, sf, old, passes=3, cooks_seq=None, **kw):
    """`passes` runs of one ResidentFit (eager, captured, replays); ``cooks_seq``: with_cooks per pass."""
    from pydeseq2_b200.pipeline import ResidentFit

    rf = (_old_glue_fit() if old else ResidentFit)(inf._ops.ctx, X, sf, **kw)
    rf.upload(counts)
    out = []
    try:
        for i in range(passes):
            if cooks_seq is not None:
                rf.with_cooks = cooks_seq[i]
            out.append(rf.run())
    finally:
        rf.close()
    return out


def _assert_same(a, b, keys=KEYS):
    for k in keys:
        np.testing.assert_array_equal(np.asarray(a[k]), np.asarray(b[k]), err_msg=k)


def _compare(inf, counts, X, sf, passes=4, keys=KEYS, **kw):
    ref = _fit(inf, counts, X, sf, True, passes=2, **kw)[-1]
    for r in _fit(inf, counts, X, sf, False, passes=passes, **kw):  # the eager pass, the captured pass and every replay
        _assert_same(r, ref, keys)
    return ref


@pytest.mark.parametrize("N,G,kind,seed", [(200, 6000, "two_level", 0), (60, 3000, "factorial", 1), (48, 3000, "continuous", 2)])
def test_new_glue_equals_old(inf, N, G, kind, seed):
    """Sorted gene order; the two-level design takes the folded launch, the other two the IRLS-initialised branch."""
    ref = _compare(inf, *_data(N, G, kind, seed))
    assert np.isfinite(ref["dispersions"]).all() and np.isfinite(ref["lfc"]).all()


@pytest.mark.parametrize("G", [37, 203])
def test_unsorted_small_shard(inf, G):
    """Below 256 genes the gene order is the caller's (no scatter); the slab still reaches the host in two halves."""
    from pydeseq2_b200.pipeline import ResidentFit

    counts, X, sf = _data(24, G, "two_level", 3)
    rf = ResidentFit(inf._ops.ctx, X, sf)
    rf.upload(counts)
    try:
        assert rf._perm is None
    finally:
        rf.close()
    _compare(inf, counts, X, sf)


def test_wide_design_unit(inf):
    """p = 9 on a lin_reg_mu design: the fold in the translation unit of the wide widths."""
    N, levels = 90, 9
    X = np.zeros((N, levels))
    X[:, 0] = 1.0
    for i in range(N):
        if i % levels:
            X[i, i % levels] = 1.0
    counts, _, sf = _data(N, 1500, "two_level", 4)
    _compare(inf, counts, X, sf)


def test_cooks_toggled_between_passes(inf):
    """with_cooks off, on, off, on, on on one ResidentFit: the Cook's vectors are scattered and copied exactly when computed."""
    counts, X, sf = _data(30, 2000, "two_level", 7)
    seq = [False, True, False, True, True]
    new = _fit(inf, counts, X, sf, False, passes=len(seq), cooks_seq=seq)
    old = _fit(inf, counts, X, sf, True, passes=len(seq), cooks_seq=seq)
    for c, a, b in zip(seq, new, old):
        _assert_same(a, b, KEYS + (COOKS_KEYS if c else ()))
        assert all((k in a) == c for k in COOKS_KEYS)


@pytest.mark.parametrize("flags", [2, 1], ids=["alpha_grid", "irls_optimizer"])
@pytest.mark.parametrize("kind", ["two_level", "factorial"])
def test_forced_fallbacks(inf, force, flags, kind):
    """Genes rewritten by the fallback kernels behind the searches (PDQ_DEBUG_FORCE_ALPHA_GRID: every gene through k_alpha_grid,
    also behind the folded launch; PDQ_DEBUG_FORCE_IRLS_OPTIMIZER: every gene through the optimiser branch) reach the caller's
    order; afterwards the control words of the folded launch carry nothing over."""
    counts, X, sf = _data(40, 700, kind, 5)
    plain = _fit(inf, counts, X, sf, False, passes=1)[0]
    force(flags)
    forced = _compare(inf, counts, X, sf)
    if flags & 2:
        assert (forced["genewise_converged"] == 0).all()
    force(0)
    _assert_same(_fit(inf, counts, X, sf, False, passes=1)[0], plain)


def test_refit_subset_after_a_pass(inf):
    """The outlier refit's genewise stage takes the folded launch too, on its own gene set."""
    counts, X, sf = _data(60, 3000, "two_level", 8)
    idx = np.arange(0, 3000, 97)
    sub = np.ascontiguousarray(counts[:, idx])
    outs = []
    for old in (False, True):
        from pydeseq2_b200.pipeline import ResidentFit

        rf = (_old_glue_fit() if old else ResidentFit)(inf._ops.ctx, X, sf)
        rf.upload(counts)
        try:
            res = rf.run()
            rf.run()
            outs.append((res, rf.refit_subset(sub, res["trend"], res["prior_var"])))
        finally:
            rf.close()
    (new, new_sub), (old, old_sub) = outs
    _assert_same(new, old)
    for k in ("normed_means", "genewise", "fitted", "disp", "lfc", "pvalue", "stat", "se"):
        np.testing.assert_array_equal(new_sub[k], old_sub[k], err_msg=k)


def test_profile_keeps_the_stage_names(inf):
    """Stage timings come from the separate launches, under their names, whatever fold_moments says."""
    from pydeseq2_b200.pipeline import ResidentFit

    counts, X, sf = _data(24, 1500, "two_level", 9)
    rf = ResidentFit(inf._ops.ctx, X, sf)
    assert rf.fold_moments and rf.lin_branch
    rf.upload(counts)
    try:
        a = rf.run()
        b = rf.run(profile=True)
        assert {"mom_dispersions", "alpha_mle_genewise", "to_caller_order"} <= set(rf.stage_ms)
        _assert_same(a, b)
    finally:
        rf.close()
