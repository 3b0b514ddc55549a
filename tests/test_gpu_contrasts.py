"""GPU suite: pdq_wald_contrasts (k_wald_contrasts) on an H100 -- the ct_* goldens of the real orchestrator through `_CudaOps`, the
device against the host emulator on seeded cases (p = 1..16; the gene-block pipeline at N = 8 000 x G = 60 000, K = 45; six rounds
of contrasts per lane at p = 12, G = 20 000, K = 45), one
contrast against pdq_mu_from_lfc_dev + pdq_wald_test_dev, the C ABI's argument checks, and `workflow.deseq2_stats` on both drivers."""
import ctypes as C

import numpy as np
import pytest

from contrast_cases import ALTS, CT, assert_tests_close, check_golden_wald, check_stats_e2e, seeded_case, stat_atol

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def inf():
    from pydeseq2_b200.inference import B200Inference

    return B200Inference(device=0)


def emulated(X, sf, disp, lfc, cs, nulls, alts):
    from emu.contrast_ops import ContrastEmuOps
    from pydeseq2_b200.inference import B200Inference

    return B200Inference(_ops=ContrastEmuOps()).wald_tests(X, sf, disp, lfc, cs, None, nulls, alts)


@pytest.mark.parametrize("name", CT)
def test_goldens_through_the_device(inf, name):
    check_golden_wald(inf, name)


@pytest.mark.parametrize("p,N,G,K", [(p, 3 * p + 12, 700, 45 if p % 2 else 7) for p in range(1, 17)]
                         + [(2, 8000, 60000, 45), (12, 200, 20000, 45)])
def test_device_against_emulator(inf, p, N, G, K):
    X, sf, disp, lfc, cs = seeded_case(p, N, G, K, seed=1000 + p + K)
    alts = [ALTS[k % 5] for k in range(K)]
    nulls = np.where(np.arange(K) % 2, 0.25, 0.0)
    got = inf.wald_tests(X, sf, disp, lfc, cs, None, nulls, alts)
    want = emulated(X, sf, disp, lfc, cs, nulls, alts)
    # the lane widths differ (the device's sums run in another order), so a statistic whose dot product cancels is compared
    # against the rounding of its terms
    assert_tests_close(got, want, 1e-12, f"p={p} N={N} G={G} K={K}", stat_atol(cs, lfc, nulls, want[2], 1e-12))


@pytest.mark.parametrize("p", [1, 3, 8, 9, 16])
def test_one_contrast_equals_mu_from_lfc_then_wald_test(inf, p):
    from pydeseq2_b200 import _lib

    N, G = 4 * p + 20, 3000
    X, sf, disp, lfc, cs = seeded_case(p, N, G, 1, seed=77 + p)
    ridge = np.diag(np.repeat(1e-6, p))
    got = inf.wald_tests(X, sf, disp, lfc, cs[0], ridge, 0.2, "greater")
    ctx = inf._ops.ctx
    L, h, cd = ctx.lib, ctx.h, _lib.c_dptr
    d = _lib.c_design()
    ctx.check(L.pdq_design_create(h, _lib.as_f64p(X), _lib.as_f64p(sf), N, p, C.byref(d)))
    bufs = [ctx.malloc(n * 8) for n in (G * p, G, N * G, G, G, G)]
    try:
        d_lfc, d_disp, d_mu, d_p, d_s, d_se = bufs
        ctx.h2d(d_lfc, lfc)
        ctx.h2d(d_disp, disp)
        ctx.check(L.pdq_mu_from_lfc_dev(h, d, cd(d_lfc), G, cd(d_mu), G))
        ctx.check(L.pdq_wald_test_dev(h, d, cd(d_disp), cd(d_lfc), cd(d_mu), G, G, _lib.as_f64p(ridge), _lib.as_f64p(cs[0]), 0.2,
                                      _lib.ALT_CODES["greater"], cd(d_p), cd(d_s), cd(d_se)))
        want = [np.empty(G) for _ in range(3)]
        for w, b in zip(want, (d_p, d_s, d_se)):
            ctx.d2h(w, b)
        ctx.sync()
    finally:
        for b in bufs:
            ctx.free(b)
        L.pdq_design_destroy(h, d)
    assert_tests_close(got, want, 1e-12, f"p={p}")


def test_c_abi_pitch_and_argument_checks(inf):
    from pydeseq2_b200._lib import as_f64p

    ops = inf._ops
    N, p, G, K = 30, 3, 500, 4
    X, sf, disp, lfc, cs = seeded_case(p, N, G, K, seed=5)
    ridge = np.diag(np.repeat(1e-6, p))
    nulls = np.zeros(K)
    alt = np.array([0, 1, 3, 4], np.int32)
    ld = G + 7
    outs = [np.full((K, ld), -1.0) for _ in range(3)]
    ops.wald_contrasts(X, sf, N, p, disp, lfc, G, ridge, K, cs, nulls, alt, *outs, ld)
    want = inf.wald_tests(X, sf, disp, lfc, cs, ridge, nulls, [ALTS[a] for a in alt])
    for o, w in zip(outs, want):
        np.testing.assert_array_equal(o[:, :G], w)       # same kernel, same lane width: identical
        assert (o[:, G:] == -1.0).all()                  # the pitch's padding is not written

    def rc(K_=K, alt_=alt, ld_=ld, p_=p, X_=X, ridge_=ridge, cs_=cs, lfc_=lfc):
        return ops.lib.pdq_wald_contrasts(ops.ctx.h, as_f64p(X_), as_f64p(sf), N, p_, as_f64p(disp), as_f64p(lfc_), G, as_f64p(ridge_),
                                          K_, as_f64p(cs_), as_f64p(nulls), alt_.ctypes.data_as(C.POINTER(C.c_int)), *(as_f64p(o) for o in outs), ld_)

    assert rc() == 0
    assert rc(K_=0) == -2
    assert rc(alt_=np.array([0, 1, 5, 4], np.int32)) == -2
    assert rc(alt_=np.array([0, -1, 3, 4], np.int32)) == -2
    assert rc(ld_=G - 1) == -2
    X17, lfc17 = np.ones((N, 17)), np.zeros((G, 17))
    assert rc(p_=17, X_=X17, ridge_=np.eye(17), cs_=np.ones((K, 17)), lfc_=lfc17) == -3


@pytest.mark.parametrize("name", ["ct_three_level_batch", "ct_outliers", "ct_ten_levels"])
@pytest.mark.parametrize("resident", [False, True])
def test_deseq2_stats_on_both_drivers(inf, name, resident):
    check_stats_e2e(inf, name, 2e-3 if name == "ct_ten_levels" else 2e-4, max_frac=0.02, resident=resident)
