"""GPU suite: the refusals of the C ABI's operation entry points, in both forms (host buffers and device pointers).  Each pins the
return code and the pdq_last_error text, including which refusal wins when several apply, and a refused host-buffer call must
stage nothing: the residency cache, the context's buffers and the launch counter are as they were."""
import ctypes as C

import numpy as np
import pytest

from pydeseq2_b200._lib import Context, as_f64p, as_i64p
from test_large_designs import paired

pytestmark = pytest.mark.gpu

INVALID, UNSUPPORTED = -2, -3
N, G = 128, 4096  # an (N, G) float64 array of 4 MiB with ld == G: the residency cache takes it
NI16 = "lfc_shrink: apeGLM shrinkage of designs with more than 16 columns is not implemented"
NI64 = "lfc_shrink: apeGLM shrinkage of designs with more than 64 columns is not implemented"
SQUARE = "The number of samples and the number of design variables are equal"


def narrow(p):
    return f"design has {p} columns; this build supports p <= 16"


def wide(p, limit):
    return f"design has {p} columns; wide designs support p <= {limit}"


class Abi:
    def __init__(self):
        self.ctx = Context(0)
        self.lib, self.h = self.ctx.lib, self.ctx.h
        rng = np.random.default_rng(3)
        self.counts = rng.poisson(30, (N, G)).astype(np.int64)
        self.mu = rng.uniform(5.0, 50.0, (N, G))
        self.vec = np.ones(G)
        self.out = [np.zeros((N, G)) for _ in range(3)]
        self.dev = self.ctx.malloc(8 << 20)  # stands in for every device buffer: a refused call launches nothing
        self.staged = []  # refusals that changed the residency statistics, the buffer epoch or the launch count

    def opt_in(self, wide=0, wide_shrink=0, large=0, large_shrink=0):
        for f, on in ((self.lib.pdq_set_wide_designs, wide), (self.lib.pdq_set_wide_shrink, wide_shrink),
                      (self.lib.pdq_set_large_designs, large), (self.lib.pdq_set_large_shrink, large_shrink)):
            assert f(self.h, on) == 0

    def state(self):
        v = [C.c_int64() for _ in range(4)]
        assert self.lib.pdq_residency_stats(self.h, *[C.byref(x) for x in v]) == 0
        return [x.value for x in v], self.lib.pdq_buffer_epoch(self.h), self.lib.pdq_launch_count(self.h)

    def refused(self, call, code, msg):
        before = self.state()
        assert call() == code
        assert self.lib.pdq_last_error(self.h) == msg.encode()
        if self.state() != before:
            self.staged.append(msg)

    def nothing_staged(self):
        staged, self.staged = self.staged, []
        assert not staged

    def design(self, X):
        d = C.c_void_p()
        X = np.ascontiguousarray(X, dtype=np.float64)
        assert self.lib.pdq_design_create(self.h, as_f64p(X), as_f64p(np.ones(X.shape[0])), X.shape[0], X.shape[1], C.byref(d)) == 0, \
            self.lib.pdq_last_error(self.h)
        return d

    # ---- host-buffer forms
    def lin_reg_mu(self, X, g=G):
        return self.lib.pdq_lin_reg_mu(self.h, as_i64p(self.counts), G, N, g, as_f64p(np.ones(N)), as_f64p(X), X.shape[1], 0.5,
                                       as_f64p(self.out[0]))

    def irls(self, X, ld=G):
        nfb = C.c_int(0)
        return self.lib.pdq_irls(self.h, as_i64p(self.counts), ld, N, G, as_f64p(np.ones(N)), as_f64p(X), X.shape[1],
                                 as_f64p(self.vec), 0.5, 1e-8, -30.0, 30.0, 250, as_f64p(np.zeros((G, X.shape[1]))),
                                 as_f64p(self.out[0]), as_f64p(self.out[1]), as_f64p(self.vec.copy()), C.byref(nfb))

    def alpha_mle(self, X, prior_reg=0, prior_var=1.0, ld_mu=G):
        return self.lib.pdq_alpha_mle(self.h, as_i64p(self.counts), G, N, G, as_f64p(X), X.shape[1], as_f64p(self.mu), ld_mu,
                                      as_f64p(self.vec), 1e-8, 10.0, prior_var, 1, prior_reg, as_f64p(np.zeros(G)), as_f64p(np.zeros(G)))

    def wald_test(self, X, alt=0, ld_mu=G):
        p = X.shape[1]
        return self.lib.pdq_wald_test(self.h, as_f64p(X), N, p, as_f64p(self.vec), as_f64p(np.zeros((G, p))), as_f64p(self.mu), ld_mu,
                                      G, as_f64p(np.eye(p)), as_f64p(np.ones(p)), 0.0, alt, *(as_f64p(np.zeros(G)) for _ in range(3)))

    def wald_contrasts(self, X, alts=(0, 0), K=2):
        p = X.shape[1]
        alt = np.asarray(alts, np.int32)
        return self.lib.pdq_wald_contrasts(self.h, as_f64p(X), as_f64p(np.ones(N)), N, p, as_f64p(self.vec),
                                           as_f64p(np.zeros((G, p))), G, as_f64p(np.eye(p)), K, as_f64p(np.ones((2, p))),
                                           as_f64p(np.zeros(2)), alt.ctypes.data_as(C.POINTER(C.c_int)),
                                           *(as_f64p(o) for o in self.out[:3]), G)

    def shrink(self, X, shrink_index=1, scale=0.4):
        p = X.shape[1]
        out = [np.zeros((G, p)), np.zeros((G, p, p)), np.zeros(G)]
        n_grid = C.c_int(0)
        return self.lib.pdq_lfc_shrink_nbinom_glm(self.h, as_f64p(X), as_i64p(self.counts), G, N, G, p, as_f64p(self.vec),
                                                  as_f64p(np.zeros(N)), 15.0, scale, shrink_index, *(as_f64p(o) for o in out),
                                                  C.byref(n_grid))

    # ---- device forms (d: a design made by pdq_design_create)
    def shrink_dev(self, d, shrink_index=1, scale=0.4, g=8):
        b = self.dev
        return self.lib.pdq_lfc_shrink_dev(self.h, d, b, g, g, b, 15.0, scale, shrink_index, b, b, b, b)


def two_column():
    return np.ascontiguousarray(np.column_stack([np.ones(N), np.arange(N) % 2]).astype(np.float64))


def p17():
    return np.ascontiguousarray(np.tile(paired(16), (N // 32, 1)))  # (N, 17)


def p65():
    return np.ascontiguousarray(paired(64))  # (N, 65)


@pytest.fixture(scope="module")
def abi():
    a = Abi()
    # warm the context: buffers allocated and the inputs resident, so that a refused call that stages shows in the state
    X = two_column()
    assert a.lin_reg_mu(X) == 0 and a.alpha_mle(X) == 0 and a.wald_test(X) == 0, a.lib.pdq_last_error(a.h)
    return a


def test_host_forms_refuse_before_staging(abi):
    X, X17 = two_column(), p17()
    abi.opt_in()
    abi.refused(lambda: abi.lin_reg_mu(X, g=0), INVALID, "pdq_lin_reg_mu: bad arguments")
    abi.refused(lambda: abi.lin_reg_mu(X17), UNSUPPORTED, narrow(17))
    abi.refused(lambda: abi.irls(X, ld=G - 1), INVALID, "pdq_irls: bad arguments")
    abi.refused(lambda: abi.irls(X17), UNSUPPORTED, narrow(17))
    abi.refused(lambda: abi.alpha_mle(X, ld_mu=G - 1), INVALID, "pdq_alpha_mle: bad arguments")
    abi.refused(lambda: abi.alpha_mle(X, prior_reg=1, prior_var=0.0), INVALID, "alpha_mle: prior_reg needs prior_disp_var > 0")
    abi.refused(lambda: abi.alpha_mle(X17, prior_reg=1, prior_var=0.0), UNSUPPORTED, narrow(17))
    abi.refused(lambda: abi.wald_test(X, ld_mu=G - 1), INVALID, "pdq_wald_test: bad arguments")
    abi.refused(lambda: abi.wald_test(X, alt=5), INVALID, "pdq_wald_test: unknown alternative")
    abi.refused(lambda: abi.wald_test(X, alt=-1), INVALID, "pdq_wald_test: unknown alternative")
    abi.refused(lambda: abi.wald_test(X17, alt=5), UNSUPPORTED, narrow(17))
    abi.refused(lambda: abi.wald_contrasts(X, K=0), INVALID, "pdq_wald_contrasts: bad arguments")
    abi.refused(lambda: abi.wald_contrasts(X17), UNSUPPORTED, "pdq_wald_contrasts: " + narrow(17))
    abi.refused(lambda: abi.wald_contrasts(X, alts=(0, 7)), INVALID, "pdq_wald_contrasts: unknown alternative 7 (contrast 1)")
    abi.refused(lambda: abi.shrink(X, shrink_index=2), INVALID, "pdq_lfc_shrink_dev: bad arguments")
    abi.refused(lambda: abi.shrink(X, scale=0.0), INVALID, "pdq_lfc_shrink_dev: bad arguments")
    # a design without columns is refused as pdq_design_create refuses it, ahead of the later checks
    X0 = np.ones((N, 0))
    abi.refused(lambda: abi.alpha_mle(X0, prior_reg=1, prior_var=0.0), INVALID, "pdq_design_create: bad arguments")
    abi.refused(lambda: abi.wald_test(X0, alt=5), INVALID, "pdq_design_create: bad arguments")
    abi.refused(lambda: abi.shrink(X0, shrink_index=0), INVALID, "pdq_design_create: bad arguments")
    Xsq = np.eye(2)
    normed = np.ones((2, G))
    abi.refused(lambda: abi.lib.pdq_fit_rough_dispersions(abi.h, as_f64p(normed), G, 2, G, as_f64p(Xsq), 2, as_f64p(np.zeros(G))),
                INVALID, SQUARE)
    abi.refused(lambda: abi.lib.pdq_fit_moments_dispersions(abi.h, as_f64p(abi.mu), G - 1, N, G, as_f64p(np.ones(N)),
                                                            as_f64p(np.zeros(G)), as_f64p(np.zeros(G))),
                INVALID, "pdq_fit_moments_dispersions: bad arguments")
    for kind, c0, msg in ((2, 1.0, "unknown kind 2 (0 parametric, 1 mean)"), (0, 0.0, "a0 must be > 0"),
                          (1, -1.0, "the mean dispersion must be > 0")):
        abi.refused(lambda: abi.lib.pdq_vst_transform(abi.h, as_i64p(abi.counts), G, N, G, as_f64p(np.ones(N)), kind, c0, 0.0,
                                                      as_f64p(abi.out[2]), G), INVALID, "pdq_vst_transform: " + msg)
    abi.nothing_staged()


def test_host_shrinkage_opt_ins(abi):
    """The width and opt-in refusals of pdq_lfc_shrink_nbinom_glm, at every combination the opt-in contract tests use."""
    X17, X65, X129 = p17(), p65(), np.ones((N, 129))
    a = abi
    # wide designs on, wide shrinkage off; and off, with and without wide shrinkage
    a.opt_in(wide=1)
    a.refused(lambda: a.shrink(X17), UNSUPPORTED, NI16)
    a.refused(lambda: a.shrink(X17, shrink_index=40), UNSUPPORTED, NI16)  # the opt-in wins over a bad shrink_index
    a.opt_in(wide=0, wide_shrink=1)
    a.refused(lambda: a.shrink(X17), UNSUPPORTED, narrow(17))
    a.opt_in()
    a.refused(lambda: a.shrink(X17), UNSUPPORTED, narrow(17))  # the width wins over the shrinkage opt-in
    # 65 columns: wide shrinkage off whatever the others; large designs off; large shrinkage off
    a.opt_in(wide=1, large=1, large_shrink=1)
    a.refused(lambda: a.shrink(X65), UNSUPPORTED, NI16)
    a.opt_in(wide=1, wide_shrink=1, large_shrink=1)
    a.refused(lambda: a.shrink(X65), UNSUPPORTED, wide(65, 64))
    a.opt_in(wide=1, wide_shrink=1, large=1)
    a.refused(lambda: a.shrink(X65), UNSUPPORTED, NI64)
    a.opt_in(wide=1, wide_shrink=1, large=1, large_shrink=1)
    a.refused(lambda: a.shrink(X129), UNSUPPORTED, wide(129, 128))
    a.refused(lambda: a.lin_reg_mu(X129), UNSUPPORTED, wide(129, 128))
    a.refused(lambda: a.wald_contrasts(X129), UNSUPPORTED, "pdq_wald_contrasts: " + wide(129, 128))
    a.opt_in(wide=1)
    a.refused(lambda: a.lin_reg_mu(X65), UNSUPPORTED, wide(65, 64))
    a.refused(lambda: a.wald_contrasts(X65), UNSUPPORTED, "pdq_wald_contrasts: " + wide(65, 64))
    a.opt_in()
    a.nothing_staged()


def test_device_forms(abi):
    a, b = abi, abi.dev
    a.opt_in(wide=1, large=1)
    d2, d17, d65, dsq = a.design(two_column()), a.design(p17()), a.design(p65()), a.design(np.eye(4))
    try:
        g = 8
        ridge, contrast = np.eye(2), np.ones(2)
        # design packs
        X17 = p17()
        dd = C.c_void_p()
        a.opt_in()
        a.refused(lambda: a.lib.pdq_design_create(a.h, as_f64p(X17), None, N, 17, C.byref(dd)), UNSUPPORTED, narrow(17))
        a.refused(lambda: a.lib.pdq_design_create(a.h, as_f64p(X17), None, 0, 17, C.byref(dd)), INVALID,
                  "pdq_design_create: bad arguments")
        # lin_reg_mu, irls and irls + Wald
        a.refused(lambda: a.lib.pdq_lin_reg_mu_dev(a.h, d2, b, g, 0, 0.5, b, g), INVALID, "pdq_lin_reg_mu_dev: bad arguments")
        irls = (0.5, 1e-8, -30.0, 30.0, 250, b, b, b, g, b, None)
        a.refused(lambda: a.lib.pdq_irls_dev(a.h, d2, b, g - 1, g, b, *irls), INVALID, "pdq_irls_dev: bad arguments")
        for alt in (-1, 5):
            a.refused(lambda: a.lib.pdq_irls_wald_dev(a.h, d2, b, g, g, b, *irls, as_f64p(ridge), as_f64p(contrast), 0.0, alt, b, b, b),
                      INVALID, "pdq_irls_wald_dev: bad arguments")
            a.refused(lambda: a.lib.pdq_wald_test_dev(a.h, d2, b, b, b, g, g, as_f64p(ridge), as_f64p(contrast), 0.0, alt, b, b, b),
                      INVALID, "pdq_wald_test_dev: bad arguments")
        # dispersion searches
        mle = (b, g, b, 1e-8, 10.0, 0.0, None, 1, 1, b, b)
        a.refused(lambda: a.lib.pdq_alpha_mle_dev(a.h, d2, b, g, g, *mle), INVALID, "alpha_mle: prior_reg needs prior_disp_var > 0")
        a.refused(lambda: a.lib.pdq_alpha_mle_hint_dev(a.h, d2, b, g, g, *mle, b, b), INVALID,
                  "alpha_mle: prior_reg needs prior_disp_var > 0")
        a.refused(lambda: a.lib.pdq_alpha_mle_dev(a.h, d2, b, g, g, b, g - 1, *mle[2:]), INVALID, "pdq_alpha_mle_dev: bad arguments")
        tail = (b, g, b, b, b, b, 1e-8, 10.0)
        fit = (0.5, 1e-8, -30.0, 30.0, 250, b, b, b, g, b, as_f64p(ridge), as_f64p(contrast), 0.0)
        a.refused(lambda: a.lib.pdq_map_irls_wald_dev(a.h, d2, b, g, g, *tail, 1.0, None, b, b, b, b, *fit, 5, b, b, b), INVALID,
                  "pdq_map_irls_wald_dev: bad arguments")
        a.refused(lambda: a.lib.pdq_map_irls_wald_dev(a.h, d2, b, g, g, *tail, 0.0, None, b, b, b, b, *fit, 0, b, b, b), INVALID,
                  "pdq_map_irls_wald_dev: needs prior_disp_var > 0")
        a.refused(lambda: a.lib.pdq_mom_dispersions_dev(a.h, dsq, b, g, g, 1e-8, 10.0, b, b, 0.5, None, 0), INVALID, SQUARE)
        a.refused(lambda: a.lib.pdq_mom_alpha_mle_dev(a.h, dsq, b, g, g, 1e-8, 10.0, 0.5, b, b, b, g, b, b, None), INVALID, SQUARE)
        # apeGLM shrinkage: a bad shrink_index or scale is a bad argument, and wins over the opt-ins
        for kw in ({"shrink_index": 2}, {"shrink_index": -1}, {"scale": 0.0}, {"scale": float("nan")}):
            a.refused(lambda: a.shrink_dev(d2, **kw), INVALID, "pdq_lfc_shrink_dev: bad arguments")
        a.refused(lambda: a.shrink_dev(d17, shrink_index=40), INVALID, "pdq_lfc_shrink_dev: bad arguments")
        a.refused(lambda: a.shrink_dev(d17, g=0), INVALID, "pdq_lfc_shrink_dev: bad arguments")
        # packs made with the opt-ins on, refused once they are off: the shrinkage opt-in first, then the width
        a.opt_in()
        a.refused(lambda: a.shrink_dev(d17), UNSUPPORTED, NI16)
        a.opt_in(wide_shrink=1)
        a.refused(lambda: a.shrink_dev(d17), UNSUPPORTED, narrow(17))
        a.opt_in(wide=1, large=1, large_shrink=1)
        a.refused(lambda: a.shrink_dev(d65), UNSUPPORTED, NI16)
        a.opt_in(wide=1, wide_shrink=1, large_shrink=1)
        a.refused(lambda: a.shrink_dev(d65), UNSUPPORTED, wide(65, 64))
        a.opt_in(wide=1, wide_shrink=1, large=1)
        a.refused(lambda: a.shrink_dev(d65), UNSUPPORTED, NI64)
        a.nothing_staged()
    finally:
        a.opt_in()
        for d in (d2, d17, d65, dsq):
            a.lib.pdq_design_destroy(a.h, d)
