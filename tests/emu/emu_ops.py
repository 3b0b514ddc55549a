"""ctypes front-end of the host emulator (tests/emu/pdq_emu.cpp) with the `_CudaOps` interface, so the
CPU suite can push the *device* algorithms through `B200Inference`'s marshalling.  Test infrastructure.

`trend_prior` is left out on purpose: without it `B200Inference.trend_and_prior` returns None, and the CPU pipeline tests fit the
dispersion trend through `trend_glm`, the path they check."""
import ctypes as C

import numpy as np

from . import build as _build

f64p = C.POINTER(C.c_double)
i64p = C.POINTER(C.c_int64)
i32p = C.POINTER(C.c_int)


def _p(a, t):
    return a.ctypes.data_as(t)


class EmuOps:
    def __init__(self, force_optimizer=False, force_grid=False, force_shrink_grid=False, lanes=1):
        self.lib = C.CDLL(_build.build())
        self.lib.emu_lgamma.restype = C.c_double
        self.lib.emu_lgamma.argtypes = [C.c_double]
        self.lib.emu_digamma.restype = C.c_double
        self.lib.emu_digamma.argtypes = [C.c_double]
        self.force_optimizer = int(force_optimizer)
        self.force_grid = int(force_grid)
        self.force_shrink_grid = int(force_shrink_grid)
        self.lanes = int(lanes)  # 2..32: one std::thread per lane of a gene, the device's exchange patterns (pdq_emu.cpp)
        self.last_status = None

    def empty(self, shape):
        return np.empty(shape, dtype=np.float64)

    def _lanes(self):
        """The library with this object's lane count selected: the count is a global of the library."""
        assert self.lib.emu_set_lanes(self.lanes) == 0
        return self.lib

    def lin_reg_mu(self, counts, ld, N, G, sf, X, p, min_mu, mu):
        rc = self._lanes().emu_lin_reg_mu(_p(counts, i64p), C.c_int64(ld), N, G, _p(sf, f64p), _p(X, f64p), p, C.c_double(min_mu),
                                          _p(mu, f64p))
        assert rc == 0

    def irls(self, counts, ld, N, G, sf, X, p, disp, min_mu, beta_tol, min_beta, max_beta, maxiter, beta, mu, hat, conv):
        status = np.zeros(G, dtype=np.int32)
        rc = self._lanes().emu_irls(_p(counts, i64p), C.c_int64(ld), N, G, _p(sf, f64p), _p(X, f64p), p, _p(disp, f64p),
                                    C.c_double(min_mu), C.c_double(beta_tol), C.c_double(min_beta), C.c_double(max_beta),
                                    maxiter, _p(beta, f64p), _p(mu, f64p), _p(hat, f64p), _p(conv, f64p), _p(status, i32p),
                                    self.force_optimizer)
        assert rc == 0
        self.last_status = status
        return int((status != 0).sum())

    def alpha_mle(self, counts, ld, N, G, X, p, mu, ld_mu, alpha_hat, min_disp, max_disp, prior_var, cr_reg, prior_reg,
                  alpha, conv):
        status = np.zeros(G, dtype=np.int32)
        rc = self._lanes().emu_alpha_mle(_p(counts, i64p), C.c_int64(ld), N, G, _p(X, f64p), p, _p(mu, f64p), C.c_int64(ld_mu),
                                         _p(alpha_hat, f64p), C.c_double(min_disp), C.c_double(max_disp), C.c_double(prior_var),
                                         cr_reg, prior_reg, _p(alpha, f64p), _p(conv, f64p), _p(status, i32p), self.force_grid)
        assert rc == 0
        self.last_status = status

    def wald_test(self, X, N, p, disp, lfc, mu, ld_mu, G, ridge, contrast, lfc_null, alt, pv, stat, se):
        rc = self._lanes().emu_wald_test(_p(X, f64p), N, p, _p(disp, f64p), _p(lfc, f64p), _p(mu, f64p), C.c_int64(ld_mu), G,
                                         _p(ridge, f64p), _p(contrast, f64p), C.c_double(lfc_null), alt, _p(pv, f64p),
                                         _p(stat, f64p), _p(se, f64p))
        assert rc == 0

    def rough(self, normed, ld, N, G, X, p, out):
        assert self._lanes().emu_rough(_p(normed, f64p), C.c_int64(ld), N, G, _p(X, f64p), p, _p(out, f64p)) == 0

    def moments(self, normed, ld, N, G, sf, out, all_zero):
        assert self._lanes().emu_moments(_p(normed, f64p), C.c_int64(ld), N, G, _p(sf, f64p), _p(out, f64p), _p(all_zero, f64p)) == 0

    def mom_from_counts(self, counts, sf, X, min_disp, max_disp):
        counts, sf, X = np.ascontiguousarray(counts), np.ascontiguousarray(sf), np.ascontiguousarray(X)
        N, G = counts.shape
        a = np.empty(G)
        m = np.empty(G)
        mu = np.empty((N, G))
        rc = self._lanes().emu_mom_from_counts(_p(counts, i64p), C.c_int64(G), N, G, _p(sf, f64p), _p(X, f64p), X.shape[1],
                                               C.c_double(min_disp), C.c_double(max_disp), _p(a, f64p), _p(m, f64p), C.c_double(0.5),
                                               _p(mu, f64p))
        assert rc == 0
        return a, m, mu

    def trend_glm(self, cov, targets):
        out = np.zeros(16)
        rc = self.lib.emu_trend_fit(_p(cov, f64p), _p(targets, f64p), C.c_size_t(len(cov)), 0, C.c_double(-np.inf),
                                    C.c_double(np.inf), 0, C.c_double(0.0), C.c_double(0.0), 0, _p(out, f64p))
        assert rc == 0
        return out[:2].copy(), out[0] + out[1] * cov, bool(out[7])

    def trend_outer(self, means, gw, lo, hi, min_disp=1e-8, trigamma_c=0.0, with_prior=True):
        out = np.zeros(16)
        assert self.lib.emu_trend_fit(_p(means, f64p), _p(gw, f64p), C.c_size_t(len(gw)), 1, C.c_double(lo), C.c_double(hi), 1,
                                      C.c_double(min_disp), C.c_double(trigamma_c), int(with_prior), _p(out, f64p)) == 0
        return out

    def lfc_shrink(self, X, counts, ld, N, G, p, size, offset, prior_no_shrink_scale, prior_scale, shrink_index, lfcs, inv_hessians,
                   conv):
        status = np.zeros(G, dtype=np.int32)
        rc = self._lanes().emu_lfc_shrink(_p(X, f64p), _p(counts, i64p), C.c_int64(ld), N, G, p, _p(size, f64p), _p(offset, f64p),
                                          C.c_double(prior_no_shrink_scale), C.c_double(prior_scale), shrink_index, _p(lfcs, f64p),
                                          _p(inv_hessians, f64p), _p(conv, f64p), _p(status, i32p), self.force_shrink_grid)
        assert rc == 0
        self.last_status = status
        return int((status != 0).sum())

    def size_factors(self, counts, ld, N, G, sf, logmeans=None):
        assert self.lib.emu_size_factors(_p(counts, i64p), C.c_int64(ld), N, G, _p(sf, f64p),
                                         None if logmeans is None else _p(logmeans, f64p)) == 0

    def size_factors_ex_rc(self, counts, ld, N, G, kind, control, sf, logmeans):
        """emu_size_factors_ex's status: 0, or -2 (PDQ_ERR_INVALID) for an unknown kind."""
        ctl = None if control is None else np.ascontiguousarray(control, dtype=np.uint8)
        return self.lib.emu_size_factors_ex(_p(counts, i64p), C.c_int64(ld), N, G, int(kind),
                                            None if ctl is None else C.c_void_p(ctl.ctypes.data), _p(sf, f64p), _p(logmeans, f64p))

    def size_factors_ex(self, counts, ld, N, G, kind, control, sf, logmeans):
        """pdq_size_factors_ex: `control` uint8 (G,) or None, `logmeans` (G,) receives the raw log means."""
        rc = self.size_factors_ex_rc(counts, ld, N, G, kind, control, sf, logmeans)
        assert rc == 0, rc

    def size_factors_from_logmeans(self, counts, ld, N, G, logmeans, sf):
        assert self.lib.emu_size_factors_from_logmeans(_p(counts, i64p), C.c_int64(ld), N, G, _p(logmeans, f64p), _p(sf, f64p)) == 0

    def vst_transform(self, counts, ld, N, G, sf, kind, c0, c1, out, ld_out):
        rc = self.lib.emu_vst_transform(_p(counts, i64p), C.c_int64(ld), N, G, _p(sf, f64p), kind, C.c_double(c0), C.c_double(c1),
                                        _p(out, f64p), C.c_int64(ld_out))
        assert rc == 0

    def wald_contrasts_rc(self, X, sf, N, p, disp, lfc, G, ridge, K, contrasts, lfc_null, alt, pv, stat, se, ld_out):
        """emu_wald_contrasts' status: 0, -2 (PDQ_ERR_INVALID) for K <= 0, an unknown alternative or ld_out < G, -3 for p > 16."""
        return self._lanes().emu_wald_contrasts(_p(X, f64p), _p(sf, f64p), N, p, _p(disp, f64p), _p(lfc, f64p), G, _p(ridge, f64p), K,
                                                _p(contrasts, f64p), _p(lfc_null, f64p), _p(alt, i32p), _p(pv, f64p), _p(stat, f64p),
                                                _p(se, f64p), C.c_int64(ld_out))

    def wald_contrasts(self, X, sf, N, p, disp, lfc, G, ridge, K, contrasts, lfc_null, alt, pv, stat, se, ld_out):
        rc = self.wald_contrasts_rc(X, sf, N, p, disp, lfc, G, ridge, K, contrasts, lfc_null, alt, pv, stat, se, ld_out)
        assert rc == 0, rc

    def elem(self, op, x, y=None):
        """The host branch of one primitive (op code of tests/gpu_probe/math_ops.h) applied elementwise."""
        x = np.ascontiguousarray(x, dtype=np.float64)
        y = np.zeros_like(x) if y is None else np.ascontiguousarray(np.broadcast_to(y, x.shape), dtype=np.float64)
        out = np.empty_like(x)
        assert self.lib.emu_math(int(op), _p(x, f64p), _p(y, f64p), _p(out, f64p), int(x.size)) == 0
        return out

    def tables(self, r, T):
        """[G][4 kPsiK]: lgamma, psi, then psi and psi' of build_psi_tri_tables at each r, built by T lane threads."""
        r = np.ascontiguousarray(r, dtype=np.float64)
        out = np.empty((r.size, 4 * 32))
        assert self.lib.emu_tables(_p(r, f64p), int(r.size), int(T), _p(out, f64p)) == 0
        return out

    def math_table(self):
        """(kMathTab as compiled into the emulator, {bits, n, split, exp_n})"""
        tab = np.empty(4096)
        layout = np.zeros(4, dtype=np.int32)
        n = self.lib.emu_math_table(_p(tab, f64p), _p(layout, i32p))
        return tab[:n].copy(), dict(zip(("bits", "n", "split", "exp_n"), (int(v) for v in layout)))

    def cooks(self, counts, ld, N, G, sf, X, p, mu, hat, ld2, cutoff, cooks, disp, outlier, replaced):
        assert self._lanes().emu_cooks(_p(counts, i64p), C.c_int64(ld), N, G, _p(sf, f64p), _p(X, f64p), p, _p(mu, f64p), _p(hat, f64p),
                                       C.c_int64(ld2), C.c_double(cutoff), _p(cooks, f64p) if cooks is not None else None,
                                       _p(disp, f64p), _p(outlier, f64p), _p(replaced, f64p)) == 0

    def cooks_cols(self, counts, ld, N, G, sf, X, p, mu, hat, ld2, cutoff, cooks, disp, outlier, replaced):
        """`cooks` with the design width at run time (emu_cooks_cols): the routine k_wide_cooks runs, for any p."""
        assert self._lanes().emu_cooks_cols(_p(counts, i64p), C.c_int64(ld), N, G, _p(sf, f64p), _p(X, f64p), p, _p(mu, f64p),
                                            _p(hat, f64p), C.c_int64(ld2), C.c_double(cutoff),
                                            _p(cooks, f64p) if cooks is not None else None, _p(disp, f64p), _p(outlier, f64p),
                                            _p(replaced, f64p)) == 0
