"""``B200Inference`` -- drop-in ``pydeseq2.inference.Inference`` backend running on one H100.

The class mirrors the reference's plugin interface (``pydeseq2/inference.py:9-362``,
default implementation ``default_inference.py:14-264``): same method names, argument meaning and
return conventions, so ``DeseqDataSet(..., inference=B200Inference())`` and
``DeseqStats(..., inference=B200Inference())`` work unchanged.  Every per-gene method is one call
through the C ABI (``include/pydeseq2_b200.h``) into hand-written sm_90a kernels batched over all
genes; host code here only marshals numpy buffers.

Deliberate differences from ``DefaultInference`` (all documented in DESIGN.md):

* ``converged`` flags are float64 0/1 (the caller stores them in a float column; a bool array
  raises under pandas >= 3, ``dds.py:796-797``).
* ``mu``/``H`` come back C-contiguous (N, G); the reference returns ``.T`` views of (G, N) arrays.
* the dispersion optimum is located by a bounded root search on the analytic derivative instead of
  scipy's L-BFGS-B, so a gene for which L-BFGS-B reports ``ABNORMAL`` and the reference substitutes
  its grid value (``utils.py:556-564``) is returned at the true optimum with ``converged = 1``.
* ``lfc_shrink_nbinom_glm`` (apeGLM, ``DeseqStats.lfc_shrink``) runs the reference's own L-BFGS-B iteration per gene.
"""
from __future__ import annotations

import ctypes as C
from abc import ABC, abstractmethod

import numpy as np

from . import _lib
from ._lib import ALT_CODES, B200Error, as_f64p, as_i64p

VST_KINDS = {"parametric": 0, "mean": 1}  # `kind` of pdq_vst_transform
SF_KINDS = {"ratio": 0, "poscounts": 1}  # `kind` of pdq_size_factors_ex


def control_mask(control_genes, G):
    """Boolean (G,) mask of control genes (DESeq2's ``controlGenes``, dds.py:628-651) from a boolean mask of length G or integer
    positions; None stays None (every gene).  Gene names are resolved by the caller (``DeseqDataSet._normalize_indices``)."""
    if control_genes is None:
        return None
    c = np.asarray(control_genes.values if hasattr(control_genes, "values") else control_genes)
    if c.dtype == bool:
        if c.shape != (G,):
            raise ValueError(f"control_genes is a mask of shape {c.shape} for {G} genes")
        return c.copy()
    if c.ndim != 1 or (c.size and c.dtype.kind not in "iu"):
        raise ValueError("control_genes must be a boolean mask or integer gene positions")
    mask = np.zeros(G, dtype=bool)
    try:
        mask[c.astype(np.int64)] = True
    except IndexError as e:
        raise ValueError(f"control_genes: {e}") from None
    return mask

try:  # the reference, when it is importable, provides the ABC we plug into
    from pydeseq2.inference import Inference as _InferenceBase  # type: ignore
except Exception:  # pragma: no cover - pydeseq2 is not installed

    class _InferenceBase(ABC):
        """Structural mirror of ``pydeseq2.inference.Inference`` (inference.py:9-362)."""

        @abstractmethod
        def lin_reg_mu(self, counts, size_factors, design_matrix, min_mu): ...

        @abstractmethod
        def irls(self, counts, size_factors, design_matrix, disp, min_mu, beta_tol, min_beta=-30, max_beta=30,
                 optimizer="L-BFGS-B", maxiter=250): ...

        @abstractmethod
        def alpha_mle(self, counts, design_matrix, mu, alpha_hat, min_disp, max_disp, prior_disp_var=None,
                      cr_reg=True, prior_reg=False, optimizer="L-BFGS-B"): ...

        @abstractmethod
        def wald_test(self, design_matrix, disp, lfc, mu, ridge_factor, contrast, lfc_null, alt_hypothesis=None): ...

        @abstractmethod
        def fit_rough_dispersions(self, normed_counts, design_matrix): ...

        @abstractmethod
        def fit_moments_dispersions(self, normed_counts, size_factors): ...

        @abstractmethod
        def dispersion_trend_gamma_glm(self, covariates, targets): ...

        @abstractmethod
        def lfc_shrink_nbinom_glm(self, design_matrix, counts, size, offset, prior_no_shrink_scale, prior_scale,
                                  optimizer, shrink_index): ...


def _f64(a, name, ndim=None):
    a = np.asarray(a.values if hasattr(a, "values") else a)
    if a.dtype != np.float64:
        a = a.astype(np.float64)
    if ndim is not None and a.ndim != ndim:
        raise ValueError(f"{name} must be {ndim}-dimensional, got shape {a.shape}")
    return a


def _rows(a, dtype, name):
    """(N, G) array with unit stride along genes; returns (array, row pitch in elements)."""
    a = np.asarray(a.values if hasattr(a, "values") else a)
    if a.ndim != 2:
        raise ValueError(f"{name} must be (samples, genes), got shape {a.shape}")
    if a.dtype != dtype:
        if dtype == np.int64 and a.dtype.kind == "f" and not np.all(np.isfinite(a)):
            raise ValueError(f"{name} contains NaN/inf")
        a = a.astype(dtype)
    item = a.dtype.itemsize
    if a.shape[1] > 1 and a.strides[1] != item or a.strides[0] % item or a.strides[0] < a.shape[1] * item:
        a = np.ascontiguousarray(a)
    return a, (a.strides[0] // item if a.shape[0] > 1 else a.shape[1])


class _CudaOps:
    """Raw ops on numpy buffers through the C ABI (host-buffer entry points)."""

    def __init__(self, device=0, lanes_per_gene=0, pinned_outputs=True):
        self.ctx = _lib.Context(device)
        self.lib = self.ctx.lib
        self.pinned_outputs = pinned_outputs
        self.h2d_bytes = 0  # bytes the calls below asked the library to copy in / out (bench.py `e2e`)
        self.d2h_bytes = 0
        if lanes_per_gene:
            self.ctx.check(self.lib.pdq_set_lanes_per_gene(self.ctx.h, int(lanes_per_gene)))

    def empty(self, shape):
        # large outputs land in recycled page-locked blocks: the D2H copy then runs at full PCIe rate
        if self.pinned_outputs and int(np.prod(shape)) >= (1 << 16):
            return self.ctx.pinned_empty(shape)
        return np.empty(shape, dtype=np.float64)

    def _io(self, ins, outs):
        self.h2d_bytes += sum(a.nbytes for a in ins)
        self.d2h_bytes += sum(a.nbytes for a in outs)

    def lin_reg_mu(self, counts, ld, N, G, sf, X, p, min_mu, mu):
        self._io((counts, sf, X), (mu,))
        self.ctx.check(self.lib.pdq_lin_reg_mu(self.ctx.h, as_i64p(counts), ld, N, G, as_f64p(sf), as_f64p(X), p, min_mu,
                                               as_f64p(mu)))

    def irls(self, counts, ld, N, G, sf, X, p, disp, min_mu, beta_tol, min_beta, max_beta, maxiter, beta, mu, hat, conv):
        nfb = C.c_int(0)
        self._io((counts, sf, X, disp), (beta, mu, hat, conv))
        self.ctx.check(self.lib.pdq_irls(self.ctx.h, as_i64p(counts), ld, N, G, as_f64p(sf), as_f64p(X), p, as_f64p(disp),
                                         min_mu, beta_tol, min_beta, max_beta, maxiter, as_f64p(beta), as_f64p(mu),
                                         as_f64p(hat), as_f64p(conv), C.byref(nfb)))
        return nfb.value

    def alpha_mle(self, counts, ld, N, G, X, p, mu, ld_mu, alpha_hat, min_disp, max_disp, prior_var, cr_reg, prior_reg,
                  alpha, conv):
        self._io((counts, mu, X, alpha_hat), (alpha, conv))
        self.ctx.check(self.lib.pdq_alpha_mle(self.ctx.h, as_i64p(counts), ld, N, G, as_f64p(X), p, as_f64p(mu), ld_mu,
                                              as_f64p(alpha_hat), min_disp, max_disp, prior_var, cr_reg, prior_reg,
                                              as_f64p(alpha), as_f64p(conv)))

    def wald_test(self, X, N, p, disp, lfc, mu, ld_mu, G, ridge, contrast, lfc_null, alt, pv, stat, se):
        self._io((X, disp, lfc, mu), (pv, stat, se))
        self.ctx.check(self.lib.pdq_wald_test(self.ctx.h, as_f64p(X), N, p, as_f64p(disp), as_f64p(lfc), as_f64p(mu), ld_mu,
                                              G, as_f64p(ridge), as_f64p(contrast), lfc_null, alt, as_f64p(pv),
                                              as_f64p(stat), as_f64p(se)))

    def wald_contrasts(self, X, sf, N, p, disp, lfc, G, ridge, K, contrasts, lfc_null, alt, pv, stat, se, ld_out):
        """pdq_wald_contrasts: `alt` int32 (K,), outputs (K, ld_out)."""
        self._io((X, sf, disp, lfc, contrasts), (pv, stat, se))
        self.ctx.check(self.lib.pdq_wald_contrasts(self.ctx.h, as_f64p(X), as_f64p(sf), N, p, as_f64p(disp), as_f64p(lfc), G,
                                                   as_f64p(ridge), K, as_f64p(contrasts), as_f64p(lfc_null),
                                                   alt.ctypes.data_as(C.POINTER(C.c_int)), as_f64p(pv), as_f64p(stat), as_f64p(se),
                                                   ld_out))

    def rough(self, normed, ld, N, G, X, p, out):
        self._io((normed, X), (out,))
        self.ctx.check(self.lib.pdq_fit_rough_dispersions(self.ctx.h, as_f64p(normed), ld, N, G, as_f64p(X), p, as_f64p(out)))

    def moments(self, normed, ld, N, G, sf, out, all_zero):
        self._io((normed, sf), (out, all_zero))
        self.ctx.check(self.lib.pdq_fit_moments_dispersions(self.ctx.h, as_f64p(normed), ld, N, G, as_f64p(sf), as_f64p(out),
                                                            as_f64p(all_zero)))


    def cooks(self, counts, ld, N, G, sf, X, p, mu, hat, ld2, cutoff, cooks, disp, outlier, replaced):
        self._io((counts, mu, hat), (disp, outlier, replaced) + ((cooks,) if cooks is not None else ()))
        self.ctx.check(self.lib.pdq_calculate_cooks(self.ctx.h, as_i64p(counts), ld, N, G, as_f64p(sf), as_f64p(X), p, as_f64p(mu),
                                                    as_f64p(hat), ld2, cutoff, as_f64p(cooks) if cooks is not None else None,
                                                    as_f64p(disp), as_f64p(outlier), as_f64p(replaced)))

    def size_factors(self, counts, ld, N, G, sf, logmeans=None):
        self._io((counts,), (sf,))
        self.ctx.check(self.lib.pdq_size_factors(self.ctx.h, as_i64p(counts), ld, N, G, as_f64p(sf),
                                                 as_f64p(logmeans) if logmeans is not None else None))

    def size_factors_ex(self, counts, ld, N, G, kind, control, sf, logmeans):
        self._io((counts,) + ((control,) if control is not None else ()), (sf, logmeans))
        self.ctx.check(self.lib.pdq_size_factors_ex(self.ctx.h, as_i64p(counts), ld, N, G, kind,
                                                    control.ctypes.data if control is not None else None, as_f64p(sf), as_f64p(logmeans)))

    def size_factors_from_logmeans(self, counts, ld, N, G, logmeans, sf):
        self._io((counts, logmeans), (sf,))
        self.ctx.check(self.lib.pdq_size_factors_from_logmeans(self.ctx.h, as_i64p(counts), ld, N, G, as_f64p(logmeans), as_f64p(sf)))

    def vst_transform(self, counts, ld, N, G, sf, kind, c0, c1, out, ld_out):
        self._io((counts, sf), (out,))
        self.ctx.check(self.lib.pdq_vst_transform(self.ctx.h, as_i64p(counts), ld, N, G, as_f64p(sf), kind, c0, c1, as_f64p(out),
                                                  ld_out))

    def lfc_shrink(self, X, counts, ld, N, G, p, size, offset, prior_no_shrink_scale, prior_scale, shrink_index, lfcs, inv_hessians,
                   conv):
        n_grid = C.c_int(0)
        self._io((counts,), (lfcs, inv_hessians, conv))
        self.ctx.check(self.lib.pdq_lfc_shrink_nbinom_glm(self.ctx.h, as_f64p(X), as_i64p(counts), ld, N, G, p, as_f64p(size),
                                                          as_f64p(offset), prior_no_shrink_scale, prior_scale, shrink_index,
                                                          as_f64p(lfcs), as_f64p(inv_hessians), as_f64p(conv), C.byref(n_grid)))
        return n_grid.value

    def trend_glm(self, cov, targets):
        n = len(cov)
        coeffs = np.empty(2)
        pred = np.empty(n)
        ok = C.c_int(0)
        self._io((cov, targets), (coeffs,))
        self.ctx.check(self.lib.pdq_dispersion_trend_gamma_glm(self.ctx.h, as_f64p(cov), as_f64p(targets), n, as_f64p(coeffs),
                                                               as_f64p(pred), C.byref(ok)))
        return coeffs, pred, bool(ok.value)


    def trend_prior(self, means, genewise, min_disp, max_disp, trigamma_c):
        n = len(means)
        out16, fitted = np.empty(16), np.empty(n)
        self._io((means, genewise), (out16, fitted))
        self.ctx.check(self.lib.pdq_trend_prior(self.ctx.h, as_f64p(means), as_f64p(genewise), n, min_disp, max_disp, trigamma_c,
                                                as_f64p(out16), as_f64p(fitted)))
        return out16, fitted


class B200Inference(_InferenceBase):
    """CUDA (H100) implementation of the reference's ``Inference`` plugin API.

    Parameters
    ----------
    device : int
        CUDA device ordinal (one backend object per GPU; gene shards across GPUs are handled by
        ``pydeseq2_b200.sharding``).
    n_cpus : int, optional
        Accepted and stored because ``DeseqDataSet``/``DeseqStats`` set it on the backend
        (``dds.py:323-333``, ``ds.py:194-204``); it has no effect on the GPU path.
    lanes_per_gene : int
        0 (default) picks the lanes cooperating on one gene from the number of genes.
    trace : bool
        Record every plugin call in ``self.trace`` (method, milliseconds, bytes requested host→device / device→host).
    """

    _TRACED = ("lin_reg_mu", "irls", "alpha_mle", "wald_test", "wald_tests", "fit_rough_dispersions", "fit_moments_dispersions",
               "dispersion_trend_gamma_glm", "lfc_shrink_nbinom_glm", "size_factors", "calculate_cooks")

    def __init__(self, device: int = 0, n_cpus: int | None = None, lanes_per_gene: int = 0, _ops=None, trace: bool = False,
                 pinned_outputs: bool = True):
        # pinned_outputs: large results are returned in page-locked numpy blocks (full-rate device-to-host copies, and full-rate
        # uploads when the caller hands them back); False returns ordinary pageable arrays
        self._ops = _ops if _ops is not None else _CudaOps(device, lanes_per_gene, pinned_outputs)
        self._n_cpus = n_cpus or 1
        self.last_irls_fallbacks = 0
        # per-call tracing (the reference prints wall-clock per phase to stderr, dds.py:626-711 ...; a backend is better served by
        # a record it can be asked for): one dict per plugin call -- method, milliseconds, bytes requested in / out
        self.trace = [] if trace else None
        if trace:
            for name in self._TRACED:
                setattr(self, name, self._traced(name, getattr(self, name)))

    def _traced(self, name, fn):
        import functools
        import time

        @functools.wraps(fn)
        def call(*a, **k):
            ops = self._ops
            h0, d0 = getattr(ops, "h2d_bytes", 0), getattr(ops, "d2h_bytes", 0)
            t0 = time.perf_counter()
            out = fn(*a, **k)
            self.trace.append({"method": name, "ms": (time.perf_counter() - t0) * 1e3,
                               "h2d_bytes": getattr(ops, "h2d_bytes", 0) - h0, "d2h_bytes": getattr(ops, "d2h_bytes", 0) - d0})
            return out

        return call

    @property
    def n_cpus(self) -> int:  # noqa: D102
        return self._n_cpus

    @n_cpus.setter
    def n_cpus(self, n_cpus: int) -> None:
        self._n_cpus = n_cpus or 1

    # ------------------------------------------------------------------ a4: inference.py:12-43
    def lin_reg_mu(self, counts, size_factors, design_matrix, min_mu):  # noqa: D102
        counts, ld = _rows(counts, np.int64, "counts")
        X = np.ascontiguousarray(_f64(design_matrix, "design_matrix", 2))
        sf = np.ascontiguousarray(_f64(size_factors, "size_factors", 1))
        N, G = counts.shape
        self._check_design(X, N, sf)
        mu = self._ops.empty((N, G))
        if G:
            self._ops.lin_reg_mu(counts, ld, N, G, sf, X, X.shape[1], float(min_mu), mu)
        return mu

    # ------------------------------------------------------------------ a1: inference.py:45-118
    def irls(self, counts, size_factors, design_matrix, disp, min_mu, beta_tol, min_beta=-30, max_beta=30,
             optimizer="L-BFGS-B", maxiter=250):  # noqa: D102
        assert optimizer in ["BFGS", "L-BFGS-B"]  # utils.py:343 (the device optimiser honours the bounds)
        counts, ld = _rows(counts, np.int64, "counts")
        X = np.ascontiguousarray(_f64(design_matrix, "design_matrix", 2))
        sf = np.ascontiguousarray(_f64(size_factors, "size_factors", 1))
        disp = np.ascontiguousarray(_f64(disp, "disp", 1))
        N, G = counts.shape
        p = X.shape[1]
        self._check_design(X, N, sf)
        if disp.shape[0] != G:
            raise ValueError(f"disp has {disp.shape[0]} entries for {G} genes")
        beta = self._ops.empty((G, p))
        mu = self._ops.empty((N, G))
        hat = self._ops.empty((N, G))
        conv = self._ops.empty((G,))
        if G:
            self.last_irls_fallbacks = self._ops.irls(counts, ld, N, G, sf, X, p, disp, float(min_mu), float(beta_tol),
                                                      float(min_beta), float(max_beta), int(maxiter), beta, mu, hat, conv)
        return beta, mu, hat, conv

    # ------------------------------------------------------------------ a2: inference.py:120-177
    def alpha_mle(self, counts, design_matrix, mu, alpha_hat, min_disp, max_disp, prior_disp_var=None, cr_reg=True,
                  prior_reg=False, optimizer="L-BFGS-B"):  # noqa: D102
        assert optimizer in ["BFGS", "L-BFGS-B"]  # utils.py:499
        if prior_reg and prior_disp_var is None:
            raise ValueError("Sigma_prior is required for prior regularization")  # utils.py:518
        counts, ld = _rows(counts, np.int64, "counts")
        mu, ld_mu = _rows(mu, np.float64, "mu")
        X = np.ascontiguousarray(_f64(design_matrix, "design_matrix", 2))
        alpha_hat = np.ascontiguousarray(_f64(alpha_hat, "alpha_hat", 1))
        N, G = counts.shape
        self._check_design(X, N)
        if mu.shape != (N, G) or alpha_hat.shape[0] != G:
            raise ValueError("counts, mu and alpha_hat disagree on the number of samples/genes")
        alpha = self._ops.empty((G,))
        conv = self._ops.empty((G,))
        if G:
            self._ops.alpha_mle(counts, ld, N, G, X, X.shape[1], mu, ld_mu, alpha_hat, float(min_disp), float(max_disp),
                                float(prior_disp_var) if prior_disp_var is not None else 1.0, int(bool(cr_reg)),
                                int(bool(prior_reg)), alpha, conv)
        return alpha, conv

    # ------------------------------------------------------------------ a3: inference.py:179-234
    def wald_test(self, design_matrix, disp, lfc, mu, ridge_factor, contrast, lfc_null, alt_hypothesis=None):  # noqa: D102
        if alt_hypothesis not in ALT_CODES:
            raise KeyError(alt_hypothesis)  # same failure mode as the dict lookup at utils.py:798-803
        X = np.ascontiguousarray(_f64(design_matrix, "design_matrix", 2))
        mu, ld_mu = _rows(mu, np.float64, "mu")
        disp = np.ascontiguousarray(_f64(disp, "disp", 1))
        lfc = np.ascontiguousarray(_f64(lfc, "lfc", 2))
        ridge = np.ascontiguousarray(_f64(ridge_factor, "ridge_factor", 2))
        contrast = np.ascontiguousarray(_f64(contrast, "contrast", 1))
        N, G = mu.shape
        p = X.shape[1]
        self._check_design(X, N)
        if lfc.shape != (G, p) or disp.shape[0] != G or ridge.shape != (p, p) or contrast.shape[0] != p:
            raise ValueError("wald_test arguments disagree on the number of genes/coefficients")
        pv = self._ops.empty((G,))
        stat = self._ops.empty((G,))
        se = self._ops.empty((G,))
        if G:
            self._ops.wald_test(X, N, p, disp, lfc, mu, ld_mu, G, ridge, contrast, float(np.asarray(lfc_null)),
                                ALT_CODES[alt_hypothesis], pv, stat, se)
        return pv, stat, se

    def wald_tests(self, design_matrix, size_factors, disp, lfc, contrasts, ridge_factor=None, lfc_null=0.0, alt_hypothesis=None):
        """Wald tests of K contrasts on one fit -- ``DeseqStats.run_wald_test`` (ds.py:303-360) once per contrast -- in one call.
        mu = size_factors * exp(X lfc) is built on the device, so only the coefficients and dispersions travel, and X^T W X is
        factored once per gene.  ``contrasts`` (K, p), or (p,) for one contrast; ``lfc_null`` (natural log, as for
        :meth:`wald_test`) and ``alt_hypothesis`` are scalars or length-K sequences; ``ridge_factor`` defaults to diag(1e-6).
        Returns (pvalue, stat, se), each (K, G), or (G,) for a 1-D contrast.  Genes whose LFC row or dispersion is not finite are
        not sent: their outputs are NaN, as NaN propagates through the reference's mu."""
        X = np.ascontiguousarray(_f64(design_matrix, "design_matrix", 2))
        sf = np.ascontiguousarray(_f64(size_factors, "size_factors", 1))
        disp = np.ascontiguousarray(_f64(disp, "disp", 1))
        lfc = np.ascontiguousarray(_f64(lfc, "lfc", 2))
        cs = _f64(contrasts, "contrasts")
        single = cs.ndim == 1
        cs = np.ascontiguousarray(cs[None, :] if single else cs)
        N, p = X.shape
        G = lfc.shape[0]
        self._check_design(X, N, sf)
        if cs.ndim != 2 or cs.shape[1] != p or cs.shape[0] == 0:
            raise ValueError(f"contrasts must be (K, {p}) or ({p},), got shape {np.shape(contrasts)}")
        K = cs.shape[0]
        if lfc.shape != (G, p) or disp.shape != (G,):
            raise ValueError("wald_tests arguments disagree on the number of genes/coefficients")
        ridge = np.diag(np.repeat(1e-6, p)) if ridge_factor is None else np.ascontiguousarray(_f64(ridge_factor, "ridge_factor", 2))
        if ridge.shape != (p, p):
            raise ValueError(f"ridge_factor must be ({p}, {p}), got shape {ridge.shape}")
        alts = list(alt_hypothesis) if isinstance(alt_hypothesis, (list, tuple, np.ndarray)) else [alt_hypothesis] * K
        nulls = np.asarray(lfc_null, dtype=np.float64)
        if len(alts) != K or nulls.ndim > 1 or (nulls.ndim == 1 and nulls.shape[0] != K):
            raise ValueError(f"lfc_null and alt_hypothesis must be scalars or have one entry per contrast ({K})")
        for a in alts:
            if a not in ALT_CODES:
                raise KeyError(a)  # same failure mode as the dict lookup at utils.py:798-803
        codes = np.array([ALT_CODES[a] for a in alts], dtype=np.int32)
        nulls = np.ascontiguousarray(np.broadcast_to(nulls, (K,)))
        ok = np.isfinite(disp) & np.isfinite(lfc).all(axis=1)
        idx = None if ok.all() else np.flatnonzero(ok)
        if idx is not None:
            disp, lfc = np.ascontiguousarray(disp[idx]), np.ascontiguousarray(lfc[idx])
        Gs = disp.shape[0]
        outs = [self._ops.empty((K, Gs)) for _ in range(3)]
        if Gs:
            self._ops.wald_contrasts(X, sf, N, p, disp, lfc, Gs, ridge, K, cs, nulls, codes, *outs, Gs)
        if idx is not None:
            full = [np.full((K, G), np.nan) for _ in range(3)]
            for f, o in zip(full, outs):
                f[:, idx] = o
            outs = full
        return tuple(o[0] for o in outs) if single else tuple(outs)

    # ------------------------------------------------------------------ a5: inference.py:236-281
    def fit_rough_dispersions(self, normed_counts, design_matrix):  # noqa: D102
        normed, ld = _rows(normed_counts, np.float64, "normed_counts")
        X = np.ascontiguousarray(_f64(design_matrix, "design_matrix", 2))
        N, G = normed.shape
        if N == X.shape[1]:  # utils.py:839-844, relied on by the reference's tests/test_edge_cases.py:141-158
            raise ValueError(
                "The number of samples and the number of design variables are "
                "equal, i.e., there are no replicates to estimate the "
                "dispersion. Please use a design with fewer variables."
            )
        self._check_design(X, N)
        out = self._ops.empty((G,))
        if G:
            self._ops.rough(normed, ld, N, G, X, X.shape[1], out)
        return out

    def fit_moments_dispersions(self, normed_counts, size_factors):  # noqa: D102
        normed, ld = _rows(normed_counts, np.float64, "normed_counts")
        sf = np.ascontiguousarray(_f64(size_factors, "size_factors", 1))
        N, G = normed.shape
        out = self._ops.empty((G,))
        all_zero = self._ops.empty((G,))
        if G:
            self._ops.moments(normed, ld, N, G, sf, out, all_zero)
        return out[all_zero == 0.0]  # the reference drops all-zero columns (utils.py:878)

    # ------------------------------------------------------------------ global (not per gene): host
    def dispersion_trend_gamma_glm(self, covariates, targets):  # noqa: D102
        """Gamma-GLM trend ``alpha ~ a0 + a1 * covariate`` (inference.py:283-307, default_inference.py:200-230).

        The whole fit (every iteration) runs in one kernel launch of one cooperative block: Fisher scoring /
        Newton with backtracking on the reference's loss ``mean(t/m + log m)`` under the reference's bounds.
        It converges to the minimiser; the reference's L-BFGS-B stops within ~4e-6 of it (DESIGN.md §6).
        """
        cov = np.ascontiguousarray(_f64(covariates, "covariates", 1))
        tgt = np.ascontiguousarray(_f64(targets, "targets", 1))
        if cov.shape != tgt.shape:
            raise ValueError("covariates and targets must have the same length")
        coeffs, pred, ok = self._ops.trend_glm(cov, tgt)
        return coeffs, pred, ok

    # ------------------------------------------------------------------ beyond the ABC
    def trend_and_prior(self, normed_means, genewise, min_disp, max_disp, n_samples, n_coeffs):
        """``fit_dispersion_trend`` (parametric, dds.py:1199-1275) and ``fit_dispersion_prior`` (dds.py:840-884) in ONE kernel
        launch on the gene-length vectors, instead of one plugin call per round of the orchestrator's outlier loop plus numpy
        medians.  Returns ``(coeffs (2,), fitted (G,), squared_logres, prior_var, n_rounds)`` or ``None`` when the parametric
        fit fails (the caller then falls back to the mean trend exactly like the orchestrator, dds.py:1243-1252) or the
        backend cannot run it."""
        if not hasattr(self._ops, "trend_prior"):
            return None
        from scipy.special import polygamma

        means = np.ascontiguousarray(_f64(normed_means, "normed_means", 1))
        gw = np.ascontiguousarray(_f64(genewise, "genewise", 1))
        if means.shape != gw.shape or not len(means):
            raise ValueError("normed_means and genewise must be non-empty vectors of the same length")
        out16, fitted = self._ops.trend_prior(means, gw, float(min_disp), float(max_disp),
                                              float(polygamma(1, (n_samples - n_coeffs) / 2)))
        if out16[2] != 0.0:
            return None
        return np.array([out16[0], out16[1]]), fitted, float(out16[8]), float(out16[9]), int(out16[3])

    def size_factors(self, counts, return_logmeans: bool = False, logmeans=None, fit_type: str = "ratio", control_genes=None):
        """Median-of-ratios size factors on the device (``preprocessing.deseq2_norm``, preprocessing.py:5-102).

        Not part of the ``Inference`` ABC -- the reference computes them in the orchestrator (``dds.py:584-711``) --
        but it is the step that precedes the plugin calls.  Returns ``(normed_counts, size_factors)`` like
        ``deseq2_norm``; raises ``ValueError`` when every gene contains a zero (the reference's cue to switch to its
        iterative estimator, ``dds.py:682-690``).

        ``fit_type="poscounts"`` fits DESeq2's poscounts estimator instead (dds.py:656-679): log means over all samples with zeros
        taken as log 1, medians over the genes with a log mean > 0 and over each sample's positive counts only, scaled to a
        geometric mean of 1.  It never raises: a sample without a usable gene makes every size factor NaN, as in numpy.
        ``control_genes`` (boolean mask of length G, or integer positions): take the medians over these genes only (DESeq2's
        ``controlGenes``, dds.py:628-651), for either fit type.  The log means returned are not masked by them; with ``"ratio"``,
        a control set without a finite log mean gives NaN size factors, and a table in which every gene holds a zero still raises.

        ``logmeans`` (G,): normalise NEW counts against the log means of an earlier fit instead
        (``deseq2_norm_transform``, preprocessing.py:59-102, with ``filtered_genes`` = the finite entries; pass -inf for a gene
        to leave out).  This is how held-out samples are normalised (dds.py:478-486): a zero count in a kept gene counts as a
        log ratio of -inf, so a sample can get size factor 0 (and infinite / NaN normalised counts), exactly as in numpy; nothing
        is raised.
        """
        if fit_type not in SF_KINDS:
            raise ValueError(f"fit_type must be one of {sorted(SF_KINDS)} on the device, got {fit_type!r}")
        if logmeans is not None and (fit_type != "ratio" or control_genes is not None):
            raise ValueError("logmeans= normalises held-out counts; it takes no fit_type or control_genes")
        counts, ld = _rows(counts, np.int64, "counts")
        N, G = counts.shape
        ctl = control_mask(control_genes, G)
        if fit_type != "ratio" or ctl is not None:
            sf, lm = np.empty(N), np.empty(G)
            self._ops.size_factors_ex(counts, ld, N, G, SF_KINDS[fit_type], None if ctl is None else ctl.astype(np.uint8), sf, lm)
            if fit_type == "ratio" and np.isinf(lm).all():
                raise ValueError("Every gene contains at least one zero, cannot compute log geometric means.")
            with np.errstate(invalid="ignore"):
                normed = counts / sf[:, None]
            return (normed, sf, lm) if return_logmeans else (normed, sf)
        if logmeans is not None:
            lm = np.ascontiguousarray(_f64(logmeans, "logmeans", 1))
            if lm.shape[0] != G:
                raise ValueError(f"logmeans has {lm.shape[0]} entries for {G} genes")
            sf = np.empty(N)
            self._ops.size_factors_from_logmeans(counts, ld, N, G, lm, sf)
            with np.errstate(divide="ignore", invalid="ignore"):
                return counts / sf[:, None], sf
        sf = np.empty(N)
        logmeans = np.empty(G) if return_logmeans else None  # what deseq2_norm_fit returns (preprocessing.py:31-59)
        self._ops.size_factors(counts, ld, N, G, sf, logmeans)
        if not np.isfinite(sf).all():
            raise ValueError("Every gene contains at least one zero, cannot compute log geometric means.")
        if return_logmeans:
            return counts / sf[:, None], sf, logmeans
        return counts / sf[:, None], sf

    def vst_transform(self, counts, size_factors, kind, coeffs):
        """Variance-stabilised counts (``DeseqDataSet.vst_transform``, dds.py:438-514) from RAW counts and size factors, one
        elementwise kernel: ``q = counts / size_factors`` (a true division, the reference's ``normed_counts`` bit for bit), then
        the parametric closed form with ``coeffs = (a0, a1)`` (``uns["vst_trend_coeffs"]``) or, for ``kind="mean"``, the asinh
        form with ``coeffs = mean_disp`` (dds.py:503-505).  Returns (N, G) float64."""
        if kind not in VST_KINDS:
            raise NotImplementedError(f"Found fit_type '{kind}'. Expected 'parametric' or 'mean'.")  # dds.py:511-514
        counts, ld = _rows(counts, np.int64, "counts")
        sf = np.ascontiguousarray(_f64(size_factors, "size_factors", 1))
        N, G = counts.shape
        if sf.shape[0] != N:
            raise ValueError(f"size_factors has {sf.shape[0]} entries for {N} samples")
        c = np.ravel(np.asarray(coeffs, dtype=np.float64))
        if len(c) != (2 if kind == "parametric" else 1) or not c[0] > 0:
            raise ValueError(f"vst_transform({kind!r}) needs " + ("(a0 > 0, a1)" if kind == "parametric" else "a mean dispersion > 0")
                             + f", got {c}")
        out = self._ops.empty((N, G))
        if G and N:
            self._ops.vst_transform(counts, ld, N, G, sf, VST_KINDS[kind], float(c[0]), float(c[1]) if len(c) > 1 else 0.0, out, G)
        return out

    def calculate_cooks(self, counts, size_factors, design_matrix, mu, hat_diagonals, return_matrix=True):
        """Cook's distances on the device (``DeseqDataSet.calculate_cooks``, dds.py:986-1040; SURVEY.md §8 f-1).

        ``mu`` / ``hat_diagonals`` are what :meth:`irls` returned for the LFC fit (``obsm["_mu_LFC"]``,
        ``obsm["_hat_diagonals"]``).  Returns ``(cooks (N, G) or None, robust_dispersions (G,), cooks_outlier (G,) bool,
        replaced (G,) bool)``: the trimmed-moments dispersions of ``utils.robust_method_of_moments_disp``, the genes whose
        p-value ``cooks_outlier()`` masks (dds.py:1066-1110, before any refit) and the genes ``_replace_outliers`` would
        refit (dds.py:1320-1323).  With ``return_matrix=False`` the (N, G) matrix never leaves the device.
        """
        from scipy.stats import f as _f

        counts, ld = _rows(counts, np.int64, "counts")
        mu, ld2 = _rows(mu, np.float64, "mu")
        hat, ld3 = _rows(hat_diagonals, np.float64, "hat_diagonals")
        if ld3 != ld2:
            hat = np.ascontiguousarray(hat)
            mu = np.ascontiguousarray(mu)
            ld2 = mu.shape[1]
        X = np.ascontiguousarray(_f64(design_matrix, "design_matrix", 2))
        sf = np.ascontiguousarray(_f64(size_factors, "size_factors", 1))
        N, G = counts.shape
        p = X.shape[1]
        self._check_design(X, N, sf)
        if mu.shape != (N, G) or hat.shape != (N, G):
            raise ValueError("counts, mu and hat_diagonals disagree on the number of samples/genes")
        cutoff = float(_f.ppf(0.99, p, N - p))
        cooks = self._ops.empty((N, G)) if return_matrix else None
        disp, outlier, replaced = np.empty(G), np.empty(G), np.empty(G)
        if G:
            self._ops.cooks(counts, ld, N, G, sf, X, p, mu, hat, ld2, cutoff, cooks, disp, outlier, replaced)
        return cooks, disp, outlier == 1.0, replaced == 1.0

    def lfc_shrink_nbinom_glm(self, design_matrix, counts, size, offset, prior_no_shrink_scale, prior_scale,
                              optimizer="L-BFGS-B", shrink_index=1):
        """apeGLM MAP log-fold changes (``inference.py:309-362`` -> ``utils.nbinomGLM`` utils.py:990-1145; SURVEY.md §8 f-3).

        Returns ``(lfcs (G, p), inv_hessians (G, p, p), l_bfgs_b_converged (G,) float 0/1)``.  The kernel walks the
        reference's own optimiser path (unconstrained L-BFGS-B, ftol = gtol = 1e-8) and, for two-column designs, refits
        the genes that did not converge on the reference's 2-D grid; ``last_shrink_grid`` counts them.  ``optimizer`` must be
        ``"L-BFGS-B"``, the only value the reference's caller passes (ds.py:400-409).
        """
        if optimizer != "L-BFGS-B":
            raise NotImplementedError(f"optimizer={optimizer!r}: only the reference's default 'L-BFGS-B' path is implemented")
        counts, ld = _rows(counts, np.int64, "counts")
        X = np.ascontiguousarray(_f64(design_matrix, "design_matrix", 2))
        N, G = counts.shape
        p = X.shape[1]
        self._check_design(X, N)
        size = np.ascontiguousarray(_f64(size, "size", 1))
        offset = np.ascontiguousarray(_f64(offset, "offset", 1))
        shrink_index = int(shrink_index)
        if size.shape != (G,) or offset.shape != (N,):
            raise ValueError("size must have one entry per gene and offset one per sample")
        if not 0 <= shrink_index < p:
            raise IndexError(f"shrink_index {shrink_index} out of range for {p} design columns")
        lfcs, ih, conv = np.empty((G, p)), np.empty((G, p, p)), np.empty(G)
        self.last_shrink_grid = 0
        if G:
            self.last_shrink_grid = self._ops.lfc_shrink(X, counts, ld, N, G, p, size, offset, float(prior_no_shrink_scale),
                                                         float(prior_scale), shrink_index, lfcs, ih, conv)
        return lfcs, ih, conv

    # ------------------------------------------------------------------ helpers
    @staticmethod
    def _check_design(X, N, sf=None):
        if X.shape[0] != N:
            raise ValueError(f"design_matrix has {X.shape[0]} rows for {N} samples")
        if X.shape[1] > _lib.PDQ_MAX_P:
            raise B200Error(f"design has {X.shape[1]} columns; this build supports p <= {_lib.PDQ_MAX_P}")
        if sf is not None and sf.shape[0] != N:
            raise ValueError(f"size_factors has {sf.shape[0]} entries for {N} samples")
