"""Hot-path drivers: the order in which ``DeseqDataSet.deseq2()`` + ``DeseqStats.run_wald_test()`` call the
``Inference`` plugin (``pydeseq2/dds.py:516-562``, ``ds.py:303-360``), without the orchestrator's
AnnData/pandas state and without the stages SURVEY.md §8 marks "next" (Cook's distances / outlier refit,
independent filtering).

Two drivers share the host glue (size factors, trend loop, dispersion prior -- global reductions over genes):

* :func:`fit_host` -- takes ANY object with the reference's ``Inference`` methods (``B200Inference``, the oracle,
  the reference's own ``DefaultInference``) and passes HOST numpy buffers, exactly like the orchestrator does.
  This is the end-to-end (``e2e``) path of ``bench.py`` and what the parity tests chain.
* :class:`ResidentFit` -- keeps counts and every (N, G) intermediate in HBM and chains the ``*_dev`` entry
  points of the C ABI; only per-gene vectors cross PCIe.  This is the ``value`` path of ``bench.py``.
"""
from __future__ import annotations

import ctypes as C
import os
import time
import warnings
from dataclasses import dataclass, field
from types import SimpleNamespace

import numpy as np
from scipy.special import polygamma
from scipy.stats import trim_mean

LN2 = float(np.log(2.0))


# --------------------------------------------------------------------------------------- host glue
def median_of_ratios(counts: np.ndarray):
    """Size factors by median of ratios (preprocessing.py:31-102). Returns (normed_counts, size_factors)."""
    with np.errstate(divide="ignore"):
        lc = np.log(counts)
    lm = lc.mean(0)
    keep = ~np.isinf(lm)
    if not keep.any():
        raise ValueError("Every gene contains at least one zero, cannot compute log geometric means.")
    sf = np.exp(np.median(lc[:, keep] - lm[keep], axis=1))
    return counts / sf[:, None], sf


def filtered_genes(logmeans: np.ndarray, fit_type: str = "ratio") -> np.ndarray:
    """``DeseqDataSet.filtered_genes`` after ``fit_size_factors``: the genes held-out samples are normalised against
    (dds.py:478-486).  Finite log means (preprocessing.py:54); for poscounts also above 0 (dds.py:663).  Never masked by control
    genes."""
    lm = np.asarray(logmeans)
    keep = ~np.isinf(lm)
    return keep & (lm > 0) if fit_type == "poscounts" else keep


def size_factors_numpy(counts: np.ndarray, fit_type: str = "ratio", control=None):
    """``fit_size_factors`` (dds.py:628-703) for ``"ratio"`` / ``"poscounts"`` in numpy, for backends without ``size_factors``.
    ``control``: boolean mask of the control genes or None.  Returns (normed_counts, size_factors, logmeans)."""
    counts = np.asarray(counts)
    use = np.ones(counts.shape[1], dtype=bool) if control is None else np.asarray(control, dtype=bool)
    with np.errstate(divide="ignore", invalid="ignore"), warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)  # np.median of an empty set: NaN, as in the reference
        if fit_type == "poscounts":
            lc = np.zeros_like(counts, dtype=float)
            np.log(counts, out=lc, where=counts != 0)
            lm = lc.mean(0)
            use = use & filtered_genes(lm, "poscounts")
            sf = np.array([np.exp(np.median(np.log(x[use & (x > 0)]) - lm[use & (x > 0)])) for x in counts])
            sf = sf / np.exp(np.mean(np.log(sf)))
        else:
            lc = np.log(counts)
            lm = lc.mean(0)
            if np.isinf(lm).all():
                raise ValueError("Every gene contains at least one zero, cannot compute log geometric means.")
            use = use & ~np.isinf(lm)
            sf = np.exp(np.median(lc[:, use] - lm[use], axis=1))
        return counts / sf[:, None], sf, lm


def size_factor_kind(fit_type: str) -> int:
    """``kind`` of pdq_size_factors_ex for a ``size_factors_fit_type`` of the drivers; "iterative" stays with the reference."""
    from .inference import SF_KINDS

    if fit_type == "iterative":
        raise NotImplementedError("iterative size factors have no device implementation; fit them with the reference")
    if fit_type not in SF_KINDS:
        raise ValueError(f"size_factors_fit_type must be one of {sorted(SF_KINDS)}, got {fit_type!r}")
    return SF_KINDS[fit_type]


def check_size_factors(sf, counts, logmeans, fit_type="ratio", control=None):
    """Raise for NaN size factors, naming the samples whose median had no entry: no usable gene, or for poscounts no positive count
    in one.  ``counts`` (N, G) host counts in the gene order of ``logmeans`` and ``control``."""
    if np.isfinite(sf).all():
        return
    usable = filtered_genes(logmeans, fit_type)
    if control is not None:
        usable = usable & control
    counts = np.asarray(counts)
    if fit_type == "poscounts":
        bad = np.flatnonzero(~(counts[:, usable] > 0).any(1))
    else:
        bad = np.arange(counts.shape[0]) if not usable.any() else np.flatnonzero(~np.isfinite(sf))
    raise ValueError(f"Size factors are NaN: sample(s) {bad.tolist()} have no usable gene ({fit_type}"
                     + (", control genes" if control is not None else "") + ")")


def lin_mu_branch(X: np.ndarray) -> bool:
    """True when #unique design rows == #columns: mu_hat comes from ``lin_reg_mu`` (dds.py:747-756)."""
    return len(np.unique(X, axis=0)) == X.shape[1]


def mean_absolute_deviation(x: np.ndarray) -> float:
    """utils.py:1210-1227 (scaled MAD)."""
    from scipy.special import erfinv  # 1 / (sqrt(2) erfinv(0.5)) = 1.4826...

    return float(np.median(np.abs(x - np.median(x))) / (np.sqrt(2.0) * erfinv(0.5)))


@dataclass
class TrendFit:
    kind: str                 # "parametric" | "mean"
    coeffs: np.ndarray        # (a0, a1) or (mean_disp, nan)
    fitted: np.ndarray        # fitted dispersion per gene
    n_iter: int = 0

    def at(self, means: np.ndarray) -> np.ndarray:
        """The trend at the normalised means ``means`` (dds.py:1267-1275); the mean trend is flat."""
        if self.kind == "parametric":
            return self.coeffs[0] + self.coeffs[1] / means
        return np.full(len(means), self.coeffs[0])


def mean_dispersion(genewise: np.ndarray, min_disp: float) -> float:
    """The mean-type trend: trimmed mean of the genewise dispersions above 10 * min_disp (dds.py:1277-1299, :503-505)."""
    g = np.asarray(genewise, dtype=float)
    return float(trim_mean(g[g > 10 * min_disp], proportiontocut=0.001))


def default_contrast(contrast, p: int) -> np.ndarray:
    """``contrast`` as a float64 vector; None selects the last coefficient."""
    if contrast is None:
        contrast = np.zeros(p)
        contrast[-1] = 1.0
    return np.ascontiguousarray(contrast, dtype=np.float64)


def fit_trend(inference, normed_means: np.ndarray, genewise: np.ndarray, min_disp: float, fit_type="parametric") -> TrendFit:
    """Dispersion trend (dds.py:799-831): parametric gamma-GLM loop (:1199-1275) or trimmed mean (:1277-1299)."""
    def mean_trend():
        m = mean_dispersion(genewise, min_disp)
        return TrendFit("mean", np.array([m, np.nan]), np.full_like(genewise, m))

    if fit_type == "mean":
        return mean_trend()
    with np.errstate(divide="ignore"):
        cov = 1.0 / normed_means
    ok = np.isfinite(cov)
    idx = np.flatnonzero(ok)
    old = np.array([0.1, 0.1])
    coeffs = np.array([1.0, 1.0])
    n_iter = 0
    while (coeffs > 1e-10).all() and (np.log(np.abs(coeffs / old)) ** 2).sum() >= 1e-6:
        old = coeffs
        coeffs, pred, converged = inference.dispersion_trend_gamma_glm(cov[idx], genewise[idx])
        coeffs = np.asarray(coeffs, dtype=float)
        n_iter += 1
        if not converged or (coeffs <= 1e-10).any():
            warnings.warn("The dispersion trend curve fitting did not converge. Switching to a mean-based dispersion trend.",
                          UserWarning, stacklevel=2)
            return mean_trend()
        ratio = genewise[idx] / np.asarray(pred, dtype=float)
        idx = idx[~((ratio < 1e-4) | (ratio >= 15))]
    fitted = coeffs[0] + coeffs[1] / normed_means
    return TrendFit("parametric", coeffs, fitted, n_iter)


def _device_trend(t16: np.ndarray, fit_type: str) -> TrendFit | None:
    """The parametric trend of the device's trend record ``t16``, or None -- the caller falls back to the mean trend -- for
    ``fit_type="mean"`` and, after the reference's warning, when the fit did not converge (dds.py:1243-1252)."""
    if fit_type != "parametric":
        return None
    if t16[2] == 0.0:
        return TrendFit("parametric", np.array([t16[0], t16[1]]), None, int(t16[3]))
    warnings.warn("The dispersion trend curve fitting did not converge. Switching to a mean-based dispersion trend.",
                  UserWarning, stacklevel=3)
    return None


def fit_prior_var(genewise: np.ndarray, fitted: np.ndarray, N: int, p: int, min_disp: float):
    """dds.py:840-884: squared MAD of log residuals, minus trigamma((N-p)/2), floored at 0.25."""
    res = np.log(genewise) - np.log(fitted)
    above = genewise >= 100 * min_disp
    sq = mean_absolute_deviation(res[above]) ** 2
    return sq, float(np.maximum(sq - polygamma(1, (N - p) / 2), 0.25))


@dataclass
class FitResult:
    size_factors: np.ndarray
    non_zero: np.ndarray
    mom: np.ndarray
    genewise: np.ndarray
    genewise_converged: np.ndarray
    trend: TrendFit
    prior_var: float
    squared_logres: float
    map: np.ndarray
    map_converged: np.ndarray
    dispersions: np.ndarray
    lfc: np.ndarray            # (G, p), natural log scale
    lfc_converged: np.ndarray
    pvalue: np.ndarray
    stat: np.ndarray
    se: np.ndarray
    timings: dict = field(default_factory=dict)
    irls_init_converged: np.ndarray | None = None  # flag of the initial mu_hat IRLS (all ones on the lin_reg_mu branch)
    # what the orchestrator keeps for the steps after the LFC fit (non-zero genes only): obsm["_mu_LFC"], obsm["_hat_diagonals"]
    # (dds.py:980-981) and var["_normed_means"] (dds.py:708)
    mu_lfc: np.ndarray | None = None
    hat: np.ndarray | None = None
    normed_means: np.ndarray | None = None


def _expand(v, nz, G_all):
    out = np.full((G_all,) + v.shape[1:], np.nan)
    out[nz] = v
    return out


def _as_is(a):
    return a


def _untimed(key, fn, *a, **k):
    return fn(*a, **k)


def genewise_stage(counts, X, inference, sf, normed, normed_means, min_mu, min_disp, max_disp, beta_tol, fresh=_as_is, timed=_untimed):
    """``fit_genewise_dispersions`` (dds.py:713-797) after the size factors: all-zero mask, method-of-moments start values
    (dds.py:1140-1162), initial mu_hat by ``lin_reg_mu`` or ``irls``, genewise ``alpha_mle``.  ``max_disp`` is the caller's
    ``max(max_disp, N)``.  Returns ``(non_zero, counts of the non-zero genes, their normalised means, mom, mu_hat,
    initial-fit converged flags, genewise dispersions (clipped), genewise converged flags)``.  Shared by :func:`fit_host`, the
    outlier refit and ``workflow.vst``."""
    # dds.py:729-731 `~(X == 0).all(0)`.  Counts are non-negative, so a gene is all-zero exactly when the mean of its normalised
    # counts is 0: with var["_normed_means"] at hand (dds.py:708) the mask costs O(G) instead of a pass over the (N, G) matrix.
    normed_means = normed.mean(0) if normed_means is None else np.asarray(normed_means)
    nz = normed_means != 0
    all_nz = bool(nz.all())
    c = counts if all_nz else counts[:, nz]              # no copy when the caller already dropped all-zero genes
    nn = normed if all_nz else normed[:, nz]
    normed_means = normed_means[nz]

    rde = timed("fit_rough_dispersions", inference.fit_rough_dispersions, nn, X)       # dds.py:1150-1157
    mde = timed("fit_moments_dispersions", inference.fit_moments_dispersions, nn, sf)
    mom = np.clip(np.minimum(rde, mde), min_disp, max_disp)
    if lin_mu_branch(X):                                 # dds.py:747-765
        mu_hat = timed("lin_reg_mu", inference.lin_reg_mu, fresh(c), sf, X, min_mu)
        init_conv = np.ones(c.shape[1])
    else:  # the orchestrator drops this call's `converged` flag (dds.py:757-765); kept here for diagnostics
        _, mu_hat, _, init_conv = timed("irls_init", inference.irls, fresh(c), sf, X, mom, min_mu, beta_tol)
    mu_hat = np.ascontiguousarray(mu_hat)                # layers["_mu_hat"][:, non_zero_idx] is a fresh C array
    gw, gw_conv = timed("alpha_mle_genewise", inference.alpha_mle, fresh(c), X, fresh(mu_hat), mom, min_disp, max_disp)
    gw = np.clip(gw, min_disp, max_disp)                 # dds.py:792-794
    return nz, c, normed_means, mom, mu_hat, init_conv, gw, gw_conv


def map_lfc_stage(c, X, inference, sf, mu_hat, gw, fitted, prior_var, sq, min_mu, min_disp, max_disp, beta_tol, fresh=_as_is,
                  timed=_untimed):
    """After the trend, on the genes of :func:`genewise_stage`: MAP dispersions, final dispersions (dds.py:886-935) and the LFC
    fit (dds.py:937-984).  ``fitted``: the trend at the genes' means.  Returns ``(map, map converged, final dispersions, lfc, mu,
    hat diagonals, lfc converged)``.  Shared by :func:`fit_host` and the outlier refit."""
    mp, mp_conv = timed("alpha_mle_map", inference.alpha_mle, fresh(c), X, fresh(mu_hat), fitted, min_disp, max_disp,
                        prior_disp_var=prior_var, cr_reg=True, prior_reg=True)
    mp = np.clip(mp, min_disp, max_disp)
    disp = mp.copy()
    outlier = np.log(gw) > np.log(fitted) + 2 * np.sqrt(sq)   # dds.py:926-932
    disp[outlier] = gw[outlier]
    lfc, mu_lfc, hat, lfc_conv = timed("irls_lfc", inference.irls, fresh(c), sf, X, disp, min_mu, beta_tol)
    return mp, mp_conv, disp, lfc, mu_lfc, hat, lfc_conv


def fit_host(counts, X, inference, contrast=None, size_factors=None, min_mu=0.5, min_disp=1e-8, max_disp=10.0,
             beta_tol=1e-8, fit_type="parametric", lfc_null=0.0, alt_hypothesis=None, timings=None, comm=None,
             normed_counts=None, normed_means=None, reuse_lfc_mu=True, fresh_copies=False) -> FitResult:
    """deseq2() + run_wald_test() hot path through the plugin API with host buffers.

    ``comm`` (``sharding.NcclComm`` / ``TorchDistComm``): this process holds one gene shard; the genewise
    dispersions and normalised means of all shards are gathered for the trend and prior (the only cross-gene
    step).  ``size_factors`` must then be given (they are per sample, global over genes).

    ``normed_counts`` / ``normed_means``: ``counts / size_factors`` and its per-gene mean when the caller already holds
    them (the orchestrator keeps both from ``fit_size_factors``: ``layers["normed_counts"]``, ``var["_normed_means"]``,
    dds.py:700-708).  ``counts`` must be non-negative (the reference validates that at construction, utils.py:100-133).  ``reuse_lfc_mu``: feed the Wald stage
    with the ``mu`` the LFC fit returned -- ``irls`` returns the UNclamped ``sf * exp(X beta)`` (utils.py:435-438),
    which is exactly what ``run_wald_test`` recomputes on the host (ds.py:320-324).  ``fresh_copies``: hand every plugin call
    a FRESH pageable copy of its (N, G) arguments, like the orchestrator's fancy-indexed ``self.X[:, self.non_zero_idx]`` /
    ``self.layers["_mu_hat"][:, self.non_zero_idx]`` (dds.py:752, 759, 779-781, 902-904, 954); the time spent copying is the
    orchestrator's, it is accumulated under ``timings["orchestrator_copies"]``."""
    T = timings if timings is not None else {}

    def fresh(a):
        if not fresh_copies:
            return a
        t0 = time.perf_counter()
        b = np.array(a)
        T["orchestrator_copies"] = T.get("orchestrator_copies", 0.0) + time.perf_counter() - t0
        return b

    def timed(key, fn, *a, **k):
        t0 = time.perf_counter()
        r = fn(*a, **k)
        T[key] = T.get(key, 0.0) + time.perf_counter() - t0
        return r

    counts = np.asarray(counts)
    X = np.ascontiguousarray(X, dtype=np.float64)
    N, G_all = counts.shape
    p = X.shape[1]
    max_disp = max(max_disp, N)  # dds.py:312
    contrast = default_contrast(contrast, p)
    if size_factors is None:
        normed, sf = timed("size_factors", median_of_ratios, counts)
    else:
        sf = np.asarray(size_factors, dtype=float)
        normed = normed_counts if normed_counts is not None else timed("normed_counts", lambda: counts / sf[:, None])
    nz, c, normed_means, mom, mu_hat, init_conv, gw, gw_conv = genewise_stage(
        counts, X, inference, sf, normed, normed_means, min_mu, min_disp, max_disp, beta_tol, fresh, timed)
    all_nz = bool(nz.all())
    # trend + prior are global over ALL genes of ALL shards (dds.py:799-884): with gene shards the two per-gene vectors are
    # all-gathered first (the only exchange on the path)
    if comm is None:
        gw_all, means_all = gw, normed_means
    else:
        assert len(gw) == len(normed_means) <= comm.sizes[comm.rank], "comm.sizes must bound the shard's non-zero genes"
        gw_all, means_all = timed("allgather", comm.allgather_pair, gw, normed_means)
        keep = ~np.isnan(means_all)  # NaN = padding of shorter shards (and nothing else: means of non-zero genes are finite)
        gw_all, means_all = gw_all[keep], means_all[keep]
    one_launch = getattr(inference, "trend_and_prior", None) if fit_type == "parametric" else None
    tp = timed("trend_prior", one_launch, means_all, gw_all, min_disp, max_disp, N, p) if one_launch is not None else None
    if tp is not None:   # backend runs the orchestrator's trend loop + prior in one launch (B200Inference.trend_and_prior)
        trend, sq, prior_var = TrendFit("parametric", tp[0], tp[1], tp[4]), tp[2], tp[3]
    else:
        trend = timed("trend", fit_trend, inference, means_all, gw_all, min_disp, fit_type)
        sq, prior_var = timed("prior", fit_prior_var, gw_all, trend.fitted, N, p, min_disp)
    if comm is not None:
        trend = TrendFit(trend.kind, trend.coeffs, trend.at(normed_means), trend.n_iter)
    mp, mp_conv, disp, lfc, mu_lfc, hat, lfc_conv = map_lfc_stage(c, X, inference, sf, mu_hat, gw, trend.fitted, prior_var, sq, min_mu,
                                                                  min_disp, max_disp, beta_tol, fresh, timed)

    # Wald stage on ALL genes, all-zero genes carry NaN (ds.py:320-347)
    lfc_all = _expand(np.asarray(lfc), nz, G_all)
    disp_all = _expand(disp, nz, G_all)
    t0 = time.perf_counter()
    if reuse_lfc_mu:
        mu_w = mu_lfc if all_nz else np.full((N, G_all), np.nan)
        if not all_nz:
            mu_w[:, nz] = mu_lfc
    else:
        mu_w = np.exp(X @ lfc_all.T) * sf[:, None]
    T["wald_mu_host"] = T.get("wald_mu_host", 0.0) + time.perf_counter() - t0
    ridge = np.diag(np.repeat(1e-6, p))
    pv, st, se = timed("wald_test", inference.wald_test, X, disp_all, lfc_all, fresh(mu_w), ridge, contrast, LN2 * lfc_null,
                       alt_hypothesis)
    return FitResult(sf, nz, mom, gw, np.asarray(gw_conv), trend, prior_var, sq, mp, np.asarray(mp_conv), disp_all,
                     lfc_all, np.asarray(lfc_conv), np.asarray(pv), np.asarray(st), np.asarray(se), T,
                     np.asarray(init_conv, dtype=float), mu_lfc, hat, normed_means)


# --------------------------------------------------------------------------------------- apeGLM shrinkage (ds.py:363-443)
def fit_shrink_prior_var(lfc_coeff: np.ndarray, se: np.ndarray, min_var: float = 1e-6, max_var: float = 400.0) -> float:
    """Prior variance of the apeGLM model from the MLE LFCs of the shrunk coefficient and their standard errors
    (``DeseqStats._fit_prior_var``, ds.py:551-585): the zero of a weighted moment equation, bracketed on [min_var, max_var]."""
    from scipy.optimize import root_scalar

    keep = ~np.isnan(lfc_coeff)
    S, D = lfc_coeff[keep] ** 2, se[keep] ** 2

    def objective(a):
        coeff = 1 / (2 * (a + D) ** 2)
        return ((S - D) * coeff).sum() / coeff.sum() - a

    if objective(min_var) < 0:
        return min_var
    return float(root_scalar(objective, bracket=(min_var, max_var)).root)


@dataclass
class ShrinkResult:
    lfc: np.ndarray          # (G, p) natural log scale; only column `coeff_idx` differs in meaning from the MLE table
    se: np.ndarray           # (G,) sqrt(|inv_hessian[k, k]|), all-zero genes NaN
    converged: np.ndarray    # (G,) 0/1, NaN for all-zero genes
    prior_scale: float
    prior_var: float


def lfc_shrink_host(fit: FitResult, counts, X, inference, coeff_idx: int, adapt: bool = True, se=None) -> ShrinkResult:
    """``DeseqStats.lfc_shrink`` (ds.py:363-443) on top of a finished fit: prior scale from the MLE LFCs and the Wald SEs of
    the shrunk coefficient (``se`` defaults to ``fit.se``, which is that coefficient's SE when the Wald contrast selected
    it), one ``lfc_shrink_nbinom_glm`` plugin call on the non-zero genes, results written over the MLE column."""
    counts = np.asarray(counts)
    nz = fit.non_zero
    prior_var, prior_scale = float("nan"), 1.0
    if adapt:
        prior_var = fit_shrink_prior_var(fit.lfc[:, coeff_idx], fit.se if se is None else np.asarray(se, dtype=float))
        prior_scale = float(np.minimum(np.sqrt(prior_var), 1))
    cz = counts if nz.all() else np.ascontiguousarray(counts[:, nz])
    lfcs, ih, conv = inference.lfc_shrink_nbinom_glm(X, cz, 1.0 / fit.dispersions[nz], np.log(fit.size_factors), 15, prior_scale,
                                                     "L-BFGS-B", coeff_idx)
    G_all = counts.shape[1]
    lfc = fit.lfc.copy()
    lfc[nz, coeff_idx] = np.asarray(lfcs)[:, coeff_idx]
    se_out = _expand(np.sqrt(np.abs(np.asarray(ih)[:, coeff_idx, coeff_idx])), nz, G_all)
    return ShrinkResult(lfc, se_out, _expand(np.asarray(conv, dtype=float), nz, G_all), prior_scale, prior_var)


# --------------------------------------------------------------------------------------- resident driver
class ResidentFit:
    """Same sequence with counts and all (N, G) intermediates resident in HBM (C ABI ``*_dev`` entry points).

    ``upload()`` places the shard's counts on the device; ``run()`` is one pass of the hot path: every kernel of
    the chain plus the host trend/prior glue on per-gene vectors.  ``comm`` (optional, see ``sharding.py``)
    gathers the per-gene vectors of all gene shards where the path needs them.
    """

    def __init__(self, ctx, X, size_factors, min_mu=0.5, min_disp=1e-8, max_disp=10.0, beta_tol=1e-8, comm=None,
                 with_cooks=False, sort_genes=True, size_factors_fit_type="ratio", control_genes=None):
        from . import _lib

        size_factor_kind(size_factors_fit_type)
        # size factors fitted on the device when none are given (device_size_factors): the estimator, and the control genes as a
        # boolean mask or integer positions over the uploaded genes in the caller's order
        self.size_factors_fit_type, self.control_genes = size_factors_fit_type, control_genes
        self._lib_mod = _lib
        self.ctx = ctx
        self.lib = ctx.lib
        self.X = np.ascontiguousarray(X, dtype=np.float64)
        self.N, self.p = self.X.shape
        self.min_mu, self.min_disp, self.beta_tol = min_mu, min_disp, beta_tol
        self.max_disp = max(max_disp, self.N)
        self.comm = comm
        self.with_cooks = with_cooks  # also compute Cook's distances (per-gene outlier flags) after the LFC fit
        self.use_graph = True         # replay the pass as one CUDA graph after the first eager pass
        self.gather = comm is not None  # end the pass with the all-gather of the result tables of all gene shards
        # MAP search, final dispersions and LFC fit + Wald test with a per-tile dependency instead of three grid-wide ones
        # (pdq_map_irls_wald_dev): the fit's kernel becomes resident while the search's last tiles run.  Bit-identical results; the
        # entry point keeps the three launches where a warp has many tiles per launch.  False: the three launches always (the
        # reference of tests/test_gpu_fused_tail.py and scripts/tail_bench.py)
        self.fuse_tail = True
        # on the lin_reg_mu branch: the start values and the genewise search in one persistent launch (pdq_mom_alpha_mle_dev), which
        # keeps each gene's start value in registers instead of draining one grid and ramping up the next.  Bit-identical results.
        # False: the two launches always (the reference of tests/test_gpu_pass_glue.py and scripts/pass_glue_bench.py)
        self.fold_moments = True
        # how gene shards exchange: "peer" = one kernel per exchange storing into every peer's HBM over NVLink (sharding.PeerWindow),
        # "nccl" = grouped NCCL all-gathers, "auto" = peer when the ranks can map each other's memory (one node), else NCCL
        self.exchange = os.environ.get("PDQ_EXCHANGE", "auto")
        self._win, self._win_key = None, None
        # Device-side gene order: columns sorted by total count at upload.  IRLS iteration counts follow the expression level and
        # the four genes of a warp iterate in lock step, so neighbours of similar expression waste fewer repeated sweeps (22 % ->
        # 4 % of the IRLS sweeps on the synthetic cohorts).  Per-gene arithmetic is position-independent: results are bit-identical
        # and are returned in the caller's order (one scatter per half of the result slab, see _place).
        self.sort_genes = sort_genes
        self._perm = self._inv = None
        self._graph, self._graph_key, self._eager_key, self._graph_epoch = None, None, None, -1
        self.design = None
        self.sf = None
        if size_factors is not None:  # None: median of ratios on the device from the uploaded counts (see upload)
            self._set_size_factors(size_factors)
        self.lin_branch = lin_mu_branch(self.X)
        self.G = 0
        self._bufs = {}
        self.stage_ms = {}

    def _set_size_factors(self, sf):
        _lib = self._lib_mod
        self.sf = np.ascontiguousarray(sf, dtype=np.float64)
        if self.design:
            self.lib.pdq_design_destroy(self.ctx.h, self.design)
        d = _lib.c_design()
        self.ctx.check(self.lib.pdq_design_create(self.ctx.h, _lib.as_f64p(self.X), _lib.as_f64p(self.sf), self.N, self.p,
                                                  C.byref(d)))
        self.design = d
        self._drop_graph()  # a captured pass holds the old design pack
        self._eager_key = None

    def device_size_factors(self):
        """Size factors from the resident counts -- median of ratios (preprocessing.py:31-102) or poscounts, over every gene or the
        control genes (``size_factors_fit_type`` / ``control_genes``, dds.py:628-703); rebuilds the design pack.
        With gene shards the medians are over the LOCAL genes only -- pass global size factors in that case."""
        from .inference import control_mask

        c_d, kind = self._lib_mod.c_dptr, self.size_factors_fit_type
        d_sf = self._dev("sf", self.N * 8)
        sf = np.empty(self.N)
        ctl = control_mask(self.control_genes, self.G)
        if kind == "ratio" and ctl is None:
            self.ctx.check(self.lib.pdq_size_factors_dev(self.ctx.h, c_d(self._main.counts), self.G, self.N, self.G, c_d(d_sf), None))
            self.ctx.d2h(sf, d_sf)
            self.ctx.sync()
            if not np.isfinite(sf).all():
                raise ValueError("Every gene contains at least one zero, cannot compute log geometric means.")
            self._set_size_factors(sf)
            return sf
        d_ctl = None
        if ctl is not None:
            ctl = ctl if self._perm is None else ctl[self._perm]  # device column j holds the caller's gene perm[j]
            d_ctl = self._dev("sf_control", self.G)
            self.ctx.h2d(d_ctl, ctl.astype(np.uint8))
        d_lm = self._dev("sf_logmeans", self.G * 8)
        self.ctx.check(self.lib.pdq_size_factors_ex_dev(self.ctx.h, c_d(self._main.counts), self.G, self.N, self.G, size_factor_kind(kind),
                                                        c_d(d_ctl) if d_ctl else None, c_d(d_sf), c_d(d_lm)))
        lm = np.empty(self.G)
        self.ctx.d2h(sf, d_sf)
        self.ctx.d2h(lm, d_lm)
        self.ctx.sync()
        if kind == "ratio" and np.isinf(lm).all():
            raise ValueError("Every gene contains at least one zero, cannot compute log geometric means.")
        if not np.isfinite(sf).all():  # the error path only: the counts come back to name the samples
            counts = np.empty((self.N, self.G), dtype=np.int64)
            self.ctx.d2h(counts, self._main.counts)
            self.ctx.sync()
            check_size_factors(sf, counts, lm, kind, ctl)
        self._set_size_factors(sf)
        return sf

    # -- memory --------------------------------------------------------------------------------
    def _dev(self, name, nbytes):
        cur = self._bufs.get(name)
        if cur is None or cur[1] < nbytes:
            if cur is not None:
                self.ctx.free(cur[0])
            self._bufs[name] = (self.ctx.malloc(nbytes), nbytes)
        return self._bufs[name][0]

    def _gene_set(self, prefix: str, G: int, d_vec: int, stride: int, names) -> SimpleNamespace:
        """Device pointers of one gene set, what the stages of a pass read and write: the (N, G) ``counts``, ``mu_hat``, ``mu`` and
        ``hat`` diagonals, the MAP search's ``hint`` and the IRLS start values ``beta0`` in buffers named ``prefix + name``; the
        per-gene vectors ``names``, then the (G, p) LFCs ``beta``, ``stride`` doubles apart from ``d_vec``."""
        ng = self.N * G * 8
        return SimpleNamespace(G=G, **{k: self._dev(prefix + k, ng) for k in ("counts", "mu_hat", "mu", "hat")},
                               hint=self._dev(prefix + "hint", 2 * G * 8), beta0=self._dev(prefix + "beta0", G * self.p * 8),
                               beta=d_vec + len(names) * stride * 8, **{k: d_vec + i * stride * 8 for i, k in enumerate(names)})

    def upload(self, counts: np.ndarray):
        """H2D of this shard's counts (genes that are all-zero must already be dropped, dds.py:729-731)."""
        counts = np.ascontiguousarray(counts, dtype=np.int64)
        assert counts.shape[0] == self.N
        self._place(counts.shape[1], lambda d: self.ctx.h2d(d, counts))
        self._h_counts = counts  # the outlier refit (refit_subset) replaces counts of a few genes on the host

    def upload_columns_dev(self, d_src, ld_src: int, cols: np.ndarray):
        """Like :meth:`upload`, from counts already in HBM: columns ``cols`` (caller's gene order) of the device (N, ld_src) int64
        table ``d_src`` are gathered on the device -- no (N, G) transfer.  The outlier refit (which edits counts on the host) is
        not available after this."""
        cols = np.ascontiguousarray(cols, dtype=np.int32)
        d_idx = self._dev("src_cols", max(len(cols), 1) * 4)
        self.ctx.h2d(d_idx, cols)
        c_d = self._lib_mod.c_dptr
        self._place(len(cols), lambda d: self.ctx.check(self.lib.pdq_gather_columns_dev(
            self.ctx.h, c_d(d_src), int(ld_src), self.N, c_d(d_idx), len(cols), c_d(d), len(cols))))
        self._h_counts = None

    def _place(self, G: int, fill):
        """Buffers for G genes; ``fill(dptr)`` enqueues the (N, G) int64 counts in the caller's gene order into ``dptr``."""
        self._drop_graph()  # buffers may move
        self._eager_key = None
        self.G = G
        G, N, p = self.G, self.N, self.p
        ng = N * G * 8
        # every per-gene result lives in ONE device slab mirrored by one page-locked host block: a pass copies it in two halves
        # (below) instead of a dozen small copies.  With gene shards every vector is laid out with the LARGEST shard's
        # length `Gs` and NaN behind this shard's last gene (written here, once): the slab then is directly the send
        # segment of the exchanges (peer-memory push kernel or equal-count NCCL all-gathers) -- no per-step padding, no staging.
        per_gene = ("mom", "means", "gw", "gw_conv", "map", "map_conv", "disp", "conv", "pv", "stat", "se", "outlier",
                    "robust_disp", "cooks_outlier", "cooks_replaced")
        Gs = self.Gs = self.comm.max_size if self.comm is not None else G
        assert Gs >= G
        total = self._slab_len = len(per_gene) * Gs + Gs * p + 16
        self.d_slab = self._dev("slab", total * 8)
        gs = self._main = self._gene_set("", G, self.d_slab, Gs, per_gene)
        self._h_slab = self.ctx.pinned_empty((total,))
        self._h_slab[:] = np.nan
        self._h = {}
        self._slab_off = {}
        off = 0
        for name in per_gene:
            self._h[name] = self._h_slab[off:off + G]
            self._slab_off[name] = (off, 1)
            off += Gs
        self._h["beta"] = self._h_slab[off:off + G * p].reshape(G, p)
        self._slab_off["beta"] = (off, p)
        off += Gs * p
        self.d_t16, self._h["t16"] = self.d_slab + off * 8, self._h_slab[off:off + 16]
        self._off_beta, self._off_t16 = off - Gs * p, off
        self._h_slab[off:off + 16] = 0.0
        self.ctx.h2d(self.d_slab, self._h_slab)  # NaN pads (and zeros) land on the device once
        self.d_nfb = self._dev("nfb", 64)
        c_d = self._lib_mod.c_dptr
        self._perm = self._inv = None
        self.d_slab_out = self.d_slab
        # The slab reaches the caller's order and the host in two halves.  The genewise half (start values, means, genewise
        # dispersions and flags) is final when the genewise search ends: it is reordered and copied to the host on a branch of the
        # stream while the trend and the tail run.  The tail half and the trend record follow at the end of the pass; the Cook's
        # vectors only when they are computed.  Segments: (offset in doubles, rows, width, permuted) for pdq_scatter_segments_dev.
        sort = self.sort_genes and G >= 256
        vec = lambda names: [(self._slab_off[k][0], G, 1, int(sort)) for k in names]  # noqa: E731
        tail = ("map", "map_conv", "disp", "conv", "pv", "stat", "se", "outlier")
        cooks = ("robust_disp", "cooks_outlier", "cooks_replaced")
        rest = [(self._off_beta, G, p, int(sort)), (self._off_t16, 16, 1, 0)]
        self._seg_gw = np.array(vec(("mom", "means", "gw", "gw_conv")), dtype=np.int64)
        self._seg_tail = {False: np.array(vec(tail) + rest, dtype=np.int64), True: np.array(vec(tail + cooks) + rest, dtype=np.int64)}
        # host ranges of the halves (all per-gene vectors are Gs long, in the order of per_gene)
        o = self._slab_off
        self._h_gw = [(0, o["map"][0])]
        self._h_tail = {False: [(o["map"][0], o["robust_disp"][0]), (self._off_beta, total)], True: [(o["map"][0], total)]}
        if sort:
            d_raw = self.ctx.malloc(ng)
            try:
                fill(d_raw)
                d_sums = self._dev("colsum", G * 8)
                self.ctx.check(self.lib.pdq_column_sums_dev(self.ctx.h, c_d(d_raw), G, N, G, c_d(d_sums)))
                sums = np.empty(G)
                self.ctx.d2h(sums, d_sums)
                self.ctx.sync()
                perm = np.argsort(sums, kind="stable").astype(np.int32)  # device column j holds the caller's gene perm[j]
                self._perm = perm
                self._inv = np.empty(G, dtype=np.int32)
                self._inv[perm] = np.arange(G, dtype=np.int32)
                self.d_perm = self._dev("perm", G * 4)
                self.ctx.h2d(self.d_perm, perm)
                self.d_inv = self._dev("inv", G * 4)  # device column of each caller-order gene: the rows the reorder gathers
                self.ctx.h2d(self.d_inv, self._inv)
                # 8-byte words are moved as they are: the same gather serves int64 counts and float64 arrays
                self.ctx.check(self.lib.pdq_gather_columns_dev(self.ctx.h, c_d(d_raw), G, N, c_d(self.d_perm), G, c_d(gs.counts), G))
                self.ctx.sync()
            finally:
                self.ctx.free(d_raw)
            self.d_slab_out = self._dev("slab_out", total * 8)  # the results in the caller's gene order
            self.ctx.h2d(self.d_slab_out, self._h_slab)
        else:
            fill(gs.counts)
        self.ctx.sync()
        if self.design is None:
            self.device_size_factors()

    def _to_caller_order(self, seg, host=False):
        """Enqueue the slab segments ``seg`` (``_seg_gw`` or ``_seg_tail``) in the caller's gene order, one launch: into
        ``d_slab_out`` (no-op when unsorted), or with ``host`` straight into the page-locked host block, with no copy behind it."""
        if self._perm is None and not host:
            return
        c_d, i64p = self._lib_mod.c_dptr, self._lib_mod.i64p
        out = self._h_slab.ctypes.data if host else self.d_slab_out
        src = c_d(self.d_inv) if self._perm is not None else None
        self.ctx.check(self.lib.pdq_scatter_segments_dev(self.ctx.h, c_d(self.d_slab), c_d(out), src, len(seg), seg.ctypes.data_as(i64p)))

    def _copy_out(self, ranges, side=False):
        """Enqueue the device-to-host copies of the caller-ordered slab's ``ranges`` ((start, end) in doubles); ``side``: on the
        branch of the stream that :meth:`run` joins at the end of the pass."""
        for a, b in ranges:
            (self.ctx.d2h_side if side else self.ctx.d2h)(self._h_slab[a:b], self.d_slab_out + a * 8)

    def _window(self, n_all):
        """The peer-memory receive window of this fit (collective on first use; None = exchange through NCCL)."""
        if self.exchange == "nccl" or not hasattr(self.comm, "open_window"):
            return None
        key = (n_all, self._slab_len)
        if self._win_key == key:
            return self._win
        from .sharding import PeerUnavailable

        if self._win is not None:
            self._drop_graph()
            self._win.close()
            self._win = None
        vec = -(-n_all * 8 // 128) * 128
        try:
            self._win = self.comm.open_window(2 * vec + self.comm.world * self._slab_len * 8)
        except PeerUnavailable:
            if self.exchange == "peer":
                raise
            self._win = None
        self._win_key = key
        return self._win

    def _drop_graph(self):
        if self._graph is not None:
            self.lib.pdq_graph_destroy(self.ctx.h, self._graph)
        self._graph, self._graph_key = None, None

    def close(self):
        self._drop_graph()
        if self._win is not None:  # collective, like the construction
            self._win.close()
            self._win, self._win_key = None, None
        for ptr, _ in self._bufs.values():
            self.ctx.free(ptr)
        self._bufs = {}
        if self.design:
            self.lib.pdq_design_destroy(self.ctx.h, self.design)
            self.design = None

    # -- one pass ----------------------------------------------------------------------------------
    def _enqueue_genewise(self, gs, check, begin, fold=True):
        """Steps 1-3 of a pass (``fit_genewise_dispersions``, dds.py:713-797) on the gene set ``gs``, enqueued without
        synchronising.  ``fold`` (with ``fold_moments``, lin_reg_mu branch): steps 1 and 3 as one launch; stage timings need the
        separate launches."""
        L, h, d, G = self.lib, self.ctx.h, self.design, gs.G
        c_d = self._lib_mod.c_dptr
        if fold and self.fold_moments and self.lin_branch:
            check(L.pdq_mom_alpha_mle_dev(h, d, c_d(gs.counts), G, G, self.min_disp, self.max_disp, self.min_mu, c_d(gs.mom),
                                          c_d(gs.means), c_d(gs.mu_hat), G, c_d(gs.gw), c_d(gs.gw_conv), c_d(gs.hint)))
            return
        # 1. method-of-moments start values + normalised means (dds.py:1140-1162, :708)
        begin("mom_dispersions")
        #    -- and, on the lin_reg_mu branch (dds.py:747-756), the initial mu_hat from the same projection
        check(L.pdq_mom_dispersions_dev(h, d, c_d(gs.counts), G, G, self.min_disp, self.max_disp, c_d(gs.mom),
                                        c_d(gs.means), self.min_mu, c_d(gs.mu_hat) if self.lin_branch else None, G))
        # 2. initial mu_hat by IRLS otherwise (dds.py:757-765)
        if not self.lin_branch:
            begin("irls_init")
            check(L.pdq_irls_dev(h, d, c_d(gs.counts), G, G, c_d(gs.mom), self.min_mu, self.beta_tol, -30.0, 30.0,
                                 250, c_d(gs.beta0), c_d(gs.mu_hat), c_d(gs.hat), G, c_d(gs.conv), c_d(self.d_nfb)))
        # 3. genewise dispersions (dds.py:778-797)
        begin("alpha_mle_genewise")
        #    (its optimum and curvature per gene are kept on the device: the MAP search of step 5 opens from them)
        check(L.pdq_alpha_mle_hint_dev(h, d, c_d(gs.counts), G, G, c_d(gs.mu_hat), G, c_d(gs.mom), self.min_disp,
                                       self.max_disp, 1.0, None, 1, 0, c_d(gs.gw), c_d(gs.gw_conv), None, c_d(gs.hint)))

    def vst_dispersions(self, fit_type="parametric"):
        """The fit stage of ``vst_fit`` (dds.py:384-436) on the resident counts: steps 1-3 of :meth:`run` and the dispersion
        trend (dds.py:1199-1299), then stop.  Returns ``(kind, coeffs, genewise)``: the final kind (``"mean"`` also after a
        parametric trend that did not converge, with the reference's warning), ``(a0, a1)`` or ``(mean_disp,)``, and the clipped
        genewise dispersions in the uploaded gene order.  Only per-gene vectors come back; :meth:`run`'s graph is left alone."""
        ctx, c_d, gs = self.ctx, self._lib_mod.c_dptr, self._main
        self._enqueue_genewise(gs, ctx.check, lambda name: None)
        if fit_type == "parametric":
            ctx.check(self.lib.pdq_trend_fit_dev(ctx.h, c_d(gs.means), c_d(gs.gw), self.G, self.min_disp, self.max_disp,
                                                 float(polygamma(1, (self.N - self.p) / 2)), c_d(self.d_t16), None))
        gw = ctx.pinned_empty((self.G,))
        ctx.d2h(gw, gs.gw)
        t16 = ctx.pinned_empty((16,))
        ctx.d2h(t16, self.d_t16)
        ctx.sync()
        gw = np.clip(gw, self.min_disp, self.max_disp)
        if self._perm is not None:  # device column j holds the caller's gene perm[j]
            out = np.empty_like(gw)
            out[self._perm] = gw
            gw = out
        trend = _device_trend(t16, fit_type)
        if trend is not None:
            return "parametric", trend.coeffs, gw
        return "mean", np.array([mean_dispersion(gw, self.min_disp)]), gw

    def run(self, contrast=None, lfc_null=0.0, alt_hypothesis=None, fit_type="parametric", profile=False, copy=True, events=None):
        """One pass of the hot path.  Every stage is enqueued on the context's stream back to back -- the trend and
        the dispersion prior run on the device too -- so the host synchronises exactly once, at the end.
        ``profile=True`` brackets every stage with CUDA events (``stage_ms``); it serialises the host against each
        stage, so never time a step with it.  ``copy=False`` returns views into the page-locked result block, which the NEXT
        pass overwrites.  ``events=(a, b)``: record the context's event slots around the device work of the pass -- first launch
        to the end of the result copy -- so that a caller can time exactly that (``ctx.elapsed_ms(a, b)`` after the call)."""
        L, ctx, h, d, G = self.lib, self.ctx, self.ctx.h, self.design, self.G
        c_d = self._lib_mod.c_dptr
        p, N = self.p, self.N
        H = self._h
        stage = [None]

        def check(rc):  # ctx.check with optional per-stage event timing
            ctx.check(rc)
            if profile and stage[0]:
                ctx.record(3)
                self.stage_ms[stage[0]] = ctx.elapsed_ms(2, 3)
                stage[0] = None

        def begin(name):
            if profile:
                stage[0] = name
                ctx.sync()
                ctx.record(2)

        gs = self._main
        contrast = default_contrast(contrast, p)
        fused = self.fuse_tail and not profile  # stage timings need the three launches: overlapping kernels have no boundaries
        trigamma_c = float(polygamma(1, (N - p) / 2))
        W = self.comm.world if self.comm is not None else 1
        rank = self.comm.rank if self.comm is not None else 0
        m = self.comm.max_size if self.comm is not None else G
        n_all = W * m
        win = self._window(n_all) if self.comm is not None else None
        if win is not None:  # the gathered vectors live in the window every peer stores into
            vec = -(-n_all * 8 // 128) * 128
            off_gw, off_means, off_table = 0, vec, 2 * vec
            d_gw_all, d_means_all = win.data + off_gw, win.data + off_means
            d_table_all = win.data + off_table if self.gather else None
        elif self.comm is not None:
            d_gw_all, d_means_all = self._dev("gw_all", n_all * 8), self._dev("means_all", n_all * 8)
            d_table_all = self._dev("table_all", W * self._slab_len * 8) if self.gather else None
        else:
            d_gw_all, d_means_all, d_table_all = gs.gw, gs.means, None
        self._d_table_all = d_table_all

        def exchange_vectors():
            if win is not None:
                win.push([(gs.gw, off_gw), (gs.means, off_means)], m)
            else:
                self.comm.allgather_dev([(gs.gw, d_gw_all), (gs.means, d_means_all)], m)

        def exchange_tables():
            if win is not None:  # without a table exchange the pass still ends with the barrier: a fast rank must not store the
                # next pass' vectors into a window whose owner is still reading this pass'
                win.push([(self.d_slab_out, off_table)] if self.gather else [], self._slab_len)
            elif d_table_all is not None:
                self.comm.allgather_dev([(self.d_slab_out, d_table_all)], self._slab_len)
        d_fit_all = self._dev("fitted_all", n_all * 8)
        d_t16 = self.d_t16
        d_fitted = d_fit_all + rank * m * 8  # this shard's slice of the fitted curve

        def enqueue():
            self._enqueue_genewise(gs, check, begin, fold=not profile)  # steps 1-3
            # the genewise half of the slab is final: to the caller's order, and to the host while the rest of the pass runs
            self._to_caller_order(self._seg_gw)
            self._copy_out(self._h_gw, side=True)
            # 4. trend + prior: global over ALL genes of ALL shards (dds.py:799-884).  With gene shards the per-gene
            #    vectors are exchanged first, device to device (peer-memory push kernel or grouped NCCL all-gathers); the fit itself
            #    is one launch (a thread-block cluster, or a cooperative grid from 65 536 genes).
            if self.comm is not None:
                begin("allgather")
                exchange_vectors()
                if profile:
                    check(0)
            if fit_type == "parametric":
                begin("trend_prior")
                check(L.pdq_trend_fit_dev(h, c_d(d_means_all), c_d(d_gw_all), n_all, self.min_disp, self.max_disp, trigamma_c,
                                          c_d(d_t16), c_d(d_fit_all)))
                self._tail(gs, d_fitted, d_t16 + 9 * 8, 0.0, contrast, lfc_null, alt_hypothesis, begin, check, fused)
                self._cooks(begin, check)
                if self.comm is None:
                    # the tail half of the results + the trend record: written into the host block by the reorder launch itself
                    begin("to_caller_order")
                    self._to_caller_order(self._seg_tail[self.with_cooks], host=True)
                    if profile:
                        check(0)
                else:
                    if self._perm is not None:
                        begin("to_caller_order")
                        self._to_caller_order(self._seg_tail[self.with_cooks])
                        if profile:
                            check(0)
                    if d_table_all is not None or win is not None:
                        # end-of-call exchange (SURVEY.md §8e / north star): ONE exchange of the whole result slab -- dispersions,
                        # coefficients, flags, Wald statistics of every shard -- after which each rank holds the full tables in HBM
                        begin("gather_results")
                        exchange_tables()
                        if profile:
                            check(0)
                    self._copy_out(self._h_tail[self.with_cooks])  # the tail half of THIS shard's results + the trend record
            ctx.side_join()

        # The pass is ~20 launches + copies with no host synchronisation in between: after one eager pass (which allocates
        # every buffer) the identical sequence is captured into a CUDA graph and replayed with a single call.
        key = (fit_type, contrast.tobytes(), float(lfc_null), alt_hypothesis, G, self.with_cooks, n_all, self.fuse_tail, self.fold_moments,
               self.gather, win is not None)
        # a captured pass holds pointers into context-owned scratch (per-gene status words, trend scratch); host-buffer calls on the
        # same context may have re-allocated it since: the context counts re-allocations, a stale graph is dropped and re-captured
        if events:
            ctx.record(events[0])
        if self._graph is not None and self._graph_epoch != L.pdq_buffer_epoch(h):
            self._drop_graph()
            self._eager_key = None
        if self.use_graph and not profile and self._graph is not None and self._graph_key == key:
            ctx.check(L.pdq_graph_launch(h, self._graph))
        elif self.use_graph and not profile and self._eager_key == key:
            self._drop_graph()
            ctx.check(L.pdq_capture_begin(h))
            try:
                enqueue()
            finally:
                g = C.c_void_p()
                ctx.check(L.pdq_capture_end(h, C.byref(g)))
            self._graph, self._graph_key, self._graph_epoch = g, key, L.pdq_buffer_epoch(h)
            ctx.check(L.pdq_graph_launch(h, self._graph))
        else:
            enqueue()
            self._eager_key = key
        if events:
            ctx.record(events[1])
        ctx.sync()  # the only host synchronisation of the pass
        if win is not None:
            win.check()
        self._check_tail()
        t16 = H["t16"]
        trend = _device_trend(t16, fit_type)
        if trend is not None:
            sq, prior_var = float(t16[8]), float(t16[9])
        else:
            # dds.py:1243-1252 / fit_type="mean": trimmed-mean trend on the host (global, G-length), then the tail again
            A = ctx.pinned_empty((2, n_all))
            ctx.d2h(A[0], d_gw_all)
            ctx.d2h(A[1], d_means_all)
            ctx.sync()
            valid = ~np.isnan(A[1])
            gw_all = np.clip(A[0][valid], self.min_disp, self.max_disp)
            trend = fit_trend(None, A[1][valid], gw_all, self.min_disp, "mean")
            sq, prior_var = fit_prior_var(gw_all, trend.fitted, N, p, self.min_disp)
            rec = ctx.pinned_empty((16,))
            rec[:] = 0.0
            rec[0], rec[2], rec[8], rec[9] = trend.coeffs[0], 0.0, sq, prior_var
            fit_all = ctx.pinned_empty((n_all,))
            fit_all[:] = trend.coeffs[0]
            ctx.h2d(d_t16, rec)
            ctx.h2d(d_fit_all, fit_all)
            self._tail(gs, d_fitted, None, prior_var, contrast, lfc_null, alt_hypothesis, begin, check, fused)
            self._cooks(begin, check)
            if self.comm is None:
                self._to_caller_order(self._seg_tail[self.with_cooks], host=True)
            else:
                self._to_caller_order(self._seg_tail[self.with_cooks])
                exchange_tables()
                self._copy_out(self._h_tail[self.with_cooks])
            ctx.sync()
            self._check_tail()
        gw = np.clip(H["gw"], self.min_disp, self.max_disp)
        means = H["means"]
        fitted = trend.at(means)
        if trend.kind == "parametric":
            trend = TrendFit("parametric", trend.coeffs, fitted, trend.n_iter)
        # the slab is reused by the next pass: hand out copies (a result dict must survive later run() calls)
        cp = np.array if copy else (lambda v: v)
        return {"mom": cp(H["mom"]), "genewise": gw, "genewise_converged": cp(H["gw_conv"]), "trend": trend, "prior_var": prior_var,
                "squared_logres": sq, "map": np.clip(H["map"], self.min_disp, self.max_disp), "map_converged": cp(H["map_conv"]),
                "dispersions": cp(H["disp"]), "lfc": cp(H["beta"]), "lfc_converged": cp(H["conv"]), "pvalue": cp(H["pv"]),
                "stat": cp(H["stat"]), "se": cp(H["se"]), "normed_means": cp(means), "fitted": fitted, "outlier": cp(H["outlier"]),
                **({"robust_dispersions": cp(H["robust_disp"]), "cooks_outlier": H["cooks_outlier"] == 1.0,
                    "cooks_replaced": H["cooks_replaced"] == 1.0} if self.with_cooks else {})}

    def gather_results(self, result: dict) -> dict:
        """Full-length per-gene tables on this rank (rank order = gene order) from the end-of-call all-gather :meth:`run` issued
        (``self.gather``): one device-to-host copy of the gathered slab, NaN pads of short shards stripped.  No-op without shards."""
        if self.comm is None:
            return result
        if not self.gather:
            raise RuntimeError("run() was told not to gather (ResidentFit.gather = False)")
        W, L = self.comm.world, self._slab_len
        tab = self.ctx.pinned_empty((W, L))
        self.ctx.d2h(tab, self._d_table_all)
        self.ctx.sync()
        sizes = self.comm.sizes
        names = {"mom": "mom", "genewise": "gw", "genewise_converged": "gw_conv", "map": "map", "map_converged": "map_conv",
                 "dispersions": "disp", "lfc": "beta", "lfc_converged": "conv", "pvalue": "pv", "stat": "stat", "se": "se",
                 "normed_means": "means", "outlier": "outlier"}
        if self.with_cooks:
            names.update(robust_dispersions="robust_disp", cooks_outlier="cooks_outlier", cooks_replaced="cooks_replaced")
        out = dict(result)
        for key, slot in names.items():
            off, w = self._slab_off[slot]
            parts = [tab[r, off:off + sizes[r] * w] for r in range(W)]
            full = np.concatenate(parts)
            out[key] = full.reshape(-1, w) if w > 1 else full
        out["genewise"] = np.clip(out["genewise"], self.min_disp, self.max_disp)
        out["map"] = np.clip(out["map"], self.min_disp, self.max_disp)
        out["fitted"] = result["trend"].at(out["normed_means"])
        for k in ("cooks_outlier", "cooks_replaced"):
            if k in out and k in names:
                out[k] = out[k] == 1.0
        return out

    # -- Cook's outlier refit on the resident state (dds.py:1301-1458) ----------------------------------------
    def gather_columns(self, which: str, idx: np.ndarray) -> np.ndarray:
        """Columns ``idx`` of the resident ``"mu"`` / ``"hat"`` array of the last pass as a host (N, len(idx)) array: the only (N, .)
        data the outlier refit needs from the device."""
        idx = np.ascontiguousarray(idx, dtype=np.int32)
        if self._inv is not None:
            idx = np.ascontiguousarray(self._inv[idx])  # caller's gene index -> device column
        R = len(idx)
        out = self.ctx.pinned_empty((self.N, R))
        if R == 0:
            return out
        d_idx, d_out = self._dev("gather_idx", R * 4), self._dev("gather_out", self.N * R * 8)
        self.ctx.h2d(d_idx, idx)
        src = {"mu": self._main.mu, "hat": self._main.hat}[which]
        c_d = self._lib_mod.c_dptr
        self.ctx.check(self.lib.pdq_gather_columns_dev(self.ctx.h, c_d(src), self.G, self.N, c_d(d_idx), R, c_d(d_out), R))
        self.ctx.d2h(out, d_out)
        self.ctx.sync()
        return out

    def refit_subset(self, sub_counts: np.ndarray, trend: "TrendFit", prior_var: float, contrast=None, lfc_null=0.0, alt_hypothesis=None):
        """``_refit_without_outliers`` (dds.py:1393-1458) for a few genes whose outlier counts were replaced: the stages of
        :meth:`run` on the compact (N, R) matrix -- genewise dispersions from scratch, the main fit's trend FUNCTION and prior
        (neither is re-estimated; the trend record of the last pass is still on the device), MAP dispersions, LFCs, Wald test.
        The tail always takes the three launches.  Returns R-length per-gene results."""
        ctx = self.ctx
        sub = np.ascontiguousarray(sub_counts, dtype=np.int64)
        R = sub.shape[1]
        assert sub.shape[0] == self.N and R > 0
        names = ("mom", "means", "gw", "gw_conv", "fitted", "map", "map_conv", "disp", "outlier", "conv", "pv", "stat", "se")
        d_vec = self._dev("refit_vec", (len(names) + self.p) * R * 8)
        gs = self._gene_set("refit_", R, d_vec, R, names)
        ctx.h2d(gs.counts, sub)
        no_stage = lambda name: None  # noqa: E731
        self._enqueue_genewise(gs, ctx.check, no_stage)
        means = np.empty(R)
        ctx.d2h(means, gs.means)
        ctx.sync()
        with np.errstate(divide="ignore"):
            fitted = trend.at(means)
        ctx.h2d(gs.fitted, np.ascontiguousarray(fitted))
        self._tail(gs, gs.fitted, None, float(prior_var), default_contrast(contrast, self.p), lfc_null, alt_hypothesis, no_stage,
                   ctx.check, False)
        host = np.empty((len(names) + self.p) * R)
        ctx.d2h(host, d_vec)
        ctx.sync()
        v = {k: host[i * R:(i + 1) * R] for i, k in enumerate(names)}
        return {"normed_means": means, "genewise": np.clip(v["gw"], self.min_disp, self.max_disp), "fitted": fitted, "disp": v["disp"],
                "lfc": host[len(names) * R:].reshape(R, self.p), "pvalue": v["pv"], "stat": v["stat"], "se": v["se"]}

    # -- apeGLM shrinkage on the resident counts ----------------------------------------------------------
    def lfc_shrink(self, result, coeff_idx: int, adapt: bool = True, se=None, prior_scale=None):
        """``DeseqStats.lfc_shrink`` (ds.py:363-443) after :meth:`run`: counts, design pack and dispersions are already in HBM,
        so the call moves 8*G bytes up (size = 1/dispersion) and 24*G down: the shrunk column, the [k, k] entries of the inverse
        Hessians (the kernel writes all p*p of them on the device) and the convergence flags.  ``result`` is what :meth:`run`
        returned; the prior scale comes from its LFC column ``coeff_idx`` and ``se`` (default: the Wald SEs of that run, i.e.
        the run's contrast must have selected the same coefficient).  With gene shards pass ``prior_scale`` computed from the
        gathered tables (the prior is global over genes).  Returns a :class:`ShrinkResult` for this shard's genes."""
        L, ctx, h, G, p = self.lib, self.ctx, self.ctx.h, self.G, self.p
        c_d = self._lib_mod.c_dptr
        prior_var = float("nan")
        if prior_scale is None:
            prior_scale = 1.0
            if adapt:
                if self.comm is not None:
                    raise ValueError("gene shards: pass prior_scale fitted on the gathered LFC / SE tables")
                prior_var = fit_shrink_prior_var(np.asarray(result["lfc"])[:, coeff_idx],
                                                 np.asarray(result["se"] if se is None else se, dtype=float))
                prior_scale = float(np.minimum(np.sqrt(prior_var), 1))
        host = ctx.pinned_empty((4 * G,))
        size, lfc_k, ih_kk, conv = host[:G], host[G:2 * G], host[2 * G:3 * G], host[3 * G:]
        disp_in = np.asarray(result["dispersions"])
        size[:] = 1.0 / (disp_in if self._perm is None else disp_in[self._perm])  # device gene order
        d_size, d_out = self._dev("shrink_size", G * 8), self._dev("shrink_out", G * (p + p * p + 1) * 8)
        d_status = self._dev("shrink_status", G * 4)
        ctx.h2d(d_size, size)
        ctx.check(L.pdq_lfc_shrink_dev(h, self.design, c_d(self._main.counts), G, G, c_d(d_size), 15.0, float(prior_scale), int(coeff_idx),
                                       c_d(d_out), c_d(d_out + G * p * 8), c_d(d_out + G * (p + p * p) * 8), c_d(d_status)))
        k = int(coeff_idx)
        ctx.d2h_strided(lfc_k, d_out + k * 8, p * 8)
        ctx.d2h_strided(ih_kk, d_out + (G * p + k * p + k) * 8, p * p * 8)
        ctx.d2h(conv, d_out + G * (p + p * p) * 8)
        ctx.sync()
        lfc = np.array(result["lfc"], copy=True)
        se_s, conv_s = np.sqrt(np.abs(ih_kk)), conv.copy()
        if self._perm is None:
            lfc[:, coeff_idx] = lfc_k
            return ShrinkResult(lfc, se_s, conv_s, float(prior_scale), prior_var)
        se_o, conv_o = np.empty(G), np.empty(G)  # back to the caller's gene order
        lfc[self._perm, coeff_idx] = lfc_k
        se_o[self._perm], conv_o[self._perm] = se_s, conv_s
        return ShrinkResult(lfc, se_o, conv_o, float(prior_scale), prior_var)

    def _check_tail(self):
        """After a stream synchronisation: raise when a tile hand-off of the fused tail launch gave up waiting."""
        st = C.c_uint64(0)
        self.ctx.check(self.lib.pdq_map_irls_status(self.ctx.h, C.byref(st)))
        if st.value:
            raise RuntimeError(f"MAP -> LFC hand-off: the LFC fit of tile {st.value - 1} never saw its dispersions")

    def _cooks(self, begin, check):
        """Optional: Cook's distances from the resident mu / hat (dds.py:986-1040); only per-gene results leave the device."""
        if self.with_cooks:
            from scipy.stats import f as _f

            L, h, d, G, gs = self.lib, self.ctx.h, self.design, self.G, self._main
            c_d = self._lib_mod.c_dptr
            begin("cooks")
            check(L.pdq_cooks_dev(h, d, c_d(gs.counts), G, G, c_d(gs.mu), c_d(gs.hat), G,
                                  float(_f.ppf(0.99, self.p, self.N - self.p)), None, G, c_d(gs.robust_disp),
                                  c_d(gs.cooks_outlier), c_d(gs.cooks_replaced)))

    def _tail(self, gs, d_fitted, d_prior_var, prior_var, contrast, lfc_null, alt_hypothesis, begin, check, fused):
        """MAP dispersions -> final dispersions -> LFC fit -> Wald on the gene set ``gs``, enqueued without host synchronisation.
        The prior variance is read from ``d_prior_var`` on the device, or is ``prior_var`` when that is None.  ``fused``: the
        kernel pair of ``pdq_map_irls_wald_dev`` instead of the three launches."""
        L, h, d, G = self.lib, self.ctx.h, self.design, gs.G
        c_d, f64p = self._lib_mod.c_dptr, self._lib_mod.as_f64p
        ridge = np.ascontiguousarray(np.diag(np.repeat(1e-6, self.p)))
        prior = (prior_var, None) if d_prior_var is None else (1.0, c_d(d_prior_var))
        wald = (f64p(ridge), f64p(contrast), LN2 * lfc_null, self._lib_mod.ALT_CODES[alt_hypothesis], c_d(gs.pv), c_d(gs.stat),
                c_d(gs.se))
        if fused:
            # steps 5-7 below with a per-tile dependency: the LFC fit of a gene tile starts when that tile's final dispersions are
            # written
            check(L.pdq_map_irls_wald_dev(h, d, c_d(gs.counts), G, G, c_d(gs.mu_hat), G, c_d(d_fitted), c_d(gs.gw), c_d(gs.hint),
                                          c_d(self.d_t16), self.min_disp, self.max_disp, *prior, c_d(gs.map), c_d(gs.map_conv),
                                          c_d(gs.disp), c_d(gs.outlier), self.min_mu, self.beta_tol, -30.0, 30.0, 250, c_d(gs.beta),
                                          c_d(gs.mu), c_d(gs.hat), G, c_d(gs.conv), *wald))
            return
        # 5. MAP dispersions (dds.py:886-935), opened from the genewise optimum and curvature
        begin("alpha_mle_map")
        check(L.pdq_alpha_mle_hint_dev(h, d, c_d(gs.counts), G, G, c_d(gs.mu_hat), G, c_d(d_fitted), self.min_disp, self.max_disp,
                                       *prior, 1, 1, c_d(gs.map), c_d(gs.map_conv), c_d(gs.hint), None))
        # final dispersions: clip(MAP), outlier genes keep the genewise value (dds.py:918-932)
        begin("select_dispersions")
        check(L.pdq_select_dispersions_dev(h, c_d(gs.gw), c_d(gs.map), c_d(d_fitted), c_d(self.d_t16), G, self.min_disp,
                                           self.max_disp, c_d(gs.disp), c_d(gs.outlier)))
        # 6. + 7. LFC fit (dds.py:937-984: beta, mu (unclamped), hat diagonal stay on the device) and the Wald test of its
        #    coefficients (ds.py:303-360) in ONE launch: the test's X^T W X is the last IRLS sweep's, so mu is not read again
        begin("irls_lfc_wald")
        check(L.pdq_irls_wald_dev(h, d, c_d(gs.counts), G, G, c_d(gs.disp), self.min_mu, self.beta_tol, -30.0, 30.0, 250,
                                  c_d(gs.beta), c_d(gs.mu), c_d(gs.hat), G, c_d(gs.conv), c_d(self.d_nfb), *wald))
