"""``DeseqDataSet.deseq2()`` + ``DeseqStats.summary()`` end to end on bare arrays, for any ``Inference`` backend.

`pipeline.fit_host` covers the hot path (dispersions, LFCs, Wald).  This module adds the steps the reference's orchestrator
runs around it, in the reference's order, so that a table computed here can be compared with ``DeseqStats.results_df``:

* Cook's distances and the outlier refit -- ``calculate_cooks`` (dds.py:986-1040), ``_replace_outliers`` (dds.py:1301-1358),
  ``_refit_without_outliers`` (dds.py:1360-1458), ``cooks_outlier`` (dds.py:1066-1110)          [SURVEY.md §8 f-1]
* p-value post-processing -- ``_cooks_filtering`` (ds.py:544-549), ``_independent_filtering`` (ds.py:486-528) with its lowess
  smoother (utils.py:1379-1442), ``_p_value_adjustment`` (ds.py:530-542)                         [SURVEY.md §8 f-4]
* the results table of ``summary()`` (ds.py:278-285), optionally with apeGLM-shrunk LFCs (ds.py:363-443).

Everything per gene and heavy goes through the backend (plugin calls + the two extra methods ``calculate_cooks`` /
``lfc_shrink_nbinom_glm``); what stays here is G-length bookkeeping on a handful of genes, exactly the part the reference keeps in
its orchestrator.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from math import ceil, floor

import warnings

import numpy as np

from .pipeline import (LN2, FitResult, check_size_factors, default_contrast, filtered_genes, fit_host, fit_shrink_prior_var, fit_trend,
                       genewise_stage, map_lfc_stage, mean_dispersion, size_factor_kind, size_factors_numpy)


def n_or_more_replicates(X: np.ndarray, min_replicates: int) -> np.ndarray:
    """Per sample: does its design row occur at least ``min_replicates`` times (utils.py:888-911)."""
    _, inv, cnt = np.unique(np.asarray(X), axis=0, return_inverse=True, return_counts=True)
    return cnt[np.ravel(inv)] >= min_replicates


def trimmed_mean_rows(x: np.ndarray, trim: float) -> np.ndarray:
    """Mean over axis 0 after dropping floor(n * trim) values at each end (utils.py:567-599, ``axis=0`` form)."""
    n = x.shape[0]
    k = floor(n * trim)
    return np.sort(x, axis=0)[k:n - k].mean(axis=0)


def lowess(x: np.ndarray, y: np.ndarray, frac: float = 2.0 / 3.0, iters: int = 3) -> np.ndarray:
    """Robust locally weighted linear regression as the reference runs it (utils.py:1379-1442): tricube weights with the
    bandwidth at the sorted distance of index ceil(frac * n), ``iters`` bisquare re-weightings; each local line comes from
    the minimum-norm solution of its 2 x 2 normal equations."""
    x, y = np.asarray(x, dtype=float), np.asarray(y, dtype=float)
    n = len(x)
    r = int(ceil(frac * n))
    dist = np.abs(x[:, None] - x[None, :])
    h = np.maximum(np.sort(dist, axis=0)[r], 1e-12)           # h[i]: distance from x[i] to its r-th neighbour
    w = np.clip(np.abs(np.nan_to_num((x[:, None] - x[None, :]) / h)), 0.0, 1.0)
    w = (1 - w**3) ** 3                                        # w[:, i]: weights of all points around x[i]
    est, delta = np.zeros(n), np.ones(n)
    for _ in range(iters):
        for i in range(n):
            wi = delta * w[:, i]
            A = np.array([[wi.sum(), (wi * x).sum()], [(wi * x).sum(), (wi * x * x).sum()]])
            b = np.array([(wi * y).sum(), (wi * y * x).sum()])
            c0, c1 = np.linalg.lstsq(A, b, rcond=None)[0]
            est[i] = c0 + c1 * x[i]
        res = y - est
        s = np.median(np.abs(res))
        delta = (np.abs(res) > 0).astype(float) if s == 0 else np.clip(res / (6.0 * s), -1, 1)
        delta = (1 - delta**2) ** 2
    return est


def bh_adjust(p: np.ndarray) -> np.ndarray:
    """Benjamini-Hochberg adjusted p-values (what ``scipy.stats.false_discovery_control(method="bh")`` returns)."""
    p = np.asarray(p, dtype=float)
    m = p.size
    order = np.argsort(p)
    adj = p[order] * m / np.arange(1, m + 1)
    adj = np.minimum.accumulate(adj[::-1])[::-1]
    out = np.empty(m)
    out[order] = np.clip(adj, 0.0, 1.0)
    return out


def filter_theta(base_mean: np.ndarray) -> np.ndarray:
    """The 50 quantile levels of the independent filter's base-mean cutoffs (ds.py:495-502)."""
    lower = float(np.mean(base_mean == 0))
    upper = 0.95 if lower < 0.95 else 1.0
    return np.linspace(lower, upper, 50)


def filter_threshold(theta: np.ndarray, num_rej: np.ndarray, lowess=lowess) -> int:
    """Index of the cutoff the independent filter keeps (ds.py:515-525): the first whose rejection count exceeds the lowess fit's
    maximum less the root mean square residual of the non-zero counts; 0 when no count exceeds 10.  ``lowess`` is the smoother
    (the project's restatement, or the reference's own ``pydeseq2.utils.lowess``)."""
    fit = lowess(theta, num_rej, frac=1 / 5)
    j = 0
    if num_rej.max() > 10:
        resid = num_rej[num_rej > 0] - fit[num_rej > 0]
        thresh = fit.max() - np.sqrt(np.mean(resid**2))
        above = np.where(num_rej > thresh)[0]
        if above.size:
            j = int(above[0])
    return j


def independent_filtering(base_mean: np.ndarray, pvalues: np.ndarray, alpha: float = 0.05) -> np.ndarray:
    """Adjusted p-values with the mean-count filter chosen to maximise rejections (ds.py:486-528)."""
    theta = filter_theta(base_mean)
    cutoffs = np.quantile(base_mean, theta)
    G = len(pvalues)
    padj = np.full((G, len(theta)), np.nan)
    tested = ~np.isnan(pvalues)
    for i, cut in enumerate(cutoffs):
        use = (base_mean >= cut) & tested
        if use.any():
            padj[use, i] = bh_adjust(pvalues[use])
    num_rej = (padj < alpha).sum(0).astype(int)
    return padj[:, filter_threshold(theta, num_rej)]


@dataclass
class Deseq2Results:
    """Columns of ``DeseqStats.results_df`` (ds.py:278-285) plus what ``DeseqDataSet.var`` holds after ``deseq2()``."""
    base_mean: np.ndarray
    log2_fold_change: np.ndarray
    lfc_se: np.ndarray           # log2 scale
    stat: np.ndarray
    pvalue: np.ndarray
    padj: np.ndarray
    lfc: np.ndarray              # (G, p) natural log
    dispersions: np.ndarray
    genewise_dispersions: np.ndarray
    fitted_dispersions: np.ndarray
    size_factors: np.ndarray
    non_zero: np.ndarray
    replaced: np.ndarray
    refitted: np.ndarray
    cooks_outlier: np.ndarray
    cooks: np.ndarray | None
    fit: FitResult = field(repr=False, default=None)
    shrink_prior_scale: float | None = None


def deseq2_results(counts, X, inference, contrast=None, size_factors=None, refit_cooks=True, min_replicates=7, cooks_filter=True,
                   independent_filter=True, alpha=0.05, lfc_null=0.0, alt_hypothesis=None, fit_type="parametric", min_mu=0.5,
                   min_disp=1e-8, max_disp=10.0, beta_tol=1e-8, shrink_coeff=None, shrink_adapt=True, keep_cooks=False,
                   comm=None, size_factors_fit_type="ratio", control_genes=None) -> Deseq2Results:
    """The reference's default analysis -- ``dds.deseq2()`` then ``DeseqStats(dds, contrast).summary()`` (and ``lfc_shrink`` when
    ``shrink_coeff`` is given) -- through ``inference``.  ``counts`` (N, G) non-negative integers, ``X`` (N, p) expanded design,
    ``contrast`` (p,) numeric contrast vector (default: last coefficient).

    ``comm`` (``sharding.TorchDistComm`` / ``NcclComm``): ``counts`` is this rank's gene shard and ``size_factors`` must be given.
    Everything per gene -- fits, Cook's distances, the outlier refit -- stays local; the three steps that look at ALL genes are
    exchanged: the dispersion trend / prior (inside ``fit_host``), the multiple-testing step (base means and p-values are
    all-gathered, adjusted identically on every rank, and the local slice is kept) and the apeGLM prior scale.

    ``size_factors_fit_type`` (``"ratio"`` or ``"poscounts"``) and ``control_genes`` (boolean mask or integer positions) select
    the size-factor estimator when ``size_factors`` is not given (``DeseqDataSet(size_factors_fit_type=, control_genes=)``,
    dds.py:584-711); anything but plain ratio goes through ``inference.size_factors``, or numpy for a backend without it."""
    from scipy.stats import f as f_dist

    counts = np.ascontiguousarray(counts, dtype=np.int64)
    X = np.ascontiguousarray(X, dtype=np.float64)
    N, G = counts.shape
    p = X.shape[1]
    contrast = _test_arguments(contrast, p, lfc_null, alt_hypothesis)
    if comm is not None and size_factors is None:
        raise ValueError("gene shards: size factors are per sample and global over genes -- pass them in")
    if size_factors is None and (size_factors_fit_type != "ratio" or control_genes is not None):
        size_factors = _fit_size_factors(counts, inference, size_factors_fit_type, control_genes)[1]
    fit = fit_host(counts, X, inference, contrast=contrast, size_factors=size_factors, min_mu=min_mu, min_disp=min_disp, max_disp=max_disp,
                   beta_tol=beta_tol, fit_type=fit_type, lfc_null=lfc_null, alt_hypothesis=alt_hypothesis, comm=comm)
    max_disp = max(max_disp, N)
    sf, nz = fit.size_factors, fit.non_zero
    lfc, disp = fit.lfc.copy(), fit.dispersions.copy()
    genewise, fitted = _full(fit.genewise, nz, G), _full(fit.trend.fitted, nz, G)
    base_mean = np.zeros(G)
    base_mean[nz] = fit.normed_means                     # all-zero genes have mean 0
    pv, stat, se = fit.pvalue.copy(), fit.stat.copy(), fit.se.copy()
    tables = dict(normed_means=base_mean, lfc=lfc, genewise=genewise, fitted=fitted, disp=disp, pvalue=pv, stat=stat, se=se)

    # ---- Cook's distances (dds.py:986-1040) on the non-zero genes
    c_nz = counts if nz.all() else np.ascontiguousarray(counts[:, nz])
    ck = inference.calculate_cooks(c_nz, sf, X, fit.mu_lfc, fit.hat)[0]
    cooks = np.full((N, G), np.nan)
    cooks[:, nz] = ck
    cutoff = f_dist.ppf(0.99, p, N - p)
    above = cooks > cutoff

    # ---- outlier replacement and refit (dds.py:1042-1064, 1301-1458)
    replaced, refitted, new_zero = np.zeros(G, bool), np.zeros(G, bool), np.zeros(G, bool)
    replace_cooks = None
    if refit_cooks:
        replaceable = n_or_more_replicates(X, min_replicates)
        if replaceable.any():
            replaced = above.any(axis=0)
        if replaced.any():
            new, zero_now = _replace_counts(counts[:, replaced], sf, replaceable[:, None] & above[:, replaced])
            ridx = np.flatnonzero(replaced)
            new_zero[ridx[zero_now]] = True
            refitted[ridx[~zero_now]] = True
            r = None
            if refitted.any():
                r = _refit_subset(np.ascontiguousarray(new[:, ~zero_now]), X, sf, inference, fit, contrast, lfc_null, alt_hypothesis,
                                  min_mu, min_disp, max_disp, beta_tol)
                replace_cooks = cooks.copy()
                replace_cooks[np.ix_(replaceable, refitted)] = 0.0
            _merge_refit(tables, refitted, new_zero, r)

    # ---- which genes lose their p-value (dds.py:1066-1110)
    outlier = _cooks_outlier(cooks if replace_cooks is None else replace_cooks, cooks, counts, X, cutoff)
    if cooks_filter:
        pv[outlier] = np.nan

    padj = _adjust(base_mean, pv, independent_filter, alpha, comm, inference)

    res = Deseq2Results(base_mean, lfc @ contrast / LN2, se / LN2, stat, pv, padj, lfc, disp, genewise, fitted, sf, nz, replaced, refitted,
                        outlier, cooks if keep_cooks else None, fit)
    if shrink_coeff is not None:   # DeseqStats.lfc_shrink (ds.py:363-443): LFC column and SE replaced, p-values untouched
        k = int(shrink_coeff)
        scale = 1.0
        if shrink_adapt:
            lk, sk = lfc[:, k], se
            if comm is not None:
                g = comm.allgather_table({"l": lk, "s": sk})
                lk, sk = g["l"], g["s"]
            scale = float(np.minimum(np.sqrt(fit_shrink_prior_var(lk, sk)), 1))
        sh, ih, _ = inference.lfc_shrink_nbinom_glm(X, c_nz, 1.0 / disp[nz], np.log(sf), 15, scale, "L-BFGS-B", k)
        lfc[nz, k] = np.asarray(sh)[:, k]
        se = se.copy()
        se[nz] = np.sqrt(np.abs(np.asarray(ih)[:, k, k]))
        res.lfc, res.log2_fold_change, res.lfc_se, res.shrink_prior_scale = lfc, lfc[:, k] / LN2, se / LN2, scale
    return res


def _test_arguments(contrast, p, lfc_null, alt_hypothesis) -> np.ndarray:
    """The drivers' contrast (default: the last coefficient); raises for a negative ``lfc_null`` with an ``*Abs`` alternative."""
    contrast = default_contrast(contrast, p)
    if lfc_null < 0 and alt_hypothesis in ("greaterAbs", "lessAbs"):
        raise ValueError(f"The alternative hypothesis being {alt_hypothesis}, please provide a positive lfc_null value (got {lfc_null}).")
    return contrast


def _replace_counts(sub, sf, mask):
    """``_replace_outliers`` (dds.py:1301-1358) on the (N, R) counts of the replaced genes: the entries of ``mask`` become the
    gene's trimmed mean of normalised counts times the sample's size factor.  Returns (new counts, genes now all zero)."""
    base = trimmed_mean_rows(sub / sf[:, None], 0.2)
    repl = (base[None, :] * sf[:, None]).astype(int)   # truncation towards zero, like DataFrame.astype(int)
    new = sub.copy()
    new[mask] = repl[mask]
    return new, (new == 0).all(axis=0)


def _cooks_outlier(flag_cooks, cooks, counts, X, cutoff):
    """``cooks_outlier`` (dds.py:1066-1110): genes with a Cook's distance of ``flag_cooks`` above ``cutoff`` in a sample of a
    design cell with at least 3 replicates, unless fewer than 3 samples have more counts than the sample of the gene's largest
    distance in ``cooks``."""
    outlier = (flag_cooks[n_or_more_replicates(X, 3)] > cutoff).any(axis=0)
    if outlier.any():
        pos = cooks[:, outlier].argmax(0)
        c = counts[:, outlier]
        outlier[outlier] = (c > c[pos, np.arange(len(pos))]).sum(0) < 3
    return outlier


def _merge_refit(tables, refitted, new_zero, refit):
    """Write an outlier refit over ``tables`` (G-length arrays under the keys of the refit's result, changed in place): the rows of
    the ``refitted`` genes from ``refit`` (None when no gene was refitted), and for genes that the replacement made all zero base
    mean 0, LFC 0 and the test of an all-zero gene, se 0, stat 0, p 1 (ds.py:355-360)."""
    if refit is not None:
        for k, v in tables.items():
            v[refitted] = refit[k]
    tables["normed_means"][new_zero] = 0.0
    tables["lfc"][new_zero] = 0.0
    tables["se"][new_zero], tables["stat"][new_zero], tables["pvalue"][new_zero] = 0.0, 0.0, 1.0


def _adjust(base_mean, pv, independent_filter, alpha, comm=None, inference=None):
    """Multiple testing (ds.py:486-542): global over the genes of all shards.  Through ``inference.adjust_pvalues`` when the
    backend has it and the genes are not sharded, else the host restatement below."""
    if comm is None and hasattr(inference, "adjust_pvalues"):
        padj = inference.adjust_pvalues(base_mean, pv, alpha, independent_filter)
        if padj is not None:
            return padj
    bm_all, pv_all = base_mean, pv
    if comm is not None:
        g = comm.allgather_table({"bm": base_mean, "pv": pv})
        bm_all, pv_all = g["bm"], g["pv"]
    if independent_filter:
        padj = independent_filtering(bm_all, pv_all, alpha)
    else:
        padj = np.full(len(pv_all), np.nan)
        ok = ~np.isnan(pv_all)
        padj[ok] = bh_adjust(pv_all[ok])
    if comm is not None:
        padj = padj[comm.local_slice()]
    return padj


def deseq2_results_resident(rf, contrast=None, refit_cooks=True, min_replicates=7, cooks_filter=True, independent_filter=True,
                            alpha=0.05, lfc_null=0.0, alt_hypothesis=None, fit_type="parametric", non_zero=None,
                            adjust=True, shrink_coeff=None, shrink_adapt=True) -> Deseq2Results:
    """:func:`deseq2_results` on a :class:`pipeline.ResidentFit` whose counts are already in HBM (``rf.upload(counts)``, all-zero
    genes dropped by the caller): the hot path, Cook's distances and their per-gene decisions run in ONE resident pass; only
    per-gene vectors come back.  For the few genes whose outlier counts get replaced (dds.py:1301-1358) the mu / hat columns are
    gathered on the device, the replacement is decided on the host (R columns), and the refit (dds.py:1360-1458) runs resident
    again on the compact matrix.  Multiple testing is G-length host work as in :func:`deseq2_results`.  ``non_zero``: boolean mask of
    the uploaded genes within the caller's full gene list (all-zero genes are not fitted but take part in the independent
    filtering with base mean 0, ds.py:486-528); the returned tables then have the full length.  ``shrink_coeff`` /
    ``shrink_adapt``: apeGLM shrinkage of that coefficient on the resident counts (:meth:`pipeline.ResidentFit.lfc_shrink`), as in
    :func:`deseq2_results`."""
    from scipy.stats import f as f_dist

    X, N, p, G = rf.X, rf.N, rf.p, rf.G
    sf = rf.sf
    contrast = _test_arguments(contrast, p, lfc_null, alt_hypothesis)
    was = rf.with_cooks
    rf.with_cooks = True
    try:
        r = rf.run(contrast=contrast, lfc_null=lfc_null, alt_hypothesis=alt_hypothesis, fit_type=fit_type)
    finally:
        rf.with_cooks = was
    base_mean = np.array(r["normed_means"])
    lfc, disp = np.array(r["lfc"]), np.array(r["dispersions"])
    genewise, fitted = np.array(r["genewise"]), np.array(r["fitted"])
    pv, stat, se = np.array(r["pvalue"]), np.array(r["stat"]), np.array(r["se"])
    tables = dict(normed_means=base_mean, lfc=lfc, genewise=genewise, fitted=fitted, disp=disp, pvalue=pv, stat=stat, se=se)
    outlier = np.array(r["cooks_outlier"], dtype=bool)
    cutoff = f_dist.ppf(0.99, p, N - p)
    replaced, refitted, new_zero = np.zeros(G, bool), np.zeros(G, bool), np.zeros(G, bool)
    if refit_cooks:
        replaceable = n_or_more_replicates(X, min_replicates)
        if replaceable.any():
            replaced = np.array(r["cooks_replaced"], dtype=bool)
        if replaced.any():
            ridx = np.flatnonzero(replaced)
            sub = np.ascontiguousarray(rf._h_counts[:, ridx])
            mu, hat = rf.gather_columns("mu", ridx), rf.gather_columns("hat", ridx)
            # Cook's distances of the replaced genes (dds.py:1022-1036) from the resident mu / hat and the device's robust dispersions
            a = np.asarray(r["robust_dispersions"])[ridx]
            V = mu + a[None, :] * mu**2
            ck = (sub - mu) ** 2 / V / p * (hat / (1 - hat) ** 2)
            new, zero_now = _replace_counts(sub, sf, replaceable[:, None] & (ck > cutoff))
            new_zero[ridx[zero_now]] = True
            refitted[ridx[~zero_now]] = True
            q = None
            if refitted.any():
                q = rf.refit_subset(np.ascontiguousarray(new[:, ~zero_now]), r["trend"], r["prior_var"], contrast, lfc_null, alt_hypothesis)
                # which refitted genes still lose their p-value (dds.py:1066-1110 on `replace_cooks`: distances of the replaceable
                # samples are zeroed for refitted genes): samples in cells of 3..min_replicates-1 replicates can still flag them
                keep = ~zero_now
                ck_r = ck[:, keep].copy()
                ck_r[replaceable] = 0.0
                outlier[ridx[keep]] = _cooks_outlier(ck_r, ck[:, keep], sub[:, keep], X, cutoff)
            _merge_refit(tables, refitted, new_zero, q)
    if cooks_filter:
        pv[outlier] = np.nan
    scale = None
    if shrink_coeff is not None:   # DeseqStats.lfc_shrink (ds.py:363-443): LFC column and SE replaced, p-values untouched
        k = int(shrink_coeff)
        scale = float(np.minimum(np.sqrt(fit_shrink_prior_var(lfc[:, k], se)), 1)) if shrink_adapt else 1.0
        sh = rf.lfc_shrink({"lfc": lfc, "se": se, "dispersions": disp}, k, prior_scale=scale)
        lfc, se = sh.lfc, sh.se
    nz = np.ones(G, bool)
    if non_zero is not None:
        nz = np.asarray(non_zero, dtype=bool)
        assert int(nz.sum()) == G, "non_zero must select exactly the uploaded genes"

        def full(v, fill):
            out = np.full((len(nz),) + v.shape[1:], fill, dtype=v.dtype if v.dtype != bool else bool)
            out[nz] = v
            return out

        base_mean, lfc = full(base_mean, 0.0), full(lfc, np.nan)
        disp, genewise, fitted = full(disp, np.nan), full(genewise, np.nan), full(fitted, np.nan)
        pv, stat, se = full(pv, np.nan), full(stat, np.nan), full(se, np.nan)
        replaced, refitted, outlier = full(replaced, False), full(refitted, False), full(outlier, False)
    # adjust=False stops where deseq2() + run_wald_test() + the Cook's filter stop (no independent filtering / BH: `padj` is NaN)
    padj = _adjust(base_mean, pv, independent_filter, alpha, None, _context_inference(rf.ctx)) if adjust else np.full(len(pv), np.nan)
    res = Deseq2Results(base_mean, lfc @ contrast / LN2, se / LN2, stat, pv, padj, lfc, disp, genewise, fitted, sf, nz, replaced, refitted,
                        outlier, None, None)
    if scale is not None:
        res.log2_fold_change, res.shrink_prior_scale = lfc[:, int(shrink_coeff)] / LN2, scale
    return res


def _context_inference(ctx):
    """A ``B200Inference`` on an existing context (the resident drivers' own), for the backend calls that follow a resident pass."""
    from .inference import B200Inference, _CudaOps

    return B200Inference(_ops=_CudaOps(ctx=ctx))


def _full(v, nz, G):
    out = np.full(G, np.nan)
    out[nz] = v
    return out


# --------------------------------------------------------------------------------------- more contrasts on one fit
def wald_tests_numpy(X, size_factors, disp, lfc, contrasts, ridge, lfc_null, alts):
    """``utils.wald_test`` (utils.py:718-811) for every gene and each of K contrasts, with mu = sf * exp(X lfc) (ds.py:320-324),
    for backends without ``wald_tests``.  ``lfc_null`` (K,) natural log, ``alts`` K alternatives.  Returns (K, G) p-values,
    statistics and standard errors; genes with a non-finite LFC row or dispersion get NaN."""
    from scipy.stats import norm

    K, G = len(contrasts), lfc.shape[0]
    pv, stat, se = (np.full((K, G), np.nan) for _ in range(3))
    ok = np.isfinite(disp) & np.isfinite(lfc).all(axis=1)
    b = lfc[ok]
    mu = np.exp(X @ b.T) * size_factors[:, None]
    W = mu / (1 + mu * disp[ok][None, :])
    M = np.einsum("ni,ng,nj->gij", X, W, X)
    H = np.linalg.inv(M + ridge)
    for k, (c, t, alt) in enumerate(zip(contrasts, lfc_null, alts)):
        Hc = H @ c
        s = np.sqrt(np.einsum("gi,gij,gj->g", Hc, M, Hc))[:, None]
        greater = lambda t: (np.fmax((b - t) / s, 0) @ c, norm.sf(np.fmax((b - t) / s, 0) @ c))  # noqa: E731
        less = lambda t: (np.fmin((b - t) / s, 0) @ c, norm.sf(np.abs(np.fmin((b - t) / s, 0) @ c)))  # noqa: E731
        if alt is None:
            st = (b - t) @ c / s[:, 0]
            p = 2 * norm.sf(np.abs(st))
        elif alt == "greaterAbs":
            st = (np.sign(b) * np.fmax((np.abs(b) - t) / s, 0)) @ c
            p = 2 * norm.sf(np.abs(st))
        elif alt == "lessAbs":
            (sa, pa), (sb, pb) = greater(-abs(t)), less(abs(t))
            st, p = np.where(np.abs(sb) < np.abs(sa), sb, sa), np.maximum(pa, pb)
        elif alt == "greater":
            st, p = greater(t)
        else:
            st, p = less(t)
        pv[k, ok], stat[k, ok], se[k, ok] = p, st, s[:, 0]
    return pv, stat, se


def deseq2_stats(res: Deseq2Results, X, inference, contrasts, lfc_null=0.0, alt_hypothesis=None, cooks_filter=True,
                 independent_filter=True, alpha=0.05, prior_lfc_var=None) -> list[Deseq2Results]:
    """``DeseqStats(dds, contrast).summary()`` for each row of ``contrasts`` (K, p) -- or one (p,) contrast -- on the fit that
    :func:`deseq2_results` or :func:`deseq2_results_resident` returned: the LFCs, dispersions, size factors, Cook's outliers and
    the outlier refit are the fit's and are not recomputed; only the Wald test depends on the contrast (ds.py:303-360), and all K
    run in ONE ``inference.wald_tests`` call (a numpy restatement for backends without it), and their p-values are adjusted in ONE
    ``inference.adjust_pvalues`` call when the backend has it.  ``lfc_null`` (log2, as for the
    drivers) and ``alt_hypothesis`` are scalars or one per contrast; ``prior_lfc_var`` (p,) sets the ridge diag(1 / var^2)
    (ds.py:327-330).  Genes whose replaced counts became all zero get se 0, stat 0, p 1 (ds.py:355-360).  Returns one
    :class:`Deseq2Results` per contrast, sharing every field but the results-table columns with ``res``."""
    import dataclasses

    if res.shrink_prior_scale is not None:
        raise ValueError("deseq2_stats needs the fit's MLE LFCs; this result holds apeGLM-shrunk LFCs (shrink_coeff)")
    X = np.ascontiguousarray(X, dtype=np.float64)
    p = X.shape[1]
    cs = np.asarray(contrasts, dtype=float)
    cs = cs[None, :] if cs.ndim == 1 else cs
    if cs.ndim != 2 or cs.shape[1] != p or cs.shape[0] == 0 or res.lfc.shape[1] != p:
        raise ValueError(f"contrasts must be (K, {p}) or ({p},) for a fit with {res.lfc.shape[1]} coefficients, got shape {np.shape(contrasts)}")
    K = cs.shape[0]
    alts = list(alt_hypothesis) if isinstance(alt_hypothesis, (list, tuple, np.ndarray)) else [alt_hypothesis] * K
    nulls = np.asarray(lfc_null, dtype=float)
    if len(alts) != K or nulls.ndim > 1 or (nulls.ndim == 1 and nulls.shape[0] != K):
        raise ValueError(f"lfc_null and alt_hypothesis must be scalars or have one entry per contrast ({K})")
    nulls = np.broadcast_to(nulls, (K,))
    for a, t in zip(alts, nulls):
        if t < 0 and a in ("greaterAbs", "lessAbs"):
            raise ValueError(f"The alternative hypothesis being {a}, please provide a positive lfc_null value (got {t}).")
    ridge = np.diag(np.repeat(1e-6, p)) if prior_lfc_var is None else np.diag(1 / np.asarray(prior_lfc_var, dtype=float) ** 2)
    if hasattr(inference, "wald_tests"):
        pv, stat, se = inference.wald_tests(X, res.size_factors, res.dispersions, res.lfc, cs, ridge, LN2 * nulls, alts)
    else:
        for a in alts:
            if a not in (None, "greaterAbs", "lessAbs", "greater", "less"):
                raise KeyError(a)
        pv, stat, se = wald_tests_numpy(X, res.size_factors, res.dispersions, res.lfc, cs, ridge, LN2 * nulls, alts)
    new_zero = res.replaced & ~res.refitted
    pv, stat, se = np.array(pv), np.array(stat), np.array(se)
    se[:, new_zero], stat[:, new_zero], pv[:, new_zero] = 0.0, 0.0, 1.0
    if cooks_filter:
        pv[:, res.cooks_outlier] = np.nan
    padj = inference.adjust_pvalues(res.base_mean, pv, alpha, independent_filter) if hasattr(inference, "adjust_pvalues") else None
    if padj is None:  # all K rows in one call above; row by row on the host here
        padj = [_adjust(res.base_mean, pv[k], independent_filter, alpha) for k in range(K)]
    return [dataclasses.replace(res, log2_fold_change=res.lfc @ cs[k] / LN2, lfc_se=se[k] / LN2, stat=stat[k], pvalue=pv[k], padj=padj[k])
            for k in range(K)]


# --------------------------------------------------------------------------------------- variance-stabilising transform
_LEAK_WARNING = ("The size factors were fitted iteratively. They will be re-computed with the counts to be transformed. In a "
                 "train/test setting with a downstream task, this would result in a leak of data from test to train set.")


@dataclass
class VstFit:
    """What ``DeseqDataSet.vst_fit()`` leaves behind (dds.py:384-436) plus ``layers["vst_counts"]``.

    ``kind`` is the final ``vst_fit_type``: ``"mean"`` also after a parametric trend that failed to converge.  ``coeffs`` is
    ``(a0, a1)`` (``uns["vst_trend_coeffs"]``) or ``(mean_disp,)`` (dds.py:503-505).  ``genewise`` has one entry per gene, NaN for
    all-zero genes (``var["vst_genewise_dispersions"]``); ``vst_counts`` covers every gene, all-zero genes included.
    ``logmeans`` / ``filtered_genes`` are ``deseq2_norm_fit``'s (preprocessing.py:31-56), None when the size factors were
    passed in without log means."""
    size_factors: np.ndarray
    logmeans: np.ndarray | None
    filtered_genes: np.ndarray | None
    kind: str
    coeffs: np.ndarray
    genewise: np.ndarray
    non_zero: np.ndarray
    vst_counts: np.ndarray | None = None
    inference: object = field(repr=False, default=None)

    def transform(self, counts) -> np.ndarray:
        """``vst_transform(counts)`` on NEW samples (dds.py:464-514): their size factors are medians of ratios against the fit's
        log means (``deseq2_norm_transform``); without log means they are re-fitted on ``counts`` with the reference's warning."""
        counts = np.ascontiguousarray(counts, dtype=np.int64)
        if self.logmeans is None:
            warnings.warn(_LEAK_WARNING, UserWarning, stacklevel=2)
            sf = _fit_size_factors(counts, self.inference)[1]
        else:
            lm = np.where(self.filtered_genes, self.logmeans, -np.inf)
            sf = self.inference.size_factors(counts, logmeans=lm)[1]
        return self.inference.vst_transform(counts, sf, self.kind, self.coeffs)


def _fit_size_factors(counts, inference, fit_type="ratio", control_genes=None):
    """(normed counts, size factors, log means) of ``fit_size_factors`` (dds.py:584-711): on the backend when it has
    ``size_factors``, else numpy.  NaN size factors raise, naming the samples without a usable gene."""
    from .inference import control_mask

    size_factor_kind(fit_type)
    ctl = control_mask(control_genes, counts.shape[1])
    if hasattr(inference, "size_factors"):
        kw = {} if fit_type == "ratio" and ctl is None else {"fit_type": fit_type, "control_genes": ctl}
        normed, sf, lm = inference.size_factors(counts, return_logmeans=True, **kw)
    else:
        normed, sf, lm = size_factors_numpy(counts, fit_type, ctl)
    check_size_factors(sf, counts, lm, fit_type, ctl)
    return normed, sf, lm


def vst(counts, X, inference, fit_type="parametric", use_design=False, size_factors=None, logmeans=None, min_mu=0.5, min_disp=1e-8,
        max_disp=10.0, beta_tol=1e-8, transform=True, size_factors_fit_type="ratio", control_genes=None) -> VstFit:
    """``DeseqDataSet.vst(use_design, fit_type)`` (dds.py:349-436) on bare arrays: median-of-ratios size factors unless
    ``size_factors`` are given (``logmeans`` then are the fit's, for :meth:`VstFit.transform`), genewise dispersions on an
    intercept-only design unless ``use_design`` (dds.py:713-797), the parametric trend loop with its fallback to the trimmed mean
    (dds.py:1199-1299), and the transform of every gene through ``inference.vst_transform``.  ``counts`` (N, G) non-negative
    integers, ``X`` (N, p) the expanded design.  ``size_factors_fit_type`` / ``control_genes``: the size-factor estimator, as in
    :func:`deseq2_results`; ``filtered_genes`` (the genes held-out samples are normalised against) follows it."""
    if fit_type not in ("parametric", "mean"):
        raise NotImplementedError(f"Found fit_type '{fit_type}'. Expected 'parametric' or 'mean'.")
    if not hasattr(inference, "vst_transform"):
        raise TypeError(f"{type(inference).__name__} has no vst_transform")
    counts = np.ascontiguousarray(counts, dtype=np.int64)
    N, G = counts.shape
    max_disp = max(max_disp, N)  # dds.py:312
    if size_factors is None:
        normed, sf, logmeans = _fit_size_factors(counts, inference, size_factors_fit_type, control_genes)
    else:
        sf = np.asarray(size_factors, dtype=float)
        normed = counts / sf[:, None]
    filtered = None if logmeans is None else filtered_genes(logmeans, size_factors_fit_type)
    if use_design:
        Xv = np.ascontiguousarray(X, dtype=np.float64)
        if fit_type == "mean":
            warnings.warn("use_design=True is only useful when fit_type='parametric'. ", UserWarning, stacklevel=2)
    else:
        Xv = np.ones((N, 1))
    nz, _, means, _, _, _, gw, _ = genewise_stage(counts, Xv, inference, sf, normed, None, min_mu, min_disp, max_disp, beta_tol)
    kind = fit_type
    if fit_type == "parametric":
        trend = fit_trend(inference, means, gw, min_disp, "parametric")  # warns and returns the mean trend when the fit fails
        kind = trend.kind
    coeffs = np.asarray(trend.coeffs, dtype=float) if kind == "parametric" else np.array([mean_dispersion(gw, min_disp)])
    fit = VstFit(sf, logmeans, filtered, kind, coeffs, _full(gw, nz, G), nz, None, inference)
    if transform:
        fit.vst_counts = inference.vst_transform(counts, sf, kind, coeffs)
    return fit


def vst_resident(inference, counts, X, fit_type="parametric", use_design=False, size_factors=None, logmeans=None, min_mu=0.5,
                 min_disp=1e-8, max_disp=10.0, beta_tol=1e-8, size_factors_fit_type="ratio", control_genes=None) -> VstFit:
    """:func:`vst` with the counts resident in HBM: they go up once, the size factors (median of ratios on the device unless
    given), the all-zero mask and the fit stage (steps 1-3 of ``ResidentFit.run`` and the trend, on a ``ResidentFit`` of the VST
    design over the non-zero genes, gathered on the device) run there, and ``pdq_vst_transform_dev`` transforms the full table
    in the caller's gene order; only ``vst_counts`` comes back.  Every other transfer is a per-sample or per-gene vector.
    ``inference`` is a ``B200Inference`` (its context is used).  ``size_factors_fit_type`` / ``control_genes`` as in :func:`vst`."""
    from . import _lib
    from .inference import VST_KINDS, control_mask
    from .pipeline import ResidentFit

    if fit_type not in ("parametric", "mean"):
        raise NotImplementedError(f"Found fit_type '{fit_type}'. Expected 'parametric' or 'mean'.")
    kind_code = size_factor_kind(size_factors_fit_type)
    ctx = inference._ops.ctx
    L, h, c_d = ctx.lib, ctx.h, _lib.c_dptr
    counts = np.ascontiguousarray(counts, dtype=np.int64)
    N, G = counts.shape
    ctl = control_mask(control_genes, G)
    plain = size_factors_fit_type == "ratio" and ctl is None
    d_counts, d_sf, d_lm, d_sums, d_out, d_ctl = (ctx.malloc(n) for n in (N * G * 8, N * 8, G * 8, G * 8, N * G * 8, G))
    rf = None
    try:
        ctx.h2d(d_counts, counts)  # the one (N, G) upload
        if size_factors is None:
            if plain:
                ctx.check(L.pdq_size_factors_dev(h, c_d(d_counts), G, N, G, c_d(d_sf), c_d(d_lm)))
            else:
                if ctl is not None:
                    ctx.h2d(d_ctl, ctl.astype(np.uint8))
                ctx.check(L.pdq_size_factors_ex_dev(h, c_d(d_counts), G, N, G, kind_code,
                                                    c_d(d_ctl) if ctl is not None else None, c_d(d_sf), c_d(d_lm)))
            sf, logmeans = np.empty(N), np.empty(G)
            ctx.d2h(sf, d_sf)
            ctx.d2h(logmeans, d_lm)
        else:
            sf = np.ascontiguousarray(size_factors, dtype=np.float64)
            ctx.h2d(d_sf, sf)
        ctx.check(L.pdq_column_sums_dev(h, c_d(d_counts), G, N, G, c_d(d_sums)))
        sums = np.empty(G)
        ctx.d2h(sums, d_sums)
        ctx.sync()
        if plain and not np.isfinite(sf).all():
            raise ValueError("Every gene contains at least one zero, cannot compute log geometric means.")
        if size_factors is None and not plain:
            if size_factors_fit_type == "ratio" and np.isinf(logmeans).all():
                raise ValueError("Every gene contains at least one zero, cannot compute log geometric means.")
            check_size_factors(sf, counts, logmeans, size_factors_fit_type, ctl)
        nz = sums != 0  # counts are non-negative (dds.py:729-731)
        if use_design:
            Xv = np.ascontiguousarray(X, dtype=np.float64)
            if fit_type == "mean":
                warnings.warn("use_design=True is only useful when fit_type='parametric'. ", UserWarning, stacklevel=2)
        else:
            Xv = np.ones((N, 1))
        rf = ResidentFit(ctx, Xv, sf, min_mu=min_mu, min_disp=min_disp, max_disp=max_disp, beta_tol=beta_tol)
        rf.upload_columns_dev(d_counts, G, np.flatnonzero(nz))
        kind, coeffs, gw = rf.vst_dispersions(fit_type)
        ctx.check(L.pdq_vst_transform_dev(h, c_d(d_counts), G, N, G, c_d(d_sf), VST_KINDS[kind], float(coeffs[0]),
                                          float(coeffs[1]) if len(coeffs) > 1 else 0.0, c_d(d_out), G))
        out = ctx.pinned_empty((N, G))
        ctx.d2h(out, d_out)  # the one (N, G) download
        ctx.sync()
    finally:
        if rf is not None:
            rf.close()
        for p in (d_counts, d_sf, d_lm, d_sums, d_out, d_ctl):
            ctx.free(p)
    filtered = None if logmeans is None else filtered_genes(logmeans, size_factors_fit_type)
    return VstFit(sf, logmeans, filtered, kind, coeffs, _full(gw, nz, G), nz, out, inference)


def _refit_subset(sub, X, sf, inference, fit: FitResult, contrast, lfc_null, alt_hypothesis, min_mu, min_disp, max_disp, beta_tol):
    """``_refit_without_outliers`` (dds.py:1393-1458) on the replaced counts, through the main fit's stages: genewise dispersions
    from scratch, the SAME trend function and prior as the main fit (neither is re-estimated), MAP dispersions, LFCs, then the
    Wald test of the refitted genes (per-gene independent: the same as re-running run_wald_test on every gene)."""
    _, c, means, _, mu_hat, _, gw, _ = genewise_stage(sub, X, inference, sf, sub / sf[:, None], None, min_mu, min_disp, max_disp,
                                                      beta_tol)
    fitted = fit.trend.at(means)
    disp, lfc = map_lfc_stage(c, X, inference, sf, mu_hat, gw, fitted, fit.prior_var, fit.squared_logres, min_mu, min_disp, max_disp,
                              beta_tol)[2:4]
    lfc = np.asarray(lfc)
    mu = np.exp(X @ lfc.T) * sf[:, None]
    pv, stat, se = inference.wald_test(X, disp, lfc, mu, np.diag(np.repeat(1e-6, X.shape[1])), contrast, LN2 * lfc_null, alt_hypothesis)
    return {"normed_means": means, "genewise": gw, "fitted": fitted, "disp": disp, "lfc": lfc, "pvalue": pv, "stat": stat, "se": se}
