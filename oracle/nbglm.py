"""CPU oracle for the per-gene negative-binomial GLM hot path.  TEST INFRASTRUCTURE.

This module is a numpy/scipy restatement of the reference's per-gene numerics
(``pydeseq2/utils.py`` and ``grid_search.py``) and of its joblib gene
fan-out (``default_inference.py``).  It exists only to *check* the CUDA path:

* importable ONLY from ``tests/``, ``__graft_entry__.smoke()`` and the
  ``cpu_baseline`` / ``--impl reference`` legs of ``bench.py``;
* never imported by ``pydeseq2_b200`` (the product fails loudly without its CUDA
  library instead of falling back to this code).

Parity pin: every function below is compared with the *real* reference, imported from a
PYDESEQ2_SRC checkout through ``oracle/refshim``, by ``oracle/make_golden.py``; the
resulting input/output vectors are committed under ``tests/golden/`` and re-checked by
``tests/test_oracle_golden.py`` (CPU suite).  Third-party arithmetic the reference
leans on and that is not part of PyDESeq2 (versions of this image):
scipy 1.18.1 ``optimize.minimize(method="L-BFGS-B")``, ``linalg.solve``,
``special.gammaln/polygamma``, ``stats.norm.sf``; numpy 2.3.5 ``linalg``;
scikit-learn 1.9.0 ``LinearRegression`` (least squares, re-expressed with
``numpy.linalg.lstsq`` here).  The same scipy/numpy wheels are used here, so the
optimiser path is the reference's own.

Every function cites the reference lines it follows.
"""
from __future__ import annotations

import os

import numpy as np
from scipy.linalg import solve as _posdef_solve
from scipy.optimize import minimize as _minimize
from scipy.special import gammaln, polygamma
from scipy.stats import norm as _norm

RIDGE = 1e-6


# --------------------------------------------------------------------------- likelihood
def nb_nll(y, mu, alpha):
    """NB negative log-likelihood of one gene (utils.py:163-234, scalar-alpha branch)."""
    r = 1.0 / alpha
    lb = gammaln(y + r) - gammaln(y + 1) - gammaln(r)
    return len(y) * r * np.log(alpha) + (-lb + (y + r) * np.log(r + mu) - y * np.log(mu)).sum()


def nb_nll_grid(y, mu, alphas):
    """NB nll of one gene on a vector of dispersions (grid_search.py:7-51).

    ``mu`` is (N,) for the alpha grid or (N, K) for the beta grid.
    """
    r = 1.0 / alphas
    lb = gammaln(y[:, None] + r) - gammaln(y + 1)[:, None] - gammaln(r)
    m = mu[:, None] if mu.ndim == 1 else mu
    body = -lb + (y[:, None] + r) * np.log(m + r) - (y[:, None] * np.log(m) if mu.ndim > 1 else (y * np.log(mu))[:, None])
    return len(y) * r * np.log(alphas) + body.sum(0)


def dnb_nll(y, mu, alpha):
    """d nll / d alpha (utils.py:237-270)."""
    r = 1.0 / alpha
    s = (polygamma(0, r) - polygamma(0, y + r) + np.log(1 + mu * alpha) + (y - mu) / (mu + r)).sum()
    return -(r * r) * s


# --------------------------------------------------------------------------- IRLS (a1)
def grid_fit_beta(y, sf, X, disp, min_mu=0.5, grid_length=60, min_beta=-30, max_beta=30):
    """Two-level 2-D grid for p == 2 (grid_search.py:145-221)."""
    gx = np.linspace(min_beta, max_beta, grid_length)
    gy = np.linspace(min_beta, max_beta, grid_length)

    def loss(B):
        mu = np.maximum(sf[:, None] * np.exp(X @ B.T), min_mu)
        return nb_nll_grid(y, mu, disp) + 0.5 * (RIDGE * B**2).sum(1)

    ll = np.zeros((grid_length, grid_length))
    for i, x in enumerate(gx):
        ll[i] = loss(np.array([[x, v] for v in gy]))
    i0, j0 = np.unravel_index(np.argmin(ll), ll.shape)
    d = gx[1] - gx[0]
    fx = np.linspace(gx[i0] - d, gx[i0] + d, grid_length)
    fy = np.linspace(gy[j0] - d, gy[j0] + d, grid_length)
    for i, x in enumerate(fx):
        ll[i] = loss(np.array([[x, v] for v in fy]))
    i1, j1 = np.unravel_index(np.argmin(ll), ll.shape)
    return np.array([fx[i1], fy[j1]])


def irls_gene(y, sf, X, disp, min_mu=0.5, beta_tol=1e-8, min_beta=-30, max_beta=30,
              optimizer="L-BFGS-B", maxiter=250, _trace=None):
    """One gene of ``Inference.irls`` (utils.py:273-438).

    Returns (beta, mu_unclamped, hat_diag, converged).  ``_trace`` (a list) receives the
    number of IRLS iterations and whether the optimiser fallback ran (test introspection).
    """
    p = X.shape[1]
    # start value (utils.py:349-357)
    if np.linalg.matrix_rank(X) == p:
        Q, R = np.linalg.qr(X)
        beta0 = _posdef_solve(R, Q.T @ np.log(y / sf + 0.1))
    else:
        beta0 = np.zeros(p)
        with np.errstate(divide="ignore"):
            beta0[0] = np.log(y / sf).mean()
    beta = beta0
    ridge = np.diag(np.repeat(RIDGE, p))
    mu = np.maximum(sf * np.exp(X @ beta), min_mu)
    dev, ratio, it, converged, fell_back = 1000.0, 1.0, 0, True, False
    while ratio > beta_tol:  # utils.py:367
        W = mu / (1.0 + mu * disp)
        z = np.log(mu / sf) + (y - mu) / mu
        beta_hat = _posdef_solve((X.T * W) @ X + ridge, X.T @ (W * z), assume_a="pos")
        it += 1
        if (np.abs(beta_hat) > max_beta).sum() > 0 or it >= maxiter:  # utils.py:374-413
            fell_back = True

            def f(b):
                m = np.maximum(sf * np.exp(X @ b), min_mu)
                return nb_nll(y, m, disp) + 0.5 * (ridge @ b**2).sum()

            def df(b):
                m = np.maximum(sf * np.exp(X @ b), min_mu)
                return -X.T @ y + ((1 / disp + y) * m / (1 / disp + m)) @ X + ridge @ b

            res = _minimize(f, beta0, jac=df, method=optimizer,
                            bounds=[(min_beta, max_beta)] * p if optimizer == "L-BFGS-B" else None)
            beta = res.x
            mu = np.maximum(sf * np.exp(X @ beta), min_mu)
            converged = res.success
            if not res.success and p <= 2:
                beta = grid_fit_beta(y, sf, X, disp)
                mu = np.maximum(sf * np.exp(X @ beta), min_mu)
            break
        beta = beta_hat
        mu = np.maximum(sf * np.exp(X @ beta), min_mu)
        old = dev
        dev = -2.0 * nb_nll(y, mu, disp)  # utils.py:418-421
        ratio = np.abs(dev - old) / (np.abs(dev) + 0.1)
    # hat diagonal from the clamped mu (utils.py:427-433); mu returned unclamped (:435-438)
    W = mu / (1.0 + mu * disp)
    Hinv = np.linalg.inv((X.T * W[None, :]) @ X + ridge)
    h = np.einsum("ij,jk,ki->i", X, Hinv, X.T)
    rw = np.sqrt(W)
    if _trace is not None:
        _trace.append((it, fell_back))
    return beta, sf * np.exp(X @ beta), rw * h * rw, converged


# --------------------------------------------------------------------------- alpha (a2)
def grid_fit_alpha(y, X, mu, alpha_hat, min_disp, max_disp, prior_disp_var=None,
                   cr_reg=True, prior_reg=False, grid_length=100):
    """Two-level 1-D grid in log(alpha) (grid_search.py:54-142). Returns log(alpha)."""
    grid = np.linspace(np.log(min_disp), np.log(max_disp), grid_length)

    def loss(la):
        a = np.exp(la)
        W = mu[:, None] / (1 + mu[:, None] * a)
        reg = 0
        if cr_reg:
            reg = reg + 0.5 * np.linalg.slogdet((X.T[:, :, None] * W).transpose(2, 0, 1) @ X)[1]
        if prior_reg:
            reg = reg + (np.log(a) - np.log(alpha_hat)) ** 2 / (2 * prior_disp_var)
        return nb_nll_grid(y, mu, a) + reg

    ll = loss(grid)
    k = np.argmin(ll)
    d = grid[1] - grid[0]
    fine = np.linspace(grid[k] - d, grid[k] + d, grid_length)
    ll = loss(fine)
    return fine[np.argmin(ll)]


def alpha_mle_gene(y, X, mu, alpha_hat, min_disp, max_disp, prior_disp_var=None,
                   cr_reg=True, prior_reg=False, optimizer="L-BFGS-B", _trace=None):
    """One gene of ``Inference.alpha_mle`` (utils.py:441-564). Returns (alpha, converged)."""
    la_hat = np.log(alpha_hat)
    nev = [0]

    def loss(la):  # utils.py:509-520
        nev[0] += 1
        a = np.exp(la)
        reg = 0.0
        if cr_reg:
            W = mu / (1 + mu * a)
            reg += 0.5 * np.linalg.slogdet((X.T * W) @ X)[1]
        if prior_reg:
            reg += (la - la_hat) ** 2 / (2 * prior_disp_var)
        return nb_nll(y, mu, a) + reg

    def dloss(la):  # utils.py:522-544
        a = np.exp(la)
        g = 0.0
        if cr_reg:
            W = mu / (1 + mu * a)
            g += 0.5 * (np.linalg.inv((X.T * W) @ X) * ((X.T * (-(W**2))) @ X)).sum() * a
        if prior_reg:
            g += (la - la_hat) / prior_disp_var
        return a * dnb_nll(y, mu, a) + g

    res = _minimize(lambda x: loss(x[0]), x0=np.asarray([la_hat]), jac=lambda x: np.asarray([dloss(x[0])]),
                    method=optimizer,
                    bounds=[(np.log(min_disp), np.log(max_disp))] if optimizer == "L-BFGS-B" else None)
    if _trace is not None:
        _trace.append((nev[0], res.success))
    if res.success:
        return np.exp(res.x[0]), res.success
    # quirk kept: the grid call drops the prior/cr flags (utils.py:556-564)
    return np.exp(grid_fit_alpha(y, X, mu, alpha_hat, min_disp, max_disp)), res.success


# --------------------------------------------------------------------------- Wald (a3)
def wald_gene(X, disp, lfc, mu, ridge, contrast, lfc_null, alt_hypothesis=None):
    """One gene of ``Inference.wald_test`` (utils.py:718-811). Returns (p, stat, se)."""
    W = mu / (1 + mu * disp)
    M = (X.T * W[None, :]) @ X
    Hc = np.linalg.inv(M + ridge) @ contrast
    se = np.sqrt(Hc.T @ M @ Hc)

    def greater(t):
        s = contrast @ np.fmax((lfc - t) / se, 0)
        return s, _norm.sf(s)

    def less(t):
        s = contrast @ np.fmin((lfc - t) / se, 0)
        return s, _norm.sf(np.abs(s))

    if alt_hypothesis is None:
        s = float(contrast @ (lfc - lfc_null) / se)
        return 2 * _norm.sf(np.abs(s)), s, se
    if alt_hypothesis == "greater":
        s, pv = greater(lfc_null)
    elif alt_hypothesis == "less":
        s, pv = less(lfc_null)
    elif alt_hypothesis == "greaterAbs":
        s = contrast @ (np.sign(lfc) * np.fmax((np.abs(lfc) - lfc_null) / se, 0))
        pv = 2 * _norm.sf(np.abs(s))
    elif alt_hypothesis == "lessAbs":
        sa, pa = greater(-abs(lfc_null))
        sb, pb = less(abs(lfc_null))
        s, pv = min(sa, sb, key=abs), max(pa, pb)
    else:
        raise KeyError(alt_hypothesis)
    return pv, s, se


# --------------------------------------------------------------------------- initialisers (a4, a5)
def lin_mu_gene(y, sf, X, min_mu=0.5):
    """One gene of ``Inference.lin_reg_mu`` (utils.py:682-715): OLS without intercept."""
    coef = np.linalg.lstsq(X, y / sf, rcond=None)[0]
    return np.maximum(sf * (X @ coef), min_mu)


def fit_rough_dispersions(normed_counts, design_matrix):
    """utils.py:814-853 (vectorised over genes in the reference as well)."""
    X = np.asarray(design_matrix, dtype=float)
    n, p = X.shape
    if n == p:
        raise ValueError(
            "The number of samples and the number of design variables are equal, i.e., there are no "
            "replicates to estimate the dispersion. Please use a design with fewer variables."
        )
    coef = np.linalg.lstsq(X, normed_counts, rcond=None)[0]
    yhat = np.maximum(X @ coef, 1)
    a = (((normed_counts - yhat) ** 2 - yhat) / ((n - p) * yhat**2)).sum(0)
    return np.maximum(a, 0)


def fit_moments_dispersions(normed_counts, size_factors):
    """utils.py:856-885."""
    nc = normed_counts[:, ~(normed_counts == 0).all(axis=0)]
    s_mean_inv = (1 / np.asarray(size_factors)).mean()
    m = nc.mean(0)
    v = nc.var(0, ddof=1)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.nan_to_num((v - s_mean_inv * m) / m**2)


def dispersion_trend_gamma_glm(covariates, targets):
    """default_inference.py:200-230 on plain arrays: returns (coeffs, predictions, converged)."""
    C = np.column_stack([np.ones(len(covariates)), np.asarray(covariates, dtype=float)])
    t = np.asarray(targets, dtype=float)

    def loss(c):
        m = C @ c
        return np.nanmean(t / m + np.log(m), axis=0)

    def grad(c):
        m = C @ c
        return -np.nanmean(((t / m - 1)[:, None] * C) / m[:, None], axis=0)

    try:
        res = _minimize(loss, x0=np.array([1.0, 1.0]), jac=grad, method="L-BFGS-B", bounds=[(1e-12, np.inf)])
    except RuntimeWarning:
        return np.array([np.nan, np.nan]), np.array([np.nan, np.nan]), False
    return res.x, C @ res.x, res.success


def deseq2_norm(counts):
    """Median-of-ratios size factors (preprocessing.py:31-102). Returns (normed, size_factors)."""
    with np.errstate(divide="ignore"):
        lc = np.log(counts)
    lm = lc.mean(0)
    keep = ~np.isinf(lm)
    sf = np.exp(np.median(lc[:, keep] - lm[keep], axis=1))
    return counts / sf[:, None], sf


# --------------------------------------------------------------------------- apeGLM LFC shrinkage (SURVEY.md §8 f-3)
def nbinom_fn(beta, X, y, size, offset, prior_no_shrink_scale, prior_scale, shrink_index=1):
    """NB negative log-likelihood + apeGLM prior (utils.py:1148-1207): zero-mean normal on every
    coefficient except `shrink_index`, which gets the Cauchy-type prior log1p((b / scale)^2)."""
    mask = np.zeros(X.shape[-1])
    mask[shrink_index] = 1.0
    xbeta = X @ beta
    prior = ((beta * (1.0 - mask)) ** 2 / (2 * prior_no_shrink_scale**2)).sum() + np.log1p((beta[shrink_index] / prior_scale) ** 2)
    nll = (y * xbeta - (y + size) * np.logaddexp(xbeta + offset, np.log(size))).sum(0)
    return prior - nll


def nbinom_grad(beta, X, y, size, offset, prior_no_shrink_scale, prior_scale, shrink_index=1):
    """utils.py:1076-1089 (unscaled)."""
    mask = np.zeros(X.shape[-1])
    mask[shrink_index] = 1.0
    xbeta = X @ beta
    d_prior = beta * (1.0 - mask) / prior_no_shrink_scale**2 + 2 * beta * mask / (prior_scale**2 + beta[shrink_index] ** 2)
    d_nll = (y - (y + size) / (1 + size * np.exp(-xbeta - offset))) @ X
    return d_prior - d_nll


def nbinom_hess(beta, X, y, size, offset, prior_no_shrink_scale, prior_scale, shrink_index=1):
    """utils.py:1091-1108 (unscaled, `cnst = 1`).

    Quirk kept on purpose: the reference builds ``h = np.diag(vector)`` and then adds ``np.diag(h)`` -- the diagonal
    extracted again, a length-p vector -- to the p x p data term, so numpy broadcasting adds ``h_j`` to every entry of
    column j rather than to the diagonal.  The result is not symmetric; only its inverse is ever used (utils.py:1143,
    ``SE = sqrt(|inv[k, k]|)`` at ds.py:421-431)."""
    mask = np.zeros(X.shape[-1])
    mask[shrink_index] = 1.0
    e = np.exp(X @ beta + offset)
    frac = (y + size) * size * e / (size + e) ** 2
    h11 = 1 / prior_no_shrink_scale**2
    h22 = 2 * (prior_scale**2 - beta[shrink_index] ** 2) / (prior_scale**2 + beta[shrink_index] ** 2) ** 2
    h = np.diag((1.0 - mask) * h11 + mask * h22)
    return (X.T * frac) @ X + np.diag(h)


def grid_fit_shrink_beta(y, offset, X, size, prior_no_shrink_scale, prior_scale, scale_cnst, grid_length=60,
                         min_beta=-30, max_beta=30):
    """2-D grid search of the shrunk fit (grid_search.py:224-318): coarse grid over [min, max]^2, then a
    fine grid of one coarse cell either side of the best node; first minimum in row-major order wins."""
    def loss(b):  # the reference leaves shrink_index at its default (1) here
        return nbinom_fn(b, X, y, size, offset, prior_no_shrink_scale, prior_scale) / scale_cnst

    xg = np.linspace(min_beta, max_beta, grid_length)
    yg = np.linspace(min_beta, max_beta, grid_length)
    ll = np.array([[loss(np.array([x, v])) for v in yg] for x in xg])
    i, j = np.unravel_index(np.argmin(ll), ll.shape)
    delta = xg[1] - xg[0]
    fx = np.linspace(xg[i] - delta, xg[i] + delta, grid_length)
    fy = np.linspace(yg[j] - delta, yg[j] + delta, grid_length)
    ll = np.array([[loss(np.array([x, v])) for v in fy] for x in fx])
    i, j = np.unravel_index(np.argmin(ll), ll.shape)
    return np.array([fx[i], fy[j]])


def nbinom_glm_gene(X, y, size, offset, prior_no_shrink_scale, prior_scale, optimizer="L-BFGS-B", shrink_index=1,
                    force_grid=False):
    """MAP LFC of one gene under the apeGLM prior (utils.py:990-1145).  Returns (beta, inv_hessian, converged)."""
    p = X.shape[-1]
    beta_init = np.ones(p) * 0.1 * (-1) ** np.arange(p)
    args = (X, y, size, offset, prior_no_shrink_scale, prior_scale, shrink_index)
    cnst = np.maximum(nbinom_fn(np.zeros(p), *args), 1)
    res = _minimize(lambda b: nbinom_fn(b, *args) / cnst, beta_init, jac=lambda b: nbinom_grad(b, *args) / cnst,
                    hess=(lambda b: nbinom_hess(b, *args) / cnst) if optimizer == "Newton-CG" else None,
                    method=optimizer, options={"ftol": 1e-8, "gtol": 1e-8})
    beta, converged = res.x, bool(res.success) and not force_grid
    if not converged and p == 2:
        beta = grid_fit_shrink_beta(y, offset, X, size, prior_no_shrink_scale, prior_scale, cnst)
    return beta, np.linalg.inv(nbinom_hess(beta, *args)), converged


def fit_shrink_prior_var(lfc, se, min_var=1e-6, max_var=400.0):
    """Prior variance of the apeGLM model from the MLE LFCs and their SEs (ds.py:551-585)."""
    from scipy.optimize import root_scalar

    keep = ~np.isnan(lfc)
    S, D = lfc[keep] ** 2, se[keep] ** 2

    def objective(a):
        coeff = 1 / (2 * (a + D) ** 2)
        return ((S - D) * coeff).sum() / coeff.sum() - a

    if objective(min_var) < 0:
        return min_var
    return root_scalar(objective, bracket=(min_var, max_var)).root


# --------------------------------------------------------------------------- gene fan-out (a6)
class OracleInference:
    """Gene fan-out with the reference's scheduling (default_inference.py:14-198).

    joblib/loky, one task per gene, ``batch_size=128``, ``inner_max_num_threads=1`` -- the
    reference's only parallelism strategy -- so that, timed on the benchmark machine's host cores, it is
    a like-for-like CPU baseline (``cpu_baseline.kind == "port"``).
    """

    def __init__(self, n_cpus=None, batch_size=128, backend="loky"):
        self.n_cpus = n_cpus or os.cpu_count() or 1
        self._batch = batch_size
        self._backend = backend

    def _map(self, fn, G, argf):
        if self.n_cpus == 1:
            return [fn(*argf(i)) for i in range(G)]
        from joblib import Parallel, delayed, parallel_backend

        with parallel_backend(self._backend, inner_max_num_threads=1):
            return Parallel(n_jobs=self.n_cpus, batch_size=self._batch)(delayed(fn)(*argf(i)) for i in range(G))

    def lin_reg_mu(self, counts, size_factors, design_matrix, min_mu):
        r = self._map(lin_mu_gene, counts.shape[1], lambda i: (counts[:, i], size_factors, design_matrix, min_mu))
        return np.array(r).T

    def irls(self, counts, size_factors, design_matrix, disp, min_mu, beta_tol,
             min_beta=-30, max_beta=30, optimizer="L-BFGS-B", maxiter=250):
        r = self._map(irls_gene, counts.shape[1],
                      lambda i: (counts[:, i], size_factors, design_matrix, disp[i], min_mu, beta_tol,
                                 min_beta, max_beta, optimizer, maxiter))
        b, m, h, c = (np.array(v) for v in zip(*r))
        return b, m.T, h.T, c.astype(float)

    def alpha_mle(self, counts, design_matrix, mu, alpha_hat, min_disp, max_disp,
                  prior_disp_var=None, cr_reg=True, prior_reg=False, optimizer="L-BFGS-B"):
        r = self._map(alpha_mle_gene, counts.shape[1],
                      lambda i: (counts[:, i], design_matrix, mu[:, i], alpha_hat[i], min_disp, max_disp,
                                 prior_disp_var, cr_reg, prior_reg, optimizer))
        a, c = (np.array(v) for v in zip(*r))
        return a, c.astype(float)

    def wald_test(self, design_matrix, disp, lfc, mu, ridge_factor, contrast, lfc_null, alt_hypothesis=None):
        r = self._map(wald_gene, mu.shape[1],
                      lambda i: (design_matrix, disp[i], lfc[i], mu[:, i], ridge_factor, contrast, lfc_null,
                                 alt_hypothesis))
        pv, st, se = (np.array(v, dtype=float) for v in zip(*r))
        return pv, st, se

    def lfc_shrink_nbinom_glm(self, design_matrix, counts, size, offset, prior_no_shrink_scale, prior_scale,
                              optimizer="L-BFGS-B", shrink_index=1):
        """default_inference.py:232-264."""
        r = self._map(nbinom_glm_gene, counts.shape[1],
                      lambda i: (design_matrix, counts[:, i], size[i], offset, prior_no_shrink_scale, prior_scale,
                                 optimizer, shrink_index))
        b, ih, c = (np.array(v) for v in zip(*r))
        return b, ih, c.astype(float)

    fit_rough_dispersions = staticmethod(fit_rough_dispersions)
    fit_moments_dispersions = staticmethod(fit_moments_dispersions)
    dispersion_trend_gamma_glm = staticmethod(dispersion_trend_gamma_glm)


# --------------------------------------------------------------------------- Cook's distance (SURVEY.md §8 f-1)
def _trimmed_mean_rows(x, trim):
    """Mean over axis 0 after dropping floor(n*trim) smallest and largest entries of every column (utils.py:567-601)."""
    n = x.shape[0]
    k = int(np.floor(n * trim))
    s = np.sort(x, axis=0)
    return s[k:n - k].mean(0)


def design_cells(X, min_replicates=3):
    """Cell id per sample (-1 when the sample's design row has fewer than `min_replicates` replicates);
    utils.py:888-912 `n_or_more_replicates` + the groupby of utils.py:935-941."""
    X = np.asarray(X, dtype=float)
    _, inv, cnt = np.unique(X, axis=0, return_inverse=True, return_counts=True)
    inv = inv.ravel()
    keep = cnt[inv] >= min_replicates
    cell = np.full(len(X), -1)
    ids = {}
    for i in np.flatnonzero(keep):
        cell[i] = ids.setdefault(inv[i], len(ids))
    return cell


def robust_method_of_moments_disp(normed_counts, X):
    """utils.py:914-960: trimmed-moments dispersion used only for Cook's distances."""
    cell = design_cells(X, 3)
    if (cell >= 0).any():
        y = normed_counts[cell >= 0]
        c = cell[cell >= 0]
        trimratio = (1 / 3, 1 / 4, 1 / 8)

        def trimfn(n):
            return 2 if n >= 23.5 else 1 if n >= 3.5 else 0

        var_est = []
        for lvl in np.unique(c):
            rows = y[c == lvl]
            k = trimfn(len(rows))
            mean = _trimmed_mean_rows(rows, trimratio[k])
            sq = (rows - mean[None, :]) ** 2
            var_est.append([2.04, 1.86, 1.51][k] * _trimmed_mean_rows(sq, trimratio[k]))
        v = np.max(var_est, axis=0)
    else:
        rm = _trimmed_mean_rows(normed_counts, 0.125)
        v = 1.51 * _trimmed_mean_rows((normed_counts - rm) ** 2, 0.125)
    m = normed_counts.mean(0)
    with np.errstate(divide="ignore", invalid="ignore"):
        alpha = (v - m) / m**2
    return np.maximum(alpha, 0.04)


def calculate_cooks(counts, normed_counts, X, mu, hat):
    """dds.py:986-1040 on the non-zero genes: returns (cooks (N, G), robust dispersions (G,))."""
    p = X.shape[1]
    disp = robust_method_of_moments_disp(normed_counts, X)
    V = mu**2 * disp[None, :] + mu
    cooks = (counts - mu) ** 2 / V / p * (hat / (1 - hat) ** 2)
    return cooks, disp


def cooks_outlier(counts, cooks, X):
    """dds.py:1066-1110 without a refit: genes whose p-value the Cook's filter masks."""
    from scipy.stats import f

    N, p = X.shape
    cutoff = f.ppf(0.99, p, N - p)
    use = design_cells(X, 3) >= 0
    out = (cooks[use] > cutoff).any(axis=0)
    pos = cooks[:, out].argmax(0)
    out[out] = (counts[:, out] > counts[:, out][pos, np.arange(len(pos))]).sum(0) < 3
    return out
