"""Extended-precision reference and checks of Cook's distances, the trimmed-moments ("robust") dispersions and the two per-gene
decisions of cooks_gene_cols (pdq_gene.cuh), which k_cooks (designs of up to 16 columns) and k_wide_cooks (17..128) run.  Used by
test_gpu_cooks.py on the device, and by test_cooks_checks.py on the CPU to show that the checks accept the float64 oracle and the
host emulator and reject subtly wrong results.

`reference` restates utils.py:567-679 and :914-960 (the dispersions), dds.py:986-1040 (the distances) and dds.py:1066-1110 with
:1320-1323 (the decisions) on exactly the doubles handed to the kernel, in np.longdouble (team_checks.require_longdouble), at
test time: no fixture is needed.  The same code in float64, with one of MUTANTS switched on, makes the wrong results the checks
must reject.

Bounds are first-order error propagation, computed per entry from the reference's own values (u = eps / 2 = 2^-53):
  * each normalised count x = y / sf carries u |x|;
  * a sum of n terms, in whatever order the lanes add them, is within n eps sum |terms| (twice the (n - 1) u worst case, which
    also covers the division that makes it a mean), times SUM_C;
  * an order statistic moves by at most the largest perturbation of its inputs, so a trimmed mean inherits the largest input
    error of its cell (sup norm) whichever tied entries the selection drops;
  * the cancellation in v - m gets an absolute term, e_v + e_m + u (|v| + |m|), before the division by m^2; the clamp at 0.04 is
    1-Lipschitz, so the bound of the unclamped value holds on either side of it;
  * Cook's distance gets COOKS_C eps relative (about a dozen roundings) plus the propagated dispersion error times mu^2 / V.
The decisions must match exactly, except for a gene whose deciding distance lies within its bound of the cutoff, or whose argmax
has a rival within bound that would decide differently: those are counted and reported ("exempt")."""
import math

import numpy as np

from team_checks import require_longdouble

LD = require_longdouble()
EPS = 2.0 ** -52
U = EPS / 2
SUM_C = 2.0
COOKS_C = 8.0
MIN_DISP = 0.04  # utils.py:958

# wrong variants of the computation the checks must reject (test_cooks_checks.py)
MUTANTS = {
    "ntrim_off_by_one": "floor(n trim) - 1 entries trimmed from each end",
    "trim_class_23_5": "cells of 24 samples trimmed as if below 23.5",
    "wrong_scale": "scale 1.51 instead of 1.86 for cells of 4..23 samples",
    "mean_over_all": "squared deviations about the mean over all samples instead of the cell's trimmed mean",
    "nan_dropped": "NaN dropped by the maxima (np.fmax): an all-zero gene gets 0.04",
    "last_argmax": "last-occurrence argmax of the distances",
    "larger_or_equal": ">= instead of > in the count of larger counts",
    "p_minus_1": "p - 1 in the denominator of the distance",
}


def cells_of(X):
    """(cells, global_mode): sample indices of every cell -- identical design rows with at least 3 replicates, by first
    appearance -- or, when there is none, one cell of every sample (utils.py:936-952)."""
    X = np.asarray(X, dtype=np.float64)
    _, first, inv, cnt = np.unique(X, axis=0, return_index=True, return_inverse=True, return_counts=True)
    inv = inv.ravel()
    keep = [k for k in np.argsort(first, kind="stable") if cnt[k] >= 3]
    if not keep:
        return [np.arange(len(X))], True
    return [np.flatnonzero(inv == k) for k in keep], False


def trim_class(n, global_mode, mutant=None):
    """(ntrim, scale) of a cell of n samples (utils.py:622-627, 645; trimmed_variance's 1/8 and 1.51 without cells)."""
    if global_mode:
        k, ratio, scale = 2, 0.125, 1.51
    else:
        edge = 24.5 if mutant == "trim_class_23_5" else 23.5
        k = 2 if n >= edge else 1 if n >= 3.5 else 0
        ratio = (1 / 3, 1 / 4, 1 / 8)[k]
        scale = (2.04, 1.51 if mutant == "wrong_scale" else 1.86, 1.51)[k]
    ntrim = int(math.floor(n * ratio))
    if mutant == "ntrim_off_by_one":
        ntrim = max(ntrim - 1, 0)
    return ntrim, scale


def _f64(a):
    return np.asarray(a, dtype=np.float64)


def dispersions(x, cells, global_mode, dtype=LD, mutant=None):
    """Trimmed-moments dispersions of the normalised counts x (N, G) (already in `dtype`) and their bounds:
    (alpha, e_alpha, m, e_m, v)."""
    N = x.shape[0]
    m = x.mean(0)
    e_m = SUM_C * N * EPS * _f64(np.abs(x).mean(0))
    e_x = U * _f64(np.abs(x))
    tvs, e_tvs = [], []
    for idx in cells:
        nc = len(idx)
        ntrim, scale = trim_class(nc, global_mode, mutant)
        xc = x[idx]
        kept = np.sort(xc, axis=0)[ntrim:nc - ntrim]
        nk = nc - 2 * ntrim
        tm = kept.mean(0)
        e_tm = e_x[idx].max(0) + SUM_C * nc * EPS * _f64(np.abs(kept).sum(0)) / nk
        dlt = xc - (m if mutant == "mean_over_all" else tm)[None, :]
        sq = dlt * dlt
        kept2 = np.sort(sq, axis=0)[ntrim:nc - ntrim]
        tv = scale * kept2.mean(0)
        e_dlt = e_x[idx] + e_tm[None, :] + U * _f64(np.abs(dlt))
        e_sq = 2 * _f64(np.abs(dlt)) * e_dlt + U * _f64(sq)
        e_tv = scale * (e_sq.max(0) + SUM_C * nc * EPS * _f64(kept2.sum(0)) / nk) + U * _f64(np.abs(tv))
        tvs.append(tv)
        e_tvs.append(e_tv)
    tvs = np.stack(tvs)
    v = np.fmax.reduce(tvs, axis=0) if mutant == "nan_dropped" else np.max(tvs, axis=0)
    e_v = np.max(e_tvs, axis=0)
    with np.errstate(divide="ignore", invalid="ignore"):
        raw = (v - m) / (m * m)
        mf, rf = _f64(np.abs(m)), _f64(np.abs(raw))
        e_alpha = (e_v + e_m + U * (_f64(np.abs(v)) + mf)) / (mf * mf) + rf * (2 * e_m / mf + 3 * U)
    alpha = np.fmax(raw, dtype(MIN_DISP)) if mutant == "nan_dropped" else np.maximum(raw, dtype(MIN_DISP))
    return alpha, e_alpha, m, e_m, v


def reference(case, dtype=LD, mutant=None, genes=None):
    """Cook's distances (N, G'), robust dispersions and the two decisions of the genes `genes` (all by default) of a case
    (cooks_cases.py: counts, sf, X, mu, hat, cutoff), with their bounds and exemptions.  dtype=np.float64 gives a plain float64
    implementation, with `mutant` (a key of MUTANTS) a wrong one."""
    sel = slice(None) if genes is None else np.asarray(genes)
    X = case["X"]
    N, p = X.shape
    y = case["counts"][:, sel]
    mu, h = case["mu"][:, sel].astype(dtype), case["hat"][:, sel].astype(dtype)
    yl = y.astype(dtype)
    x = yl / case["sf"].astype(dtype)[:, None]
    cells, global_mode = cells_of(X)
    alpha, e_alpha, _, _, _ = dispersions(x, cells, global_mode, dtype, mutant)
    V = mu + alpha[None, :] * mu * mu
    pd = dtype(p - 1 if mutant == "p_minus_1" else p)
    with np.errstate(divide="ignore", invalid="ignore"):
        ck = (yl - mu) ** 2 / V / pd * (h / (dtype(1) - h) ** 2)
        muf = _f64(mu)
        e_ck = _f64(np.abs(ck)) * (COOKS_C * EPS + e_alpha[None, :] * muf * muf / _f64(V))
    cutoff = case["cutoff"]
    ckf = _f64(ck)
    replaced = (ckf > cutoff).any(axis=0)
    use = np.zeros(N, dtype=bool)
    if not global_mode:
        use[np.concatenate(cells)] = True
    cand = (ckf[use] > cutoff).any(axis=0)
    G = ckf.shape[1]
    if mutant == "last_argmax":
        pos = N - 1 - np.argmax(ckf[::-1], axis=0)
    else:
        pos = np.argmax(ckf, axis=0)  # numpy: the first maximum, or the first NaN
    cols = np.arange(G)
    ypos = y[pos, cols]
    larger = ((y >= ypos) if mutant == "larger_or_equal" else (y > ypos)).sum(axis=0)
    outlier = cand & (larger < 3)
    # exemptions: a deciding distance within its bound of the cutoff, or an argmax rival within bound that decides differently
    with np.errstate(invalid="ignore"):
        near_cut = np.abs(ckf - cutoff) <= e_ck
        best, e_best = ckf[pos, cols], e_ck[pos, cols]
        rival = (best[None, :] - ckf <= e_best[None, :] + e_ck) & (ckf != best[None, :])
    rival_flip = np.zeros(G, dtype=bool)
    for g in np.flatnonzero(cand & rival.any(axis=0)):
        small = np.array([(y[:, g] > y[j, g]).sum() < 3 for j in np.flatnonzero(rival[:, g])])
        rival_flip[g] = (small != (larger[g] < 3)).any()
    exempt_outlier = (near_cut[use].any(axis=0)) | (cand & rival_flip)
    exempt_replaced = near_cut.any(axis=0)
    return {"cooks": ck, "e_cooks": e_ck, "disp": alpha, "e_disp": e_alpha, "outlier": outlier, "replaced": replaced,
            "exempt_outlier": exempt_outlier, "exempt_replaced": exempt_replaced, "global_mode": global_mode, "pos": pos}


def as_result(ref):
    """A reference's values in float64, in the (cooks, disp, outlier, replaced) form the kernels return."""
    return _f64(ref["cooks"]), _f64(ref["disp"]), ref["outlier"].copy(), ref["replaced"].copy()


def _ratio(got, want, bound):
    """Per entry error / bound; inf where the NaN patterns differ, 0 for exact agreement (a zero bound demands it)."""
    want = _f64(want)
    got = np.asarray(got, dtype=np.float64)
    nan_w, nan_g = np.isnan(want), np.isnan(got)
    err = np.abs(got - want)
    err[nan_w | nan_g] = 0.0
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(err == 0.0, 0.0, err / bound)
    r[nan_w != nan_g] = np.inf
    return r


def ratios(got, ref):
    """{"disp": (G,), "cooks": (N, G) or None} error / bound, and the genes whose decisions differ outside the exemptions."""
    ck, disp, outlier, replaced = got
    rd = _ratio(disp, ref["disp"], ref["e_disp"])
    d = np.asarray(disp, dtype=np.float64)
    rd[~np.isnan(d) & (d < MIN_DISP)] = np.inf
    rc = None if ck is None else _ratio(ck, ref["cooks"], ref["e_cooks"])
    bad_o = (np.asarray(outlier, dtype=bool) != ref["outlier"]) & ~ref["exempt_outlier"]
    bad_r = (np.asarray(replaced, dtype=bool) != ref["replaced"]) & ~ref["exempt_replaced"]
    return {"disp": rd, "cooks": rc}, {"outlier": bad_o, "replaced": bad_r}


def worst(r):
    return 0.0 if r is None or r.size == 0 else float(np.max(r))


def check(got, ref, what):
    """Every value within its bound and every decision equal outside the exemptions; returns the worst ratios and the number of
    exempted genes."""
    r, bad = ratios(got, ref)
    for q, a in r.items():
        if a is not None and not worst(a) <= 1.0:
            idx = np.unravel_index(int(np.argmax(a)), a.shape)
            raise AssertionError(f"{what}: {q} is {worst(a):.3g} x its bound at {tuple(int(i) for i in idx)}")
    for q, b in bad.items():
        if b.any():
            raise AssertionError(f"{what}: {q} differs from the reference at genes {np.flatnonzero(b)[:10].tolist()}")
    return {"disp": worst(r["disp"]), "cooks": worst(r["cooks"]),
            "exempt": int((ref["exempt_outlier"] | ref["exempt_replaced"]).sum())}
