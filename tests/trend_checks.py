"""Extended-precision reference and checks of the dispersion trend + prior launch (pdq_trend.cuh: trend_fit_outer, trend_prior /
trend_prior_dev), of the fitted dispersions k_trend_eval builds from its record and of select_disp's outlier rule.  Used by
test_gpu_trend_ref.py on the device, and by test_trend_checks.py on the CPU to show that the checks accept the host emulator
and the pinned records and reject subtly wrong results.

`reference` restates the semantics, not a solver's path, in np.longdouble (team_checks.require_longdouble) on exactly the doubles
handed to the kernel:
  * one fit (default_inference.py:200-230) is the exact minimiser of mean(t/m + log m), m = c0 + c1 x, under c >= 1e-12: Newton
    (Fisher scoring where the Hessian is indefinite) on the covariate less its smallest value, then the KKT conditions on the
    edges c0 = 1e-12 and c1 = 1e-12.  A covariate that is exactly constant identifies m only: the fit is then the minimiser
    nearest its start, start + (mean(t) - m_start) (1, x) / (1 + x^2).  Fewer than two genes make no fit (not converged);
  * the outer loop of dds.py:1199-1275: first round from (1, 1), stop on sum log(c / old)^2 < 1e-6, failure when a fit does not
    converge or a coefficient is <= 1e-10, drop a gene when its ratio to the round's fit is < 1e-4 or >= 15; targets clipped to
    [min_disp, max_disp]; genes whose covariate is NaN or infinite are left out;
  * the prior (dds.py:840-884, utils.py:1210-1227): residuals log(clip(gw)) - log(c0 + c1 / mean) over the genes with clipped
    genewise >= 100 min_disp and a mean that is not NaN, exact medians, MAD / norm.ppf(0.75) squared,
    prior_var = max(sq - trigamma, 0.25) with NaN propagating;
  * the consumers: fitted = c0 + c1 / mean, and select_disp's outlier rule log(gw) > log(fitted) + 2 sqrt(sq) (dds.py:918-932).
The same code in float64, with one of MUTANTS switched on, makes the wrong results the checks must reject.

Bounds are first-order error propagation computed from the reference's own values (eps = 2^-52):
  * each gradient sum of n terms carries SUM_C n eps sum |term| (any summation order) plus TERM_C eps per term for the fast
    reciprocal and the products that build it; the coefficients carry |H^-1| times that, plus the stopping rule's 1e-12 relative
    step; a coefficient on its bound is exact, and only the free one is bounded (its 1-D curvature);
  * a residual log(t) - log(fit) carries LOG_C eps (|log t| + |log fit|) plus the fit's relative error; an order statistic moves
    by at most the largest perturbation of its inputs, so the MAD moves by at most twice the largest residual error.
Decisions (status, rounds, genes used, prior genes, every select_disp flag) must match exactly, except where the deciding value
lies within its bound of its threshold: those are counted ("exempt").  A value exactly on its threshold is decided by the rule."""
import math

import numpy as np

from team_checks import require_longdouble

LD = require_longdouble()
EPS = 2.0 ** -52
LB = 1e-12
SUM_C = 2.0
TERM_C = 8.0
LOG_C = 4.0
STOP_REL = 1e-12
FIELDS = ("c0", "c1", "status", "n_outer", "n_used", "n_iter", "loss", "last_converged", "squared_logres", "prior_var", "n_above")

MUTANTS = {
    "gt_15": "> instead of >= at a ratio of 15",
    "le_1e4": "<= instead of < at a ratio of 1e-4",
    "drop_prev_round": "drops computed against the previous round's fit",
    "gt_100_min_disp": "> instead of >= at 100 min_disp",
    "upper_median": "the upper median alone for an even count",
    "mad_1_4826": "the MAD scaled by 1.4826 instead of 1 / norm.ppf(0.75)",
    "no_floor": "no 0.25 floor on the prior variance",
    "floor_eats_nan": "a floor that swallows NaN (np.fmax)",
    "unclipped_residuals": "residuals against the unclipped genewise",
    "c0_off_1e9": "c0 off by 1e-9 relative",
}
# the threshold variants change a decision only at a ratio exactly on 15 or 1e-4; drop_rule is checked on such ratios directly
RULE_MUTANTS = ("gt_15", "le_1e4")


def _f64(a):
    return np.asarray(a, dtype=np.float64)


def mad_scale(dtype):
    # 1 / norm.ppf(0.75) = 1 / (sqrt(2) erfinv(1/2)) to 25 digits
    return dtype("1.482602218505601860547076") if dtype is LD else dtype(1.4826022185056018)


# ---- one fit ----------------------------------------------------------------------------------------------------------------
def _sums(x, t, c0, c1, xc):
    m = c0 + c1 * x
    r = t / m
    z = x - xc
    gi = (1 - r) / m
    hi = (2 * r - 1) / (m * m)
    fi = 1 / (m * m)
    g = np.array([gi.sum(), (gi * z).sum()])
    H = np.array([[hi.sum(), (hi * z).sum()], [(hi * z).sum(), (hi * z * z).sum()]])
    F = np.array([[fi.sum(), (fi * z).sum()], [(fi * z).sum(), (fi * z * z).sum()]])
    return (r + np.log(m)).sum(), g, H, F, m


def _solve(M, g):
    det = M[0, 0] * M[1, 1] - M[0, 1] * M[1, 0]
    return np.array([-(M[1, 1] * g[0] - M[0, 1] * g[1]) / det, -(M[0, 0] * g[1] - M[1, 0] * g[0]) / det])


def _pd(M):
    return M[0, 0] > 0 and M[0, 0] * M[1, 1] - M[0, 1] ** 2 > 0


def _newton(x, t, c, xc, free, dt):
    """Damped Newton / Fisher on the coordinates `free` ((0, 1), (0,) or (1,)) in (c0 + c1 xc, c1); returns c."""
    c = np.array(c, dtype=dt)
    for _ in range(200):
        L, g, H, F, _ = _sums(x, t, c[0], c[1], xc)
        gc = np.array([g[0], g[1] + xc * g[0]])  # d/dc
        if free == (0, 1):
            M = H if _pd(H) else F
            e = _solve(M, g)
            d = np.array([e[0] - xc * e[1], e[1]])
        else:
            i = free[0]
            # curvature in c_i alone: sum w, or sum w x^2 = sum w (z + xc)^2
            M = H if H[0, 0] > 0 and H[0, 0] * xc * xc + 2 * H[0, 1] * xc + H[1, 1] > 0 else F
            curv = M[0, 0] if i == 0 else M[0, 0] * xc * xc + 2 * M[0, 1] * xc + M[1, 1]
            d = np.zeros(2, dtype=dt)
            d[i] = -gc[i] / curv
        step = dt(1)
        for _ in range(80):
            n = c + step * d
            with np.errstate(invalid="ignore", divide="ignore"):
                Ln = _sums(x, t, n[0], n[1], xc)[0] if (n[0] + n[1] * x > 0).all() else dt(np.inf)
            if Ln <= L + dt(1e-4) * step * (gc @ d):
                break
            step /= 2
        else:
            return c
        done = np.all(np.abs(n - c) <= dt(1e3) * dt(np.finfo(dt).eps) * np.abs(n))
        c = n
        if done:
            return c
    return c


def fit_once(x, t, start, dtype=LD):
    """The exact minimiser of one fit: (c (2,), converged, kind) with kind 'interior', 'c0_bound', 'c1_bound', 'corner' or
    'degenerate' (constant covariate)."""
    dt = dtype
    x, t = np.asarray(x, dtype=dt), np.asarray(t, dtype=dt)
    start = np.asarray(start, dtype=dt)
    if len(x) < 2:
        return start.copy(), False, "too_few"
    lb = dt(LB)
    if x.min() == x.max():
        xv = x[0]
        m_star = t.mean()
        c = start + (m_star - (start[0] + start[1] * xv)) / (1 + xv * xv) * np.array([dt(1), xv])
        if (c >= lb).all():
            return c, True, "degenerate"
        # the nearest minimiser on a bound
        c = np.array([lb, (m_star - lb) / xv]) if c[0] < lb else np.array([m_star - lb * xv, lb])
        return c, True, "c0_bound" if c[0] == lb else "c1_bound"
    xc = x.min()
    c = _newton(x, t, start, xc, (0, 1), dt)
    if (c >= lb).all() and np.isfinite(c).all():
        return c, True, "interior"
    cands = []
    for i, kind in ((0, "c1_bound"), (1, "c0_bound")):
        s0 = np.array([t.mean(), lb]) if i == 0 else np.array([lb, t.mean() / x.mean()])
        ci = _newton(x, t, s0, xc, (i,), dt)
        if ci[i] < lb:
            continue
        _, g, _, _, _ = _sums(x, t, ci[0], ci[1], xc)
        gc = np.array([g[0], g[1] + xc * g[0]])
        if gc[1 - i] >= 0:  # KKT: the bound coefficient is pushed outward
            cands.append((_sums(x, t, ci[0], ci[1], xc)[0], kind, ci))
    if not cands:
        return np.array([lb, lb]), True, "corner"
    _, kind, c = min(cands, key=lambda v: v[0])
    return c, True, kind


def coeff_bound(x, t, c, kind):
    """First-order bound of a fit's coefficients at the minimiser c (float64 (2,)); for 'degenerate' the bound of m = c0 + c1 x
    in entry 0."""
    x, t = np.asarray(x, dtype=LD), np.asarray(t, dtype=LD)
    m = c[0] + c[1] * x
    r = t / m
    a = _f64((np.abs(r) + 1) / np.abs(m))
    xf = np.abs(_f64(x))
    n = len(x)
    eg = (SUM_C * n * EPS + TERM_C * EPS) * np.array([a.sum(), (a * xf).sum()])
    w = _f64(1 / (m * m))
    F = np.array([[w.sum(), (w * xf).sum()], [(w * xf).sum(), (w * xf * xf).sum()]])  # curvature at the minimiser: t/m ~ 1
    cf = np.abs(_f64(c))
    if kind == "degenerate":
        return np.array([eg[0] / F[0, 0] + STOP_REL * abs(float(m[0])), np.inf])
    if kind == "interior":
        Hs = _f64(_sums(x, t, c[0], c[1], LD(0))[2])
        M = Hs if _pd(Hs) else F
        inv = np.abs(np.linalg.inv(M))
        return inv @ eg + STOP_REL * cf
    e = np.zeros(2)
    i = 0 if kind == "c1_bound" else 1
    e[i] = eg[i] / F[i, i] + STOP_REL * cf[i]
    return e


# ---- the outer loop and the prior --------------------------------------------------------------------------------------------
def drop_rule(ratio, dtype=LD, mutant=None):
    """dds.py:1255-1265: a gene leaves the fit when its ratio to the round's fit is < 1e-4 or >= 15."""
    lo = ratio <= dtype(1e-4) if mutant == "le_1e4" else ratio < dtype(1e-4)
    hi = ratio > dtype(15) if mutant == "gt_15" else ratio >= dtype(15)
    return lo | hi


def outer(x, t, dtype=LD, mutant=None, outer_loop=True):
    """dds.py:1199-1275 on prepared vectors: x covariate (float64), t clipped targets (NaN = not fitted).  Returns a dict."""
    dt = dtype
    ok = np.isfinite(x) & ~np.isnan(t)
    idx = np.flatnonzero(ok)
    old, c = np.array([dt(0.1), dt(0.1)]), np.array([dt(1), dt(1)])
    prev = None
    rounds, status, last_conv, kind = 0, 0, False, None
    exempt = 0
    info = []
    while True:
        with np.errstate(divide="ignore"):
            crit = (np.log(np.abs(c / old)) ** 2).sum()
        if not ((c > dt(1e-10)).all() and crit >= dt(1e-6)):
            break
        old = c
        c, conv, kind = fit_once(x[idx], t[idx], c, dt)
        rounds += 1
        last_conv = conv
        eb = coeff_bound(x[idx], t[idx], c, kind) if conv else np.full(2, np.inf)
        info.append((idx.copy(), c.copy(), kind, eb))
        if not conv or (c <= dt(1e-10)).any():
            status = 1
            break
        if not outer_loop:
            break
        basis = prev if (mutant == "drop_prev_round" and prev is not None) else c
        mfit = basis[0] + basis[1] * np.asarray(x[idx], dtype=dt)
        ratio = np.asarray(t[idx], dtype=dt) / mfit
        # exemptions: a ratio within its bound of a threshold (a degenerate fit bounds m directly), unless it lies on the
        # threshold exactly in this precision
        em = eb[0] if kind == "degenerate" else eb[0] + eb[1] * np.abs(_f64(x[idx]))
        er = np.abs(_f64(ratio)) * (em / np.abs(_f64(mfit)) + 2 * EPS)
        near = np.zeros(len(idx), dtype=bool)
        for thr in (15, 1e-4):
            near |= (np.abs(_f64(ratio - dt(thr))) <= er) & (ratio != dt(thr))
        exempt += int(near.sum())
        prev = c
        idx = idx[~drop_rule(ratio, dt, mutant)]
    # the stop rule near its threshold
    if rounds >= 2 and status == 0:
        with np.errstate(divide="ignore"):
            lg = np.abs(_f64(np.log(np.abs(c / old))))
        e_rel = info[-1][3] / np.abs(_f64(c)) + info[-2][3] / np.abs(_f64(old))
        if not np.isfinite(e_rel).all():
            e_rel = np.where(np.isfinite(e_rel), e_rel, 0.0) + 1e-12
        if abs(float(crit) - 1e-6) <= 2 * float((lg * e_rel).sum()) + 1e-15:
            exempt += 1
    return {"c": c, "status": status, "n_outer": rounds, "n_used": len(idx), "last_converged": last_conv, "kind": kind,
            "bound": info[-1][3] if info else np.full(2, np.inf), "idx": idx, "exempt": exempt, "x": x, "t": t,
            "rounds": [v[1] for v in info]}


def _median(v, mutant=None):
    v = np.sort(v)
    n = len(v)
    if n == 0:
        return v.dtype.type(np.nan)
    if n % 2 or mutant == "upper_median":
        return v[n // 2]
    return (v[n // 2 - 1] + v[n // 2]) / 2


def prior(means, gw, min_disp, max_disp, trigamma_c, c, dtype=LD, mutant=None):
    """(sq, prior_var, n_above, residuals (NaN = not in the prior), the residuals' bound) at coefficients c."""
    dt = dtype
    tc = np.clip(gw, min_disp, max_disp)
    above = tc > 100 * min_disp if mutant == "gt_100_min_disp" else tc >= 100 * min_disp
    use = above & ~np.isnan(means)
    tv = np.asarray(gw if mutant == "unclipped_residuals" else tc, dtype=dt)[use]
    mv = np.asarray(means, dtype=dt)[use]
    fit = dt(c[0]) + dt(c[1]) / mv
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.log(tv) - np.log(fit)
        er = LOG_C * EPS * (np.abs(_f64(np.log(tv))) + np.abs(_f64(np.log(fit)))) + 3 * EPS
    med = _median(r, mutant)
    scale = dt(1.4826) if mutant == "mad_1_4826" else mad_scale(dt)
    mad = _median(np.abs(r - med), mutant) * scale
    sq = mad * mad
    pv = sq - dt(trigamma_c)
    if mutant == "floor_eats_nan":
        pv = np.fmax(pv, dt(0.25))
    elif mutant != "no_floor":
        pv = np.maximum(pv, dt(0.25))
    return sq, pv, int(use.sum()), r, er


def prepare(means, gw, min_disp, max_disp, x_is_mean=True, clip=True):
    with np.errstate(divide="ignore"):
        x = 1.0 / means if x_is_mean else np.asarray(means, dtype=np.float64)
    t = np.clip(gw, min_disp, max_disp) if clip else np.asarray(gw, dtype=np.float64).copy()
    t = np.where(np.isfinite(x), t, np.nan)
    return x, t


def reference(case, dtype=LD, mutant=None):
    """The trend + prior record of a case (means, gw, min_disp, max_disp, trigamma_c) with its bounds and exemptions."""
    means, gw, min_disp, max_disp, trig = case
    x, t = prepare(means, gw, min_disp, max_disp)
    o = outer(x, t, dtype, mutant)
    c = o["c"]
    if mutant == "c0_off_1e9":
        c = c.copy()
        c[0] *= dtype(1 + 1e-9)
        o["c"] = c
    o["loss"] = _loss(x, t, o["idx"], c) if o["status"] == 0 or o["last_converged"] else np.nan
    if o["status"] == 0:
        sq, pv, n_above, r, er = prior(means, gw, min_disp, max_disp, trig, c, dtype, mutant)
        o.update(sq=sq, prior_var=pv, n_above=n_above)
    else:
        o.update(sq=np.nan, prior_var=np.nan, n_above=np.nan)
    o["case"] = case
    return o


def _loss(x, t, idx, c):
    m = LD(c[0]) + LD(c[1]) * np.asarray(x[idx], dtype=LD)
    return (np.asarray(t[idx], dtype=LD) / m + np.log(m)).mean()


def as_record(ref):
    """A reference's values in the 16-double TrendOut layout (n_iter = 1)."""
    rec = np.zeros(16)
    rec[0], rec[1] = _f64(ref["c"])
    rec[2], rec[3], rec[4], rec[5] = ref["status"], ref["n_outer"], ref["n_used"], 1.0
    rec[6] = float(ref["loss"])
    rec[7] = 1.0 if ref["last_converged"] else 0.0
    rec[8], rec[9], rec[10] = float(ref["sq"]), float(ref["prior_var"]), float(ref["n_above"])
    return rec


def _ratio(got, want, bound):
    got, want = float(got), float(want)
    if np.isnan(got) or np.isnan(want):
        return 0.0 if np.isnan(got) and np.isnan(want) else np.inf
    err = abs(got - want)
    return 0.0 if err == 0.0 else (err / bound if bound > 0 else np.inf)


def check_record(rec, ref, what):
    """Every decision equal (outside the exemptions) and every value within its bound; returns the worst ratio per quantity and
    the number of exemptions."""
    rec = np.asarray(rec, dtype=np.float64)
    ex = ref["exempt"]
    # An exempt drop or stop decision changes the genes of every later round, and so the rounds, the genes used, the status and
    # the loss's gene set downstream of it: the whole chain of decisions is then not comparable, only the values at the record's
    # own coefficients are.  The kernel keeps its drop and prior masks in scratch: they are compared through n_used, n_above
    # and the coefficients, which a swapped drop moves far outside their bounds (see the drop_prev_round variant).
    if ex == 0:
        assert rec[2] == ref["status"], f"{what}: status {rec[2]} != {ref['status']}"
        assert rec[3] == ref["n_outer"], f"{what}: {rec[3]} outer rounds != {ref['n_outer']}"
        assert rec[4] == ref["n_used"], f"{what}: {rec[4]} genes used != {ref['n_used']}"
    assert rec[5] > 0, f"{what}: no iteration counted"
    assert np.isfinite(rec[:2]).all(), f"{what}: coefficients {rec[:2]}"
    # last_converged: 1 whenever the fit reached a minimiser, interior or on a bound
    assert rec[7] == (1.0 if ref["last_converged"] else 0.0), f"{what}: last_converged {rec[7]}"
    assert rec[2] == 0.0 or not (rec[7] == 1.0 and (rec[:2] > 1e-10).all()), f"{what}: a converged interior fit reported failure"
    out = {}
    c, eb, kind = _f64(ref["c"]), ref["bound"], ref["kind"]
    if ref["last_converged"]:
        out["c"] = coeff_ratio(rec[:2], ref)
        # the loss at the record's own coefficients
        x, t, idx = ref["x"], ref["t"], ref["idx"]
        m = rec[0] + rec[1] * np.asarray(x[idx], dtype=LD)
        terms = np.asarray(t[idx], dtype=LD) / m + np.log(m)
        el = (SUM_C * len(idx) * EPS + TERM_C * EPS) * float(np.abs(terms).mean())
        out["loss"] = _ratio(rec[6], terms.mean(), el) if ex == 0 else 0.0
    if ref["status"] != 0 or rec[2] != 0:
        assert rec[2] == ref["status"] or ex, f"{what}: status"
        assert np.isnan(rec[8]) and np.isnan(rec[9]), f"{what}: a failed fit carries a prior"
        return _verdict(out, ex, what)
    out.update(prior_ratios(rec[:2], rec[8], rec[9], rec[10], ref, what))
    return _verdict(out, ex, what)


def prior_ratios(cg, sq_got, pv_got, n_above_got, ref, what):
    """squared_logres and prior_var of coefficients cg against the prior recomputed at cg, and against the reference's prior
    through the residuals' sensitivity to the coefficients; n_above exactly (None: not reported)."""
    means, gw, min_disp, max_disp, trig = ref["case"]
    c, eb, kind = _f64(ref["c"]), ref["bound"], ref["kind"]
    rec = np.array([cg[0], cg[1], 0, 0, 0, 0, 0, 0, sq_got, pv_got], dtype=np.float64)
    out = {}
    # the prior at the record's own coefficients ...
    sq, pv, n_above, r, er = prior(means, gw, min_disp, max_disp, trig, rec[:2])
    if n_above_got is not None:
        assert n_above_got == n_above, f"{what}: {n_above_got} prior genes != {n_above}"
    e_sq = _sq_bound(sq, er)
    out["sq"] = _ratio(rec[8], sq, e_sq)
    out["prior_var"] = _pv_ratio(rec[9], pv, sq, trig, e_sq, what)
    # ... and at the reference's, through the residuals' sensitivity to the coefficients
    sq2, pv2, _, _, er2 = prior(means, gw, min_disp, max_disp, trig, ref["c"])
    use = (np.clip(gw, min_disp, max_disp) >= 100 * min_disp) & ~np.isnan(means)
    mv = np.asarray(means, dtype=np.float64)[use]
    if kind == "degenerate":
        efit = eb[0] / np.abs(c[0] + c[1] / mv)
    else:
        efit = (eb[0] + eb[1] / np.abs(mv)) / np.abs(c[0] + c[1] / mv)
    e_sq2 = _sq_bound(sq2, er2 + efit)
    out["sq_ref"] = _ratio(rec[8], sq2, e_sq2)
    out["prior_var_ref"] = _pv_ratio(rec[9], pv2, sq2, trig, e_sq2, what)
    return out


def _verdict(out, ex, what):
    for q, v in out.items():
        assert v <= 1.0, f"{what}: {q} is {v:.3g} x its bound"
    out["exempt"] = ex
    return out


def coeff_ratio(c, ref):
    """Worst error / bound of coefficients c against the last fit of an `outer` result: m = c0 + c1 x for a constant covariate,
    the free coefficient alone (and the bound one exactly) on a bound."""
    eb, kind = ref["bound"], ref["kind"]
    if kind == "degenerate":
        x0 = ref["x"][ref["idx"]][0]
        return _ratio(c[0] + c[1] * x0, float(LD(ref["c"][0]) + LD(ref["c"][1]) * LD(x0)), eb[0])
    rs = []
    for i in (0, 1):
        if eb[i] == 0.0:  # on its bound: exact
            rs.append(0.0 if c[i] == LB else np.inf)
        else:
            rs.append(_ratio(c[i], _f64(ref["c"][i]), eb[i]))
    return max(rs)


def _sq_bound(sq, er):
    if len(er) == 0 or np.isnan(float(sq)):
        return 0.0
    mad = math.sqrt(float(sq))
    e_mad = 2 * float(np.max(er[np.isfinite(er)], initial=0.0)) * 1.4826022185056018 + 4 * EPS * mad
    return 2 * mad * e_mad + e_mad ** 2 + 2 * EPS * float(sq)


def _pv_ratio(got, pv, sq, trig, e_sq, what):
    pv = float(pv)
    if np.isnan(pv):
        assert np.isnan(got), f"{what}: prior_var {got} where NaN is due"
        return 0.0
    raw = float(sq) - trig
    if abs(raw - 0.25) <= e_sq + 2 * EPS:  # at the floor, either side is right
        return 0.0 if abs(got - max(raw, 0.25)) <= e_sq + 2 * EPS else np.inf
    return _ratio(got, pv, e_sq + 2 * EPS * abs(pv))


# ---- the consumers -------------------------------------------------------------------------------------------------------------
def check_fitted(fitted, rec, means, what):
    """fitted = c0 + c1 / mean at the record's coefficients: two roundings."""
    with np.errstate(divide="ignore", invalid="ignore"):
        want = LD(rec[0]) + LD(rec[1]) / np.asarray(means, dtype=LD)
    bound = 2 * EPS * np.abs(_f64(want))
    with np.errstate(invalid="ignore"):
        err = np.abs(np.asarray(fitted) - _f64(want))
    nan_ok = np.isnan(fitted) == np.isnan(_f64(want))
    assert nan_ok.all(), f"{what}: NaN pattern of fitted"
    with np.errstate(invalid="ignore", divide="ignore"):
        r = np.where(err == 0, 0.0, err / bound)
    r = r[~np.isnan(r)]
    w = float(r.max(initial=0.0))
    assert w <= 1.0, f"{what}: fitted is {w:.3g} x its bound"
    return w


def select_reference(gw, mp, fitted, sq, lo, hi, mutant=None):
    """(dispersions, outlier flags, exempt mask) of select_disp (dds.py:918-932) at the given fitted values and sq."""
    g = np.clip(gw, lo, hi).astype(LD)
    m = np.clip(mp, lo, hi)
    with np.errstate(divide="ignore", invalid="ignore"):
        lhs = np.log(g)
        rhs = np.log(np.asarray(fitted, dtype=LD)) + 2 * np.sqrt(LD(sq))
        out = lhs > rhs
        e = LOG_C * EPS * (np.abs(_f64(lhs)) + np.abs(_f64(rhs)) + 1.0)
        # a value exactly on the threshold in long double, or an infinite one, is decided by the rule
        exempt = (np.abs(_f64(lhs - rhs)) <= e) & (lhs != rhs) & np.isfinite(_f64(lhs - rhs))
    disp = np.where(out, _f64(g), m)
    return disp, out, exempt


def check_select(disp, outlier, gw, mp, fitted, sq, lo, hi, what):
    want, out, exempt = select_reference(gw, mp, fitted, sq, lo, hi)
    bad = (np.asarray(outlier, dtype=bool) != out) & ~exempt
    assert not bad.any(), f"{what}: outlier flags differ at {np.flatnonzero(bad)[:10].tolist()}"
    ok = ~exempt
    assert np.array_equal(np.asarray(disp)[ok], want[ok]), f"{what}: dispersions differ"
    return int(exempt.sum())
