"""Inputs, extended-precision references and checks of the team building blocks of pdq_team.cuh (the wide-design kernels'
cooperative linear algebra and collectives).  Used by test_gpu_team.py on the GPU probe's team unit, and by test_team_checks.py
on the CPU to show the checks accept correctly rounded float64 results and reject subtly wrong ones.

Every reference is computed at test time from seeded inputs in np.longdouble (64-bit significand: eps 1.08e-19, 2048 times
finer than float64), so no fixture is needed.  The matrices handed to the kernels are doubles, and the references are of
exactly those doubles.

Three kinds of check:
  * backward errors of the factor and the solve, which do not depend on the condition number and are the sharp checks;
  * forward errors against the reference, in the forms of test_gpu_math.spd_bounds;
  * bit-identity: the primitives that give every entry a fixed sequential operation order whoever owns it must return the
    same bits at every team width W, and every team total must be the same in every thread.  A missing barrier or a wrong
    owner breaks these long before a normwise bound notices."""
import math

import numpy as np

EPS = 2.0 ** -52
# Backward errors ||A - L L^T||_F <= c p eps ||A||_F and ||b - A x|| <= c p eps ||A|| ||x||.  Cholesky's componentwise backward
# error is (p + 1) eps |L||L^T| and, for the solve, (3p + 1) eps |L||L^T|; for an SPD matrix (|L||L^T|)_ij <= sqrt(a_ii a_jj),
# so in norm the worst case is p eps trace(A) ~ p^1.5 eps ||A||_F, while rounding errors that do not conspire give ~ sqrt(p)
# eps ||A||.  c = 4 leaves room for that (the H100's team kernels measure at most 0.13 of it, LAPACK's float64 results 0.22)
# and still rejects one entry of L off by 1e-9 relative by four orders of magnitude.
BACKWARD_C = 4.0
# Forward errors: test_gpu_math.spd_bounds' constant, c p eps times kappa (solve, inverse) or the sum of the magnitudes of
# the terms (products, sums); N replaces p for the accumulators, whose sums run over the samples.  The logdet bound adds to
# spd_bounds' kappa_eq term the rounding of its own sum, 2 sum_i log L_ii over p terms: c p eps sum_i 2 |log L_ii|.  Without
# it, kappa = 1 at p = 101 measured 1.25 x the bound on the H100 (there logdet = p log(lambda) is large and kappa_eq is 1);
# at the narrow tier's p <= 16 the term never mattered.
FORWARD_C = 8.0
# Team<W>::sum: five butterfly levels and W - 1 additions across the warps, each adding at most eps times the partial sums'
# magnitudes, bounded by sum |v|.
SUM_LEVELS = 5

P_LIST = [1, 2, 16, 17, 31, 32, 33, 63, 64, 65, 80, 96, 97, 101, 127, 128]
WARPS = [1, 2, 4, 8]
KAPPAS = [1.0, 1e4, 1e8, 1e12]
N_LIST = [1, 2, 31, 32, 33, 63, 64, 65, 255, 256, 257, 8000]  # and 10 p + 1 (acc_sizes)
RIDGE = 1e-6  # the IRLS ridge (kRidge), and the Wald ridge of the design-like problems


def require_longdouble():
    """np.longdouble, when it is at least the x87 / IEEE quad format; the references are meaningless in plain float64."""
    eps = float(np.finfo(np.longdouble).eps)
    if eps > 1.1e-19:
        raise RuntimeError(f"the team references need an extended-precision np.longdouble (eps <= 1.1e-19); this platform's "
                           f"has eps = {eps:.3g}")
    return np.longdouble


LD = require_longdouble()


# ---- packed storage --------------------------------------------------------------------------------------------------
def packed(M):
    """Lower triangle of (..., p, p), row by row: the kernels' tri(i, j) order."""
    p = M.shape[-1]
    i, j = np.tril_indices(p)
    return M[..., i, j]


def unpack(a, p, dtype=None):
    """Symmetric (..., p, p) from packed lower triangles."""
    a = np.asarray(a)
    M = np.zeros(a.shape[:-1] + (p, p), dtype=dtype or a.dtype)
    i, j = np.tril_indices(p)
    M[..., i, j] = a
    M[..., j, i] = a
    return M


def unpack_lower(a, p, dtype=None):
    a = np.asarray(a)
    M = np.zeros(a.shape[:-1] + (p, p), dtype=dtype or a.dtype)
    i, j = np.tril_indices(p)
    M[..., i, j] = a
    return M


# ---- inputs ----------------------------------------------------------------------------------------------------------
def random_spd(p, kappa, rng):
    """Geometric spectrum from 1 to 1 / kappa (times a random scale) in a random orthogonal basis, as make_math_golden.py
    builds the narrow tier's cases."""
    Q, _r = np.linalg.qr(rng.normal(size=(p, p)))
    lam = np.geomspace(1.0, 1.0 / kappa, p) * np.exp(rng.normal())
    A = (Q * lam) @ Q.T
    return (A + A.T) / 2


def nb_weights(n, rng):
    mu = np.exp(rng.normal(3.0, 1.5, n))
    return mu / (1.0 + mu * 0.1)


def paired_design(p, rng):
    """Intercept, p - 2 subject indicators and a condition: p - 1 subjects with one sample per condition (p >= 3)."""
    S = p - 1
    X = np.zeros((2 * S, p))
    X[:, 0] = 1.0
    for s in range(1, S):
        X[2 * s:2 * s + 2, s] = 1.0
    X[1::2, p - 1] = 1.0
    return X


def levels_design(p, rng):
    """Intercept and p - 1 level indicators of a p-level factor, three samples per level."""
    X = np.zeros((3 * p, p))
    X[:, 0] = 1.0
    for lv in range(1, p):
        X[3 * lv:3 * lv + 3, lv] = 1.0
    return X


def continuous_design(p, rng, N=None):
    """Intercept, a covariate on the scale of 1e3 and alternating indicator / standard normal columns."""
    N = N or max(4 * p, 12)
    X = np.ones((N, p))
    if p > 1:
        X[:, 1] = rng.normal(0.0, 1e3, N)
    for j in range(2, p):
        X[:, j] = rng.integers(0, 2, N) if j % 2 else rng.normal(size=N)
    return X


def xtwx(X, w):
    return packed((X.T * w) @ X)


def spd_inputs(p, seed=0):
    """Two batches of problems for k_team_spd: "scalar" (ridge added to the diagonal; the Wald inverse of A alone) and "tri"
    (a packed ridge triangle, used by the factor and by the Wald inverse).  Each: name, A, b, S, P, c, ridge / ridge_tri."""
    rng = np.random.default_rng([seed, p])
    sc = [(f"kappa={k:g}", packed(random_spd(p, k, rng)), 0.0) for k in KAPPAS]
    tr = []
    if p >= 3:
        X = paired_design(p, rng)
        tr.append(("paired", xtwx(X, nb_weights(X.shape[0], rng))))
    if p >= 2:
        X = levels_design(p, rng)
        w = nb_weights(X.shape[0], rng)
        w[X[:, p - 1] == 1.0] = 1e-10  # a level without a single count
        M = xtwx(X, w)
        sc.append(("empty_level", M, RIDGE))
        tr.append(("empty_level", M))
    X = continuous_design(p, rng)
    M = xtwx(X, nb_weights(X.shape[0], rng))
    sc.append(("continuous", M, RIDGE))
    tr.append(("continuous", M))

    def batch(names, A, ridge, ridge_tri):
        n = len(names)
        A = np.array(A)
        return {"names": names, "A": A, "b": rng.normal(size=(n, p)) * np.exp(rng.normal(size=(n, 1))),
                "S": packed(unpack(rng.normal(size=A.shape), p)), "P": rng.normal(size=(n, p, p)),
                "c": rng.normal(size=(n, p)), "ridge": np.asarray(ridge, dtype=np.float64), "ridge_tri": ridge_tri}

    ridge_tri = np.broadcast_to(packed(np.eye(p) * RIDGE), (len(tr), p * (p + 1) // 2)).copy()
    return {"scalar": batch([s[0] for s in sc], [s[1] for s in sc], [s[2] for s in sc], None),
            "tri": batch([t[0] for t in tr], [t[1] for t in tr], np.zeros(len(tr)), ridge_tri)}


def pivot_inputs(p, seed=0):
    """SPD matrices (kappa 100) whose pivot m is made negative, for m = 0, p // 2 and p - 1: (A packed, b, m)."""
    rng = np.random.default_rng([seed, p, 7])
    As, bs, ms = [], [], sorted({0, p // 2, p - 1})
    for m in ms:
        A = random_spd(p, 100.0, rng)
        if m:
            d = A[m, m] - A[m, :m] @ np.linalg.solve(A[:m, :m], A[:m, m])
        else:
            d = A[0, 0]
        A[m, m] -= d + abs(d)  # Schur complement pivot -|d|
        As.append(packed(A))
        bs.append(rng.normal(size=p))
    return np.array(As), np.array(bs), ms


def acc_sizes(p):
    return sorted(set(N_LIST + [10 * p + 1]))


def acc_inputs(p, N, seed=0):
    """A design (N, p) and three weight / response sets: log-uniform weights from 1e-10 to 1e6 with exact zeros, IRLS-like
    weights, and weights of exactly 1e6; responses of mixed sign and scale.  Above 2000 samples only the first set: the
    longdouble reference is a plain loop (8 s per set at p = 128, N = 8000)."""
    rng = np.random.default_rng([seed, p, N])
    X = continuous_design(p, rng, N)
    w = np.empty((3, N))
    w[0] = np.exp(rng.uniform(np.log(1e-10), np.log(1e6), N))
    w[0, rng.random(N) < 0.2] = 0.0
    w[1] = nb_weights(N, rng)
    w[2] = 1e6
    z = rng.normal(size=(3, N)) * np.exp(rng.uniform(-5, 5, (3, N)))
    k = 1 if N > 2000 else 3
    return X, w[:k], z[:k]


# ---- extended-precision references -----------------------------------------------------------------------------------
def chol_ld(A):
    """Lower Cholesky factor of a (p, p) longdouble matrix (NaN from a non-positive pivot on)."""
    A = np.asarray(A, dtype=LD)
    p = A.shape[0]
    L = np.zeros_like(A)
    with np.errstate(invalid="ignore"):
        for j in range(p):
            d = A[j, j] - L[j, :j] @ L[j, :j]
            L[j, j] = np.sqrt(d)
            L[j + 1:, j] = (A[j + 1:, j] - L[j + 1:, :j] @ L[j, :j]) / L[j, j]
    return L


def lower_inverse_ld(L):
    p = L.shape[0]
    Li = np.zeros_like(L)
    eye = np.eye(p, dtype=LD)
    for i in range(p):
        Li[i] = (eye[i] - L[i, :i] @ Li[:i]) / L[i, i]
    return Li


def spd_reference(batch, p):
    """Per problem, in longdouble: Ae = A + ridge, its factor, x = Ae^-1 b, H = Ae^-1, logdet Ae, A b, P b, sum A_ij S_ij and
    the Wald SE sqrt(c^T H_w A H_w c) (H_w = (A + ridge_tri)^-1, or A^-1 in the scalar batch); plus kappa(Ae), the equilibrated
    kappa and the magnitudes the forward bounds need."""
    n = len(batch["names"])
    A = unpack(batch["A"], p).astype(LD)
    out = {k: [] for k in ("Ae", "x", "H", "logdet", "logdet_terms", "matvec", "pinv", "symdot", "se", "q_scale", "kappa",
                           "kappa_eq", "kappa_w")}
    for g in range(n):
        if batch["ridge_tri"] is not None:
            R = unpack(batch["ridge_tri"][g], p).astype(LD)
            Rw = R
        else:
            R = np.eye(p, dtype=LD) * LD(batch["ridge"][g])
            Rw = np.zeros((p, p), dtype=LD)
        Ae = A[g] + R
        L = chol_ld(Ae)
        Li = lower_inverse_ld(L)
        H = Li.T @ Li
        b = batch["b"][g].astype(LD)
        out["Ae"].append(Ae)
        out["x"].append(H @ b)
        out["H"].append(H)
        out["logdet"].append(2 * np.log(np.diag(L)).sum())
        out["logdet_terms"].append(float(2 * np.abs(np.log(np.diag(L))).sum()))
        out["matvec"].append(A[g] @ b)
        out["pinv"].append(batch["P"][g].astype(LD) @ b)
        out["symdot"].append((A[g] * unpack(batch["S"][g], p).astype(LD)).sum())
        Aw = A[g] + Rw
        Hw = lower_inverse_ld(chol_ld(Aw))
        Hw = Hw.T @ Hw
        u = Hw @ batch["c"][g].astype(LD)
        out["se"].append(np.sqrt(u @ (A[g] @ u)))
        u64 = np.abs(u.astype(np.float64))
        out["q_scale"].append(np.linalg.norm(u64) * np.linalg.norm(np.abs(A[g].astype(np.float64)) @ u64))
        Ae64 = Ae.astype(np.float64)
        d = np.sqrt(np.diag(Ae64))
        out["kappa"].append(np.linalg.cond(Ae64))
        out["kappa_eq"].append(np.linalg.cond(Ae64 / d[:, None] / d[None, :]))
        out["kappa_w"].append(np.linalg.cond(Aw.astype(np.float64)))
    return out


def acc_reference(X, w, z):
    """X^T W X (packed) and X^T z in longdouble, and the sums of the magnitudes of their terms."""
    Xl = X.astype(LD)
    M = np.stack([packed((Xl.T * wi.astype(LD)) @ Xl) for wi in w])
    v = np.stack([Xl.T @ zi.astype(LD) for zi in z])
    Xa = np.abs(X)
    Ms = np.stack([packed((Xa.T * np.abs(wi)) @ Xa) for wi in w])
    vs = np.abs(z) @ Xa
    return {"M": M, "v": v, "M_scale": Ms, "v_scale": vs}


# ---- checks ----------------------------------------------------------------------------------------------------------
def _fail(what, ratio, names):
    i = int(np.nanargmax(np.where(np.isfinite(ratio), ratio, np.inf)))
    raise AssertionError(f"{what}: problem {names[i]!r} is {ratio[i]:.3g} x its bound")


def spd_ratios(got, batch, ref, p):
    """Error / bound of every quantity of every problem (<= 1 passes).  `got` is a TeamProbe.spd result: the per-thread
    scalars are taken from thread 0 (check_team_identical covers the others)."""
    n = len(batch["names"])
    k = FORWARD_C * p * EPS
    r = {q: np.empty(n) for q in ("factor", "solve_backward", "solve", "inverse", "logdet", "matvec", "symdot", "quad",
                                  "pinv", "wald_se")}
    A = unpack(batch["A"], p)
    for g in range(n):
        Ae = ref["Ae"][g]
        nA = float(np.linalg.norm(Ae.astype(np.float64)))
        L = unpack_lower(got["L"][g], p).astype(LD)
        r["factor"][g] = float(np.linalg.norm((Ae - L @ L.T).astype(np.float64))) / (BACKWARD_C * p * EPS * nA)
        x = got["x"][g]
        res = Ae @ x.astype(LD) - batch["b"][g].astype(LD)
        n2 = float(np.linalg.norm(Ae.astype(np.float64), 2))
        r["solve_backward"][g] = float(np.linalg.norm(res.astype(np.float64))) / (BACKWARD_C * p * EPS * n2 * np.linalg.norm(x))
        xr = ref["x"][g]
        r["solve"][g] = float(np.linalg.norm((x - xr).astype(np.float64)) / np.linalg.norm(xr.astype(np.float64))) / (k * ref["kappa"][g])
        H = ref["H"][g]
        Hg = unpack(got["H"][g], p)
        r["inverse"][g] = float(np.linalg.norm((Hg - H).astype(np.float64)) / np.linalg.norm(H.astype(np.float64))) / (k * ref["kappa"][g])
        r["logdet"][g] = float(abs(got["logdet"][g, 0] - ref["logdet"][g])) / (k * (max(ref["kappa_eq"][g], 1.0) + ref["logdet_terms"][g]))
        b = batch["b"][g]
        r["matvec"][g] = float(np.max(np.abs(got["matvec"][g] - ref["matvec"][g]).astype(np.float64) / (k * (np.abs(A[g]) @ np.abs(b)) + 1e-300)))
        r["pinv"][g] = float(np.max(np.abs(got["pinv"][g] - ref["pinv"][g]).astype(np.float64) / (k * (np.abs(batch["P"][g]) @ np.abs(b)) + 1e-300)))
        S = unpack(batch["S"][g], p)
        r["symdot"][g] = float(abs(got["symdot"][g, 0] - ref["symdot"][g])) / (k * float(np.abs(A[g] * S).sum()) + 1e-300)
        # quad_w(H, b) against the exact quadratic form of the H the kernel returned: the check of quad_w alone
        bl = b.astype(LD)
        qx = bl @ (Hg.astype(LD) @ bl)
        r["quad"][g] = float(abs(got["quad"][g, 0] - qx)) / (k * float(np.abs(b) @ np.abs(Hg) @ np.abs(b)) + 1e-300)
        # SE^2 = u^T A u, u = H_w c: u carries kappa(A + ridge) eps of relative error, which ||u|| || |A| |u| || bounds
        se = got["se"][g, 0]
        r["wald_se"][g] = float(abs(LD(se) * LD(se) - ref["se"][g] ** 2)) / (k * ref["kappa_w"][g] * ref["q_scale"][g] + 1e-300)
    return r


def check_spd(got, batch, ref, p):
    """Every quantity within its bound; returns the worst ratio of each."""
    worst = {}
    for q, ratio in spd_ratios(got, batch, ref, p).items():
        if not (np.isfinite(ratio).all() and ratio.max() <= 1.0):
            _fail(f"{q}, p = {p}", ratio, batch["names"])
        worst[q] = float(ratio.max())
    return worst


def acc_ratios(got, ref, N):
    """Worst error / bound of X^T W X and X^T z per weight set: c N eps times the sums of the magnitudes of the terms."""
    k = FORWARD_C * max(N, 1) * EPS
    rM = np.abs(got["M"] - ref["M"]).astype(np.float64) / (k * ref["M_scale"] + 1e-300)
    rv = np.abs(got["v"] - ref["v"]).astype(np.float64) / (k * ref["v_scale"] + 1e-300)
    return {"xtwx": rM.max(axis=1), "xtwz": rv.max(axis=1)}


def check_acc(got, ref, N, p):
    worst = {}
    for q, ratio in acc_ratios(got, ref, N).items():
        if not (np.isfinite(ratio).all() and ratio.max() <= 1.0):
            raise AssertionError(f"{q}, p = {p}, N = {N}: worst error {np.max(ratio):.3g} x its bound")
        worst[q] = float(ratio.max())
    return worst


def check_team_identical(scal, what):
    """Every thread of a team holds the same bits of a team-wide value (scal: (problems, threads))."""
    s = np.asarray(scal)
    same = (s.view(np.int64) == s[:, :1].view(np.int64)).all(axis=1)
    if not same.all():
        g = int(np.flatnonzero(~same)[0])
        t = int(np.flatnonzero(s[g].view(np.int64) != s[g, 0].view(np.int64))[0])
        raise AssertionError(f"{what}: thread {t} of problem {g} holds {s[g, t]!r}, thread 0 {s[g, 0]!r}")


def check_w_invariant(by_w, keys, what):
    """by_w: {W: result dict}; the arrays under `keys` are bit-identical across the team widths (NaNs included)."""
    ws = sorted(by_w)
    for key in keys:
        a = np.ascontiguousarray(by_w[ws[0]][key])
        for W in ws[1:]:
            b = np.ascontiguousarray(by_w[W][key])
            diff = a.view(np.int64) != b.view(np.int64)
            if diff.any():
                idx = np.unravel_index(int(np.flatnonzero(diff)[0]), a.shape)
                raise AssertionError(f"{what}: {key} differs between W = {ws[0]} and W = {W} at {idx}: {a[idx]!r} vs {b[idx]!r}")


def pivot_pattern(p, m):
    """NaN pattern of the packed factor when pivot m is the first non-positive one: the columns from m on."""
    i, j = np.tril_indices(p)
    return j >= m


# ---- collectives -----------------------------------------------------------------------------------------------------
MAXN = 300


def coll_inputs(W, seed=0):
    """One block per vector length 1..300 (wdot / wmaxabs), each with its own five collective inputs of 32 W values and
    votes, of every kind: random signs over 40 binades, all equal, few distinct values, NaN lanes in the max inputs (all of
    them in some blocks), a single voter anywhere in the block, none."""
    rng = np.random.default_rng([seed, W])
    NT, count = 32 * W, MAXN
    v = rng.normal(size=(count, 5, NT)) * np.exp(rng.uniform(-20, 20, (count, 5, NT)))
    kind = np.arange(count) % 6
    v[kind == 1] = 3.25
    v[kind == 2] = rng.integers(-2, 3, v[kind == 2].shape)
    mx = v[:, [1, 3]]
    mx[rng.random(mx.shape) < 0.1] = np.nan
    mx[kind == 3] = np.nan
    mx[kind == 4, 0, :] = -np.inf
    v[:, [1, 3]] = mx
    flag = (rng.random((count, NT)) < 0.01).astype(np.int32)
    flag[kind == 1] = 0
    flag[kind == 5] = 0
    one = np.flatnonzero(kind == 5)
    flag[one, rng.integers(0, NT, one.size)] = 1
    flag[one[::2], NT - 1] = 1  # the last thread of the last warp
    lens = np.arange(1, count + 1)
    a = rng.normal(size=(count, MAXN)) * np.exp(rng.uniform(-10, 10, (count, MAXN)))
    b = rng.normal(size=(count, MAXN))
    nan_rows = np.flatnonzero(kind == 4)
    a[nan_rows, rng.integers(0, lens[nan_rows])] = np.nan  # wmaxabs ignores NaN (fmax); wdot propagates it
    return {"v": v, "flag": flag, "a": a, "b": b, "lens": lens}


def check_coll(out, inp, W):
    """out (count, 8, 32 W) from TeamProbe.coll.  Sums: the same bits in every thread, within (5 + W) eps sum|v| of the exact
    sum.  Max: exactly np.fmax.reduce (NaN lanes ignored, all-NaN gives NaN).  Any: the exact vote of the block.  wdot: the
    same bits in every thread, within (ceil(n / 32 W) + 5 + W) eps sum |a_j b_j|.  wmaxabs: exactly max(0, fmax |a_j|)."""
    NT = 32 * W
    v, flag, a, b, lens = inp["v"], inp["flag"], inp["a"], inp["b"], inp["lens"]
    for col in range(8):
        check_team_identical(out[:, col, :], f"W = {W}, output {col}")
    o = out[:, :, 0]
    for col, src in ((0, 0), (2, 2), (5, 4)):
        for g in range(v.shape[0]):
            x = v[g, src]
            err = abs(o[g, col] - math.fsum(x))
            bound = (SUM_LEVELS + W) * EPS * float(np.abs(x).sum())
            if not err <= bound:
                raise AssertionError(f"W = {W}: sum #{col} of block {g} off by {err:.3g} (bound {bound:.3g})")
    for col, src in ((1, 1), (4, 3)):
        want = np.fmax.reduce(v[:, src], axis=1)
        np.testing.assert_array_equal(o[:, col], want, err_msg=f"W = {W}: max #{col}")
    np.testing.assert_array_equal(o[:, 3] != 0, flag.any(axis=1), err_msg=f"W = {W}: any")
    for g in range(v.shape[0]):
        n = int(lens[g])
        t = a[g, :n] * b[g, :n]
        if np.isnan(t).any():
            if not np.isnan(o[g, 6]):
                raise AssertionError(f"W = {W}: wdot of block {g} ignores a NaN component")
        else:
            err = abs(o[g, 6] - math.fsum(t))
            bound = (-(-n // NT) + SUM_LEVELS + W) * EPS * float(np.abs(t).sum())
            if not err <= bound:
                raise AssertionError(f"W = {W}: wdot over n = {n} off by {err:.3g} (bound {bound:.3g})")
        want = np.fmax.reduce(np.abs(a[g, :n]), initial=0.0)
        if not (o[g, 7] == want or (np.isnan(want) and np.isnan(o[g, 7]))):
            raise AssertionError(f"W = {W}: wmaxabs over n = {n} is {o[g, 7]!r}, want {want!r}")
