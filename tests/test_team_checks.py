"""CPU tests of the team checks (tests/team_checks.py) that test_gpu_team.py applies to the GPU probe's team unit: the
longdouble references agree with mpmath, the checks accept correctly rounded float64 results, and they reject the subtly wrong
results a broken team primitive gives -- a perturbed factor entry, swapped rows, a dropped chunk, a value read before the
barrier that publishes it, one thread's total differing in its last bit."""
import math

import numpy as np
import pytest
import scipy.linalg as sl

import team_checks as tc

P_CPU = [1, 2, 17, 33, 64, 97, 128]


def numpy_spd(batch, p, NT=1):
    """The outputs of TeamProbe.spd computed with LAPACK / numpy in float64 (the scalars replicated over NT threads)."""
    out = {k: [] for k in ("L", "x", "H", "Li", "matvec", "pinv", "logdet", "symdot", "quad", "se")}
    for g in range(len(batch["names"])):
        A = tc.unpack(batch["A"][g], p)
        tri = batch["ridge_tri"] is not None
        R = tc.unpack(batch["ridge_tri"][g], p) if tri else np.eye(p) * batch["ridge"][g]
        L = np.linalg.cholesky(A + R)
        Li = sl.solve_triangular(L, np.eye(p), lower=True)
        H = Li.T @ Li
        b = batch["b"][g]
        Hw = np.linalg.inv(A + R) if tri else np.linalg.inv(A)
        u = Hw @ batch["c"][g]
        out["L"].append(tc.packed(L))
        out["Li"].append(tc.packed(Li))
        out["H"].append(tc.packed(H))
        out["x"].append(sl.cho_solve((L, True), b))
        out["matvec"].append(A @ b)
        out["pinv"].append(batch["P"][g] @ b)
        out["logdet"].append([2.0 * np.log(np.diag(L)).sum()] * NT)
        out["symdot"].append([(A * tc.unpack(batch["S"][g], p)).sum()] * NT)
        out["quad"].append([b @ H @ b] * NT)
        out["se"].append([np.sqrt(u @ A @ u)] * NT)
    return {k: np.array(v) for k, v in out.items()}


def chol_team(A, stale=None):
    """chol_w's operation order in float64 (right-looking: per column step j, sqrt of the pivot, scale the column, update the
    trailing triangle; numpy rounds each product where the kernel fuses it into an fma).  `stale` = (j, i, k): at step j,
    entry (i, k) is updated with L[k, j] as it was before step j scaled it -- the value of the previous column step, which a
    missing barrier would let it read."""
    L = np.tril(np.array(A, dtype=np.float64))
    p = L.shape[0]
    for j in range(p):
        old = L[:, j].copy()
        with np.errstate(invalid="ignore"):
            d = np.sqrt(L[j, j])
        L[j + 1:, j] /= d
        L[j, j] = d
        for i in range(j + 1, p):
            col = L[j + 1:i + 1, j].copy()
            if stale is not None and stale[0] == j and stale[1] == i:
                col[stale[2] - (j + 1)] = old[stale[2]]
            L[i, j + 1:i + 1] -= L[i, j] * col
    return L


@pytest.fixture(scope="module")
def cases():
    out = {}
    for p in P_CPU:
        inp = tc.spd_inputs(p)
        out[p] = {m: (b, tc.spd_reference(b, p)) for m, b in inp.items() if b["names"]}
    return out


def test_longdouble_is_extended():
    assert np.finfo(tc.LD).eps <= 1.1e-19


@pytest.mark.parametrize("p", [1, 5, 17, 24])
def test_references_agree_with_mpmath(p):
    """Factor, solve, inverse and logdet of the longdouble references against mpmath at 40 digits, on the kappa = 1e8 and
    design-like problems: within 64 p eps_ld kappa (the references' own rounding), far inside the float64 bounds."""
    mp = pytest.importorskip("mpmath")
    mp.mp.dps = 40
    eps_ld = float(np.finfo(tc.LD).eps)
    for mode, batch in tc.spd_inputs(p).items():
        ref = tc.spd_reference(batch, p)
        for g, name in enumerate(batch["names"]):
            if name not in ("kappa=1e+08", "empty_level", "paired", "continuous"):
                continue
            Ae = ref["Ae"][g]
            Am = mp.matrix([[mp.mpf(float(Ae[i, j])) + mp.mpf(float(Ae[i, j] - LDf(Ae[i, j]))) for j in range(p)] for i in range(p)])
            Lm = mp.cholesky(Am)
            L = tc.chol_ld(Ae)
            tol = 64 * p * eps_ld * ref["kappa"][g]
            assert max(abs(float(L[i, j]) - float(Lm[i, j])) for i in range(p) for j in range(i + 1)) <= tol * float(mp.mnorm(Lm, 1))
            xm = mp.cholesky_solve(Am, mp.matrix([mp.mpf(float(v)) for v in batch["b"][g]]))
            xs = np.array([float(xm[i]) for i in range(p)])
            assert np.linalg.norm(ref["x"][g].astype(np.float64) - xs) <= tol * np.linalg.norm(xs), (mode, name)
            Hm = mp.inverse(Am)
            Hs = np.array([[float(Hm[i, j]) for j in range(p)] for i in range(p)])
            assert np.linalg.norm(ref["H"][g].astype(np.float64) - Hs) <= tol * np.linalg.norm(Hs), (mode, name)
            assert abs(float(ref["logdet"][g]) - float(mp.log(mp.det(Am)))) <= 64 * p * eps_ld * max(ref["kappa_eq"][g], 1.0)


def LDf(x):
    return tc.LD(float(x))


@pytest.mark.parametrize("p", P_CPU)
def test_checks_accept_float64(cases, p):
    """LAPACK / numpy float64 results pass every bound (they are backward stable, as the kernels must be)."""
    for mode, (batch, ref) in cases[p].items():
        worst = tc.check_spd(numpy_spd(batch, p), batch, ref, p)
        assert max(worst.values()) < 0.5, (mode, worst)


@pytest.mark.parametrize("p", [17, 64, 128])
def test_checks_accept_team_order(cases, p):
    """chol_w's own operation order, emulated in float64, passes the factor's backward bound."""
    for mode, (batch, ref) in cases[p].items():
        got = numpy_spd(batch, p)
        for g in range(len(batch["names"])):
            Ae = ref["Ae"][g].astype(np.float64)
            got["L"][g] = tc.packed(chol_team(Ae))
        assert tc.check_spd(got, batch, ref, p)["factor"] < 0.5


def _rejected(fn, match):
    with pytest.raises(AssertionError, match=match):
        fn()


@pytest.mark.parametrize("p", [2, 17, 64, 128])
def test_rejects_perturbed_factor_entry(cases, p):
    """One entry of L off by 1e-9 relative at kappa = 1 (the largest entry of the last row, a diagonal one)."""
    batch, ref = cases[p]["scalar"]
    got = numpy_spd(batch, p)
    k = p * (p + 1) // 2 - 1
    got["L"][0, k] *= 1.0 + 1e-9
    _rejected(lambda: tc.check_spd(got, batch, ref, p), "factor")


@pytest.mark.parametrize("p", [2, 17, 64, 128])
def test_rejects_swapped_inverse_rows(cases, p):
    """Two rows of H swapped (then packed: the lower triangle of the wrong matrix)."""
    batch, ref = cases[p]["scalar"]
    got = numpy_spd(batch, p)
    H = tc.unpack(got["H"][0], p)
    H[[0, p - 1]] = H[[p - 1, 0]]
    got["H"][0] = tc.packed(H)
    _rejected(lambda: tc.check_spd(got, batch, ref, p), "inverse")


@pytest.mark.parametrize("p", [17, 64, 128])
def test_rejects_stale_factor_entry(cases, p):
    """One trailing-update entry computed from the previous column step's value: what a missing barrier between the column
    scaling and the update gives.  At kappa = 1 the off-diagonal entries are rounding noise, so a stale read of one changes
    nothing measurable; every other problem, random or design-like, is rejected (a later pivot may even turn negative).  The
    row is p - 2: the last row of the design with an empty level is ~1e-5 of the rest, where a normwise bound sees nothing --
    the bit-identity across W is what covers it on the GPU."""
    batch, ref = cases[p]["scalar"]
    for g in range(1, len(batch["names"])):
        got = numpy_spd(batch, p)
        j = p // 3
        got["L"][g] = tc.packed(chol_team(ref["Ae"][g].astype(np.float64), stale=(j, p - 2, j + 1)))
        _rejected(lambda: tc.check_spd(got, batch, ref, p), "factor")


@pytest.mark.parametrize("W", tc.WARPS)
@pytest.mark.parametrize("p", [17, 128])
def test_rejects_dropped_last_chunk(p, W):
    """X^T W X and X^T W z without the samples of the last, partial chunk of 32 W."""
    NT = 32 * W
    for N in (NT + 1, 10 * p + 1):
        if N % NT == 0:
            continue
        X, w, z = tc.acc_inputs(p, N)
        ref = tc.acc_reference(X, w, z)
        good = {"M": np.stack([tc.xtwx(X, wi) for wi in w]), "v": z @ X}
        tc.check_acc(good, ref, N, p)
        keep = N - N % NT
        bad = {"M": np.stack([tc.xtwx(X[:keep], wi[:keep]) for wi in w]), "v": z[:, :keep] @ X[:keep]}
        _rejected(lambda: tc.check_acc(bad, ref, N, p), "xtw")


def test_rejects_thread_sum_off_by_one_ulp():
    """One thread's total differing in its last bit: within every bound, but not the same in every thread."""
    for W in tc.WARPS:
        inp = tc.coll_inputs(W)
        out = emulate_coll(inp, W)
        tc.check_coll(out, inp, W)
        out[5, 0, 32 * W - 1] = np.nextafter(out[5, 0, 32 * W - 1], np.inf)
        _rejected(lambda: tc.check_coll(out, inp, W), "thread")


def test_rejects_nan_propagating_max_and_wrong_vote():
    W = 2
    inp = tc.coll_inputs(W)
    out = emulate_coll(inp, W)
    g = int(np.flatnonzero(np.isnan(inp["v"][:, 1]).any(axis=1) & ~np.isnan(inp["v"][:, 1]).all(axis=1))[0])
    bad = out.copy()
    bad[g, 1, :] = np.nan  # max instead of fmax
    _rejected(lambda: tc.check_coll(bad, inp, W), "max")
    bad = out.copy()
    g = int(np.flatnonzero(inp["flag"][:, 32:].any(axis=1) & ~inp["flag"][:, :32].any(axis=1))[0])
    bad[g, 3, :] = 0.0  # the vote of the first warp only
    _rejected(lambda: tc.check_coll(bad, inp, W), "any")


def test_rejects_w_variance():
    a = {"L": np.array([[1.0, 2.0, 3.0]])}
    b = {"L": np.array([[1.0, np.nextafter(2.0, 3.0), 3.0]])}
    tc.check_w_invariant({1: a, 2: {"L": a["L"].copy()}}, ["L"], "same")
    _rejected(lambda: tc.check_w_invariant({1: a, 2: b}, ["L"], "one ulp"), "differs")


def emulate_coll(inp, W):
    """What correct collectives return: correctly rounded sums, fmax, the block's vote, identical in every thread."""
    NT = 32 * W
    v, a, b, lens = inp["v"], inp["a"], inp["b"], inp["lens"]
    count = v.shape[0]
    o = np.empty((count, 8))
    for g in range(count):
        o[g, 0], o[g, 2], o[g, 5] = (math.fsum(v[g, k]) for k in (0, 2, 4))
        o[g, 1], o[g, 4] = np.fmax.reduce(v[g, 1]), np.fmax.reduce(v[g, 3])
        o[g, 3] = float(inp["flag"][g].any())
        n = lens[g]
        t = a[g, :n] * b[g, :n]
        o[g, 6] = np.nan if np.isnan(t).any() else math.fsum(t)
        o[g, 7] = np.fmax.reduce(np.abs(a[g, :n]), initial=0.0)
    return np.repeat(o[:, :, None], NT, axis=2)
