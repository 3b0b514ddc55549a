#!/usr/bin/env python
"""Writes tests/golden/math_ref.npz: high-precision references of the FP64 building blocks of pdq_fast.cuh / pdq_math.cuh /
pdq_gene.cuh, for tests/test_math_ref.py (host branches, through the emulator) and tests/test_gpu_math.py (device branches,
through the GPU probe).  Run once on a machine with mpmath; the fixture is committed.

Every scalar reference is computed with mpmath at 160 bits from the double input and stored as its nearest double `*_hi` and
the remainder in ulps of that double, `*_lou` (float16, |.| <= 1/2: resolved to 2^-11 ulp, far finer than any bound), so the tests can measure
errors in ulps with plain float64 arithmetic.  The table and SPD references are compared against bounds far above an ulp and
keep the nearest double only.  The file stays small (a few hundred kB): dense where the edges are, thin random fill.  The inputs aim at the places where these
routines go wrong -- table-interval ends, the sqrt(2) split of the log tables, exponent edges, the rint half-way points of the exp
reduction, the shift threshold of the special functions -- with random fill on top."""
import os

import mpmath as mp
import numpy as np

mp.mp.prec = 160
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "math_ref.npz")
rng = np.random.default_rng(20261015)
LN2 = np.log(2.0)
TAB_BITS, TAB_N, TAB_SPLIT = 9, 512, 213  # pdq_tables.h


def ulp_of(hi):
    """the spacing of the doubles at |hi| (tests/math_checks.py decodes `*_lou` with the same function)"""
    return np.maximum(np.ldexp(1.0, np.frexp(np.abs(hi))[1] - 53), 2.0 ** -1074)


def dd(f, xs, b=None):
    """(hi, remainder in ulps of hi as float16) of f evaluated in mpmath at each double of xs (and of b)."""
    hi, lo = np.empty(len(xs)), np.empty(len(xs))
    for i, x in enumerate(xs):
        v = f(mp.mpf(float(x))) if b is None else f(mp.mpf(float(x)), mp.mpf(float(b[i])))
        h = float(v)
        hi[i], lo[i] = h, float(v - h)
    lou = (lo / ulp_of(hi)).astype(np.float16)
    assert np.all(np.abs(lou) <= 0.5)
    return hi, lou


def from_bits(hi_word, lo_word):
    u = (np.asarray(hi_word, dtype=np.uint64) << np.uint64(32)) | np.asarray(lo_word, dtype=np.uint64)
    return u.view(np.float64)


def nudge(x, ks):
    """x moved by k ulps for each k of ks (flattened)."""
    x = np.asarray(x, dtype=np.float64)
    out = []
    for k in ks:
        y = x.copy()
        d = np.inf if k > 0 else -np.inf
        for _ in range(abs(k)):
            y = np.nextafter(y, d)
        out.append(y)
    return np.concatenate([np.ravel(o) for o in out])


def log_inputs():
    exps = np.array([-1022, -1, 0, 1023])
    i = np.arange(TAB_N, dtype=np.float64)
    starts = 1.0 + i / TAB_N
    ends = np.nextafter(1.0 + (i + 1) / TAB_N, 0.0)
    mids = 1.0 + (i + 0.5) / TAB_N
    m = np.concatenate([starts, ends, mids])
    xs = [np.ldexp(m[None, :], exps[:, None]).ravel()]
    # the two intervals around the table's sqrt(2) split, densely
    for e in (-1, 0, 5):
        xs.append(np.ldexp(1.0 + (TAB_SPLIT - 1 + rng.uniform(0, 2, 150)) / TAB_N, e))
    # fast_log's own split: high words 0x3ff6a09e / 0x3ff6a09f with low words at both ends and in between
    lo_words = np.concatenate([[0, 1, 0x7fffffff, 0xfffffffe, 0xffffffff], rng.integers(0, 2**32, 10)])
    for hw in (0x3ff6a09e, 0x3ff6a09f, 0x3ff6a0a0):
        base = from_bits(np.full(lo_words.size, hw), lo_words)
        xs.append(np.ldexp(base[None, :], np.array([-1000, -1, 0, 1, 600])[:, None]).ravel())
    xs.append(nudge(np.array([1.0]), range(-64, 65)))  # 1 +- k ulp
    pw = np.ldexp(1.0, np.unique(np.concatenate([np.arange(-1022, 1024, 16), [-1021, -1, 0, 1, 1023]])))
    xs += [pw, nudge(pw, [-1, 1, 2])]
    xs.append(np.array([np.finfo(np.float64).max, np.finfo(np.float64).tiny, np.sqrt(2.0), np.sqrt(0.5), np.e]))
    xs.append(np.exp2(rng.uniform(-1022, 1024, 1000)))
    x = np.concatenate(xs)
    x = x[np.isfinite(x) & (x >= np.finfo(np.float64).tiny)]
    return np.unique(x)


def exp_inputs():
    step = LN2 / 64
    ks = np.concatenate([np.arange(-64 * 4, 64 * 4), rng.integers(-64 * 1009, 64 * 1009, 100)])
    on = ks * step
    half = (ks + 0.5) * step  # rint half-way points of x * 64 / ln2
    xs = [on, half, nudge(half, [-2, -1, 1, 2])]
    edge = np.array([699.99, -699.99, 699.999999, -699.999999, np.nextafter(700.0, 0.0), -np.nextafter(700.0, 0.0), 500.0, -500.0])
    tiny = np.array([1e-300, 1e-200, 2.0 ** -60, 1e-17, 1e-12, 1e-8, 1e-4])
    xs += [edge, tiny, -tiny, [0.0], rng.uniform(-700, 700, 500), rng.uniform(-1, 1, 300), rng.uniform(-1e-3, 1e-3, 100)]
    x = np.concatenate([np.ravel(np.asarray(v, dtype=np.float64)) for v in xs])
    return np.unique(x[np.abs(x) < 700.0])


def edge_mantissas(emin, emax, n_exp):
    """Mantissas next to all zeros and all ones across exponents emin..emax, both signs, plus random ones."""
    e = np.unique(np.concatenate([np.linspace(emin, emax, n_exp).astype(int), [emin, emax, 0, 1, -1]]))
    k = np.arange(0, 6, dtype=np.uint64)
    m_lo = (np.uint64(0x3ff0000000000000) + k).view(np.float64)
    m_hi = (np.uint64(0x3fffffffffffffff) - k).view(np.float64)
    m_rand = 1.0 + rng.random(3)
    m = np.concatenate([m_lo, m_hi, m_rand])
    x = np.ldexp(m[None, :], e[:, None]).ravel()
    return np.concatenate([x, -x])


def special_inputs():
    xs = [np.geomspace(1e-4, 1e9, 500), nudge(np.array([10.0]), [-3, -2, -1, 1, 2, 3]), [10.0, 9.99, 10.01, 9.5, 10.5],
          1.4616321449683623 + np.linspace(-1e-3, 1e-3, 41), 1.0 + np.linspace(-1e-3, 1e-3, 21), 2.0 + np.linspace(-1e-3, 1e-3, 21),
          nudge(np.array([1.0, 2.0]), [-2, -1, 1, 2]), np.arange(1, 41, dtype=np.float64), np.arange(1, 41) - 0.5,
          np.exp(rng.uniform(np.log(1e-4), np.log(1e9), 300))]
    x = np.concatenate([np.ravel(np.asarray(v, dtype=np.float64)) for v in xs])
    return np.unique(x)


def packed(M):
    P = M.shape[0]
    return np.array([M[i, j] for i in range(P) for j in range(i + 1)])


def unpack(a, P):
    M = np.empty((P, P))
    k = 0
    for i in range(P):
        for j in range(i + 1):
            M[i, j] = M[j, i] = a[k]
            k += 1
    return M


def spd_cases(P):
    """SPD matrices at condition numbers 1 .. 1e12 and design-like X'WX with a continuous covariate on the scale of 1e3."""
    mats = []
    for kappa in (1.0, 1e4, 1e8, 1e12):
        Q, _r = np.linalg.qr(rng.normal(size=(P, P)))
        lam = np.geomspace(1.0, 1.0 / kappa, P) * np.exp(rng.normal())
        A = (Q * lam) @ Q.T
        mats.append((A + A.T) / 2)
    N = max(4 * P, 12)
    X = np.ones((N, P))
    if P > 1:
        X[:, 1] = rng.normal(0, 1e3, N)
    for j in range(2, P):
        X[:, j] = rng.integers(0, 2, N) if j % 2 else rng.normal(size=N)
    mu = np.exp(rng.normal(3, 1.5, N))
    w = mu / (1.0 + mu * 0.1)
    mats.append((X.T * w) @ X)
    # sym_dot's second operand is the (rounded) exact inverse, so no other matrix needs storing
    out = {k: [] for k in ("A", "b", "x", "inv", "logdet", "quad", "matvec", "dot", "kappa", "kappa_scaled")}
    for A in mats:
        a = packed(A)
        A = unpack(a, P)  # exactly the doubles the kernels get
        if np.linalg.eigvalsh(A).min() <= 0:
            continue
        b = rng.normal(size=P) * np.exp(rng.normal())
        Am, bm = mp.matrix(A.tolist()), mp.matrix(b.tolist())
        x = mp.lu_solve(Am, bm)
        inv = mp.inverse(Am)
        d = np.sqrt(np.diag(A))
        out["A"].append(a)
        out["b"].append(b)
        out["x"].append([float(x[i]) for i in range(P)])
        S = np.array([[float(inv[i, j]) for j in range(P)] for i in range(P)])
        out["inv"].append(packed(S))
        out["logdet"].append(float(mp.log(mp.det(Am))))
        out["quad"].append(float(mp.fsum(mp.mpf(b[i]) * mp.mpf(A[i, j]) * mp.mpf(b[j]) for i in range(P) for j in range(P))))
        out["matvec"].append([float(mp.fsum(mp.mpf(A[i, j]) * mp.mpf(b[j]) for j in range(P))) for i in range(P)])
        out["dot"].append(float(mp.fsum(mp.mpf(A[i, j]) * mp.mpf(S[i, j]) for i in range(P) for j in range(P))))
        out["kappa"].append(np.linalg.cond(A))
        out["kappa_scaled"].append(np.linalg.cond(A / d[:, None] / d[None, :]))
    return {f"spd{P}_{k}": np.array(v) for k, v in out.items()}


def main():
    z = {}
    z["log_x"] = log_inputs()
    z["log_hi"], z["log_lou"] = dd(mp.log, z["log_x"])
    z["exp_x"] = exp_inputs()
    z["exp_hi"], z["exp_lou"] = dd(mp.exp, z["exp_x"])
    z["rcp_x"] = edge_mantissas(-1000, 999, 24)
    z["rcp_hi"], z["rcp_lou"] = dd(lambda v: 1 / v, z["rcp_x"])
    a = edge_mantissas(-500, 500, 16)
    b = rng.permutation(edge_mantissas(-500, 500, 16))
    z["div_a"], z["div_b"] = a, b
    z["div_hi"], z["div_lou"] = dd(lambda u, v: u / v, a, b)
    z["sf_x"] = special_inputs()
    z["lgamma_hi"], z["lgamma_lou"] = dd(mp.loggamma, z["sf_x"])
    z["digamma_hi"], z["digamma_lou"] = dd(mp.digamma, z["sf_x"])
    z["trigamma_hi"], z["trigamma_lou"] = dd(lambda v: mp.psi(1, v), z["sf_x"])
    z["nsf_x"] = np.unique(np.concatenate([np.linspace(-10, 37.5, 600), rng.uniform(-40, 37.5, 150), [0.0, 1.959963984540054]]))
    z["nsf_hi"], z["nsf_lou"] = dd(lambda v: mp.erfc(v / mp.sqrt(2)) / 2, z["nsf_x"])
    # per-gene tables: r = 1/alpha over alpha in [min_disp, max(10, N)], k < kPsiK
    r = np.unique(np.concatenate([np.geomspace(1e-4, 1e8, 40), [0.5, 1.0, 2.5, 9.99, 10.0, 31.5, 1e-3, 0.1]]))
    z["tab_r"] = r
    for name, f in (("lgamma", mp.loggamma), ("psi", mp.digamma), ("tri", lambda v: mp.psi(1, v))):
        z[f"tab_{name}"] = np.array([[float(f(mp.mpf(float(rg)) + k)) for k in range(32)] for rg in r])
    for P in range(1, 17):
        z.update(spd_cases(P))
    np.savez_compressed(OUT, **z)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
