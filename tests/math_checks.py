"""Accuracy checks of the FP64 building blocks (pdq_fast.cuh, pdq_math.cuh, the per-gene tables of pdq_gene.cuh) against the
high-precision references of tests/golden/math_ref.npz (scripts/make_math_golden.py).  Shared by the host-branch tests
(test_math_ref.py, through the emulator) and the device-branch tests (test_gpu_math.py, through the GPU probe): `ops` is
anything with `elem(op, x, y=None)` and `tables(r, T)`."""
import numpy as np

from conftest import load_golden

EPS = 2.0 ** -52
# op codes of tests/gpu_probe/math_ops.h, in order
OPS = {name: i for i, name in enumerate(
    ["fast_rcp", "fast_div", "fast_log", "fast_log_nb", "fast_exp", "fast_exp_nb", "tlog", "tlog_nb", "texp", "texp_nb",
     "lgamma_pos", "digamma_pos", "trigamma_pos", "lgamma_digamma_pos.lg", "lgamma_digamma_pos.dg", "lgamma_asym",
     "digamma_asym", "trigamma_asym", "norm_sf"])}

# documented worst cases, in ulps of the correctly rounded result
ULP_BOUNDS = {"fast_log": 2.0, "fast_log_nb": 2.0, "tlog": 1.5, "tlog_nb": 1.5,
              "fast_exp": 2.0, "fast_exp_nb": 2.0, "texp": 1.5, "texp_nb": 1.5,
              "fast_rcp": 1.0, "fast_div": 1.0}
ULP_REF = {"fast_log": "log", "fast_log_nb": "log", "tlog": "log", "tlog_nb": "log", "fast_exp": "exp", "fast_exp_nb": "exp",
           "texp": "exp", "texp_nb": "exp", "fast_rcp": "rcp", "fast_div": "div"}
# special functions: |err| <= atol + rtol |f|  (lgamma / digamma: the bounds of test_emu_parity.py::test_special_functions)
SF_BOUNDS = {"lgamma_pos": ("lgamma", 2e-14, 3e-14), "digamma_pos": ("digamma", 2e-14, 3e-14),
             "trigamma_pos": ("trigamma", 4e-15, 0.0), "lgamma_digamma_pos.lg": ("lgamma", 2e-14, 3e-14),
             "lgamma_digamma_pos.dg": ("digamma", 2e-14, 3e-14), "lgamma_asym": ("lgamma", 2e-14, 3e-14),
             "digamma_asym": ("digamma", 2e-14, 3e-14), "trigamma_asym": ("trigamma", 4e-15, 0.0)}
TABLE_C = 4.0  # constant of the tables' forward-error bounds

_REF = None


def ref():
    """The fixture, with each `*_lou` (remainder in ulps of `*_hi`, float16) decoded into `*_lo` (the double-double's low part)."""
    global _REF
    if _REF is None:
        z = load_golden("math_ref")
        for key in [k for k in z if k.endswith("_lou")]:
            hi = z[key[:-4] + "_hi"]
            ulp = np.maximum(np.ldexp(1.0, np.frexp(np.abs(hi))[1] - 53), 2.0 ** -1074)
            z[key[:-1]] = z.pop(key).astype(np.float64) * ulp
        _REF = z
    return _REF


def ulp_err(got, hi, lo):
    """|got - (hi + lo)| in ulps of the exact value (hi, lo), to within the fixture's 2^-11 ulp resolution of lo."""
    hi, lo = np.asarray(hi, dtype=np.float64), np.asarray(lo, dtype=np.float64)
    m, e = np.frexp(np.abs(hi))
    ulp = np.ldexp(1.0, e - 53)
    ulp = np.where((m == 0.5) & (lo * np.sign(hi) < 0), ulp / 2, ulp)  # exact value just below a power of two
    ulp = np.maximum(ulp, 2.0 ** -1074)
    with np.errstate(invalid="ignore"):
        return np.abs((got - hi) - lo) / ulp


def inputs(name):
    z = ref()
    kind = ULP_REF[name]
    if kind == "div":
        return z["div_a"], z["div_b"], z["div_hi"], z["div_lo"]
    x = z[kind + "_x"]
    return x, None, z[kind + "_hi"], z[kind + "_lo"]


def check_ulp(ops, name):
    """Worst error of `name` over the fixture's inputs, in ulps; fails above the documented bound."""
    x, y, hi, lo = inputs(name)
    err = ulp_err(ops.elem(OPS[name], x, y), hi, lo)
    assert not np.isnan(err).any(), f"{name}: non-finite result at x = {x[np.isnan(err)][:5]}"
    i = int(np.argmax(err))
    where = f"x = {x[i]!r}" + ("" if y is None else f", y = {y[i]!r}")
    assert err[i] <= ULP_BOUNDS[name], f"{name}: {err[i]:.3f} ulp > {ULP_BOUNDS[name]} at {where}"
    return float(err[i])


def check_special(ops, name):
    """Worst |err| / (atol + rtol |f|) of a special function over the fixture's inputs (<= 1 passes)."""
    z = ref()
    key, rtol, atol = SF_BOUNDS[name]
    x = z["sf_x"]
    keep = x >= 10.0 if name.endswith("_asym") else np.ones(x.size, dtype=bool)
    x, hi, lo = x[keep], z[key + "_hi"][keep], z[key + "_lo"][keep]
    got = ops.elem(OPS[name], x, np.log(x))  # the *_asym series take log(x) as their second argument
    err = np.abs((got - hi) - lo)
    ratio = err / (atol + rtol * np.abs(hi))
    assert np.isfinite(ratio).all(), f"{name}: non-finite result"
    i = int(np.argmax(ratio))
    assert ratio[i] <= 1.0, f"{name}: error {err[i]:.3g} at x = {x[i]!r} (bound atol {atol:g} + rtol {rtol:g} |f|)"
    return float(np.max(err / np.maximum(np.abs(hi), 1.0)))


def norm_sf_bound(x):
    """Relative bound of 0.5 erfc(x / sqrt 2): a few ulps of erfc, plus the rounding of x / sqrt 2 (relative error <= eps)
    amplified by the condition number of erfc, 2 t^2 = x^2 in the tail."""
    return (8.0 + 1.5 * x * x) * EPS


def check_norm_sf(ops):
    z = ref()
    x, hi, lo = z["nsf_x"], z["nsf_hi"], z["nsf_lo"]
    assert hi.min() < 1e-300  # the fixture reaches the far tail
    got = ops.elem(OPS["norm_sf"], x)
    rel = np.abs((got - hi) - lo) / hi
    ratio = rel / norm_sf_bound(x)
    i = int(np.argmax(ratio))
    assert ratio[i] <= 1.0, f"norm_sf: relative error {rel[i]:.3g} at x = {x[i]!r}"
    return float(rel.max())


def table_refs():
    """(r, [(name, column offset in the probe output, exact (G, 32), bound (G, 32))]) for the four tables of math_ops.h."""
    z = ref()
    r = z["tab_r"]
    k = np.arange(32)
    lg, psi, tri = z["tab_lgamma"], z["tab_psi"], z["tab_tri"]  # nearest doubles: the bounds are many ulps wide
    rk = r[:, None] + k[None, :]

    def excl(a):
        return np.concatenate([np.zeros((a.shape[0], 1)), np.cumsum(a, axis=1)[:, :-1]], axis=1)

    # entry k = f(r) -/+ sum_{j<k} term(r + j): the start value's own error plus, per addition, eps times the magnitudes involved
    def bound(f0_err, f0, terms):
        return f0_err[:, None] + TABLE_C * EPS * (k[None, :] + 1) * (np.abs(f0)[:, None] + excl(np.abs(terms)))

    b_lg = bound(3e-14 + 2e-14 * np.abs(lg[:, 0]), lg[:, 0], np.log(rk))
    b_psi = bound(3e-14 + 2e-14 * np.abs(psi[:, 0]), psi[:, 0], 1.0 / rk)
    b_tri = bound(4e-15 * tri[:, 0], tri[:, 0], rk ** -2.0)
    return r, [("lgamma", 0, lg, b_lg), ("psi", 32, psi, b_psi), ("psi_tri", 64, psi, b_psi), ("psi'", 96, tri, b_tri)]


def check_tables(out, r, refs, T):
    """Worst |err| / bound per table (<= 1 passes) for tables built by T lanes."""
    worst = {}
    for name, off, exact, bnd in refs:
        got = out[:, off:off + 32]
        ratio = np.abs(got - exact) / bnd
        assert np.isfinite(ratio).all(), f"{name} table, T = {T}: non-finite entry"
        g, k = np.unravel_index(int(np.argmax(ratio)), ratio.shape)
        assert ratio[g, k] <= 1.0, (f"{name} table, T = {T}: entry k = {k} at r = {r[g]!r} is {got[g, k]!r}, exact "
                                    f"{exact[g, k]!r} (error {abs(got[g, k] - exact[g, k]):.3g}, bound {bnd[g, k]:.3g})")
        worst[name] = float(ratio[g, k])
    return worst


def check_tables_agree(out, out1, r, refs, T):
    """Tables built by T lanes against those built by one lane, within the same bound."""
    for name, off, _exact, bnd in refs:
        d = np.abs(out[:, off:off + 32] - out1[:, off:off + 32]) / bnd
        assert d.max() <= 1.0, f"{name} table: T = {T} differs from T = 1 by {d.max():.3g} x the bound"


# IEEE / libm semantics of the guarded versions on special inputs
SPECIAL_LOG_X = np.array([0.0, -0.0, -1.0, -1e-300, -np.inf, np.inf, np.nan, 5e-324, 1e-310, 2.2250738585072009e-308,
                          np.finfo(np.float64).max])
SPECIAL_EXP_X = np.array([np.inf, -np.inf, np.nan, 700.0, -700.0, 709.78, 709.8, -708.5, -740.0, -746.0, 800.0, -800.0])


def check_special_inputs(ops):
    """log of <= 0, denormal, inf, NaN and exp of |x| >= 700, inf, NaN through the guarded versions follow np.log / np.exp:
    the same NaN / inf / zero pattern and finite values within 2 ulp."""
    with np.errstate(all="ignore"):
        for names, x, f in ((("fast_log", "tlog"), SPECIAL_LOG_X, np.log), (("fast_exp", "texp"), SPECIAL_EXP_X, np.exp)):
            want = f(x)
            for name in names:
                got = ops.elem(OPS[name], x)
                np.testing.assert_array_equal(np.isnan(got), np.isnan(want), err_msg=f"{name}: NaN pattern, x = {x}")
                fin = np.isfinite(want)
                np.testing.assert_array_equal(got[~fin & ~np.isnan(want)], want[~fin & ~np.isnan(want)], err_msg=name)
                np.testing.assert_array_equal(got[want == 0], want[want == 0], err_msg=name)
                nz = fin & (want != 0)
                err = np.abs(got[nz] - want[nz]) / np.spacing(np.abs(want[nz]))
                assert err.max() <= 2.0, f"{name}: {err.max():.2f} ulp from numpy on special inputs {x[nz]}"


def sweep_worst(ops, n, seed=0):
    """Random sweep of the log / exp ops against np.log / np.exp, in ulps of numpy's result (itself within 1 ulp)."""
    rng = np.random.default_rng(seed)
    xl = np.exp2(rng.uniform(-1022, 1024, n))
    xl[: n // 4] = rng.uniform(0.5, 2.0, n // 4)
    xl = xl[np.isfinite(xl) & (xl >= np.finfo(np.float64).tiny)]
    xe = rng.uniform(-699.9, 699.9, n)
    xe[: n // 4] = rng.uniform(-1.0, 1.0, n // 4)
    out = {}
    for names, x, f in ((("fast_log", "fast_log_nb", "tlog", "tlog_nb"), xl, np.log),
                        (("fast_exp", "fast_exp_nb", "texp", "texp_nb"), xe, np.exp)):
        want = f(x)
        sp = np.spacing(np.abs(want))
        sp = np.where(want == 0, 2.0 ** -1074, sp)
        for name in names:
            out[name] = float(np.max(np.abs(ops.elem(OPS[name], x) - want) / sp))
    return out
