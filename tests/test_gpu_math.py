"""GPU suite (`-m gpu`): the DEVICE branches of the FP64 building blocks, through the GPU probe (tests/gpu_probe), against
high-precision references (tests/golden/math_ref.npz, scripts/make_math_golden.py).

The host emulator compiles the other side of every `#if defined(__CUDA_ARCH__)` (IEEE division for fast_rcp / fast_div, memcpy
bit handling in tlog_nb, ldexp in texp_nb / fast_exp_nb, one-lane collectives), and end-to-end parity is far too coarse to see an
ulp-level regression, so these are the only checks of what the kernels actually execute.  Both probe units run: the default one
(fully unrolled) and the one with the wide units' flags (-DPDQ_TU_P=16 -Xptxas -O1), whose kernels use the same primitives."""
import math

import numpy as np
import pytest

import math_checks as mc

pytestmark = pytest.mark.gpu

UNITS = ["narrow", "wide"]
LANES = [1, 2, 4, 8, 16, 32]


@pytest.fixture(scope="module")
def probes():
    from gpu_probe.probe import Probe

    return {u: Probe(u) for u in UNITS}


@pytest.mark.parametrize("unit", UNITS)
@pytest.mark.parametrize("name", sorted(mc.ULP_BOUNDS))
def test_device_primitive_ulp(probes, unit, name):
    """fast_log / fast_exp and their _nb forms <= 2 ulp, tlog / texp <= 1.5 ulp, fast_rcp / fast_div <= 1 ulp, on every table
    interval end and midpoint, the sqrt(2) splits, exponent edges, the rint half-way points and every residue k & 63."""
    mc.check_ulp(probes[unit], name)


@pytest.mark.parametrize("unit", UNITS)
@pytest.mark.parametrize("name", sorted(mc.SF_BOUNDS))
def test_device_special_function(probes, unit, name):
    mc.check_special(probes[unit], name)


@pytest.mark.parametrize("unit", UNITS)
def test_device_norm_sf(probes, unit):
    mc.check_norm_sf(probes[unit])


@pytest.mark.parametrize("unit", UNITS)
def test_device_special_inputs(probes, unit):
    mc.check_special_inputs(probes[unit])


@pytest.mark.parametrize("unit", UNITS)
def test_device_random_sweep(probes, unit):
    """10^6 random points per op against numpy (itself within 1 ulp): the documented bound plus one ulp."""
    for name, w in mc.sweep_worst(probes[unit], 1_000_000, seed=1).items():
        assert w <= mc.ULP_BOUNDS[name] + 1.0, f"{name}: {w:.3f} ulp from numpy"


@pytest.mark.parametrize("unit", UNITS)
@pytest.mark.parametrize("T", LANES)
def test_device_tables(probes, unit, T):
    """lgamma / psi / psi' tables of one gene per group of T lanes (the kernels' lane layout, stitched with excl_scan): every
    entry within the forward-error bound of its recurrence, and the same within that bound as the single-lane build.  An
    off-by-one in the scan or a lane writing the wrong segment is an error of order one."""
    r, refs = mc.table_refs()
    out = probes[unit].tables(r, T)
    mc.check_tables(out, r, refs, T)
    if T > 1:
        mc.check_tables_agree(out, probes[unit].tables(r, 1), r, refs, T)


def group_values(n_warps, rng):
    """Lane values with groups of every kind: random signs and magnitudes, all equal, repeated extremes, integers (ties)."""
    v = rng.normal(size=n_warps * 32) * np.exp(rng.uniform(-20, 20, n_warps * 32))
    kind = np.arange(n_warps) % 5
    w = v.reshape(n_warps, 32)
    w[kind == 1] = 3.25                                                  # every lane equal
    w[kind == 2] = rng.integers(-2, 3, (int((kind == 2).sum()), 32))     # few distinct values: many tied extremes
    w[kind == 3] = rng.uniform(0, 1, (int((kind == 3).sum()), 32)).round(1)
    flag = (rng.random(n_warps * 32) < 0.02).astype(np.int32)
    fw = flag.reshape(n_warps, 32)
    fw[kind == 4] = 0                                                    # no lane votes
    fw[kind == 1] = 0
    fw[np.flatnonzero(kind == 1), rng.integers(0, 32, int((kind == 1).sum()))] = 1  # exactly one lane votes
    return v, flag


@pytest.mark.parametrize("T", LANES)
def test_device_group_collectives(probes, T):
    """Group::sum / excl_scan / argext / any on every lane: sum bit-identical across the lanes of a group and within
    T eps sum|v| of the exact sum, excl_scan the ordered prefix sums, argext exact with ties to the smaller si, and any the
    exact vote over the whole warp (a superset of the group's: the branches it guards contain full-mask shuffles)."""
    rng = np.random.default_rng(T)
    n_warps = 160
    v, flag = group_values(n_warps, rng)
    res = probes["narrow"].group(T, v, flag)
    gpw = 32 // T
    for wi in range(n_warps):
        for slot in range(gpw):
            lanes = wi * 32 + slot + gpw * np.arange(T)  # ordered by si
            x = v[lanes]
            scale = T * mc.EPS * np.abs(x).sum()
            s = res["sum"][lanes]
            assert (s == s[0]).all(), f"T = {T}: lanes of a group hold different sums {s}"
            assert abs(s[0] - math.fsum(x)) <= scale, (T, s[0], math.fsum(x))
            pre = np.array([math.fsum(x[:i]) for i in range(T)])
            assert res["scan"][lanes][0] == 0.0
            np.testing.assert_array_less(np.abs(res["scan"][lanes] - pre), scale + 1e-300, err_msg=f"excl_scan, T = {T}")
            amin, amax = int(np.flatnonzero(x == x.min())[0]), int(np.flatnonzero(x == x.max())[0])
            assert (res["argmin"][lanes] == amin).all(), (T, x, res["argmin"][lanes])
            assert (res["argmax"][lanes] == amax).all(), (T, x, res["argmax"][lanes])
            assert (res["any"][lanes] == bool(flag[wi * 32:(wi + 1) * 32].any())).all(), (T, wi, flag[wi * 32:(wi + 1) * 32])


def spd_case(P):
    z = mc.ref()
    c = {k: z[f"spd{P}_{k}"] for k in ("A", "b", "x", "inv", "logdet", "quad", "matvec", "dot", "kappa", "kappa_scaled")}
    c["S"] = c["inv"]  # sym_dot's second operand: the rounded exact inverse (the fixture's `dot` is sum A_ij inv_ij)
    return c


def unpack(a, P):
    M = np.empty(a.shape[:-1] + (P, P))
    k = 0
    for i in range(P):
        for j in range(i + 1):
            M[..., i, j] = M[..., j, i] = a[..., k]
            k += 1
    return M


def spd_bounds(c, P):
    """Per-quantity error bounds: solve / inverse normwise c P eps kappa(A); logdet c P eps kappa(D^-1 A D^-1), D = diag(A)^1/2
    (Cholesky's backward error is componentwise, so the equilibrated condition number governs the pivots); the quadratic form,
    matrix-vector product and Frobenius dot c P eps times the sum of the magnitudes of their terms."""
    A, b, S = unpack(c["A"], P), c["b"], unpack(c["S"], P)
    k = 8.0 * P * mc.EPS
    return {"solve": k * c["kappa"], "inv": k * c["kappa"], "logdet": k * np.maximum(c["kappa_scaled"], 1.0),
            "quad": k * np.einsum("ni,nij,nj->n", np.abs(b), np.abs(A), np.abs(b)),
            "matvec": k * np.einsum("nij,nj->ni", np.abs(A), np.abs(b)), "dot": k * np.abs(A * S).sum(axis=(1, 2))}


def spd_errors(got, c, P):
    """Error of each quantity in the units of spd_bounds."""
    x, inv = c["x"], unpack(c["inv"], P)
    return {"solve": np.linalg.norm(got["solve"] - x, axis=1) / np.linalg.norm(x, axis=1),
            "inv": np.linalg.norm(unpack(got["inv"], P) - inv, axis=(1, 2)) / np.linalg.norm(inv, axis=(1, 2)),
            "logdet": np.abs(got["logdet"] - c["logdet"]), "quad": np.abs(got["quad"] - c["quad"]),
            "matvec": np.abs(got["matvec"] - c["matvec"]), "dot": np.abs(got["dot"] - c["dot"])}


@pytest.mark.parametrize("unit", UNITS)
@pytest.mark.parametrize("P", range(1, 17))
def test_device_spd_algebra(probes, unit, P):
    """chol / chol_solve / chol_inverse / chol_logdet / sym_quad / sym_matvec / sym_dot at condition numbers 1 .. 1e12 and on
    design-like X'WX, against mpmath.  The default unit instantiates p = 1..8, the wide-unit build p = 1..16."""
    pr = probes[unit]
    if P > pr.max_p:
        pytest.skip(f"the {unit} unit instantiates p <= {pr.max_p}")
    c = spd_case(P)
    got = pr.spd(P, c["A"], c["b"], c["S"])
    bnd = spd_bounds(c, P)
    for q, err in spd_errors(got, c, P).items():
        ratio = err / bnd[q]
        assert np.isfinite(ratio).all() and ratio.max() <= 1.0, f"{q}, P = {P}: worst error {ratio.max():.3g} x its bound"


@pytest.mark.parametrize("P", range(1, 9))
def test_device_spd_units_agree(probes, P):
    """The unrolled and the looped (wide-unit) code agree within the same bounds; bit equality is not expected, contraction
    into FMAs can differ between them."""
    c = spd_case(P)
    a, b = probes["narrow"].spd(P, c["A"], c["b"], c["S"]), probes["wide"].spd(P, c["A"], c["b"], c["S"])
    bnd = spd_bounds(c, P)
    for q in bnd:
        scale = {"solve": np.linalg.norm(c["x"], axis=1), "inv": np.linalg.norm(unpack(c["inv"], P), axis=(1, 2))}.get(q, 1.0)
        d = np.abs(a[q] - b[q])
        d = np.linalg.norm(d.reshape(d.shape[0], -1), axis=1) / scale if q in ("solve", "inv") else d
        assert (d <= bnd[q]).all(), f"{q}, P = {P}: units differ by {np.max(d / bnd[q]):.3g} x the bound"
