"""CPU suite: the extended-precision reference of the dispersion trend + prior (trend_checks.py) against mpmath and the oracle's
scipy fit; the checks reject subtly wrong variants; the host emulator (pdq_trend.cuh compiled with g++) passes every case; and
every record pinned in tests/golden/trend_prior_ref.npz passes the checks, so that a fixture re-recorded from a broken kernel fails
here."""
import functools

import mpmath
import numpy as np
import pytest

import trend_checks as tk
import trend_prior_cases as tc
from conftest import load_golden
from emu.emu_ops import EmuOps
from oracle import nbglm

CPU_CASES = [n for n in list(tc.CASES) + list(tc.REF_CASES) if n != "plain_1000000"]


@functools.lru_cache(maxsize=None)
def _ref(name):
    return tk.reference(tc.case(name))


@pytest.fixture(scope="module")
def ops():
    return EmuOps()


def _mp_fit(x, t, start):
    """The interior minimiser by Newton in 40-digit arithmetic, from `start`."""
    mpmath.mp.dps = 40
    xs, ts = [mpmath.mpf(float(v)) for v in x], [mpmath.mpf(float(v)) for v in t]
    c = [mpmath.mpf(v) for v in start]
    for _ in range(100):
        g, H = [0, 0], [[0, 0], [0, 0]]
        for xv, tv in zip(xs, ts):
            m = c[0] + c[1] * xv
            gi, hi = (1 - tv / m) / m, (2 * tv / m - 1) / (m * m)
            for a, va in enumerate((1, xv)):
                g[a] += gi * va
                for b, vb in enumerate((1, xv)):
                    H[a][b] += hi * va * vb
        det = H[0][0] * H[1][1] - H[0][1] ** 2
        d = [-(H[1][1] * g[0] - H[0][1] * g[1]) / det, -(H[0][0] * g[1] - H[0][1] * g[0]) / det]
        step = 1
        while any(c[0] + step * d[0] + (c[1] + step * d[1]) * xv <= 0 for xv in xs):
            step /= 2
        c = [c[0] + step * d[0], c[1] + step * d[1]]
        if max(abs(v) for v in d) < mpmath.mpf(10) ** -35 or det == 0:
            break
    return c


@pytest.mark.parametrize("seed", [0, 1, 4])
def test_fit_matches_mpmath(seed):
    rng = np.random.default_rng(seed)
    means = np.exp(rng.normal(3, 1.5, 30))
    x = 1 / means
    t = (3 * x + 0.2) * np.exp(rng.normal(0, 0.4, 30))
    c, conv, kind = tk.fit_once(x, t, np.ones(2))
    assert conv and kind == "interior"
    got = [mpmath.mpf(str(v)) for v in c]
    want = _mp_fit(x, t, [float(v) for v in c])
    for i in (0, 1):
        assert abs(float((got[i] - want[i]) / want[i])) < 1e-16


@pytest.mark.parametrize("name", ["plain_1000", "plain_2000", "scattered_22", "flat_tail_20000"])
def test_fit_matches_oracle_within_lbfgsb_slack(name):
    means, gw, lo, hi, _ = tc.case(name)
    x, t = tk.prepare(means, gw, lo, hi)
    ok = np.isfinite(x) & ~np.isnan(t)
    c, conv, kind = tk.fit_once(x[ok], t[ok], np.ones(2))
    oc, _, oconv = nbglm.dispersion_trend_gamma_glm(x[ok], t[ok])
    assert conv and oconv and kind == "interior"
    np.testing.assert_allclose(np.asarray(c, dtype=np.float64), oc, rtol=1e-4)


def test_constant_covariate_is_the_nearest_minimiser():
    x, t = np.full(50, 0.1), np.random.default_rng(3).uniform(0.1, 1.0, 50)
    c, conv, kind = tk.fit_once(x, t, np.ones(2))
    assert conv and kind == "degenerate"
    assert abs(float(c[0] + c[1] * tk.LD(0.1) - t.astype(tk.LD).mean())) < 1e-18
    assert abs(float((c[0] - 1) * tk.LD(0.1) - (c[1] - 1))) < 1e-18  # moved along (1, x) from the start


# cases on which each wrong variant must be rejected (the variant changes a decision or a value there, and the correct float64
# computation passes on the same case: the control of test_wrong_variants_are_rejected)
MUTANT_CASES = {
    "gt_15": "exact_15", "drop_prev_round": "planted_3001", "gt_100_min_disp": "planted_3001", "upper_median": "plain_1000",
    "mad_1_4826": "plain_1000", "no_floor": "dof_2", "floor_eats_nan": "no_prior", "unclipped_residuals": "clipped_high",
    "c0_off_1e9": "plain_1000",
}


def _mutant_case(name):
    # exact_15: a constant covariate (x = 1 / 8) and targets whose mean is exact in both precisions, 2 (28 genes at 1, one at 30):
    # the fit is m = 2 and the gene at 30 sits at a ratio of exactly 15
    if name == "exact_15":
        t = np.ones(29)
        t[0] = 30.0
        return np.full(29, 8.0), t, 1e-12, 60.0, 0.1
    return tc.case(name)


@pytest.mark.parametrize("mutant", list(MUTANT_CASES))
def test_wrong_variants_are_rejected(mutant):
    case = _mutant_case(MUTANT_CASES[mutant])
    ref = tk.reference(case)
    tk.check_record(tk.as_record(ref), ref, "reference")  # the reference passes its own checks ...
    tk.check_record(tk.as_record(tk.reference(case, np.float64)), ref, "float64")  # ... and so does the correct float64 one
    bad = tk.as_record(tk.reference(case, np.float64, mutant))
    with pytest.raises(AssertionError):
        tk.check_record(bad, ref, mutant)


@pytest.mark.parametrize("mutant", tk.RULE_MUTANTS)
def test_threshold_variants_change_the_drop_rule(mutant):
    """The drop rule at ratios exactly on, and one long-double ulp either side of, 15 and 1e-4: the threshold variants decide
    differently exactly on their threshold, and only there."""
    thr = tk.LD(15) if mutant == "gt_15" else tk.LD(1e-4)
    r = np.array([np.nextafter(thr, tk.LD(0)), thr, np.nextafter(thr, tk.LD(np.inf))])
    want = [False, True, True] if mutant == "gt_15" else [True, False, False]
    assert tk.drop_rule(r).tolist() == want
    got = tk.drop_rule(r, tk.LD, mutant).tolist()
    assert got[0] == want[0] and got[2] == want[2] and got[1] != want[1]


def test_float64_reference_passes():
    for name in ("plain_1000", "planted_3001", "spread_0.0", "flat_tail_20000"):
        ref = _ref(name)
        tk.check_record(tk.as_record(tk.reference(tc.case(name), np.float64)), ref, name)


@pytest.mark.parametrize("name", CPU_CASES)
def test_emulator_passes(ops, name):
    means, gw, lo, hi, trig = tc.case(name)
    rec = ops.trend_outer(means, gw, lo, hi, lo, trig)
    ref = _ref(name)
    r = tk.check_record(rec, ref, f"emu/{name}")
    assert r["exempt"] == 0
    # the plugin's single fit: no clipping, no outer loop
    x = 1.0 / means
    c, pred, conv = ops.trend_glm(x, gw)
    x1, t1 = tk.prepare(means, gw, -np.inf, np.inf)
    o = tk.outer(x1, t1, outer_loop=False)
    assert conv == o["last_converged"]
    assert np.isfinite(c).all()
    if o["last_converged"] and o["kind"] != "degenerate":
        # Unclipped targets (down to 1e-8 and up to 120 here) can leave the fit's last steps on Fisher scoring, which converges
        # linearly: a last step below 1e-12 then leaves up to ~2e-10 relative (scattered_50), beyond the first-order bound of
        # the clipped fits, so the plugin's coefficients are held to 1e-9 relative
        free = o["bound"] > 0
        np.testing.assert_allclose(c[free], np.asarray(o["c"], dtype=np.float64)[free], rtol=1e-9, atol=0)
        assert (c[~free] == tk.LB).all()
    if rec[2] == 0.0:
        fitted = rec[0] + rec[1] / means
        tk.check_fitted(fitted, rec, means, name)


@pytest.mark.parametrize("name", list(tc.CASES))
@pytest.mark.parametrize("mode", ["0", "1"])
def test_pinned_records_pass(name, mode):
    rec = load_golden("trend_prior_ref")[f"{name}__grid{mode}"]
    r = tk.check_record(rec, _ref(name), f"golden/{name}/grid{mode}")
    assert r["exempt"] == 0


def test_select_disp_flags_at_planted_genes():
    """Genes 1e-6 either side of log(fitted) + 2 sqrt(sq): the flags follow the rule, and no gene is exempt."""
    means, gw, lo, hi, trig = tc.case("plain_2000")
    ref = _ref("plain_2000")
    rec = tk.as_record(ref)
    fitted = rec[0] + rec[1] / means
    edge = np.exp(np.log(fitted[:4]) + 2 * np.sqrt(rec[8]) + np.array([1e-6, -1e-6, 2e-6, -2e-6]))
    g = gw.copy()
    g[:4] = edge
    mp = np.clip(g * 0.9, lo, hi)
    disp, out, exempt = tk.select_reference(g, mp, fitted, rec[8], lo, hi)
    assert out[:4].tolist() == [True, False, True, False] and not exempt.any()
    bad = out.copy()
    bad[0] = False
    with pytest.raises(AssertionError):
        tk.check_select(np.where(bad, np.clip(g, lo, hi), mp), bad, g, mp, fitted, rec[8], lo, hi, "flipped")
