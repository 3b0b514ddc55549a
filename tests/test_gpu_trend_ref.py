"""The dispersion trend + prior launch against the extended-precision reference of trend_checks.py, through every entry point that
runs it: pdq_trend_fit_dev (with the fitted dispersions of k_trend_eval), pdq_trend_prior (host vectors), the plugin's single fit
pdq_dispersion_trend_gamma_glm, pdq_select_dispersions_dev on the record, and B200Inference.trend_and_prior -- on the one-cluster
kernel and the grid kernel, and on a subset of cases at every forced thread count and cluster size.

Set PDQ_TREND_REPORT to a file path to have the worst error / bound per quantity, kernel and shape, and the exemption counts,
written there as JSON."""
import functools
import json
import os

import numpy as np
import pytest

import trend_checks as tk
import trend_prior_cases as tc

REPORT = {}
CASES = list(tc.CASES) + list(tc.REF_CASES)
SHAPE_CASES = ["plain_900", "plain_16000", "planted_3001", "spread_0.0", "spread_1e-06", "flat_trend", "few_3", "clipped_ties_20000"]
SHAPES = ([("grid", v) for v in ("0", "1")] + [("cluster", v) for v in ("1", "2", "4", "8", "16")]
          + [("threads", v) for v in ("256", "512", "1024")])
ENV = {"grid": "PDQ_TREND_GRID", "cluster": "PDQ_TREND_CLUSTER", "threads": "PDQ_TREND_THREADS"}


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    path = os.environ.get("PDQ_TREND_REPORT")
    if path:
        with open(path, "w") as f:
            json.dump(REPORT, f, indent=1, sort_keys=True)


def _record(source, r):
    for q, v in r.items():
        key = f"{source}/{q}"
        REPORT[key] = (REPORT.get(key, 0) + v) if q == "exempt" else max(REPORT.get(key, 0.0), v)


@functools.lru_cache(maxsize=None)
def _ref(name):
    return tk.reference(tc.case(name))


@pytest.fixture(scope="module")
def ctx():
    from pydeseq2_b200 import _lib

    c = _lib.Context(0)
    yield c
    c.close()


@pytest.fixture
def shape_env(request):
    """Sets the launcher's shape hooks for one test and restores them."""
    saved = {k: os.environ.get(k) for k in ENV.values()}

    def set_(**kv):
        for k, v in kv.items():
            os.environ[ENV[k]] = v

    yield set_
    for k, v in saved.items():
        if v is None:
            os.environ.pop(k, None)
        else:
            os.environ[k] = v


def _trend_dev(ctx, means, gw, min_disp, max_disp, trig):
    from pydeseq2_b200 import _lib

    n = len(means)
    dm, dg, dout, dfit = ctx.malloc(n * 8), ctx.malloc(n * 8), ctx.malloc(128), ctx.malloc(n * 8)
    try:
        ctx.h2d(dm, means)
        ctx.h2d(dg, gw)
        ctx.check(ctx.lib.pdq_trend_fit_dev(ctx.h, _lib.c_dptr(dm), _lib.c_dptr(dg), n, min_disp, max_disp, trig, _lib.c_dptr(dout),
                                            _lib.c_dptr(dfit)))
        out, fitted = np.zeros(16), np.zeros(n)
        ctx.d2h(out, dout)
        ctx.d2h(fitted, dfit)
        ctx.sync()
        return out, fitted
    finally:
        for p in (dm, dg, dout, dfit):
            ctx.free(p)


def _select_dev(ctx, gw, mp, fitted, rec, lo, hi):
    from pydeseq2_b200 import _lib

    n = len(gw)
    bufs = [ctx.malloc(n * 8) for _ in range(5)] + [ctx.malloc(128)]
    try:
        for b, v in zip(bufs, (gw, mp, fitted)):
            ctx.h2d(b, np.ascontiguousarray(v))
        ctx.h2d(bufs[5], np.ascontiguousarray(rec))
        ctx.check(ctx.lib.pdq_select_dispersions_dev(ctx.h, *(_lib.c_dptr(b) for b in (bufs[0], bufs[1], bufs[2], bufs[5])), n, lo, hi,
                                                     _lib.c_dptr(bufs[3]), _lib.c_dptr(bufs[4])))
        disp, out = np.zeros(n), np.zeros(n)
        ctx.d2h(disp, bufs[3])
        ctx.d2h(out, bufs[4])
        ctx.sync()
        return disp, out != 0.0
    finally:
        for b in bufs:
            ctx.free(b)


def _check_dev(ctx, name, source):
    means, gw, lo, hi, trig = tc.case(name)
    rec, fitted = _trend_dev(ctx, means, gw, lo, hi, trig)
    r = tk.check_record(rec, _ref(name), f"{source}/{name}")
    r["fitted"] = tk.check_fitted(fitted, rec, means, f"{source}/{name}")
    _record(source, r)
    if name not in tc.PLANTED:
        assert r["exempt"] == 0, f"{source}/{name}: {r['exempt']} exempted decisions"
    return rec, fitted


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["0", "1"])
@pytest.mark.parametrize("name", CASES)
def test_gpu_trend_fit_dev(ctx, shape_env, name, mode):
    shape_env(grid=mode)
    rec, fitted = _check_dev(ctx, name, f"grid{mode}")
    if rec[2] != 0.0:
        return
    # the final dispersions on the record (select_disp): a MAP vector near the genewise one
    means, gw, lo, hi, _ = tc.case(name)
    mp = gw * np.exp(np.random.default_rng(len(gw)).normal(0.0, 0.1, len(gw)))
    disp, out = _select_dev(ctx, gw, mp, fitted, rec, lo, hi)
    ex = tk.check_select(disp, out, gw, mp, fitted, rec[8], lo, hi, f"select/grid{mode}/{name}")
    _record(f"grid{mode}", {"select_exempt": ex})
    if name != "few_2":  # two genes: the fit runs through both, so both sit on log(fitted) + 2 sqrt(0) to rounding
        assert ex == 0


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [f"{k}{v}" for k, v in SHAPES[2:]])
@pytest.mark.parametrize("name", SHAPE_CASES)
def test_gpu_trend_forced_shapes(ctx, shape_env, name, shape):
    key = "cluster" if shape.startswith("cluster") else "threads"
    shape_env(grid="0", **{key: shape[len(key):]})
    _check_dev(ctx, name, shape)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["plain_1000", "plain_65536", "planted_3001", "spread_0.0", "spread_1e-09", "inverse_trend",
                                  "few_1", "no_prior", "flat_tail_150001"])
def test_gpu_trend_prior_host_vectors(ctx, name):
    from pydeseq2_b200.inference import B200Inference

    means, gw, lo, hi, trig = tc.case(name)
    out16, fitted = B200Inference(device=0)._ops.trend_prior(means, gw, lo, hi, trig)
    r = tk.check_record(out16, _ref(name), f"host/{name}")
    if out16[2] == 0.0:
        r["fitted"] = tk.check_fitted(fitted, out16, means, f"host/{name}")
    _record("host", r)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["plain_1000", "plain_20000", "plain_65536", "spread_0.0", "spread_1e-09", "spread_1e-06",
                                  "spread_0.001", "flat_trend", "inverse_trend", "few_2", "planted_3001"])
def test_gpu_plugin_single_fit(name):
    """pdq_dispersion_trend_gamma_glm: one fit, no clipping, NaN targets skipped, infinite covariates left out; its `converged`
    equals the single fit's, its coefficients are the minimiser's and its predictions c0 + c1 x."""
    from pydeseq2_b200.inference import B200Inference

    means, gw, _, _, _ = tc.case(name)
    with np.errstate(divide="ignore"):
        x = 1.0 / means
    t = gw.copy()
    t[::97] = np.nan
    inf = B200Inference(device=0)
    coeffs, pred, conv = inf.dispersion_trend_gamma_glm(x, t)
    xp, tp = tk.prepare(x, t, -np.inf, np.inf, x_is_mean=False, clip=False)
    o = tk.outer(xp, tp, outer_loop=False)
    assert conv == o["last_converged"], name
    assert np.isfinite(coeffs).all()
    r = {"c": tk.coeff_ratio(coeffs, o) if o["last_converged"] else 0.0}
    assert r["c"] <= 1.0, f"plugin/{name}: coefficients {r['c']:.3g} x their bound"
    _record("plugin", r)
    with np.errstate(invalid="ignore"):
        np.testing.assert_array_equal(pred, coeffs[0] + coeffs[1] * x)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["plain_2000", "planted_3001", "spread_0.0", "spread_1e-06", "flat_trend", "no_prior"])
def test_gpu_inference_trend_and_prior(name):
    """B200Inference.trend_and_prior returns None exactly when the reference's fit fails, and otherwise the minimiser's
    coefficients, c0 + c1 / mean, the prior of the reference and its rounds."""
    from scipy.special import polygamma

    from pydeseq2_b200.inference import B200Inference

    means, gw, lo, hi, _ = tc.case(name)
    ref = tk.reference((means, gw, lo, hi, float(polygamma(1, (60 - 3) / 2))))
    got = B200Inference(device=0).trend_and_prior(means, gw, lo, hi, 60, 3)
    assert (got is None) == (ref["status"] != 0), name
    if got is None:
        return
    coeffs, fitted, sq, pv, rounds = got
    r = {"c": tk.coeff_ratio(coeffs, ref)}
    r.update(tk.prior_ratios(coeffs, sq, pv, None, ref, f"inference/{name}"))
    for q, v in r.items():
        assert v <= 1.0, f"inference/{name}: {q} is {v:.3g} x its bound"
    rec = np.zeros(16)
    rec[:2] = coeffs
    r["fitted"] = tk.check_fitted(fitted, rec, means, f"inference/{name}")
    assert rounds == ref["n_outer"]
    _record("inference", r)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["0", "1"])
@pytest.mark.parametrize("name", ["plain_2000", "planted_70000"])
def test_gpu_select_disp_at_planted_genes(ctx, shape_env, name, mode):
    """pdq_select_dispersions_dev on the device's own record, with genes planted 1e-6 and 2e-6 either side of
    log(fitted) + 2 sqrt(squared_logres): every flag follows the rule, and none is exempt."""
    shape_env(grid=mode)
    means, gw, lo, hi, trig = tc.case(name)
    rec, fitted = _trend_dev(ctx, means, gw, lo, hi, trig)
    assert rec[2] == 0.0
    g = gw.copy()
    planted = np.arange(100, 104)
    g[planted] = np.exp(np.log(fitted[planted]) + 2 * np.sqrt(rec[8]) + np.array([1e-6, -1e-6, 2e-6, -2e-6]))
    mp = np.clip(gw * 0.9, lo, hi)
    disp, out = _select_dev(ctx, g, mp, fitted, rec, lo, hi)
    assert out[planted].tolist() == [True, False, True, False]
    assert tk.check_select(disp, out, g, mp, fitted, rec[8], lo, hi, f"select/planted/grid{mode}/{name}") == 0
