"""CPU suite: the extended-precision reference of Cook's distances (cooks_checks.py) against mpmath and the reference's own tape
goldens; the checks accept the float64 oracle with margin and reject subtly wrong variants; and the host emulator runs every case
through cooks_gene_cols -- the narrow cases at 1..32 lanes per gene, every case with the design width at run time at the 32
lanes of k_wide_cooks.

Set PDQ_COOKS_REPORT to a file path to have the worst error / bound of every source and quantity written there as JSON."""
import functools
import json
import os

import mpmath
import numpy as np
import pytest
from scipy.stats import f as f_dist

import cooks_cases as cs
import cooks_checks as cc
from conftest import load_golden
from emu.emu_ops import EmuOps
from oracle import nbglm
from pydeseq2_b200.inference import B200Inference

LANES = [1, 2, 4, 8, 16, 32]
TAPES = ("tape_single_factor", "tape_multi_factor", "tape_continuous", "tape_wide")
REPORT = {}


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    path = os.environ.get("PDQ_COOKS_REPORT")
    if path:
        with open(path, "w") as f:
            json.dump(REPORT, f, indent=1, sort_keys=True)


def _record(source, worst):
    for q in ("disp", "cooks"):
        key = f"{source}/{q}"
        REPORT[key] = max(REPORT.get(key, 0.0), worst[q])
    assert worst["exempt"] == 0, f"{source}: {worst['exempt']} genes exempted at the cutoff or an argmax tie"


@functools.lru_cache(maxsize=None)
def _case(name):
    return cs.make(name)


@functools.lru_cache(maxsize=None)
def _ref(name):
    return cc.reference(_case(name))


def _oracle(c):
    with np.errstate(divide="ignore", invalid="ignore"):
        ck, disp = nbglm.calculate_cooks(c["counts"], c["counts"] / c["sf"][:, None], c["X"], c["mu"], c["hat"])
        return ck, disp, nbglm.cooks_outlier(c["counts"], ck, c["X"]), (ck > c["cutoff"]).any(axis=0)


def _mp_gene(c, g):
    """Robust dispersion and distances of gene g in 40-digit arithmetic, on the same doubles."""
    X = c["X"]
    N, p = X.shape
    cells, global_mode = cc.cells_of(X)
    x = [mpmath.mpf(int(c["counts"][n, g])) / mpmath.mpf(float(c["sf"][n])) for n in range(N)]
    m = mpmath.fsum(x) / N
    v = None
    for idx in cells:
        nc = len(idx)
        ntrim, scale = cc.trim_class(nc, global_mode)
        kept = sorted(x[i] for i in idx)[ntrim:nc - ntrim]
        tm = mpmath.fsum(kept) / len(kept)
        sq = sorted((x[i] - tm) ** 2 for i in idx)[ntrim:nc - ntrim]
        tv = mpmath.mpf(scale) * mpmath.fsum(sq) / len(sq)
        v = tv if v is None else max(v, tv)
    alpha = max((v - m) / (m * m), mpmath.mpf(cc.MIN_DISP))
    ck = []
    for n in range(N):
        mu, h = mpmath.mpf(float(c["mu"][n, g])), mpmath.mpf(float(c["hat"][n, g]))
        ck.append((int(c["counts"][n, g]) - mu) ** 2 / (mu + alpha * mu * mu) / p * (h / (1 - h) ** 2))
    return alpha, ck


@pytest.mark.parametrize("name", ["cells_3_to_200", "cells_mixed_singletons", "nocell_n17", "width_p70_levels"])
def test_longdouble_reference_agrees_with_mpmath(name):
    """The longdouble reference within 1 % of the float64 bounds of 40-digit arithmetic, on the special genes and a few others."""
    c, ref = _case(name), _ref(name)
    G = c["counts"].shape[1]
    with mpmath.workdps(40):
        assert np.isnan(ref["disp"][0])  # the all-zero gene: 0 / 0
        for g in list(range(1, len(cs.SPECIAL))) + [G // 3, G // 2, G - 1]:
            alpha, ck = _mp_gene(c, g)
            assert float(abs(mpmath.mpf(float(ref["disp"][g])) - alpha)) <= 0.01 * ref["e_disp"][g], (name, g)
            for n in range(len(ck)):
                err = float(abs(mpmath.mpf(float(ref["cooks"][n, g])) - ck[n]))
                assert err <= 0.01 * ref["e_cooks"][n, g], (name, g, n)


@pytest.mark.parametrize("name", TAPES)
def test_reference_matches_the_tape_goldens(name):
    """The restatement on the layers the real orchestrator recorded: its distances, robust dispersions, outlier and replaced
    genes; and the checks pass the recorded values."""
    t = load_golden(name)
    nz = t["final_non_zero"] == 1
    X = t["design"]
    N, p = X.shape
    c = {"X": X, "sf": t["final_size_factors"], "counts": np.ascontiguousarray(t["counts"][:, nz]),
         "mu": np.ascontiguousarray(t["final_mu_LFC"]), "hat": np.ascontiguousarray(t["final_hat"]),
         "cutoff": float(f_dist.ppf(0.99, p, N - p))}
    ref = cc.reference(c)
    np.testing.assert_allclose(ref["disp"].astype(np.float64), t["final_robust_disp"], rtol=1e-10)
    np.testing.assert_allclose(ref["cooks"].astype(np.float64), t["final_cooks"][:, nz], rtol=1e-9)
    np.testing.assert_array_equal(ref["outlier"], t["final_cooks_outlier"][nz] == 1)
    np.testing.assert_array_equal(ref["replaced"], t["final_replaced"][nz] == 1)
    _record("tape goldens", cc.check((t["final_cooks"][:, nz], t["final_robust_disp"], t["final_cooks_outlier"][nz] == 1,
                                      t["final_replaced"][nz] == 1), ref, name))


@pytest.mark.parametrize("name", list(cs.CASES))
def test_float64_oracle_passes_with_margin(name):
    """oracle.nbglm's calculate_cooks / cooks_outlier, and the float64 form of the restatement, within a quarter of every bound,
    with the special genes deciding as planted."""
    c, ref = _case(name), _ref(name)
    for src, got in (("oracle", _oracle(c)), ("float64 restatement", cc.as_result(cc.reference(c, np.float64)))):
        w = cc.check(got, ref, f"{name}, {src}")
        assert w["disp"] <= 0.25 and w["cooks"] <= 0.25, (src, w)
        _record(src, w)
    out, rep = ref["outlier"], ref["replaced"]
    assert np.isnan(ref["disp"][0]) and not out[0] and not rep[0]  # all-zero gene
    assert rep[1:5].all() and not rep[5]
    assert out[1:3].all() == (not ref["global_mode"]) and not out[3] and out[4] == (not ref["global_mode"]) and not out[5]


@pytest.mark.parametrize("mutant", list(cc.MUTANTS))
def test_checks_reject_wrong_results(mutant):
    """Each wrong variant of cc.MUTANTS: values off by orders of magnitude more than their bounds, or decisions that differ."""
    worst, wrong_decisions, rejected = 0.0, 0, 0
    for name in cs.CASES:
        ref = _ref(name)
        got = cc.as_result(cc.reference(_case(name), np.float64, mutant))
        r, bad = cc.ratios(got, ref)
        worst = max(worst, cc.worst(r["disp"]), cc.worst(r["cooks"]))
        wrong_decisions += int(bad["outlier"].sum() + bad["replaced"].sum())
        try:
            cc.check(got, ref, name)
        except AssertionError:
            rejected += 1
    assert rejected > 0, cc.MUTANTS[mutant]
    if mutant in ("last_argmax", "larger_or_equal"):
        assert wrong_decisions > 0
    else:
        assert worst >= 1e3, (mutant, worst)


@pytest.fixture(scope="module", params=LANES, ids=[f"T{T}" for T in LANES])
def emu(request):
    return B200Inference(_ops=EmuOps(lanes=request.param)), request.param


@pytest.mark.parametrize("name", cs.NARROW)
def test_emulator_narrow_cases_at_every_lane_width(emu, name):
    """cooks_gene<P> at T = 1..32 lanes: within bounds, decisions exact, and the same bits without the distance matrix."""
    inf, T = emu
    c = _case(name)
    got = inf.calculate_cooks(c["counts"], c["sf"], c["X"], c["mu"], c["hat"])
    _record(f"emulator/narrow/T={T}", cc.check(got, _ref(name), f"{name}, T = {T}"))
    _, disp, outl, repl = inf.calculate_cooks(c["counts"], c["sf"], c["X"], c["mu"], c["hat"], return_matrix=False)
    np.testing.assert_array_equal(disp.view(np.int64), got[1].view(np.int64))
    np.testing.assert_array_equal(outl, got[2])
    np.testing.assert_array_equal(repl, got[3])


@pytest.mark.parametrize("name", list(cs.CASES))
def test_emulator_runtime_width_at_32_lanes(name):
    """cooks_gene_cols with p at run time, the routine of k_wide_cooks, at its 32 lanes on every case; on the narrow ones the
    same bits as the template width."""
    c = _case(name)
    ops = EmuOps(lanes=32)
    N, G = c["counts"].shape
    out = [np.empty((N, G)), np.empty(G), np.empty(G), np.empty(G)]
    ops.cooks_cols(c["counts"], G, N, G, c["sf"], c["X"], c["X"].shape[1], c["mu"], c["hat"], G, c["cutoff"], *out)
    got = (out[0], out[1], out[2] == 1.0, out[3] == 1.0)
    _record(f"emulator/{c['tier']}/T=32", cc.check(got, _ref(name), name))
    if c["tier"] == "narrow":
        ref_ops = [np.empty((N, G)), np.empty(G), np.empty(G), np.empty(G)]
        ops.cooks(c["counts"], G, N, G, c["sf"], c["X"], c["X"].shape[1], c["mu"], c["hat"], G, c["cutoff"], *ref_ops)
        for a, b in zip(out, ref_ops):
            np.testing.assert_array_equal(a.view(np.int64), b.view(np.int64))
