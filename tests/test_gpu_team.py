"""GPU suite (`-m gpu`): the team building blocks of pdq_team.cuh -- the cooperative linear algebra and collectives every
kernel of designs of 17..128 columns is built from -- through the GPU probe's team unit (tests/gpu_probe/team_probe.cu), against
extended-precision references computed here (tests/team_checks.py), at p = 1..128 around the places where thread ownership
wraps (32 W) and the packed triangle gets its pad slot, each at team widths W = 1, 2, 4 and 8.

Set PDQ_TEAM_REPORT to a file path to have the worst error / bound of every quantity at every p and W written there as JSON."""
import json
import os

import numpy as np
import pytest

import team_checks as tc

pytestmark = pytest.mark.gpu

# the primitives that give every entry a fixed sequential operation order whoever owns it (bit-identical across W); symdot_w,
# wald_se_w, wdot and Team::sum change their cross-warp order with W and get only the bounds
W_INVARIANT_SPD = ["L", "x", "H", "Li", "matvec", "pinv", "quad", "logdet"]
TEAM_SCALARS = ["logdet", "symdot", "quad", "se"]

REPORT = {}


@pytest.fixture(scope="module")
def team():
    from gpu_probe.probe import TeamProbe

    yield TeamProbe()
    path = os.environ.get("PDQ_TEAM_REPORT")
    if path:
        with open(path, "w") as f:
            json.dump(REPORT, f, indent=1, sort_keys=True)


def _record(p, W, worst):
    for q, r in worst.items():
        key = f"{q}/p={p}/W={W}"
        REPORT[key] = max(REPORT.get(key, 0.0), r)


def test_team_rejects_bad_shapes(team):
    """p outside 1..128 or W outside {1, 2, 4, 8}: cudaErrorInvalidValue (1) before anything is read or launched."""
    for p, W in ((0, 1), (129, 1), (129, 8), (17, 3), (17, 16)):
        assert team.lib.team_spd(p, W, None, None, None, None, None, None, None, 1, None, None) == 1
        assert team.lib.team_acc(p, W, 4, None, None, None, 1, None) == 1
    assert team.lib.team_coll(3, None, None, None, None, None, 4, 1, None) == 1
    assert team.ws_bytes(128, 8) == 210432  # 3 packed 128 x 128 triangles + 8 vectors + 2 chunk buffers of 256 doubles


@pytest.mark.parametrize("p", tc.P_LIST)
def test_team_spd_algebra(team, p):
    """factor_ridged / chol_solve_w / chol_inverse_w / logdet / matvec_w / symdot_w / quad_w / apply_pinv / wald_se_w on random SPD
    matrices at kappa 1 .. 1e12 and on design-like X^T W X (paired, a level without counts plus the 1e-6 ridge in both ridge
    modes, covariates on the scale of 1e3): backward and forward errors within their bounds at every W, the W-invariant
    outputs bit-identical across W, the team-wide scalars bit-identical in every thread."""
    for mode, batch in tc.spd_inputs(p).items():
        if not batch["names"]:
            continue
        ref = tc.spd_reference(batch, p)
        by_w = {}
        for W in tc.WARPS:
            got = team.spd(p, W, batch["A"], batch["b"], batch["S"], batch["P"], batch["c"], batch["ridge"], batch["ridge_tri"])
            for q in TEAM_SCALARS:
                tc.check_team_identical(got[q], f"{q}, p = {p}, W = {W} ({mode} ridge)")
            _record(p, W, tc.check_spd(got, batch, ref, p))
            by_w[W] = {k: v[:, 0] if k in TEAM_SCALARS else v for k, v in got.items()}
        tc.check_w_invariant(by_w, W_INVARIANT_SPD, f"p = {p} ({mode} ridge)")


@pytest.mark.parametrize("p", tc.P_LIST)
def test_team_nonpositive_pivot(team, p):
    """A non-positive pivot m: the factor is NaN from column m on and finite before it, the same at every W; the solve,
    inverse and logdet are NaN where the narrow tier's chol<P> (probe unit "narrow", p <= 8) makes them NaN."""
    A, b, ms = tc.pivot_inputs(p)
    n = len(ms)
    S, P, c = np.zeros_like(A), np.eye(p), np.ones((n, p))
    by_w = {W: team.spd(p, W, A, b, S, P, c) for W in tc.WARPS}
    for W in tc.WARPS:
        by_w[W] = {k: v[:, 0] if k in TEAM_SCALARS else v for k, v in by_w[W].items()}
    for W, got in by_w.items():
        for g, m in enumerate(ms):
            np.testing.assert_array_equal(np.isnan(got["L"][g]), tc.pivot_pattern(p, m), err_msg=f"L, p = {p}, W = {W}, m = {m}")
    tc.check_w_invariant(by_w, ["L", "x", "H", "Li", "logdet"], f"p = {p}, non-positive pivot")
    if p <= 8:
        from gpu_probe.probe import Probe

        nar = Probe("narrow").spd(p, A, b, S)
        got = by_w[1]
        np.testing.assert_array_equal(np.isnan(got["x"]), np.isnan(nar["solve"]), err_msg=f"solve, p = {p}")
        np.testing.assert_array_equal(np.isnan(got["H"]), np.isnan(nar["inv"]), err_msg=f"inverse, p = {p}")
        np.testing.assert_array_equal(np.isnan(got["logdet"]), np.isnan(nar["logdet"]), err_msg=f"logdet, p = {p}")


@pytest.mark.parametrize("p", tc.P_LIST)
def test_team_accumulators(team, p):
    """rank_chunk / vec_chunk (X^T W X and X^T W z), staged chunk by chunk as irls_sweep_w stages them, at N from 1 to 8000
    around the chunk size 32 W and at 10 p + 1, weights from 0 to 1e6: within c N eps of the exact sums, bit-identical across W."""
    for N in tc.acc_sizes(p):
        X, w, z = tc.acc_inputs(p, N)
        ref = tc.acc_reference(X, w, z)
        by_w = {W: team.acc(p, W, X, w, z) for W in tc.WARPS}
        for W, got in by_w.items():
            _record(p, W, tc.check_acc(got, ref, N, p))
        tc.check_w_invariant(by_w, ["M", "v"], f"p = {p}, N = {N}")


@pytest.mark.parametrize("W", tc.WARPS)
def test_team_collectives(team, W):
    """Team<W>::sum / max / sum / any / max / sum back to back on every thread (reusing the shared slots), then wdot / wmaxabs
    over 1..300 components: see team_checks.check_coll."""
    inp = tc.coll_inputs(W)
    tc.check_coll(team.coll(W, inp["v"], inp["flag"], inp["a"], inp["b"], inp["lens"]), inp, W)
