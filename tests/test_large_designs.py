"""CPU suite: the host-side linear algebra of designs of 65..128 columns (pdq_design_pinv_large) against numpy.

The large-design kernels (the team-per-gene instantiation of pdq_wide.cu) are cooperative block code with no host emulation;
tests/test_gpu_large_designs.py checks them against the oracle on an H100."""
import ctypes as C
import os

import numpy as np
import pytest

from large_cases import LARGE_E2E, MULTIMODAL_REASON, check_large_e2e
from pydeseq2_b200 import _lib


def _lib_or_build():
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as g

        g.build()
    return _lib.load()


def _pinv(X, fn="pdq_design_pinv_large"):
    N, p = X.shape
    X = np.ascontiguousarray(X, dtype=np.float64)
    out, fr = np.empty((p, p)), C.c_int(-1)
    rc = getattr(_lib_or_build(), fn)(_lib.as_f64p(X), N, p, _lib.as_f64p(out), C.byref(fr))
    return rc, out, fr.value


def paired(subjects):
    """~subject + condition: intercept, subject dummies, condition."""
    N = 2 * subjects
    subj = np.repeat(np.arange(subjects), 2)
    cols = [np.ones(N)] + [(subj == s).astype(float) for s in range(1, subjects)] + [np.tile([0.0, 1.0], subjects)]
    return np.stack(cols, axis=1)


@pytest.mark.parametrize("X", [paired(64), paired(100), paired(127), np.random.default_rng(6).normal(size=(300, 128))],
                         ids=["p65", "p101", "p128", "dense_p128"])
def test_design_pinv_large_matches_numpy(X):
    rc, pinv, full_rank = _pinv(X)
    assert rc == 0
    assert full_rank == int(np.linalg.matrix_rank(X) == X.shape[1]) == 1
    want = np.linalg.pinv(X.T @ X)
    np.testing.assert_allclose(pinv, want, rtol=0, atol=1e-10 * np.abs(want).max())


def test_design_pinv_large_rank_deficient():
    X = paired(99)
    X = np.concatenate([X, X[:, 3:4] + X[:, 5:6]], axis=1)  # p = 101, rank 100
    assert np.linalg.matrix_rank(X) == 100
    rc, pinv, full_rank = _pinv(X)
    assert rc == 0 and full_rank == 0
    want = np.linalg.pinv(X.T @ X)
    np.testing.assert_allclose(pinv, want, rtol=0, atol=1e-9 * np.abs(want).max())


def test_limits():
    """pdq_design_pinv keeps its p <= 64 contract; the large entry point stops at 128."""
    assert (_lib.PDQ_MAX_P_WIDE, _lib.PDQ_MAX_P_LARGE) == (64, 128)
    assert _pinv(np.ones((70, 65)), "pdq_design_pinv")[0] == -2
    assert _pinv(np.ones((300, 129)))[0] == -2


def test_large_designs_needs_wide_designs():
    from pydeseq2_b200.inference import B200Inference

    with pytest.raises(ValueError, match="large_designs=True needs wide_designs=True"):
        B200Inference(device=0, large_designs=True)


@pytest.mark.parametrize("name", [n if n != "large_paired_p128" else
                                  pytest.param(n, marks=pytest.mark.xfail(strict=True, reason=MULTIMODAL_REASON)) for n in LARGE_E2E])
def test_oracle_against_the_large_fixtures(name):
    """The oracle, through the workflow's host logic, against the final tables the real reference wrote for designs of 65..128
    columns (scripts/make_large_golden.py): decisions and NaN patterns identical, values at the e2e tolerance within the measured
    per-fixture budget of tests/large_cases.py."""
    from test_wide_designs import _OracleBackend

    check_large_e2e(_OracleBackend(), name)
