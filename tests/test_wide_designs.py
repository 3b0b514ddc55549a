"""CPU suite: the host-side linear algebra of designs of 17..64 columns (pdq_design_pinv) against numpy.

The wide-design kernels themselves (pdq_wide.cu) are cooperative warp code with no host emulation; tests/test_gpu_wide_designs.py
checks them against the oracle on an H100."""
import ctypes as C
import os

import numpy as np
import pytest

from pydeseq2_b200 import _lib
from wide_cases import WIDE_E2E, check_wide_e2e


def _lib_or_build():
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as g

        g.build()
    return _lib.load()


def _pinv(X):
    N, p = X.shape
    X = np.ascontiguousarray(X, dtype=np.float64)
    out, fr = np.empty((p, p)), C.c_int(-1)
    rc = _lib_or_build().pdq_design_pinv(_lib.as_f64p(X), N, p, _lib.as_f64p(out), C.byref(fr))
    return rc, out, fr.value


def _paired(subjects, covariate=False, seed=0):
    """~subject + condition (+ a continuous covariate): intercept, subject dummies, condition."""
    rng = np.random.default_rng(seed)
    N = 2 * subjects
    subj = np.repeat(np.arange(subjects), 2)
    cols = [np.ones(N)] + [(subj == s).astype(float) for s in range(1, subjects)] + [np.tile([0.0, 1.0], subjects)]
    if covariate:
        cols.append(rng.normal(0, 1, N))
    return np.stack(cols, axis=1)


@pytest.mark.parametrize("X", [_paired(16), _paired(20), _paired(31, covariate=True), _paired(63),
                               np.random.default_rng(5).normal(size=(150, 48))], ids=["p17", "p21", "p33", "p64", "dense_p48"])
def test_design_pinv_matches_numpy(X):
    rc, pinv, full_rank = _pinv(X)
    assert rc == 0
    assert full_rank == int(np.linalg.matrix_rank(X) == X.shape[1])
    want = np.linalg.pinv(X.T @ X)
    np.testing.assert_allclose(pinv, want, rtol=0, atol=1e-10 * np.abs(want).max())


def test_design_pinv_rank_deficient():
    X = _paired(20)
    X = np.concatenate([X, X[:, 3:4] + X[:, 5:6]], axis=1)  # p = 22, rank 21
    rc, pinv, full_rank = _pinv(X)
    assert rc == 0 and full_rank == 0
    want = np.linalg.pinv(X.T @ X)
    np.testing.assert_allclose(pinv, want, rtol=0, atol=1e-9 * np.abs(want).max())


def test_design_pinv_rejects_more_than_64_columns():
    assert _pinv(np.ones((70, 65)))[0] == -2
    assert _lib.PDQ_MAX_P_WIDE == 64


class _OracleBackend:
    """The oracle plus Cook's distances, which the deseq2() drivers ask the backend for (as tests/test_workflow.py)."""

    def __new__(cls, n_cpus=4):
        from oracle import nbglm

        class Backend(nbglm.OracleInference):
            def calculate_cooks(self, counts, size_factors, design_matrix, mu, hat, return_matrix=True):
                return nbglm.calculate_cooks(counts, counts / size_factors[:, None], design_matrix, mu, hat)

        return Backend(n_cpus=n_cpus)


@pytest.mark.parametrize("name", WIDE_E2E)
def test_oracle_against_the_wide_fixtures(name):
    """The oracle, through the workflow's host logic, against the final tables the real reference wrote for designs of 17..64
    columns (scripts/make_wide_golden.py): decisions and NaN patterns identical, values at the e2e tolerance within the measured
    per-fixture budget of tests/wide_cases.py."""
    check_wide_e2e(_OracleBackend(), name)
