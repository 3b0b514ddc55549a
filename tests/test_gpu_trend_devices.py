"""GPU suite, needs >= 2 devices (skipped otherwise): the trend + prior launch (`pdq_trend_fit_dev`) from two contexts on two devices
of one process.  Both kernels take more than 48 KB of dynamic shared memory at these sizes (the fit's vectors, per thread), an
opt-in that belongs to the kernel on each device: the launch on the second device, after one on the first, must still succeed and
give the first device's record."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

FIELDS_EXACT = [2, 3, 4, 5, 7, 10]  # status, rounds, used, iterations, converged, n_above


def _n_devices():
    try:
        import torch

        return torch.cuda.device_count()
    except Exception:
        return 0


def _record(ctx, means, gw):
    from pydeseq2_b200 import _lib

    n = len(means)
    dm, dg, dout, dfit = ctx.malloc(n * 8), ctx.malloc(n * 8), ctx.malloc(128), ctx.malloc(n * 8)
    try:
        ctx.h2d(dm, means)
        ctx.h2d(dg, gw)
        ctx.check(ctx.lib.pdq_trend_fit_dev(ctx.h, _lib.c_dptr(dm), _lib.c_dptr(dg), n, 1e-8, 200.0, 0.0101,
                                            _lib.c_dptr(dout), _lib.c_dptr(dfit)))
        out, fitted = np.zeros(16), np.zeros(n)
        ctx.d2h(out, dout)
        ctx.d2h(fitted, dfit)
        ctx.sync()
        return out, fitted
    finally:
        for p in (dm, dg, dout, dfit):
            ctx.free(p)


# 60 000 genes: one cluster of 16 x 1024 threads, 64 KB of vectors per block; 500 000 genes: the grid kernel, 64 KB per block
@pytest.mark.parametrize("n,grid", [(60000, "0"), (500000, "1")])
def test_trend_fit_on_two_devices_of_one_process(n, grid, monkeypatch):
    if _n_devices() < 2:
        pytest.skip("needs 2 GPUs")
    from pydeseq2_b200 import _lib

    monkeypatch.setenv("PDQ_TREND_GRID", grid)
    rng = np.random.default_rng(5)
    means = np.exp(rng.normal(4, 2, n) * np.log(2))
    gw = (4 / means + 0.1) * np.exp(rng.normal(0, 0.5, n))
    c0, c1 = _lib.Context(0), _lib.Context(1)
    try:
        a, fa = _record(c0, means, gw)
        b, fb = _record(c1, means, gw)
        a2, _ = _record(c0, means, gw)
    finally:
        c1.close()
        c0.close()
    assert a[2] == 0.0 and a[4] > 0.9 * n
    for r in (b, a2):
        np.testing.assert_array_equal(r[FIELDS_EXACT], a[FIELDS_EXACT])
        # the cluster kernel sums in a fixed order; the grid kernel's atomics may move the coefficients in the last bits
        np.testing.assert_allclose(r[[0, 1, 8, 9]], a[[0, 1, 8, 9]], rtol=0 if grid == "0" else 1e-10)
    np.testing.assert_allclose(fb, fa, rtol=0 if grid == "0" else 1e-10)
