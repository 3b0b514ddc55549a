"""Record the `TrendOut` record (16 doubles) of `pdq_trend_fit_dev` for every case of tests/trend_prior_cases.py, through the
one-cluster kernel (PDQ_TREND_GRID=0) and the cooperative grid kernel (PDQ_TREND_GRID=1), into tests/golden/trend_prior_ref.npz.

    python scripts/make_trend_prior_golden.py [OUT.npz]

Needs the GPU.  Each configuration runs three times; the script reports configurations whose repeats differ (the grid kernel adds
its per-block partial sums with global atomics, so its coefficients may move in the last bits from run to run).
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

import trend_prior_cases as tc  # noqa: E402
from pydeseq2_b200 import _lib  # noqa: E402


def trend_record(ctx, means, gw, min_disp, max_disp, trigamma_c):
    n = len(means)
    dm, dg, dout = ctx.malloc(n * 8), ctx.malloc(n * 8), ctx.malloc(128)
    try:
        ctx.h2d(dm, means)
        ctx.h2d(dg, gw)
        ctx.check(ctx.lib.pdq_trend_fit_dev(ctx.h, _lib.c_dptr(dm), _lib.c_dptr(dg), n, min_disp, max_disp, trigamma_c,
                                            _lib.c_dptr(dout), _lib.c_dptr(0)))
        out = np.zeros(16)
        ctx.d2h(out, dout)
        ctx.sync()
        return out
    finally:
        for p in (dm, dg, dout):
            ctx.free(p)


def records(ctx, repeats=1):
    """{"<case>__grid<0|1>": [record, ...]} for every case and both kernels."""
    res = {}
    for name in tc.CASES:
        args = tc.case(name)
        for mode in ("0", "1"):
            os.environ["PDQ_TREND_GRID"] = mode
            try:
                res[f"{name}__grid{mode}"] = [trend_record(ctx, *args) for _ in range(repeats)]
            finally:
                del os.environ["PDQ_TREND_GRID"]
    return res


def main():
    out_path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "trend_prior_ref.npz")
    ctx = _lib.Context(0)
    print("device", ctx.info()["name"])
    rec = records(ctx, repeats=3)
    ctx.close()
    for k, v in rec.items():
        same = all(np.array_equal(v[0].view(np.uint64), r.view(np.uint64)) for r in v[1:])
        print(f"{k:32s} status {v[0][2]:.0f} rounds {v[0][3]:.0f} iters {v[0][5]:.0f} n_above {v[0][10]:.0f} "
              f"sq {v[0][8]!r} {'' if same else 'REPEATS DIFFER'}")
    np.savez(out_path, **{k: v[0] for k, v in rec.items()})
    print("wrote", out_path)


if __name__ == "__main__":
    main()
