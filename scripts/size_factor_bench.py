"""Size factors on one GPU: prints one JSON line.

    python scripts/size_factor_bench.py [--reps 50] [--warmup 5]

For each shape (samples x genes: 200 x 20 000, 500 x 60 000, 2 000 x 7 500) at zero fractions 0 and 0.7, and each estimator --
median of ratios, poscounts, each over every gene and over 10 % control genes -- the time of one `pdq_size_factors_ex_dev` call on
device-resident counts (CUDA events around `--reps` calls after `--warmup`), and the check of its output against the reference's
numpy expressions (restated below: size factors to rtol 1e-12 with the same NaN pattern).  Ratio over every gene
is also timed through the existing `pdq_size_factors_dev`.  A ratio table in which every gene holds a zero has NaN size factors
(the reference switches to its iterative estimator there); it is timed all the same and checked for all-NaN.  The device name and
power limit are read in the same run.  There is no CPU fallback: without a GPU the script fails."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from pydeseq2_b200 import _lib  # noqa: E402

SHAPES = [(200, 20000), (500, 60000), (2000, 7500)]
KINDS = [("ratio", False), ("poscounts", False), ("ratio", True), ("poscounts", True)]


def power_limit_w(index=0):
    try:
        out = subprocess.run(["nvidia-smi", f"--id={index}", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:
        return None


def reference_size_factors(counts, fit_type, control):
    """The reference's expressions (dds.py:656-703): poscounts, or median of ratios over the finite log means, over every gene or
    the control genes.  NaN where a sample has no usable gene."""
    use = np.ones(counts.shape[1], dtype=bool) if control is None else control.copy()
    with np.errstate(divide="ignore", invalid="ignore"), warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)  # np.median([]) = nan
        if fit_type == "poscounts":
            lc = np.zeros_like(counts, dtype=float)
            np.log(counts, out=lc, where=counts != 0)
            lm = lc.mean(0)
            use &= (~np.isinf(lm)) & (lm > 0)
            sf = np.array([np.exp(np.median(np.log(x[use & (x > 0)]) - lm[use & (x > 0)])) for x in counts])
            return sf / np.exp(np.mean(np.log(sf)))
        lc = np.log(counts)
        lm = lc.mean(0)
        use &= ~np.isinf(lm)
        return np.exp(np.median(lc[:, use] - lm[use], axis=1))


def seeded(N, G, zero_frac, seed):
    rng = np.random.default_rng(seed)
    mu = np.exp(rng.normal(3.0, 1.5, G))
    counts = rng.negative_binomial(4, 4 / (4 + mu[None, :] * rng.uniform(0.5, 2.0, (N, 1))))
    counts[rng.random((N, G)) < zero_frac] = 0
    return np.ascontiguousarray(counts, dtype=np.int64)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    assert args.reps >= 1
    ctx = _lib.Context(0)
    L, h, c_d = ctx.lib, ctx.h, _lib.c_dptr
    res = {"metric": "size_factors", "device": ctx.info()["name"], "power_limit_w": power_limit_w(), "reps": args.reps, "cases": []}
    for N, G in SHAPES:
        d_counts, d_sf, d_lm, d_ctl = (ctx.malloc(n) for n in (N * G * 8, N * 8, G * 8, G))
        try:
            for zf in (0.0, 0.7):
                counts = seeded(N, G, zf, seed=N + G)
                ctx.h2d(d_counts, counts)
                ctl = np.zeros(G, dtype=bool)
                ctl[np.random.default_rng(G).choice(G, G // 10, replace=False)] = True
                ctx.h2d(d_ctl, ctl.astype(np.uint8))
                calls = [(f"{k}{'+control' if c else ''}", k, c) for k, c in KINDS] + [("ratio (pdq_size_factors_dev)", "ratio", None)]
                for label, kind, with_ctl in calls:
                    if with_ctl is None:
                        def call():
                            ctx.check(L.pdq_size_factors_dev(h, c_d(d_counts), G, N, G, c_d(d_sf), c_d(d_lm)))
                    else:
                        def call(kind=kind, with_ctl=with_ctl):
                            ctx.check(L.pdq_size_factors_ex_dev(h, c_d(d_counts), G, N, G, 1 if kind == "poscounts" else 0,
                                                                c_d(d_ctl) if with_ctl else None, c_d(d_sf), c_d(d_lm)))
                    for _ in range(args.warmup):
                        call()
                    ctx.sync()
                    ctx.record(0)
                    for _ in range(args.reps):
                        call()
                    ctx.record(1)
                    ctx.sync()
                    ms = ctx.elapsed_ms(0, 1) / args.reps
                    sf = np.empty(N)
                    ctx.d2h(sf, d_sf)
                    ctx.sync()
                    want = reference_size_factors(counts, kind, ctl if with_ctl else None)
                    same_nan = bool(np.array_equal(np.isnan(sf), np.isnan(want)))
                    ok = ~np.isnan(want)
                    err = float(np.max(np.abs(sf[ok] / want[ok] - 1))) if ok.any() else 0.0
                    res["cases"].append({"N": N, "G": G, "zero_frac": zf, "kind": label, "ms": round(ms, 4), "nan": int(np.isnan(sf).sum()),
                                         "max_rel_err": err, "ok": same_nan and err <= 1e-12})
                    print(f"# {N}x{G} zeros={zf} {label:30s} {ms:8.3f} ms  NaN={int(np.isnan(sf).sum())}  rel.err={err:.1e}",
                          file=sys.stderr)
        finally:
            for p in (d_counts, d_sf, d_lm, d_ctl):
                ctx.free(p)
    res["all_ok"] = all(c["ok"] for c in res["cases"])
    print(json.dumps(res))
    if not res["all_ok"]:
        sys.exit(1)


if __name__ == "__main__":
    main()
