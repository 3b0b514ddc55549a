"""Time the dispersion trend + prior launch (`pdq_trend_fit_dev`) with the prior on and off.

    python scripts/trend_prior_bench.py [--reps 300] [--warmup 20] [--sizes 20000,50000,125000]

The input is the synthetic vector of scripts/trend_microbench.py (log2 means ~ N(4, 2), genewise dispersions scattered
log-normally, sd 0.5, around 4 / mean + 0.1).  Vectors below 65 536 genes run the one-cluster kernel (`k_trend_prior`), larger
ones the cooperative grid kernel (`k_trend_prior_grid`).  `PDQ_TREND_PRIOR=0` skips the prior; the difference of the two times is
what the prior's two medians cost.  Each time is the mean over `--reps` back-to-back launches between two CUDA events, after
`--warmup` launches.  The device name and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
from scipy.special import polygamma  # noqa: E402

from pydeseq2_b200 import _lib  # noqa: E402


def gpu_card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return [s.strip() for s in q.split(",")]
    except Exception as e:  # pragma: no cover - reported, not fatal
        return [f"nvidia-smi unavailable: {e}"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--sizes", default="20000,50000,125000")
    args = ap.parse_args()
    ctx = _lib.Context(0)
    L, cd = ctx.lib, _lib.c_dptr
    print("device", ctx.info()["name"], "| nvidia-smi name, power limit, max SM clock:", ", ".join(gpu_card()), flush=True)
    trig = float(polygamma(1, 99))
    rows = []
    for n in (int(s) for s in args.sizes.split(",")):
        rng = np.random.default_rng(0)
        means = np.exp(rng.normal(4, 2, n) * np.log(2))
        gw = (4 / means + 0.1) * np.exp(rng.normal(0, 0.5, n))
        dm, dg, dout = ctx.malloc(n * 8), ctx.malloc(n * 8), ctx.malloc(128)
        ctx.h2d(dm, means)
        ctx.h2d(dg, gw)
        ctx.sync()
        row = {"n": n, "kernel": "grid" if n >= 65536 else "cluster"}
        for prior in ("0", "1"):
            os.environ["PDQ_TREND_PRIOR"] = prior
            try:
                def launch():
                    ctx.check(L.pdq_trend_fit_dev(ctx.h, cd(dm), cd(dg), n, 1e-8, 200.0, trig, cd(dout), cd(0)))
                for _ in range(args.warmup):
                    launch()
                ctx.sync()
                ctx.record(0)
                for _ in range(args.reps):
                    launch()
                ctx.record(1)
                ctx.sync()
                ms = ctx.elapsed_ms(0, 1) / args.reps
            finally:
                del os.environ["PDQ_TREND_PRIOR"]
            out = np.zeros(16)
            ctx.d2h(out, dout)
            ctx.sync()
            row["fit_ms" if prior == "0" else "fit_prior_ms"] = round(ms, 4)
            if prior == "1":
                row.update(n_outer=int(out[3]), n_iter=int(out[5]), n_used=int(out[4]), n_above=int(out[10]),
                           squared_logres=float(out[8]))
        row["prior_ms"] = round(row["fit_prior_ms"] - row["fit_ms"], 4)
        rows.append(row)
        print(json.dumps(row), flush=True)
        for p in (dm, dg, dout):
            ctx.free(p)
    ctx.close()


if __name__ == "__main__":
    main()
