"""Time the multiple-testing step of ``DeseqStats.summary()`` (ds.py:486-542) on the GPU (fails without one):

  host    ``workflow.independent_filtering`` on one row (the host restatement the drivers ran per contrast before);
  adjust  ``B200Inference.adjust_pvalues`` on all K rows: host clock around the call, which ends in a device synchronise;
  device  the two device calls alone (``pdq_padj_rejections``, ``pdq_padj_bh``, each with its copies), CUDA events.

    python scripts/padj_bench.py [--reps R] [--out results.json]

Workloads: G in {20 000, 60 000, 125 000, 10^6} genes, K in {1, 6, 45} rows of p-values (45 = the pairwise contrasts of a
ten-level factor); log-normal base means with 2 % exact zeros, p-values with signal in a third of the better expressed genes and
5 % NaN, seeded.  The host restatement works row by row, so it is timed on one row (``host_ms_per_row``).  Every output is checked
in the same run: the cutoffs against ``np.quantile`` on every workload, and the rejection counts and adjusted p-values of the first
and last row against scipy's ``false_discovery_control`` at every cutoff.  The card's name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

GENES = (20_000, 60_000, 125_000, 1_000_000)
ROWS = (1, 6, 45)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def workload(G, K, seed=0):
    rng = np.random.default_rng(seed)
    bm = np.exp(rng.normal(3.0, 2.0, G))
    bm[rng.random(G) < 0.02] = 0.0
    pv = np.empty((K, G))
    for k in range(K):
        signal = (rng.random(G) < 0.3) & (bm > np.quantile(bm, 0.4))
        pv[k] = np.where(signal, rng.beta(0.1, 8.0, G), rng.random(G))
        pv[k, rng.random(G) < 0.05] = np.nan
    return bm, pv


def timed(fn, reps):
    fn()  # warm-up
    best = np.inf
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        best = min(best, time.perf_counter() - t0)
    return best * 1e3


def check_row(bm, p, cutoffs, num_rej, padj, alpha, workflow):
    """num_rej and padj of one row against scipy at every cutoff and the project's threshold rule; True when all are bit-equal."""
    from scipy.stats import false_discovery_control

    cols = np.full((50, len(p)), np.nan)
    for i, c in enumerate(cutoffs):
        use = (bm >= c) & ~np.isnan(p)
        if use.any():
            cols[i, use] = false_discovery_control(p[use], method="bh")
    want = (cols < alpha).sum(1)
    j = workflow.filter_threshold(workflow.filter_theta(bm), want)
    return bool(np.array_equal(want, num_rej) and np.array_equal(cols[j].view(np.int64), padj.view(np.int64)))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", help="also write the table and the card as JSON to this file")
    args = ap.parse_args()
    from pydeseq2_b200 import _lib, workflow
    from pydeseq2_b200.inference import B200Inference

    if _lib.load().pdq_device_count() < 1:
        sys.exit("padj_bench.py needs a CUDA device")
    inf = B200Inference(device=0)
    ops, ctx = inf._ops, inf._ops.ctx
    rows, alpha = [], 0.05
    for G in GENES:
        host_ms = None
        for K in ROWS:
            bm, pv = workload(G, K, seed=G + K)
            if host_ms is None:
                host_ms = timed(lambda: workflow.independent_filtering(bm, pv[0], alpha), 1 if G > 200_000 else args.reps)
            out = {}

            def adjust():
                out["padj"] = inf.adjust_pvalues(bm, pv, alpha)
                ctx.sync()

            adjust_ms = timed(adjust, args.reps)
            theta = workflow.filter_theta(bm)
            cutoffs, num_rej = np.empty(50), np.empty((K, 50), dtype=np.int32)
            cut_k, padj = np.full(K, -np.inf), ops.empty((K, G))
            ev = {"rejections": [], "bh": []}
            for rep in range(args.reps + 1):
                ctx.record(0)
                ops.padj_rejections(bm, G, pv, G, K, theta, 50, alpha, cutoffs, num_rej)
                ctx.record(1)
                ops.padj_bh(bm, G, pv, G, K, cut_k, padj, G)
                ctx.record(2)
                ctx.sync()
                if rep:
                    ev["rejections"].append(ctx.elapsed_ms(0, 1))
                    ev["bh"].append(ctx.elapsed_ms(1, 2))
            ok = bool(np.array_equal(cutoffs.view(np.int64), np.quantile(bm, theta).view(np.int64)))
            for k in sorted({0, K - 1}):
                ok &= check_row(bm, pv[k], cutoffs, num_rej[k], out["padj"][k], alpha, workflow)
            row = dict(genes=G, K=K, host_ms_per_row=host_ms, adjust_ms=adjust_ms, host_over_adjust=K * host_ms / adjust_ms,
                       rejections_ms=float(np.median(ev["rejections"])), bh_ms=float(np.median(ev["bh"])), bit_equal=ok)
            print(json.dumps(row), flush=True)
            rows.append(row)
    res = dict(card=card(), rows=rows)
    print(json.dumps({"card": res["card"]}))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    if not all(r["bit_equal"] for r in rows):
        sys.exit("padj_bench.py: an output differs from numpy / scipy")


if __name__ == "__main__":
    main()
