"""Time K Wald contrasts on one fit, three ways, on the GPU (fails without one):

  (a) one ``pdq_wald_contrasts`` call for all K (``B200Inference.wald_tests``: mu built on the device);
  (b) K rounds of the drop-in path before it: host mu = exp(X @ LFC.T) * sf (ds.py:320-324), then ``B200Inference.wald_test``;
  (c) K x ``ResidentFit.run(contrast=...)``: the whole resident pass once per contrast, the way the drivers key a second contrast.

    python scripts/contrast_bench.py [--reps R] [--out results.json]

Workloads at user sizes: 20 000 genes x 200 samples with a 4-level factor (K = 6), 60 000 x 500 with a 6-level factor (K = 15) and
20 000 x 200 with 10 levels (K = 45), all pairwise contrasts.  Times are host clocks around work that ends in a device
synchronise, after one warm-up of each path; (a) returns page-locked arrays, (b) uploads mu from an ordinary numpy array.  Also
reported: the largest relative difference between (a) and (b), and the card's name and power limit read in the same run.
"""
from __future__ import annotations

import argparse
import itertools
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

WORKLOADS = [("20000x200_4lvl", 20000, 200, 4), ("60000x500_6lvl", 60000, 500, 6), ("20000x200_10lvl", 20000, 200, 10)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def workload(G, N, levels, seed=0):
    rng = np.random.default_rng(seed)
    lv = np.arange(N) % levels
    X = np.zeros((N, levels))
    X[:, 0] = 1.0
    for j in range(1, levels):
        X[:, j] = lv == j
    beta = np.c_[rng.normal(5, 1.5, G), rng.normal(0, 0.7, (G, levels - 1))]
    sf = np.exp(rng.normal(0, 0.2, N))
    mu = sf[:, None] * np.exp(X @ beta.T)
    d = (0.05 + 2.0 / np.exp(beta[:, 0])) * np.exp(rng.normal(0, 0.3, G))
    counts = rng.negative_binomial(1 / d, 1 / (1 + mu * d)).astype(np.int64)
    pairs = []
    for i, j in itertools.combinations(range(levels), 2):
        v = np.zeros(levels)
        v[j] += 1.0
        if i:
            v[i] -= 1.0
        pairs.append(v)
    return counts, X, np.array(pairs)


def timed(fn, reps):
    fn()  # warm-up
    best = np.inf
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        best = min(best, time.perf_counter() - t0)
    return best * 1e3


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", help="also write the table and the card as JSON to this file")
    args = ap.parse_args()
    from pydeseq2_b200 import _lib
    from pydeseq2_b200.inference import B200Inference
    from pydeseq2_b200.pipeline import ResidentFit

    if _lib.load().pdq_device_count() < 1:
        sys.exit("contrast_bench.py needs a CUDA device")
    inf = B200Inference(device=0)
    ctx = inf._ops.ctx
    rows = []
    for name, G, N, levels in WORKLOADS:
        counts, X, cs = workload(G, N, levels)
        K, p = cs.shape
        nz = ~(counts == 0).all(0)
        rf = ResidentFit(ctx, X, None)
        rf.upload(np.ascontiguousarray(counts[:, nz]))
        try:
            r = rf.run(contrast=cs[0])
            lfc, disp, sf = np.ascontiguousarray(r["lfc"]), np.ascontiguousarray(r["dispersions"]), np.asarray(rf.sf)
            ridge = np.diag(np.repeat(1e-6, p))
            out_a = {}

            def path_a():
                out_a["r"] = inf.wald_tests(X, sf, disp, lfc, cs, ridge)
                ctx.sync()

            out_b = {}

            def path_b():
                res = []
                for c in cs:
                    mu = np.exp(X @ lfc.T) * sf[:, None]  # a pageable numpy array, as DeseqStats builds it
                    res.append(inf.wald_test(X, disp, lfc, mu, ridge, c, 0.0, None))
                ctx.sync()
                out_b["r"] = res

            def path_c():
                for c in cs:
                    rf.run(contrast=c)
                ctx.sync()

            ta, tb = timed(path_a, args.reps), timed(path_b, args.reps)
            tc = timed(path_c, max(1, args.reps // 2))
            worst = [0.0, 0.0, 0.0]  # p-value, statistic, SE
            for k in range(K):
                for i, want in enumerate(out_b["r"][k]):
                    got = out_a["r"][i][k]
                    ok = np.isfinite(want) & (want != 0)
                    if ok.any():
                        worst[i] = max(worst[i], float(np.max(np.abs(got[ok] - want[ok]) / np.abs(want[ok]))))
        finally:
            rf.close()
        row = dict(workload=name, genes=int(nz.sum()), samples=N, K=K, a_ms=ta, b_ms=tb, c_ms=tc, b_over_a=tb / ta, c_over_a=tc / ta,
                   max_rel_diff_a_b=dict(zip(("pvalue", "stat", "se"), worst)))
        print(json.dumps(row), flush=True)
        rows.append(row)
    res = dict(card=card(), rows=rows)
    print(json.dumps({"card": res["card"]}))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
