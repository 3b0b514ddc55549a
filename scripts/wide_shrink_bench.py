#!/usr/bin/env python
"""Timings of apeGLM shrinkage on designs of 17..64 columns (B200Inference(wide_designs=True, wide_shrink=True)): paired designs
~subject + condition at p = 21, 33 and 64, N = 2 (p - 1) samples, G genes (default 20 000), shrinking the condition column with
the adapted prior scale.  The dispersions and MLE tables come from one ResidentFit pass.  Per shape, one JSON line:

* ``plugin_ms``: ``lfc_shrink_nbinom_glm`` on host buffers, with its full (G, p, p) inverse-Hessian output.
* ``resident_ms``: ``ResidentFit.lfc_shrink`` on the resident counts (downloads column k, the [k, k] entries and the flags).
  Both are the median of --steps calls after one warm-up call; each call ends in a device synchronise, so the host clock around it
  is the call's time.
* ``oracle_ms_extrapolated``: the oracle port (scipy's L-BFGS-B per gene, the reference's joblib fan-out over every host core) on a
  --oracle-genes subset, scaled by G / subset.  ``nfev_median`` / ``nfev_max``: scipy's objective evaluations per gene on the first
  --count-genes genes (the kernel walks the same iteration, so it makes about as many sweeps).
The card's name, power limit and maximum SM clock are read in the same run.

    python scripts/wide_shrink_bench.py [--genes 20000] [--ps 21,33,64] [--steps 5]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from pydeseq2_b200.inference import B200Inference  # noqa: E402
from pydeseq2_b200.pipeline import ResidentFit, fit_shrink_prior_var, median_of_ratios  # noqa: E402


def paired(subjects):  # the shapes and counts of scripts/wide_design_bench.py
    subj = np.repeat(np.arange(subjects), 2)
    cols = [np.ones(2 * subjects)] + [(subj == s).astype(float) for s in range(1, subjects)] + [np.tile([0.0, 1.0], subjects)]
    return np.stack(cols, axis=1)


def counts_for(X, G, seed):
    rng = np.random.default_rng(seed)
    beta = np.c_[rng.normal(5.0, 1.5, G), rng.normal(0.0, 0.5, (G, X.shape[1] - 1)) * (rng.random((G, 1)) < 0.4)]
    sf = np.exp(rng.normal(0.0, 0.2, X.shape[0]))
    mu = sf[:, None] * np.exp(X @ beta.T)
    d = (0.05 + 2.0 / np.exp(beta[:, 0])) * np.exp(rng.normal(0, 0.3, G))
    c = rng.negative_binomial(1 / d, 1 / (1 + mu * d)).astype(np.int64)
    return np.ascontiguousarray(c[:, ~(c == 0).all(0)])


ap =argparse.ArgumentParser()
ap.add_argument("--genes", type=int, default=20000)
ap.add_argument("--ps", default="21,33,64")
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("--oracle-genes", type=int, default=1000, help="0 skips the oracle port")
ap.add_argument("--count-genes", type=int, default=200)
a = ap.parse_args()


def median_ms(fn, steps):
    fn()  # warm-up (module load, allocations)
    times = []
    for _ in range(steps):
        t0 = time.perf_counter()
        fn()
        times.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(times))


try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                          text=True, timeout=30).stdout.strip().splitlines()[0]
except Exception as e:  # the query is a label, not a measurement
    card = f"unknown ({e})"
inf = B200Inference(device=0, wide_designs=True, wide_shrink=True)
ctx = inf._ops.ctx
for p in (int(v) for v in a.ps.split(",")):
    X = paired(p - 1)
    N, k = X.shape[0], p - 1
    counts = counts_for(X, a.genes, seed=p)
    G = counts.shape[1]
    sf = median_of_ratios(counts)[1]
    rf = ResidentFit(ctx, X, sf)
    rf.upload(counts)
    r = rf.run(contrast=np.eye(p)[k])
    disp = np.asarray(r["dispersions"])
    scale = float(np.minimum(np.sqrt(fit_shrink_prior_var(np.asarray(r["lfc"])[:, k], np.asarray(r["se"]))), 1))
    size, offset = 1.0 / disp, np.log(sf)
    plugin = median_ms(lambda: inf.lfc_shrink_nbinom_glm(X, counts, size, offset, 15, scale, "L-BFGS-B", k), a.steps)
    resident = median_ms(lambda: rf.lfc_shrink(r, k, prior_scale=scale), a.steps)
    conv = rf.lfc_shrink(r, k, prior_scale=scale).converged
    rf.close()
    out = dict(p=p, N=N, genes=G, card=card, prior_scale=scale, converged=float(np.mean(conv)), plugin_ms=plugin,
               plugin_genes_per_s=G / (plugin / 1e3), resident_ms=resident, resident_genes_per_s=G / (resident / 1e3))
    if a.oracle_genes:
        from oracle import nbglm

        sub = slice(0, a.oracle_genes)
        ora = nbglm.OracleInference(n_cpus=os.cpu_count())
        cs = np.ascontiguousarray(counts[:, sub])
        t0 = time.perf_counter()
        ora.lfc_shrink_nbinom_glm(X, cs, size[sub], offset, 15, scale, "L-BFGS-B", k)
        ms = (time.perf_counter() - t0) * 1e3
        inner, seen = nbglm._minimize, []

        def counted(*args, **kw):
            res = inner(*args, **kw)
            seen.append(int(res.nfev))
            return res

        nbglm._minimize = counted
        try:
            for i in range(min(a.count_genes, G)):
                nbglm.nbinom_glm_gene(X, counts[:, i], size[i], offset, 15, scale, "L-BFGS-B", k)
        finally:
            nbglm._minimize = inner
        out.update(oracle_genes=cs.shape[1], oracle_ms=ms, oracle_ms_extrapolated=ms * G / cs.shape[1], host_cores=os.cpu_count(),
                   nfev_median=float(np.median(seen)), nfev_max=int(np.max(seen)))
    print(json.dumps(out), flush=True)
