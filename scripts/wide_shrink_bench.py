#!/usr/bin/env python
"""Timings of apeGLM shrinkage on designs of 17..128 columns (B200Inference(wide_designs=True, wide_shrink=True), and
large_designs=True, large_shrink=True as well when a --ps width is above 64): paired designs ~subject + condition at p = 21, 33 and
64 by default, N = 2 (p - 1) samples, G genes (default 20 000), shrinking the condition column with the adapted prior scale.  The
dispersions and MLE tables come from one ResidentFit pass.  Above 64 columns every W of --warps (warps per gene, the
PDQ_LARGE_WARPS tuning hook, read when a design pack is made) gets its own context and resident fit, and the W are timed
alternately inside each of --rounds rounds.  Per shape (and W), one JSON line:

* ``plugin_ms``: ``lfc_shrink_nbinom_glm`` on host buffers, with its full (G, p, p) inverse-Hessian output.
* ``resident_ms``: ``ResidentFit.lfc_shrink`` on the resident counts (downloads column k, the [k, k] entries and the flags).
  Both are the median of --steps calls (per round, over every round) after one warm-up call; each call ends in a device
  synchronise, so the host clock around it is the call's time.  At p = 128 the plugin call returns G p^2 doubles of inverse
  Hessians (2.6 GB at 20 000 genes), which the resident call does not download.
* ``oracle_ms_extrapolated``: the oracle port (scipy's L-BFGS-B per gene, the reference's joblib fan-out over every host core) on a
  --oracle-genes subset, scaled by G / subset.  ``nfev_median`` / ``nfev_max``: scipy's objective evaluations per gene on the first
  --count-genes genes (the kernel walks the same iteration, so it makes about as many sweeps).
The card's name, power limit and maximum SM clock are read in the same run.

    python scripts/wide_shrink_bench.py [--genes 20000] [--ps 21,33,64] [--steps 5]
    python scripts/wide_shrink_bench.py --ps 65,81,101,128 [--warps 2,4,8] [--rounds 3] --oracle-genes 0"""
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
ap.add_argument("--warps", default="2,4,8", help="warps per gene timed above 64 columns")
ap.add_argument("--rounds", type=int, default=1)
a = ap.parse_args()


def times_ms(fn, steps):
    times = []
    for _ in range(steps):
        t0 = time.perf_counter()
        fn()
        times.append((time.perf_counter() - t0) * 1e3)
    return times


try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                          text=True, timeout=30).stdout.strip().splitlines()[0]
except Exception as e:  # the query is a label, not a measurement
    card = f"unknown ({e})"
ps = [int(v) for v in a.ps.split(",")]
large = max(ps) > 64
for p in ps:
    X = paired(p - 1)
    N, k = X.shape[0], p - 1
    counts = counts_for(X, a.genes, seed=p)
    G = counts.shape[1]
    sf = median_of_ratios(counts)[1]
    size = offset = scale = None
    runs = {}  # W (None: the built-in choice) -> backend, resident fit, its pass, plugin / resident times
    for w in ([int(v) for v in a.warps.split(",")] if p > 64 else [None]):
        if w:
            os.environ["PDQ_LARGE_WARPS"] = str(w)
        inf = B200Inference(device=0, wide_designs=True, wide_shrink=True, large_designs=large, large_shrink=large)
        rf = ResidentFit(inf._ops.ctx, X, sf)
        rf.upload(counts)
        r = rf.run(contrast=np.eye(p)[k])
        if size is None:  # every W shrinks the first fit's dispersions on the plugin path
            disp = np.asarray(r["dispersions"])
            scale = float(np.minimum(np.sqrt(fit_shrink_prior_var(np.asarray(r["lfc"])[:, k], np.asarray(r["se"]))), 1))
            size, offset = 1.0 / disp, np.log(sf)
        inf.lfc_shrink_nbinom_glm(X, counts, size, offset, 15, scale, "L-BFGS-B", k)  # warm-up; makes the plugin's pack with W
        conv = rf.lfc_shrink(r, k, prior_scale=scale).converged  # warm-up
        os.environ.pop("PDQ_LARGE_WARPS", None)
        runs[w] = dict(inf=inf, rf=rf, r=r, conv=conv, plugin=[], resident=[])
    for _ in range(a.rounds):
        for w, u in runs.items():  # alternating: every round times every W
            u["plugin"] += times_ms(lambda: u["inf"].lfc_shrink_nbinom_glm(X, counts, size, offset, 15, scale, "L-BFGS-B", k), a.steps)
            u["resident"] += times_ms(lambda: u["rf"].lfc_shrink(u["r"], k, prior_scale=scale), a.steps)
    for w, u in runs.items():
        u["rf"].close()
        plugin, resident = float(np.median(u["plugin"])), float(np.median(u["resident"]))
        out = dict(p=p, N=N, genes=G, card=card, prior_scale=scale, converged=float(np.mean(u["conv"])), plugin_ms=plugin,
                   plugin_genes_per_s=G / (plugin / 1e3), resident_ms=resident, resident_genes_per_s=G / (resident / 1e3))
        if w:
            out.update(warps=w, rounds=a.rounds, plugin_ms_all=[round(t, 1) for t in u["plugin"]],
                       resident_ms_all=[round(t, 1) for t in u["resident"]])
        print(json.dumps(out), flush=True)
    runs.clear()
    if a.oracle_genes:
        out = dict(p=p, N=N, genes=G)
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
