#!/usr/bin/env python
"""Timings of designs of 17..64 columns (B200Inference(wide_designs=True)): paired designs ~subject + condition at p = 21, 33 and
64, N = 2 (p - 1) samples, G genes (default 20 000).  Per shape, one JSON line:

* ``resident_ms``: one ResidentFit pass (counts in HBM), median of --steps passes after one warm-up; the pass ends in a device
  synchronise, so the host clock around it is the pass's time.  ``stages_ms``: the per-stage split of one profiled pass (CUDA events
  around each stage; the stages are serialised for it).
* ``plugin_ms``: the same fit through the plugin calls with host buffers (pipeline.fit_host), median of --plugin-steps.
* ``oracle_ms_extrapolated``: the oracle port (per-gene numpy / scipy with the reference's joblib fan-out over every host core) on a
  --oracle-genes subset, scaled by G / subset, as BASELINE.md §3 does for C4 / C5.
The card's name, power limit and maximum SM clock are read in the same run.

    python scripts/wide_design_bench.py [--genes 20000] [--ps 21,33,64] [--steps 5]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from pydeseq2_b200.inference import B200Inference  # noqa: E402
from pydeseq2_b200.pipeline import ResidentFit, fit_host, median_of_ratios  # noqa: E402


def paired(subjects):
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


ap = argparse.ArgumentParser()
ap.add_argument("--genes", type=int, default=20000)
ap.add_argument("--ps", default="21,33,64")
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("--plugin-steps", type=int, default=2)
ap.add_argument("--oracle-genes", type=int, default=2000, help="0 skips the oracle port")
a = ap.parse_args()

try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                          text=True, timeout=30).stdout.strip().splitlines()[0]
except Exception as e:  # the query is a label, not a measurement
    card = f"unknown ({e})"
inf = B200Inference(device=0, wide_designs=True)
ctx = inf._ops.ctx
for p in (int(v) for v in a.ps.split(",")):
    X = paired(p - 1)
    N = X.shape[0]
    counts = counts_for(X, a.genes, seed=p)
    G = counts.shape[1]
    sf = median_of_ratios(counts)[1]
    rf = ResidentFit(ctx, X, sf)
    rf.upload(counts)
    rf.run()  # warm-up (module load, allocations)
    times = []
    for _ in range(a.steps):
        t0 = time.perf_counter()
        rf.run()
        times.append((time.perf_counter() - t0) * 1e3)
    rf.run(profile=True)
    stages = {k: round(v, 3) for k, v in rf.stage_ms.items()}
    rf.close()
    fit_host(counts[:, :256], X, inf, size_factors=sf)  # warm-up
    plug = []
    for _ in range(a.plugin_steps):
        t0 = time.perf_counter()
        fit_host(counts, X, inf, size_factors=sf)
        plug.append((time.perf_counter() - t0) * 1e3)
    out = dict(p=p, N=N, genes=G, card=card, resident_ms=float(np.median(times)), resident_genes_per_s=G / (np.median(times) / 1e3),
               stages_ms=stages, plugin_ms=float(np.median(plug)), plugin_genes_per_s=G / (np.median(plug) / 1e3))
    if a.oracle_genes:
        from oracle import nbglm

        sub = np.ascontiguousarray(counts[:, :a.oracle_genes])
        ora = nbglm.OracleInference(n_cpus=os.cpu_count())
        t0 = time.perf_counter()
        fit_host(sub, X, ora, size_factors=sf)
        ms = (time.perf_counter() - t0) * 1e3
        out.update(oracle_genes=sub.shape[1], oracle_ms=ms, oracle_ms_extrapolated=ms * G / sub.shape[1], host_cores=os.cpu_count())
    print(json.dumps(out), flush=True)
