#!/usr/bin/env python
"""Timings of designs of 65..128 columns (B200Inference(wide_designs=True, large_designs=True)): paired designs
~subject + condition at p = 65, 81, 101 and 128, N = 2 (p - 1) samples, G genes (default 20 000), with the 17..64 tier at p = 64 as
the anchor.  Every W of {2, 4, 8} warps per gene is timed in the same run, alternating W inside each round (the PDQ_LARGE_WARPS
tuning hook is read when a design pack is made).

Per (p, W), one JSON line with the median over --rounds of the per-stage kernel times of one profiled ResidentFit pass (CUDA
events around each stage; the stages are serialised for it): IRLS (`irls_init`), the genewise search (`alpha_mle_genewise`),
MAP + LFC + Wald (`alpha_mle_map` + `select_dispersions` + `irls_lfc_wald`) and Cook's distances (`cooks`), plus the whole pass (`resident_ms`, host
clock around a pass that ends in a device synchronise).  The card's name, power limit and maximum SM clock are read in the same
run.

    python scripts/large_design_bench.py [--genes 20000] [--ps 64,65,81,101,128] [--warps 2,4,8] [--rounds 3]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from pydeseq2_b200.inference import B200Inference  # noqa: E402
from pydeseq2_b200.pipeline import ResidentFit, median_of_ratios  # noqa: E402


def paired(subjects):
    subj = np.repeat(np.arange(subjects), 2)
    cols = [np.ones(2 * subjects)] + [(subj == s).astype(float) for s in range(1, subjects)] + [np.tile([0.0, 1.0], subjects)]
    return np.stack(cols, axis=1)


def counts_for(X, G, seed):  # as scripts/wide_design_bench.py
    rng = np.random.default_rng(seed)
    beta = np.c_[rng.normal(5.0, 1.5, G), rng.normal(0.0, 0.5, (G, X.shape[1] - 1)) * (rng.random((G, 1)) < 0.4)]
    sf = np.exp(rng.normal(0.0, 0.2, X.shape[0]))
    mu = sf[:, None] * np.exp(X @ beta.T)
    d = (0.05 + 2.0 / np.exp(beta[:, 0])) * np.exp(rng.normal(0, 0.3, G))
    c = rng.negative_binomial(1 / d, 1 / (1 + mu * d)).astype(np.int64)
    return np.ascontiguousarray(c[:, ~(c == 0).all(0)])


GROUPS = {"irls": ("irls_init",), "genewise": ("alpha_mle_genewise",), "map_lfc_wald": ("alpha_mle_map", "select_dispersions", "irls_lfc_wald"),
          "cooks": ("cooks",)}


def grouped(stage_ms):
    out = {}
    for g, keys in GROUPS.items():
        hit = [v for k, v in stage_ms.items() if any(k.startswith(s) for s in keys)]
        out[g] = round(sum(hit), 3) if hit else None
    return out


ap = argparse.ArgumentParser()
ap.add_argument("--genes", type=int, default=20000)
ap.add_argument("--ps", default="64,65,81,101,128")
ap.add_argument("--warps", default="2,4,8")
ap.add_argument("--rounds", type=int, default=3)
a = ap.parse_args()

try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                          text=True, timeout=30).stdout.strip().splitlines()[0]
except Exception as e:  # the query is a label, not a measurement
    card = f"unknown ({e})"
inf = B200Inference(device=0, wide_designs=True, large_designs=True)
ctx = inf._ops.ctx
for p in (int(v) for v in a.ps.split(",")):
    X = paired(p - 1)
    counts = counts_for(X, a.genes, seed=p)
    G = counts.shape[1]
    sf = median_of_ratios(counts)[1]
    variants = [int(w) for w in a.warps.split(",")] if p > 64 else [1]
    res = {w: dict(stages=[], passes=[]) for w in variants}
    for _ in range(a.rounds):
        for w in variants:  # alternating: every round times every W once
            os.environ["PDQ_LARGE_WARPS"] = str(w)
            rf = ResidentFit(ctx, X, sf, with_cooks=True)
            rf.upload(counts)
            rf.run()  # warm-up (module load, allocations)
            t0 = time.perf_counter()
            rf.run()
            res[w]["passes"].append((time.perf_counter() - t0) * 1e3)
            rf.run(profile=True)
            res[w]["stages"].append(dict(rf.stage_ms))
            rf.close()
    os.environ.pop("PDQ_LARGE_WARPS", None)
    for w in variants:
        keys = res[w]["stages"][0].keys()
        med = {k: float(np.median([s[k] for s in res[w]["stages"]])) for k in keys}
        print(json.dumps(dict(p=p, N=X.shape[0], genes=G, warps=w, card=card, rounds=a.rounds,
                              resident_ms=round(float(np.median(res[w]["passes"])), 3), stages_ms=grouped(med),
                              all_stages_ms={k: round(v, 3) for k, v in med.items()})), flush=True)
