#!/usr/bin/env python
"""A/B of the resident pass' tail: (a) MAP search, final dispersions and LFC fit + Wald test as three launches against (b) the
kernel pair with per-tile hand-off (ResidentFit.fuse_tail), alternated pass by pass in one process on the shapes bench.py
measures.  CUDA events around the device work of a pass, L2 flushed before each; card name and power limit read in the same run.
    PDQ_LIB=pydeseq2_b200/libvariant.so python scripts/tail_bench.py --steps 40 [--shapes C2,C3]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from pydeseq2_b200 import _lib  # noqa: E402
from pydeseq2_b200.inference import B200Inference  # noqa: E402
from pydeseq2_b200.pipeline import ResidentFit, median_of_ratios  # noqa: E402
from pydeseq2_b200.synth import make_counts  # noqa: E402

SHAPES = {"C2": (20000, 200, "two_level"), "C3": (60000, 500, "factorial"), "C4_shard": (7500, 2000, "continuous"),
          "C5_shard": (125000, 1000, "two_level")}

ap = argparse.ArgumentParser()
ap.add_argument("--shapes", default="C2,C3,C4_shard,C5_shard")
ap.add_argument("--steps", type=int, default=40)
a = ap.parse_args()

try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                          text=True, timeout=30).stdout.strip().splitlines()[0]
except Exception as e:  # the query is a label, not a measurement
    card = f"unknown ({e})"
inf = B200Inference(device=0)
ctx = inf._ops.ctx
flush = ctx.malloc(256 << 20)
for name in a.shapes.split(","):
    G, N, design = SHAPES[name]
    counts, X, _ = make_counts(N, G, design, seed=0, sample_seed=0)
    counts = np.ascontiguousarray(counts[:, ~(counts == 0).all(0)])
    sf = median_of_ratios(counts)[1]
    fits = {}
    for label, fused in (("separate", False), ("fused", True)):
        rf = fits[label] = ResidentFit(ctx, X, sf)
        rf.fuse_tail = fused
        rf.upload(counts)
        for _ in range(3):
            last = rf.run()
        fits[label + "_out"] = last
    same = all(np.array_equal(fits["separate_out"][k], fits["fused_out"][k], equal_nan=True)
               for k in ("map", "dispersions", "lfc", "pvalue", "stat", "se", "outlier"))
    ms = {"separate": [], "fused": []}
    for _ in range(a.steps):
        for label in ("separate", "fused"):
            ctx.check(ctx.lib.pdq_memset(ctx.h, _lib.c_dptr(flush), 1, 256 << 20))
            ctx.sync()
            fits[label].run(events=(0, 1), copy=False)
            ms[label].append(ctx.elapsed_ms(0, 1))
    rec = {"lib": os.environ.get("PDQ_LIB", "default"), "card": card, "shape": name, "genes": int(counts.shape[1]), "samples": N,
           "design": design, "steps": a.steps, "bit_identical": bool(same)}
    for label, v in ms.items():
        v = np.asarray(v)
        rec[label] = {"mean_ms": round(float(v.mean()), 4), "median_ms": round(float(np.median(v)), 4),
                      "min_ms": round(float(v.min()), 4), "max_ms": round(float(v.max()), 4)}
    rec["fused_over_separate"] = round(rec["fused"]["median_ms"] / rec["separate"]["median_ms"], 4)
    print(json.dumps(rec), flush=True)
    for label in ("separate", "fused"):
        fits[label].close()
