#!/usr/bin/env python
"""The CPU baseline `bench.py` times is the oracle PORT (the benchmark does not depend on the reference).  This script, run with
PYDESEQ2_SRC naming a PyDESeq2 0.5.3 source checkout, times the REAL reference's DefaultInference and the port through the same host glue (pipeline.fit_host) on the same
input, so that the record shows the port is not slower than the code it stands for.  Output: one JSON line."""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
os.environ["PYTHONPATH"] = os.pathsep.join([os.path.join(ROOT, "oracle", "refshim"), ROOT, os.environ.get("PYTHONPATH", "")])
sys.path.insert(0, os.path.join(ROOT, "oracle", "refshim"))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402


class FloatFlags:
    """The reference's backend with `converged` returned as float64 (pandas >= 3, SURVEY.md §8c)."""

    def __init__(self, inner):
        self.inner = inner

    def __getattr__(self, name):
        fn = getattr(self.inner, name)
        if name in ("irls", "alpha_mle"):
            def wrapped(*a, **k):
                out = list(fn(*a, **k))
                out[-1] = np.asarray(out[-1], dtype=float)
                return tuple(out)
            return wrapped
        if name == "dispersion_trend_gamma_glm":  # the orchestrator hands it pandas objects (dds.py:1240)
            import pandas as pd

            def trend(cov, targets):
                co, pred, ok = fn(pd.Series(np.asarray(cov)), pd.Series(np.asarray(targets)))
                return np.asarray(co, dtype=float), np.asarray(pred, dtype=float), ok
            return trend
        return fn


def main():
    from pydeseq2.default_inference import DefaultInference  # the real reference, read-only checkout

    from oracle import nbglm
    from pydeseq2_b200.pipeline import fit_host, median_of_ratios
    from pydeseq2_b200.synth import make_counts

    G, N = int(os.environ.get("PVR_GENES", 3000)), 200
    counts, X, _ = make_counts(N, G, "two_level", seed=0)
    counts = np.ascontiguousarray(counts[:, ~(counts == 0).all(0)])
    sf = median_of_ratios(counts)[1]
    cores = os.cpu_count() or 1
    res = {}
    for name, inf in (("reference DefaultInference", FloatFlags(DefaultInference(n_cpus=cores))), ("oracle port", nbglm.OracleInference(n_cpus=cores))):
        fit_host(counts[:, :256], X, inf, size_factors=sf)  # pool start-up
        t0 = time.perf_counter()
        r = fit_host(counts, X, inf, size_factors=sf)
        dt = time.perf_counter() - t0
        res[name] = {"seconds": round(dt, 2), "genes_per_s": round(counts.shape[1] / dt, 1), "lfc_checksum": float(np.nansum(np.abs(r.lfc)))}
    print(json.dumps({"workload": f"{counts.shape[1]} genes x {N} samples, two-level design", "cores": cores, **res}))


if __name__ == "__main__":
    main()
