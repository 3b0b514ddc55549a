"""Times the four large host-buffer plugin calls for several gene-block pipeline depths (PDQ_PIPELINE).
Run on an H100:  python scripts/pipe_microbench.py [G] [N]"""
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pydeseq2_b200.inference import B200Inference  # noqa: E402
from pydeseq2_b200.pipeline import median_of_ratios  # noqa: E402
from pydeseq2_b200.synth import make_counts  # noqa: E402

G = int(sys.argv[1]) if len(sys.argv) > 1 else 20000
N = int(sys.argv[2]) if len(sys.argv) > 2 else 200
counts, X, _ = make_counts(N, G, "two_level", 0)
counts = np.ascontiguousarray(counts[:, ~(counts == 0).all(0)])
sf = median_of_ratios(counts)[1]
rng = np.random.default_rng(0)
disp = np.exp(rng.normal(-1.5, 1.0, counts.shape[1]))


def best(f, n=7):
    ts = []
    for _ in range(n):
        t = time.perf_counter()
        f()
        ts.append((time.perf_counter() - t) * 1e3)
    return min(ts), float(np.median(ts))


for depth in (0, 2, 3, 4, 6, 8, 16):
    os.environ["PDQ_PIPELINE"] = str(depth)
    inf = B200Inference(device=0)
    ctx = inf._ops.ctx
    c_host = ctx.pinned_empty(counts.shape, np.int64)
    c_host[...] = counts
    mu = inf.lin_reg_mu(c_host, sf, X, 0.5)
    beta, mu2, hat, conv = inf.irls(c_host, sf, X, disp, 0.5, 1e-8)
    ridge = np.diag(np.repeat(1e-6, X.shape[1]))
    contrast = np.array([0.0, 1.0])
    row = {
        "lin_reg_mu": best(lambda: inf.lin_reg_mu(c_host, sf, X, 0.5)),
        "alpha_mle": best(lambda: inf.alpha_mle(c_host, X, mu, disp, 1e-8, float(N))),
        "irls": best(lambda: inf.irls(c_host, sf, X, disp, 0.5, 1e-8)),
        "wald": best(lambda: inf.wald_test(X, disp, beta, mu2, ridge, contrast, 0.0, None)),
    }
    print(f"depth {depth:2d}: " + "  ".join(f"{k} {v[0]:.3f}/{v[1]:.3f}" for k, v in row.items()), flush=True)
    del inf
