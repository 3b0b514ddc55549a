"""Shared helpers of tests/test_padj.py and tests/test_gpu_padj.py: bit-for-bit comparison, seeded base means and p-values, and
numpy / scipy restatements of one row of the multiple-testing step."""
import glob
import os

import numpy as np
from scipy.stats import false_discovery_control

from conftest import GOLDEN

PADJ = sorted(os.path.basename(f)[:-4] for f in glob.glob(os.path.join(GOLDEN, "padj_*.npz")))


def same(a, b):
    """bit for bit, NaN where NaN"""
    a, b = np.asarray(a, dtype=float), np.asarray(b, dtype=float)
    return a.shape == b.shape and np.array_equal(a.view(np.int64), b.view(np.int64))


def rejections(ops, bm, pv, theta, alpha):
    pv = np.ascontiguousarray(np.atleast_2d(pv), dtype=float)
    K, G = pv.shape
    cut, num = np.empty(len(theta)), np.empty((K, len(theta)), dtype=np.int32)
    ops.padj_rejections(np.ascontiguousarray(bm, dtype=float), G, pv, G, K, np.ascontiguousarray(theta), len(theta), alpha, cut, num)
    return cut, num


def scipy_bh(bm, p, cutoff):
    out = np.full(len(p), np.nan)
    use = ~np.isnan(p) & ((bm >= cutoff) | (cutoff == -np.inf))
    if use.any():
        out[use] = false_discovery_control(p[use], method="bh")
    return out


def vectors(G, seed, ties=False):
    rng = np.random.default_rng(seed)
    if ties:
        bm = rng.choice([0.0, 0.25, 1.0, 7.0, 7.5], G)
        p = rng.choice([0.0, 1e-5, 0.01, 0.049, 0.05, 0.2, 1.0], G)
    else:
        bm = np.exp(rng.normal(2.0, 2.0, G)) * (rng.random(G) > 0.1)
        p = np.where(rng.random(G) < 0.3, rng.beta(0.2, 5.0, G), rng.random(G))
    p[rng.random(G) < 0.1] = np.nan
    return bm, p
