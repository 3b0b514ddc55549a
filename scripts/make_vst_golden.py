"""Generate tests/golden/vst_*.npz from the REAL reference orchestrator (``DeseqDataSet.vst`` / ``vst_fit`` / ``vst_transform``,
dds.py:349-514).  TEST INFRASTRUCTURE: writes only the ``vst_*`` fixtures, every other golden stays untouched.

    PYDESEQ2_SRC=<PyDESeq2 0.5.3 checkout> python scripts/make_vst_golden.py

The reference is imported through the shims of ``oracle/make_golden.py`` (same setup as every other fixture).  Each file holds the
counts, the design, the options, and what the orchestrator left behind: ``layers["vst_counts"]`` (every gene),
``var["vst_genewise_dispersions"]``, ``uns["vst_trend_coeffs"]`` or the mean dispersion of the transform, the final
``vst_fit_type``, the size factors and ``logmeans``.  Train/test cases also hold the held-out counts and their transform.
"""
from __future__ import annotations

import os
import sys
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import make_golden as mg  # noqa: E402  (sets up the reference's import path; exits without PYDESEQ2_SRC)
import numpy as np  # noqa: E402
import pandas as pd  # noqa: E402
from scipy.stats import trim_mean  # noqa: E402

REF = mg.REF
OUT = mg.OUT


def _dataset(counts, X, names=None):
    from pydeseq2.dds import DeseqDataSet

    N, G = counts.shape
    idx = [f"s{i}" for i in range(N)]
    counts_df = pd.DataFrame(counts, index=idx, columns=names or [f"g{i}" for i in range(G)])
    design_df = pd.DataFrame(X, index=idx, columns=[f"x{j}" for j in range(X.shape[1])])
    meta = pd.DataFrame({"dummy": np.arange(N)}, index=idx)
    return DeseqDataSet(counts=counts_df, metadata=meta, design=design_df, inference=mg.ref_inference(), quiet=True)


def _record(dds, counts, X, use_design, fit_type, vst_counts, caught):
    kind = dds.vst_fit_type
    gd = dds.var["vst_genewise_dispersions"].values
    out = dict(counts=np.asarray(counts, dtype=np.int64), design=np.asarray(X, dtype=float), use_design=np.float64(use_design),
               fit_type=np.array(fit_type), vst_fit_type=np.array(kind), vst_counts=np.asarray(vst_counts, dtype=float),
               vst_genewise_dispersions=gd, size_factors=dds.obs["size_factors"].values, logmeans=np.asarray(dds.logmeans, dtype=float),
               fell_back=np.float64(any("did not converge" in str(w.message) for w in caught)))
    if kind == "parametric":
        out["vst_trend_coeffs"] = np.asarray(dds.uns["vst_trend_coeffs"], dtype=float)
    else:
        out["mean_disp"] = np.float64(trim_mean(gd[gd > 10 * dds.min_disp], proportiontocut=0.001))
    return out


def gen(name, counts, X, use_design=False, fit_type="parametric", after_deseq2=False, n_train=None, extra=None, expect_fallback=False):
    held = None
    if n_train is not None:
        counts, held = counts[:n_train], counts[n_train:]
        X = X[:n_train]
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        dds = _dataset(counts, X)
        if after_deseq2:
            dds.deseq2()
        if held is None:
            dds.vst(use_design=use_design, fit_type=fit_type)
            vst_counts = dds.layers["vst_counts"]
        else:
            dds.vst_fit_type = fit_type
            dds.vst_fit(use_design=use_design)
            vst_counts = dds.vst_transform()
    out = _record(dds, counts, X, use_design, fit_type, vst_counts, caught)
    if expect_fallback:
        assert out["fell_back"] == 1.0 and str(out["vst_fit_type"]) == "mean", f"{name}: the parametric VST trend did not fall back"
    if held is not None:
        out["heldout_counts"] = np.asarray(held, dtype=np.int64)
        out["heldout_vst"] = np.asarray(dds.vst_transform(np.asarray(held, dtype=np.int64)), dtype=float)
    out.update(extra or {})
    np.savez_compressed(os.path.join(OUT, f"vst_{name}.npz"), **out)
    print(f"vst_{name}: N={counts.shape[0]} G={counts.shape[1]} use_design={use_design} fit_type={fit_type} -> {out['vst_fit_type']}"
          + (f", held-out {held.shape[0]}" if held is not None else ""))


def fallback_counts(seed=7, N=12, G=400):
    """Counts whose genewise dispersions RISE with the mean: the gamma-GLM trend a0 + a1 / mean wants a1 < 0, hits the bound, and
    the reference switches to the mean trend (dds.py:1243-1252)."""
    rng = np.random.default_rng(seed)
    mean = np.exp(rng.uniform(np.log(5), np.log(5000), G))
    disp = 0.002 * mean ** 0.8
    n = 1.0 / disp
    return rng.negative_binomial(n[None, :], (n / (n + mean))[None, :], size=(N, G)).astype(np.int64), np.ones((N, 1))


def main():
    # the reference's shipped 100 x 10 dataset, with R DESeq2's own vst() outputs (tests/data/single_factor/r_*vst*.csv)
    counts_df = pd.read_csv(f"{REF}/datasets/synthetic/test_counts.csv", index_col=0).T
    meta = pd.read_csv(f"{REF}/datasets/synthetic/test_metadata.csv", index_col=0)
    counts = counts_df.to_numpy().astype(np.int64)
    X = np.stack([np.ones(len(meta)), (meta["condition"] == "B").to_numpy(dtype=float)], axis=1)
    rdir = f"{REF}/tests/data/single_factor"
    for fit_type, use_design, rfile in (("parametric", False, "r_vst.csv"), ("parametric", True, "r_vst_with_design.csv"),
                                        ("mean", False, "r_mean_vst.csv"), ("mean", True, None)):
        extra = {"r_vst": pd.read_csv(f"{rdir}/{rfile}", index_col=0).to_numpy().T.astype(float)} if rfile else None
        gen(f"single_factor_{fit_type}{'_design' if use_design else ''}", counts, X, use_design, fit_type, extra=extra)

    # seeded synthetic tables
    c, X2, _ = mg.synth(24, 300, "two_level", seed=31)
    c[:, [5, 77, 150]] = 0  # all-zero genes: no dispersion, but a transformed value like every other gene
    gen("two_level_n24", c, X2)
    gen("two_level_n24_design", c, X2, use_design=True)
    c, X3, _ = mg.synth(20, 300, "factorial", seed=32)
    gen("factorial_n20_design", c, X3, use_design=True)
    c, X4, _ = mg.synth(30, 300, "continuous", seed=33)
    gen("continuous_n30", c, X4)
    gen("continuous_n30_mean", c, X4, fit_type="mean")

    # the parametric trend fails and the transform uses the mean dispersion
    c, X5 = fallback_counts()
    gen("fallback_to_mean", c, X5, expect_fallback=True)

    # vst() after deseq2(): the size factors of the fit are there already
    c, X6, _ = mg.synth(16, 300, "two_level", seed=34)
    gen("after_deseq2", c, X6, after_deseq2=True)

    # train/test: vst_fit on the first samples, vst_transform on the rest.  The last held-out sample has zeros in more than half of
    # the filtered genes: its size factor is 0 and its transformed counts are inf / NaN
    c, X7, _ = mg.synth(24, 300, "two_level", seed=35)
    c[-1, : 200] = 0
    gen("train_test", c, X7, n_train=18)
    gen("train_test_mean", c, X7, fit_type="mean", n_train=18)


if __name__ == "__main__":
    main()
