"""Shared by tests/test_size_factors.py (host emulator) and tests/test_gpu_size_factors.py (device): the sf_* goldens of the real
orchestrator (scripts/make_size_factor_golden.py), a numpy restatement of the reference pinned by them, and how a result is
compared with them."""
import functools
import glob
import os
import warnings

import numpy as np
from scipy.stats import rankdata

from conftest import GOLDEN

SF_CASES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN, "sf_*.npz"))
                  if not os.path.basename(p).startswith(("sf_e2e_", "sf_vst_")))
SF_E2E = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN, "sf_e2e_*.npz")))
SF_VST = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN, "sf_vst_*.npz")))


def fit_size_factors(counts, fit_type="ratio", control=None):
    """``DeseqDataSet.fit_size_factors`` (dds.py:628-703) for ``"ratio"`` and ``"poscounts"``, over every gene or the genes of the
    boolean mask ``control``, restated in numpy.  Returns (size_factors, logmeans, filtered_genes); filtered_genes is not masked by
    ``control``."""
    # the orchestrator's X is the column-major `.values` of a DataFrame: its per-gene means then sum the samples pairwise
    counts = np.asfortranarray(counts)
    use = np.ones(counts.shape[1], dtype=bool) if control is None else np.asarray(control, dtype=bool).copy()
    with np.errstate(divide="ignore", invalid="ignore"), warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)  # np.median([]) = nan
        if fit_type == "poscounts":
            lc = np.zeros_like(counts, dtype=float)
            np.log(counts, out=lc, where=counts != 0)
            lm = lc.mean(0)
            filtered = (~np.isinf(lm)) & (lm > 0)
            use &= filtered
            sf = np.array([np.exp(np.median(np.log(x[use & (x > 0)]) - lm[use & (x > 0)])) for x in counts])
            return sf / np.exp(np.mean(np.log(sf))), lm, filtered
        lm = np.log(counts).mean(0)
        filtered = ~np.isinf(lm)
        use &= filtered
        return np.exp(np.median(np.log(counts)[:, use] - lm[use], axis=1)), lm, filtered


def case_args(z):
    """(fit_type, control) of a golden: control as the reference was given it -- mask, positions or names resolved to positions."""
    if not z["has_control"]:
        return str(z["fit_type"]), None
    given = z["control_given"]
    if given.dtype == bool:
        return str(z["fit_type"]), given
    if given.dtype.kind in "US":
        return str(z["fit_type"]), np.array([int(s[1:]) for s in given])
    return str(z["fit_type"]), given.astype(np.int64)


def assert_size_factors(sf, want, rtol=1e-12):
    """Same NaN pattern, the same ranking of the samples, and within rtol."""
    sf, want = np.asarray(sf), np.asarray(want)
    np.testing.assert_array_equal(np.isnan(sf), np.isnan(want))
    ok = ~np.isnan(want)
    np.testing.assert_array_equal(rankdata(sf[ok]), rankdata(want[ok]))
    np.testing.assert_allclose(sf[ok], want[ok], rtol=rtol)


def assert_logmeans(lm, want, atol=1e-13):
    lm, want = np.asarray(lm), np.asarray(want)
    np.testing.assert_array_equal(np.isneginf(lm), np.isneginf(want))
    ok = np.isfinite(want)
    np.testing.assert_allclose(lm[ok], want[ok], rtol=0, atol=atol)


def check_sf_e2e(monkeypatch, check_e2e, inf, g, rtol, name, max_frac=0.0, resident=False):
    """parity.check_e2e with the golden's size-factor estimator: `workflow.deseq2_results` and the resident fit are called with
    size_factors_fit_type / control_genes (the control mask follows the non-zero genes the resident check uploads)."""
    from pydeseq2_b200 import pipeline, workflow

    kind = str(g["size_factors_fit_type"])
    ctl = g["control"] if g["has_control"] else None
    monkeypatch.setattr(workflow, "deseq2_results",
                        functools.partial(workflow.deseq2_results, size_factors_fit_type=kind, control_genes=ctl))
    nz = ~(np.asarray(g["counts"]) == 0).all(0)
    base = pipeline.ResidentFit

    class Fit(base):
        def __init__(self, ctx, X, size_factors, **kw):
            super().__init__(ctx, X, size_factors, size_factors_fit_type=kind, control_genes=None if ctl is None else ctl[nz], **kw)

    monkeypatch.setattr(pipeline, "ResidentFit", Fit)
    return check_e2e(inf, g, rtol, name, max_frac=max_frac, resident=resident)
