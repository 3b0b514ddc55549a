"""The wiring a PyDESeq2 maintainer adds for the steps that are NOT behind the ``Inference`` plugin API but have a device
implementation here (SURVEY.md §8 f-1, f-2): Cook's distances, median-of-ratios size factors, the variance-stabilising
transform (``vst()`` / ``vst_transform(counts)``), the Wald test of a contrast from the fitted coefficients and the adjusted
p-values (independent filtering / Benjamini-Hochberg).

``pydeseq2`` is imported lazily -- this module is only usable where the reference package is installed::

    from pydeseq2_b200 import B200Inference
    from pydeseq2_b200.integration import b200_dataset_class

    DeseqDataSet = b200_dataset_class()                      # subclass of pydeseq2.dds.DeseqDataSet
    dds = DeseqDataSet(counts=..., metadata=..., design=..., inference=B200Inference(device=0))
    dds.deseq2()                                             # size factors and Cook's distances now come from the GPU too

Everything else -- state handling, the refit, the statistics -- is the reference's own code, untouched.
"""
from __future__ import annotations

import numpy as np


def b200_dataset_class(all_size_factors=False):
    """Returns a ``DeseqDataSet`` subclass whose ``fit_size_factors`` (plain median-of-ratios case), ``calculate_cooks`` and
    ``vst_transform`` call the backend when it offers ``size_factors`` / ``calculate_cooks`` / ``vst_transform`` (``B200Inference``
    does), and fall back to the reference's own implementation otherwise (other fit types, control genes, a missing VST fit,
    held-out counts after iteratively fitted size factors, a different backend).

    ``all_size_factors=True`` also sends ``"poscounts"`` and control genes (with ``"ratio"`` or ``"poscounts"``, dds.py:628-679) to
    the backend.  It is opt-in so that the size factors of existing code do not change unnoticed; ``"iterative"``, and ratio when
    every gene holds a zero, stay with the reference either way."""
    from pydeseq2.dds import DeseqDataSet

    from .pipeline import filtered_genes

    class B200DeseqDataSet(DeseqDataSet):
        def fit_size_factors(self, fit_type=None, control_genes=None):  # dds.py:584-711
            kind = self.size_factors_fit_type if fit_type is None else fit_type
            # an explicit control_genes= overrides the attribute set at init, which the reference always sets (None by default)
            control = control_genes if control_genes is not None else getattr(self, "control_genes", None)
            plain = kind == "ratio" and control is None
            device = (plain or (all_size_factors and kind in ("ratio", "poscounts"))) and hasattr(self.inference, "size_factors") \
                and isinstance(self.X, np.ndarray)
            if device:
                kw = {}
                if not plain:
                    mask = None
                    if control is not None:  # masks, positions or var names, resolved as the reference does (dds.py:641-647)
                        mask = np.zeros(self.X.shape[1], dtype=bool)
                        mask[self._normalize_indices((slice(None), control))[1]] = True
                    kw = {"fit_type": kind, "control_genes": mask}
                try:
                    normed, sf, logmeans = self.inference.size_factors(self.X, return_logmeans=True, **kw)
                except ValueError:  # every gene holds a zero: the reference switches to its iterative estimator (dds.py:682-690)
                    return super().fit_size_factors(fit_type=fit_type, control_genes=control_genes)
                # what the reference keeps (dds.py:663, 679, 693): vst_fit / vst_transform normalise NEW counts with them
                self.logmeans, self.filtered_genes = logmeans, filtered_genes(logmeans, kind)
                self.layers["normed_counts"] = normed
                self.obs["size_factors"] = sf
                self.var["_normed_means"] = normed.mean(0)
                return None
            return super().fit_size_factors(fit_type=fit_type, control_genes=control_genes)

        def calculate_cooks(self):  # dds.py:986-1040
            if not hasattr(self.inference, "calculate_cooks"):
                return super().calculate_cooks()
            if "dispersions" not in self.var:
                self.fit_MAP_dispersions()
            nz = self.var["non_zero"].values
            cooks = self.inference.calculate_cooks(self.X[:, nz], self.obs["size_factors"].values, self.obsm["design_matrix"].values,
                                                   self.obsm["_mu_LFC"], self.obsm["_hat_diagonals"])[0]
            if self.low_memory:
                del self.obsm["_mu_LFC"]
                del self.obsm["_hat_diagonals"]
            self.layers["cooks"] = np.full((self.n_obs, self.n_vars), np.nan)
            self.layers["cooks"][:, nz] = cooks
            return None

        def vst_transform(self, counts=None):  # dds.py:438-514
            # The fit (vst_fit) stays the reference's: it already reaches the backend through the plugin calls.  The transform
            # runs on the device from the raw counts and the size factors: every size-factor path of the reference sets
            # normed_counts = X / size_factors exactly (dds.py:676-678, 698-703, 1548).
            inf, kind = self.inference, getattr(self, "vst_fit_type", None)
            ok = (hasattr(inf, "vst_transform") and kind in ("parametric", "mean") and "size_factors" in self.obs
                  and isinstance(self.X, np.ndarray) and (kind == "mean" or "vst_trend_coeffs" in self.uns))
            if ok and counts is not None:  # held-out samples: normalised against the fit's log means on the device
                ok = (isinstance(counts, np.ndarray) and counts.dtype.kind in "iu" and getattr(self, "logmeans", None) is not None
                      and getattr(self, "filtered_genes", None) is not None)
            if ok:
                if kind == "parametric":
                    coeffs = np.asarray(self.uns["vst_trend_coeffs"], dtype=float)
                    ok = coeffs[0] > 0
                else:
                    from scipy.stats import trim_mean

                    gd = self.var["vst_genewise_dispersions"]
                    coeffs = float(trim_mean(gd[gd > 10 * self.min_disp], proportiontocut=0.001))
                    ok = coeffs > 0
            if not ok:  # missing fit (the reference's errors), iterative size factors with new counts, other backends
                return super().vst_transform(counts)
            if counts is None:
                return inf.vst_transform(self.X, self.obs["size_factors"].values, kind, coeffs)
            sf = inf.size_factors(counts, logmeans=np.where(self.filtered_genes, self.logmeans, -np.inf))[1]
            return inf.vst_transform(counts, sf, kind, coeffs)

    return B200DeseqDataSet


def b200_stats_class():
    """Returns a ``DeseqStats`` subclass whose ``run_wald_test`` (ds.py:303-360) sends the fit's coefficients, dispersions, size
    factors and the contrast to ``inference.wald_tests``: mu is built on the device instead of as an (N, G) host array per
    contrast.  The outputs and the override for genes whose replaced counts became all zero are the reference's.  A backend
    without ``wald_tests``, or a dataset without size factors, runs the reference's own method.

    ``_independent_filtering`` and ``_p_value_adjustment`` (ds.py:486-542) go through ``inference.adjust_pvalues``: the cutoffs,
    the rejection counts and the BH values come from the device, bit for bit those of numpy and scipy, and the cutoff is chosen
    with the reference's own ``pydeseq2.utils.lowess``.  A backend without ``adjust_pvalues`` runs the reference's methods::

        DeseqStats = b200_stats_class()
        for c in contrasts:                                  # one fit, any number of comparisons
            ds = DeseqStats(dds, contrast=c, inference=B200Inference(device=0))
            ds.summary()
    """
    import sys

    import pandas as pd
    from pydeseq2.ds import DeseqStats

    class B200DeseqStats(DeseqStats):
        def run_wald_test(self):  # ds.py:303-360
            if not hasattr(self.inference, "wald_tests") or "size_factors" not in self.dds.obs:
                return super().run_wald_test()
            if self.shrunk_LFCs and not self.quiet:
                print("Note: running Wald test on shrunk LFCs. Some sequencing datasets show better performance with the testing "
                      "separated from the use of the LFC prior.", file=sys.stderr)
            p = self.design_matrix.shape[1]
            ridge = np.diag(1 / self.prior_LFC_var**2) if self.prior_LFC_var is not None else np.diag(np.repeat(1e-6, p))
            pv, stat, se = self.inference.wald_tests(self.design_matrix.values, self.dds.obs["size_factors"].values,
                                                     self.dds.var["dispersions"].values, self.LFC.values,
                                                     np.asarray(self.contrast_vector, dtype=float), ridge,
                                                     np.log(2) * self.lfc_null, self.alt_hypothesis)
            self.p_values = pd.Series(pv, index=self.dds.var_names)
            self.statistics = pd.Series(stat, index=self.dds.var_names)
            self.SE = pd.Series(se, index=self.dds.var_names)
            if self.dds.refit_cooks and self.dds.var["replaced"].sum() > 0:
                self.SE.loc[self.dds.new_all_zeroes_genes] = 0.0
                self.statistics.loc[self.dds.new_all_zeroes_genes] = 0.0
                self.p_values.loc[self.dds.new_all_zeroes_genes] = 1.0
            return None

        def _independent_filtering(self):  # ds.py:486-528
            if not self._device_padj(True):
                return super()._independent_filtering()
            return None

        def _p_value_adjustment(self):  # ds.py:529-542
            if not self._device_padj(False):
                return super()._p_value_adjustment()
            return None

        def _device_padj(self, independent_filter):
            """Sets self.padj through the backend; False when it has no adjust_pvalues or cannot run it."""
            if not hasattr(self.inference, "adjust_pvalues"):
                return False
            from pydeseq2.utils import lowess

            if not hasattr(self, "p_values"):
                self.run_wald_test()
            padj = self.inference.adjust_pvalues(np.asarray(self.base_mean, dtype=float), np.asarray(self.p_values, dtype=float),
                                                 self.alpha, independent_filter, lowess=lowess)
            if padj is None:
                return False
            self.padj = pd.Series(padj, index=self.dds.var_names)
            return True

    return B200DeseqStats
