"""Generate tests/golden/large_shrink*.npz from the REAL reference: apeGLM shrinkage (``lfc_shrink_nbinom_glm``) of designs of
65..128 columns.  TEST INFRASTRUCTURE: writes only the ``large_shrink*`` fixtures, every other golden stays untouched.

    PYDESEQ2_SRC=<PyDESeq2 0.5.3 checkout> python scripts/make_large_shrink_golden.py

The generators and layouts are those of scripts/make_wide_shrink_golden.py (``gen_calls`` / ``gen_tape`` with the ``large_``
prefix), run on the reference's own final state of the ``large_*`` fixtures (scripts/make_large_golden.py), whose contrasts each
select the one coefficient shrunk here.  ``HEAD_BYTES`` keeps the full inverse Hessians to the first genes (3 at p = 65 and 70, 1 at
p = 101 and 128); column ``shrink_index`` is stored for every gene.

* ``large_shrink_<case>`` -- one ``lfc_shrink_nbinom_glm`` call each: paired p = 65, 101 (adapted and with prior scale 1) and 128
  shrinking the condition column, and the 70-level outlier fit shrinking level 3.
* ``large_shrinktape_paired_p101`` -- ``deseq2()``, ``summary()`` and ``lfc_shrink(coeff=condition)`` through the real orchestrator on
  the paired p = 101 design (the width whose unshrunk end-to-end tables match; at p = 65 and 128 a few genes' genewise dispersion
  has two minima).
"""
from __future__ import annotations

import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_wide_shrink_golden as mws  # noqa: E402  (the reference's import path and the generators)


def main():
    mws.gen_calls("paired_p65", "large_paired_p65", 64, prefix="large_")
    mws.gen_calls("paired_p101", "large_paired_p101", 100, prefix="large_")
    mws.gen_calls("paired_p101_noadapt", "large_paired_p101", 100, adapt=False, prefix="large_")
    mws.gen_calls("paired_p128", "large_paired_p128", 127, prefix="large_")
    mws.gen_calls("levels_p70_outliers", "large_levels_p70_outliers", 3, prefix="large_")
    mws.gen_tape("paired_p101", "large_paired_p101", 100, prefix="large_")


if __name__ == "__main__":
    main()
