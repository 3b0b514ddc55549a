#!/usr/bin/env python
"""Prints the measured worst cases of the FP64 building blocks against tests/golden/math_ref.npz: ulps for log / exp /
reciprocal / division, errors relative to max(|f|, 1) for the special functions, and the worst table error over its bound for
each lane count T.  `--device` measures the device branches through the GPU probe (needs a GPU), otherwise the host branches
through the emulator.  The numbers quoted in pdq_fast.cuh / pdq_math.cuh come from this script."""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.join(HERE, ".."), os.path.join(HERE, "..", "tests")]

import math_checks as mc  # noqa: E402


def measure(f):
    """f()'s worst case, or the message of the bound it breaks"""
    try:
        return f()
    except AssertionError as e:
        return "FAILS: " + str(e).splitlines()[0]


def main():
    if "--device" in sys.argv:
        from gpu_probe.probe import Probe

        units = {u: Probe(u) for u in ("narrow", "wide")}
    else:
        from emu.emu_ops import EmuOps

        units = {"host": EmuOps()}
    rep = {}
    for unit, ops in units.items():
        u = rep[unit] = {"ulp": {}, "special_rel": {}, "tables": {}}
        for name in sorted(mc.ULP_BOUNDS):
            u["ulp"][name] = measure(lambda: round(mc.check_ulp(ops, name), 3))
        for name in sorted(mc.SF_BOUNDS):
            u["special_rel"][name] = measure(lambda: float(f"{mc.check_special(ops, name):.3g}"))
        u["special_rel"]["norm_sf"] = measure(lambda: float(f"{mc.check_norm_sf(ops):.3g}"))
        u["sweep_ulp_vs_numpy"] = {k: round(v, 3) for k, v in mc.sweep_worst(ops, 1_000_000).items()}
        r, refs = mc.table_refs()
        for T in (1, 2, 4, 8, 16, 32):
            out = ops.tables(r, T)
            worst = measure(lambda: mc.check_tables(out, r, refs, T))
            if isinstance(worst, str):
                u["tables"][f"T={T}"] = worst
                continue
            abs_err = {name: float(f"{abs(out[:, off:off + 32] - ex).max():.3g}") for name, off, ex, _b in refs}
            u["tables"][f"T={T}"] = {k: {"worst_over_bound": round(v, 4), "max_abs_err": abs_err[k]} for k, v in worst.items()}
    print(json.dumps(rep, indent=1))


if __name__ == "__main__":
    main()
