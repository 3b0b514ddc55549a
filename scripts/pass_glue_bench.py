#!/usr/bin/env python
"""Where the glue of the resident pass spends its time, and the pass with the old glue against the new, on the shapes bench.py
measures.  Per shape, each piece captured as a CUDA graph and timed with CUDA events behind an L2 flush (the flush is enqueued
first, so the pieces' launches are queued before it ends):
  * end:     what follows the tail -- the old three caller-order nodes and one copy of the whole slab; the new single launch that
             writes the tail half (no Cook's vectors) into the page-locked host block; and, for comparison, the same tail half
             reordered on the device and copied;
  * genewise: the genewise half's reorder and copy, which the new pass runs while the trend and the tail do (copy on a branch);
  * fold:    k_mom_from_counts + k_alpha_mle (+ the memset node between them) against k_mom_alpha (lin_reg_mu branch only);
  * pass:    whole passes (ResidentFit.run, CUDA graph replays), old glue and new alternated pass by pass, L2 flushed before each.
Card name, power limit and SM clock are read in the same run.
    python scripts/pass_glue_bench.py --steps 40 [--shapes C2,C3]"""
import argparse
import ctypes as C
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
KEYS = ("mom", "genewise", "genewise_converged", "map", "map_converged", "dispersions", "lfc", "lfc_converged", "pvalue", "stat", "se",
        "normed_means", "outlier")


class OldGlue(ResidentFit):
    """The pass as it was: start values as a launch of their own, the whole slab scattered at the end (two row scatters and a copy
    of the trend record), one copy of the whole slab."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.fold_moments = False

    def _to_caller_order(self, seg, host=False):  # the tail half's output step: the old reorder and one copy
        if seg is self._seg_gw:
            return
        old_end(self)

    def _copy_out(self, ranges, side=False):  # single-GPU passes copy the genewise half only, on the side branch
        pass


def old_reorder(rf):
    L, h, c_d = rf.lib, rf.ctx.h, _lib.c_dptr
    rf.ctx.check(L.pdq_scatter_rows_dev(h, c_d(rf.d_slab), c_d(rf.d_slab_out), c_d(rf.d_perm), rf.G, 15, rf.Gs, 1))
    rf.ctx.check(L.pdq_scatter_rows_dev(h, c_d(rf.d_slab + rf._off_beta * 8), c_d(rf.d_slab_out + rf._off_beta * 8), c_d(rf.d_perm),
                                        rf.G, 1, rf.Gs, rf.p))
    rf.ctx.check(L.pdq_memcpy_d2d(h, c_d(rf.d_slab_out + rf._off_t16 * 8), c_d(rf.d_t16), 16 * 8))


def old_end(rf):
    if rf._perm is not None:
        old_reorder(rf)
    rf.ctx.d2h(rf._h_slab, rf.d_slab_out)


def stats(v):
    v = np.asarray(v)
    return {"median_ms": round(float(np.median(v)), 4), "min_ms": round(float(v.min()), 4), "max_ms": round(float(v.max()), 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="C2,C3,C4_shard,C5_shard")
    ap.add_argument("--steps", type=int, default=40, help="timed repetitions of every piece and passes of each arm (>= 30 for the pass)")
    a = ap.parse_args()
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # the query is a label, not a measurement
        card = f"unknown ({e})"
    inf = B200Inference(device=0)
    ctx = inf._ops.ctx
    L, h, c_d = ctx.lib, ctx.h, _lib.c_dptr
    flush = ctx.malloc(256 << 20)

    def capture(fn):
        ctx.check(L.pdq_capture_begin(h))
        try:
            fn()
        finally:
            g = C.c_void_p()
            ctx.check(L.pdq_capture_end(h, C.byref(g)))
        return g

    def time_graphs(graphs):
        """{label: graph} timed alternately, `steps` times each."""
        ms = {k: [] for k in graphs}
        for g in graphs.values():  # warm-up
            ctx.check(L.pdq_graph_launch(h, g))
        ctx.sync()
        for _ in range(a.steps):
            for k, g in graphs.items():
                ctx.check(L.pdq_memset(h, c_d(flush), 1, 256 << 20))
                ctx.record(0)
                ctx.check(L.pdq_graph_launch(h, g))
                ctx.record(1)
                ms[k].append(ctx.elapsed_ms(0, 1))
        for g in graphs.values():
            L.pdq_graph_destroy(h, g)
        return {k: stats(v) for k, v in ms.items()}

    for name in a.shapes.split(","):
        G, N, design = SHAPES[name]
        counts, X, _ = make_counts(N, G, design, seed=0, sample_seed=0)
        counts = np.ascontiguousarray(counts[:, ~(counts == 0).all(0)])
        sf = median_of_ratios(counts)[1]
        fits = {"old": OldGlue(ctx, X, sf), "new": ResidentFit(ctx, X, sf)}
        last = {}
        for label, rf in fits.items():
            rf.upload(counts)
            for _ in range(3):
                last[label] = rf.run()
        same = all(np.array_equal(last["old"][k], last["new"][k], equal_nan=True) for k in KEYS)
        rf = fits["new"]
        gs, d, Gd = rf._main, rf.design, rf.G
        rec = {"card": card, "shape": name, "genes": int(Gd), "samples": N, "design": design, "steps": a.steps, "bit_identical": bool(same),
               "slab_mb": round(rf._slab_len * 8 / 1e6, 3)}
        # -- end of the pass, and the genewise half
        tail, gw = rf._seg_tail[False], rf._seg_gw

        def tail_device_then_copy():
            rf._to_caller_order(tail)
            rf._copy_out(rf._h_tail[False])

        def gw_half():
            rf._to_caller_order(gw)
            rf._copy_out(rf._h_gw)
        rec["end"] = time_graphs({"old_reorder_and_whole_copy": capture(lambda: old_end(rf)),
                                  "new_tail_to_host": capture(lambda: rf._to_caller_order(tail, host=True)),
                                  "tail_reorder_then_copy": capture(tail_device_then_copy)})
        rec["genewise"] = time_graphs({"reorder_and_copy": capture(gw_half)})
        mb = lambda rs: round(sum(e - s for s, e in rs) * 8 / 1e6, 3)  # noqa: E731
        rec["mb"] = {"whole_slab": rec["slab_mb"], "tail_half": mb(rf._h_tail[False]), "genewise_half": mb(rf._h_gw)}
        # -- fold
        if rf.lin_branch:
            def separate():
                ctx.check(L.pdq_mom_dispersions_dev(h, d, c_d(gs.counts), Gd, Gd, rf.min_disp, rf.max_disp, c_d(gs.mom), c_d(gs.means),
                                                    rf.min_mu, c_d(gs.mu_hat), Gd))
                ctx.check(L.pdq_alpha_mle_hint_dev(h, d, c_d(gs.counts), Gd, Gd, c_d(gs.mu_hat), Gd, c_d(gs.mom), rf.min_disp,
                                                   rf.max_disp, 1.0, None, 1, 0, c_d(gs.gw), c_d(gs.gw_conv), None, c_d(gs.hint)))

            def folded():
                ctx.check(L.pdq_mom_alpha_mle_dev(h, d, c_d(gs.counts), Gd, Gd, rf.min_disp, rf.max_disp, rf.min_mu, c_d(gs.mom),
                                                  c_d(gs.means), c_d(gs.mu_hat), Gd, c_d(gs.gw), c_d(gs.gw_conv), c_d(gs.hint)))
            rec["fold"] = time_graphs({"mom_then_alpha_mle": capture(separate), "mom_alpha_folded": capture(folded)})
        # -- whole pass, alternated
        ms = {"old": [], "new": []}
        for _ in range(a.steps):
            for label in ("old", "new"):
                ctx.check(L.pdq_memset(h, c_d(flush), 1, 256 << 20))
                ctx.sync()
                fits[label].run(events=(0, 1), copy=False)
                ms[label].append(ctx.elapsed_ms(0, 1))
        rec["pass"] = {k: stats(v) for k, v in ms.items()}
        rec["pass"]["new_over_old"] = round(rec["pass"]["new"]["median_ms"] / rec["pass"]["old"]["median_ms"], 4)
        print(json.dumps(rec), flush=True)
        for f in fits.values():
            f.close()


if __name__ == "__main__":
    main()
