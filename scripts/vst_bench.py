"""Variance-stabilising transform on one GPU: prints one JSON line.

    python scripts/vst_bench.py [--reps 200] [--e2e-reps 3]

For C2 (20 000 genes x 200 samples) and C3 (60 000 x 500): the time of one k_vst_transform launch on device-resident counts
(CUDA events around `--reps` launches after warm-up), its achieved bandwidth from the 16 bytes per (sample, gene) it must move
(8 read, 8 written), the device-to-device copy bandwidth measured in the same run on the same bytes, the whole
`workflow.vst()` through the plugin calls (host buffers, wall clock), the whole `workflow.vst_resident()` (counts up once,
transformed counts down once, wall clock), and the numpy closed form on the host with its core count.
The device name and power limit are read in the same run.  There is no CPU fallback: without a GPU the script fails."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from pydeseq2_b200 import _lib  # noqa: E402
from pydeseq2_b200.inference import B200Inference  # noqa: E402
from pydeseq2_b200.synth import make_counts  # noqa: E402
from pydeseq2_b200.workflow import vst, vst_resident  # noqa: E402

SHAPES = {"C2": (200, 20000), "C3": (500, 60000)}


def power_limit_w(index=0):
    try:
        out = subprocess.run(["nvidia-smi", f"--id={index}", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:
        return None


def numpy_vst(normed, a0, a1):
    return np.log2((1 + a1 + 2 * a0 * normed + 2 * np.sqrt(a0 * normed * (1 + a1 + a0 * normed))) / (4 * a0))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--e2e-reps", type=int, default=3)
    a = ap.parse_args()
    inf = B200Inference(device=0)
    ctx = inf._ops.ctx
    c_d = _lib.c_dptr
    res = {"metric": "vst", "device": ctx.info()["name"], "power_limit_w": power_limit_w(), "host_cores": os.cpu_count(), "shapes": {}}
    for tag, (N, G) in SHAPES.items():
        counts, X, _ = make_counts(N, G, "two_level", seed=3)
        _, sf = inf.size_factors(counts)
        a0, a1 = 0.02, 1.5
        nbytes = N * G * 8
        dc, ds, do = ctx.malloc(nbytes), ctx.malloc(N * 8), ctx.malloc(nbytes)
        try:
            ctx.h2d(dc, np.ascontiguousarray(counts))
            ctx.h2d(ds, sf)

            def launch():
                ctx.check(ctx.lib.pdq_vst_transform_dev(ctx.h, c_d(dc), G, N, G, c_d(ds), 0, a0, a1, c_d(do), G))

            def copy():
                ctx.check(ctx.lib.pdq_memcpy_d2d(ctx.h, c_d(do), c_d(dc), nbytes))

            def timed(fn):
                for _ in range(10):
                    fn()
                ctx.sync()
                ctx.record(0)
                for _ in range(a.reps):
                    fn()
                ctx.record(1)
                ctx.sync()
                return ctx.elapsed_ms(0, 1) / a.reps

            t_k, t_c = timed(launch), timed(copy)
            launch()  # the copies overwrote the output
            out = np.empty((N, G))
            ctx.d2h(out, do)
            ctx.sync()
        finally:
            for p in (dc, ds, do):
                ctx.free(p)
        normed = counts / sf[:, None]
        t0 = time.perf_counter()
        want = numpy_vst(normed, a0, a1)
        t_np = time.perf_counter() - t0
        err = float(np.max(np.abs(out - want) / np.maximum(np.abs(want), 1.0)))
        t_e2e, t_res = [], []
        for run, times in ((lambda: vst(counts, X, inf), t_e2e), (lambda: vst_resident(inf, counts, X), t_res)):
            run()  # warm-up: library state, caches, pinned blocks
            for _ in range(a.e2e_reps):
                t0 = time.perf_counter()
                run()
                times.append(time.perf_counter() - t0)
        moved = 16.0 * N * G
        res["shapes"][tag] = {
            "N": N, "G": G, "kernel_ms": t_k, "kernel_gbps": moved / t_k / 1e6, "d2d_copy_ms": t_c, "d2d_copy_gbps": moved / t_c / 1e6,
            "kernel_vs_copy": t_c / t_k, "max_rel_err_vs_numpy": err, "vst_plugin_calls_s": float(np.median(t_e2e)),
            "vst_resident_s": float(np.median(t_res)),
            "numpy_transform_s": t_np}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
