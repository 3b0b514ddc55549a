"""Build ``libpydeseq2_b200.so`` in-tree with nvcc for sm_90a (cross-compiles without a GPU)."""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libpydeseq2_b200.so")
# translation units: (source, object tag, extra defines).  pdq_kernels.cu holds the per-gene kernels of designs of up to 16 columns
# and is compiled once for p = 1..8 and once per wide design width p = 9..16 (see the note at its top); pdq_wide.cu holds the
# kernels of designs of 17..128 columns, one build for every width (p is a run-time argument there; 65..128 columns are its
# team-per-gene instantiations); pdq_common.cu holds the kernels that do not depend on the design width.  The units are independent
# and compile in parallel.
WIDE_P = tuple(range(9, 17))
UNITS = [("pdq_api.cu", "pdq_api", ()), ("pdq_dispatch.cu", "pdq_dispatch", ()), ("pdq_io.cpp", "pdq_io", ()), ("pdq_padj.cu", "pdq_padj", ()), ("pdq_wide.cu", "pdq_wide", ()),
         ("pdq_common.cu", "pdq_common", ()), ("pdq_kernels.cu", "pdq_kernels_p1to8", ())] + \
        [("pdq_kernels.cu", f"pdq_kernels_p{p}", (f"-DPDQ_TU_P={p}", "-Xptxas", "-O1")) for p in WIDE_P]
# (ptxas -O1 for the wide widths: 12 s instead of 85 s per unit; their kernels keep the small matrices in local memory anyway)
SOURCES = sorted({u[0] for u in UNITS})
HEADERS = ["pdq_math.cuh", "pdq_fast.cuh", "pdq_tables.h", "pdq_trend.cuh", "pdq_gene.cuh", "pdq_shrink.cuh", "pdq_vst.cuh", "pdq_padj.cuh", "pdq_team.cuh", "pdq_launch.cuh", "pdq_internal.h",
           "pdq_host_linalg.h", os.path.join("..", "..", "include", "pydeseq2_b200.h")]
NVCC_FLAGS = ["-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
              "-Xcompiler", "-fPIC,-fopenmp", "--expt-relaxed-constexpr"]


def _nvcc() -> str:
    nv = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nv):
        raise RuntimeError("nvcc not found: the CUDA extension cannot be built")
    return nv


def _stale(target: str, deps) -> bool:
    return not os.path.exists(target) or any(os.path.getmtime(d) > os.path.getmtime(target) for d in deps)


def build(force: bool = False, verbose: bool = False, defines=(), out: str | None = None) -> str:
    """`defines` / `out` build a tuning variant (e.g. ("-DPDQ_ALPHA_MINB=5",), "libpdq_a5.so") next to the default library."""
    global OUT
    tag = "".join(d.replace("-D", "_").replace("=", "") for d in defines)
    objdir = os.path.join(HERE, "build" + tag)
    target = os.path.join(HERE, out) if out else OUT
    hdrs = [os.path.join(CSRC, h) for h in HEADERS]
    # the library is newer than every source: nothing to do (the object directory does not travel with gpurun snapshots)
    if not force and not _stale(target, [os.path.join(CSRC, s) for s in SOURCES] + hdrs):
        return target
    os.makedirs(objdir, exist_ok=True)
    objs, todo = [], []
    for src, name, unit_defs in UNITS:
        s = os.path.join(CSRC, src)
        o = os.path.join(objdir, name + ".o")
        objs.append(o)
        if force or _stale(o, [s] + hdrs):
            todo.append([_nvcc()] + NVCC_FLAGS + list(defines) + list(unit_defs) + (["-Xptxas", "-v"] if verbose else []) + ["-c", s, "-o", o])
    jobs = max(1, min(len(todo), int(os.environ.get("PDQ_BUILD_JOBS", os.cpu_count() or 1))))
    running, failed = [], None
    while todo or running:
        while todo and len(running) < jobs:
            cmd = todo.pop(0)
            log = open(cmd[-1] + ".log", "w+")
            running.append((cmd, subprocess.Popen(cmd, stdout=log, stderr=subprocess.STDOUT), log))
        still = []
        for cmd, pr, log in running:
            if pr.poll() is None:
                still.append((cmd, pr, log))
                continue
            log.seek(0)
            out = log.read()
            log.close()
            if verbose or pr.returncode:
                sys.stderr.write(out)
            if pr.returncode and failed is None:
                failed = cmd
        running = still
        if running:
            time.sleep(0.2)
    if failed is not None:
        raise RuntimeError("nvcc failed: " + " ".join(failed))
    if force or _stale(target, objs):
        cmd = [_nvcc(), "-shared", "-o", target] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-lcudart_static",
                                                        "-ldl", "-lrt", "-lpthread", "-lgomp"]
        subprocess.run(cmd, check=True)
    return target


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
