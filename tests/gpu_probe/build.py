"""Build the GPU probe (test infrastructure) with nvcc for sm_90a; cross-compiles without a GPU.  See pdq_probe.cu.

Two shared libraries, mirroring the units of the CUDA library (pydeseq2_b200/build.py): the default unit, whose loops over the
design columns are fully unrolled, and one with the wide units' flags (-DPDQ_TU_P=16 -Xptxas -O1: loops, local memory)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT_DIR = os.path.join(HERE, "_build")
SRC = os.path.join(HERE, "pdq_probe.cu")
UNITS = {"narrow": ("libpdq_probe.so", []), "wide": ("libpdq_probe_wide.so", ["-DPDQ_TU_P=16", "-Xptxas", "-O1"])}


def _library_build():
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from pydeseq2_b200 import build as lib_build

    return lib_build


def build(force=False):
    """Returns {unit: path}; a library is rebuilt when its source, math_ops.h or one of the library's headers is newer."""
    lb = _library_build()
    deps = [SRC, os.path.join(HERE, "math_ops.h")] + [os.path.join(lb.CSRC, h) for h in lb.HEADERS]
    os.makedirs(OUT_DIR, exist_ok=True)
    outs, procs = {}, []
    for unit, (name, defs) in UNITS.items():
        out = os.path.join(OUT_DIR, name)
        outs[unit] = out
        if force or lb._stale(out, deps):
            cmd = [lb._nvcc()] + lb.NVCC_FLAGS + defs + ["-shared", SRC, "-o", out, "-lcudart_static", "-ldl", "-lrt", "-lpthread"]
            procs.append((cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    for cmd, pr in procs:
        log = pr.communicate()[0]
        if pr.returncode:
            sys.stderr.write(log.decode(errors="replace"))
            raise RuntimeError("nvcc failed: " + " ".join(cmd))
    return outs


if __name__ == "__main__":
    print(build(force=True))
