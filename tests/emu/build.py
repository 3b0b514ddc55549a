"""Build the host emulator (test infrastructure) with g++.  See pdq_emu.cpp."""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_build", "libpdq_emu.so")
SRC = os.path.join(HERE, "pdq_emu.cpp")
DEPS = [SRC] + [os.path.join(HERE, "..", "..", "pydeseq2_b200", "csrc", f)
                for f in ("pdq_gene.cuh", "pdq_math.cuh", "pdq_host_linalg.h", "pdq_trend.cuh", "pdq_fast.cuh", "pdq_shrink.cuh",
                          "pdq_tables.h", "pdq_vst.cuh")] + [os.path.join(HERE, "..", "gpu_probe", "math_ops.h")]


def build(force=False, defines=None):
    """`defines` (or the environment variable PDQ_EMU_DEFINES, space separated, e.g. "-DPDQ_IRLS_UNROLL=4") builds a variant of the
    emulator next to the default one -- the CPU check of a kernel experiment before it gets GPU time."""
    defines = list(defines) if defines is not None else os.environ.get("PDQ_EMU_DEFINES", "").split()
    out = OUT if not defines else OUT.replace(".so", "".join(d.replace("-D", "_").replace("=", "") for d in defines) + ".so")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    if not force and os.path.exists(out) and all(os.path.getmtime(out) >= os.path.getmtime(d) for d in DEPS):
        return out
    # -ffp-contract=off: fma() calls stay explicit, nothing else is fused, so results do not depend on g++'s mood
    cmd = ["g++", "-O2", "-std=c++20", "-pthread", "-fPIC", "-shared", "-ffp-contract=off"] + defines + ["-x", "c++", SRC, "-o", out, "-lm"]
    subprocess.run(cmd, check=True)
    return out


if __name__ == "__main__":
    print(build(force=True))
