"""Host emulator of the VST kernels (tests/emu/vst_emu.cpp) added to the `EmuOps` interface, so that the CPU suite can push
`workflow.vst` and the `vst_transform` override through `B200Inference`'s marshalling.  Test infrastructure."""
import ctypes as C
import os
import subprocess

from .emu_ops import EmuOps, _p, f64p, i64p

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_build", "libpdq_vst_emu.so")
SRC = os.path.join(HERE, "vst_emu.cpp")
DEPS = [SRC] + [os.path.join(HERE, "..", "..", "pydeseq2_b200", "csrc", f)
                for f in ("pdq_vst.cuh", "pdq_trend.cuh", "pdq_math.cuh", "pdq_fast.cuh", "pdq_tables.h")]


def build(force=False):
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    if not force and os.path.exists(OUT) and all(os.path.getmtime(OUT) >= os.path.getmtime(d) for d in DEPS):
        return OUT
    # -ffp-contract=off as for the main emulator: no fused multiply-adds the source does not write
    subprocess.run(["g++", "-O2", "-std=c++20", "-fPIC", "-shared", "-ffp-contract=off", "-x", "c++", SRC, "-o", OUT, "-lm"], check=True)
    return OUT


class VstEmuOps(EmuOps):
    def __init__(self, **kw):
        super().__init__(**kw)
        self.vst_lib = C.CDLL(build())

    def vst_transform(self, counts, ld, N, G, sf, kind, c0, c1, out, ld_out):
        rc = self.vst_lib.emu_vst_transform(_p(counts, i64p), C.c_int64(ld), N, G, _p(sf, f64p), kind, C.c_double(c0), C.c_double(c1),
                                            _p(out, f64p), C.c_int64(ld_out))
        assert rc == 0

    def size_factors_from_logmeans(self, counts, ld, N, G, logmeans, sf):
        assert self.vst_lib.emu_size_factors_from_logmeans(_p(counts, i64p), C.c_int64(ld), N, G, _p(logmeans, f64p), _p(sf, f64p)) == 0
