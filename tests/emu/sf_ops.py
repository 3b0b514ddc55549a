"""Host emulator of the size-factor kernels (tests/emu/sf_emu.cpp) added to the `VstEmuOps` interface as `size_factors_ex`, so that
the CPU suite can push poscounts and control-gene size factors through `B200Inference`'s marshalling.  A separate class: the
`EmuOps` that tests/test_integration.py uses keeps the methods it had.  Test infrastructure."""
import ctypes as C
import os
import subprocess

import numpy as np

from .emu_ops import _p, f64p, i64p
from .vst_ops import VstEmuOps

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_build", "libpdq_sf_emu.so")
SRC = os.path.join(HERE, "sf_emu.cpp")
DEPS = [SRC] + [os.path.join(HERE, "..", "..", "pydeseq2_b200", "csrc", f)
                for f in ("pdq_trend.cuh", "pdq_math.cuh", "pdq_fast.cuh", "pdq_tables.h")]


def build(force=False):
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    if not force and os.path.exists(OUT) and all(os.path.getmtime(OUT) >= os.path.getmtime(d) for d in DEPS):
        return OUT
    # -ffp-contract=off as for the main emulator: no fused multiply-adds the source does not write
    subprocess.run(["g++", "-O2", "-std=c++20", "-fPIC", "-shared", "-ffp-contract=off", "-x", "c++", SRC, "-o", OUT, "-lm"], check=True)
    return OUT


class SfEmuOps(VstEmuOps):
    def __init__(self, **kw):
        super().__init__(**kw)
        self.sf_lib = C.CDLL(build())

    def size_factors_ex_rc(self, counts, ld, N, G, kind, control, sf, logmeans):
        """emu_size_factors_ex's status: 0, or -2 (PDQ_ERR_INVALID) for an unknown kind."""
        ctl = None if control is None else np.ascontiguousarray(control, dtype=np.uint8)
        return self.sf_lib.emu_size_factors_ex(_p(counts, i64p), C.c_int64(ld), N, G, int(kind),
                                               None if ctl is None else C.c_void_p(ctl.ctypes.data), _p(sf, f64p), _p(logmeans, f64p))

    def size_factors_ex(self, counts, ld, N, G, kind, control, sf, logmeans):
        """pdq_size_factors_ex: `control` uint8 (G,) or None, `logmeans` (G,) receives the raw log means."""
        rc = self.size_factors_ex_rc(counts, ld, N, G, kind, control, sf, logmeans)
        assert rc == 0, rc
