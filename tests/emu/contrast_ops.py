"""Host emulator of `k_wald_contrasts` (emu_wald_contrasts in tests/emu/contrast_emu.cpp) added to the `SfEmuOps` interface as
`wald_contrasts`, so that the CPU suite can push `B200Inference.wald_tests` and the drivers built on it through the device algorithm.
A separate class and library: the emulator classes other tests use keep the methods they had.  Test infrastructure."""
import ctypes as C
import os
import subprocess

from . import build as _build
from .emu_ops import _p, f64p
from .sf_ops import SfEmuOps

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_build", "libpdq_contrast_emu.so")
SRC = os.path.join(HERE, "contrast_emu.cpp")
DEPS = [SRC] + _build.DEPS


def build(force=False):
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    if not force and os.path.exists(OUT) and all(os.path.getmtime(OUT) >= os.path.getmtime(d) for d in DEPS):
        return OUT
    # the flags of the main emulator (tests/emu/build.py): -ffp-contract=off, no fused multiply-adds the source does not write
    subprocess.run(["g++", "-O2", "-std=c++20", "-pthread", "-fPIC", "-shared", "-ffp-contract=off", "-x", "c++", SRC, "-o", OUT, "-lm"],
                   check=True)
    return OUT


class ContrastEmuOps(SfEmuOps):
    def __init__(self, **kw):
        super().__init__(**kw)
        self.contrast_lib = C.CDLL(build())

    def wald_contrasts_rc(self, X, sf, N, p, disp, lfc, G, ridge, K, contrasts, lfc_null, alt, pv, stat, se, ld_out):
        """emu_wald_contrasts' status: 0, -2 (PDQ_ERR_INVALID) for K <= 0, an unknown alternative or ld_out < G, -3 for p > 16."""
        assert self.contrast_lib.emu_set_lanes(self.lanes) == 0
        return self.contrast_lib.emu_wald_contrasts(_p(X, f64p), _p(sf, f64p), N, p, _p(disp, f64p), _p(lfc, f64p), G, _p(ridge, f64p), K,
                                                    _p(contrasts, f64p), _p(lfc_null, f64p), alt.ctypes.data_as(C.POINTER(C.c_int)),
                                                    _p(pv, f64p), _p(stat, f64p), _p(se, f64p), C.c_int64(ld_out))

    def wald_contrasts(self, X, sf, N, p, disp, lfc, G, ridge, K, contrasts, lfc_null, alt, pv, stat, se, ld_out):
        rc = self.wald_contrasts_rc(X, sf, N, p, disp, lfc, G, ridge, K, contrasts, lfc_null, alt, pv, stat, se, ld_out)
        assert rc == 0, rc
