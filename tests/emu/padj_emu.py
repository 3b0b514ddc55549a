"""Build (g++) and bind the host emulator of the multiple-testing entry points (tests/emu/padj_emu.cpp) with the `_CudaOps`
interface of `padj_rejections` / `padj_bh`, so that the CPU suite can push pdq_padj.cuh through `B200Inference.adjust_pvalues`.
Test infrastructure."""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_build", "libpadj_emu.so")
SRC = os.path.join(HERE, "padj_emu.cpp")
DEPS = [SRC, os.path.join(HERE, "..", "..", "pydeseq2_b200", "csrc", "pdq_padj.cuh")]

f64p = C.POINTER(C.c_double)
i32p = C.POINTER(C.c_int)


def build(force=False):
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    if not force and os.path.exists(OUT) and all(os.path.getmtime(OUT) >= os.path.getmtime(d) for d in DEPS):
        return OUT
    # -ffp-contract=off: nothing is fused into an FMA, so the roundings are numpy's and scipy's
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-x", "c++", SRC, "-o", OUT, "-lm"], check=True)
    return OUT


def _p(a, t):
    return a.ctypes.data_as(t)


class PadjEmuOps:
    def __init__(self):
        self.lib = C.CDLL(build())

    def empty(self, shape):
        return np.empty(shape, dtype=np.float64)

    def padj_rejections_rc(self, base_mean, G, pv, ld, K, theta, n_theta, alpha, cutoffs, num_rej):
        """emu_padj_rejections' status: 0, or -2 (PDQ_ERR_INVALID) for bad shapes or a p-value outside [0, 1]."""
        return self.lib.emu_padj_rejections(_p(base_mean, f64p), G, _p(pv, f64p), C.c_int64(ld), K, _p(theta, f64p), n_theta,
                                            C.c_double(alpha), _p(cutoffs, f64p), _p(num_rej, i32p))

    def padj_rejections(self, *a):
        rc = self.padj_rejections_rc(*a)
        assert rc == 0, rc

    def padj_bh_rc(self, base_mean, G, pv, ld, K, cutoff, padj, ld_out):
        """emu_padj_bh's status: 0, or -2 (PDQ_ERR_INVALID) for bad shapes or a p-value outside [0, 1]."""
        return self.lib.emu_padj_bh(_p(base_mean, f64p), G, _p(pv, f64p), C.c_int64(ld), K, _p(cutoff, f64p), _p(padj, f64p),
                                    C.c_int64(ld_out))

    def padj_bh(self, *a):
        rc = self.padj_bh_rc(*a)
        assert rc == 0, rc


if __name__ == "__main__":
    print(build(force=True))
