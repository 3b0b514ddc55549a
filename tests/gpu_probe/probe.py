"""ctypes front-end of the GPU probe (pdq_probe.cu).  Test infrastructure: every call copies its inputs to the device, runs
one kernel and copies the result back."""
import ctypes as C

import numpy as np

from . import build as _build

f64p = C.POINTER(C.c_double)
i32p = C.POINTER(C.c_int)
KTAB = 4 * 32  # doubles per gene written by the table kernel (math_ops.h: kTabOut)


def _d(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def _p(a, t=f64p):
    return a.ctypes.data_as(t)


class Probe:
    """The elementwise / table / collective / SPD kernels of one probe unit ("narrow" or "wide")."""

    def __init__(self, unit="narrow"):
        self.unit = unit
        self.lib = C.CDLL(_build.build()[unit])
        self.max_p = self.lib.probe_max_p()

    def _check(self, rc, what):
        if rc != 0:
            raise RuntimeError(f"probe {what}: CUDA error {rc}")

    def elem(self, op, x, y=None):
        x = _d(x)
        y = np.zeros_like(x) if y is None else _d(np.broadcast_to(y, x.shape))
        out = np.empty_like(x)
        self._check(self.lib.probe_elem(int(op), _p(x), _p(y), _p(out), int(x.size)), "elem")
        return out

    def tables(self, r, T):
        r = _d(r)
        out = np.empty((r.size, KTAB))
        self._check(self.lib.probe_tables(_p(r), int(r.size), int(T), _p(out)), "tables")
        return out

    def group(self, T, v, flag):
        v = _d(v)
        flag = np.ascontiguousarray(flag, dtype=np.int32)
        out = np.empty((5, v.size))
        self._check(self.lib.probe_group(int(T), _p(v), _p(flag, i32p), _p(out), int(v.size)), "group")
        return {"sum": out[0], "scan": out[1], "argmin": out[2].astype(np.int64), "argmax": out[3].astype(np.int64),
                "any": out[4] != 0}

    def spd(self, P, A, b, S):
        A, b, S = _d(A), _d(b), _d(S)
        n, nt = A.shape[0], P * (P + 1) // 2
        out = np.empty((n, 2 * P + nt + 3))
        self._check(self.lib.probe_spd(int(P), _p(A), _p(b), _p(S), _p(out), int(n)), "spd")
        return {"solve": out[:, :P], "inv": out[:, P:P + nt], "logdet": out[:, P + nt], "quad": out[:, P + nt + 1],
                "matvec": out[:, P + nt + 2:2 * P + nt + 2], "dot": out[:, 2 * P + nt + 2]}
