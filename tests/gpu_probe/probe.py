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


class TeamProbe:
    """The SPD / accumulator / collective kernels of the team unit (team_probe.cu): one block of 32 W threads per problem."""

    def __init__(self):
        self.lib = C.CDLL(_build.build()["team"])
        self.lib.team_ws_bytes.restype = C.c_size_t
        self.max_p = self.lib.team_max_p()

    def _check(self, rc, what):
        if rc != 0:
            raise RuntimeError(f"team probe {what}: CUDA error {rc}")

    def ws_bytes(self, p, W):
        return int(self.lib.team_ws_bytes(int(p), int(W)))

    def spd(self, p, W, A, b, S, P, c, ridge=None, ridge_tri=None):
        """Per problem (rows of A, S, ridge_tri packed; b, c of p; P dense p x p): L of A + ridge, the solve x, H = (A + ridge)^-1
        and L^-1 (chol_inverse_w), A b (matvec_w), P b (apply_pinv); and every thread's logdet, symdot(A, S), quad(H, b) and Wald
        SE of c against A (wald_inverse_w with ridge_tri, or with none when the ridge is a scalar), each (n, 32 W)."""
        A, b, S, c = _d(A), _d(b), _d(S), _d(c)
        n, nt, NT = A.shape[0], p * (p + 1) // 2, 32 * W
        P = _d(np.broadcast_to(P, (n, p, p)))
        ridge = _d(np.broadcast_to(0.0 if ridge is None else ridge, (n,)))
        rt = None if ridge_tri is None else _d(np.broadcast_to(ridge_tri, (n, nt)))
        out = np.empty((n, 3 * nt + 3 * p))
        scal = np.empty((n, 4, NT))
        self._check(self.lib.team_spd(int(p), int(W), _p(A), _p(b), _p(S), _p(P), _p(c), _p(ridge),
                                      None if rt is None else _p(rt), int(n), _p(out), _p(scal)), "spd")
        o = np.cumsum([0, nt, p, nt, nt, p, p])
        names = ["L", "x", "H", "Li", "matvec", "pinv"]
        res = {k: out[:, o[i]:o[i + 1]] for i, k in enumerate(names)}
        res.update({k: scal[:, i] for i, k in enumerate(["logdet", "symdot", "quad", "se"])})
        return res

    def acc(self, p, W, X, w, z):
        """X (N, p) through design_pack; w, z (count, N): {"M": X^T W X packed (count, p(p+1)/2), "v": X^T z (count, p)}."""
        X, w, z = _d(X), _d(np.atleast_2d(w)), _d(np.atleast_2d(z))
        N, nt = X.shape[0], p * (p + 1) // 2
        out = np.empty((w.shape[0], nt + p))
        self._check(self.lib.team_acc(int(p), int(W), int(N), _p(X), _p(w), _p(z), int(w.shape[0]), _p(out)), "acc")
        return {"M": out[:, :nt], "v": out[:, nt:]}

    def coll(self, W, v, flag, a, b, lens):
        """Per block: v (5, 32 W), flag (32 W), a / b (maxn), lens: every thread's [sum v0, max v1, sum v2, any flag, max v3,
        sum v4, wdot(a, b), wmaxabs(a)] over the first lens[g] components, (count, 8, 32 W)."""
        v, a, b = _d(v), _d(a), _d(b)
        flag = np.ascontiguousarray(flag, dtype=np.int32)
        lens = np.ascontiguousarray(lens, dtype=np.int32)
        count, maxn = a.shape
        out = np.empty((count, 8, 32 * W))
        self._check(self.lib.team_coll(int(W), _p(v), _p(flag, i32p), _p(a), _p(b), _p(lens, i32p), int(maxn), int(count),
                                       _p(out)), "coll")
        return out
