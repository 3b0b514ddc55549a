"""Unconstrained L-BFGS-B, restated.  TEST INFRASTRUCTURE (see oracle/nbglm.py for the import rules).

The reference fits the apeGLM MAP with ``scipy.optimize.minimize(method="L-BFGS-B", options={"ftol": 1e-8, "gtol": 1e-8})``
(``pydeseq2/utils.py:1110-1120``) and keeps whatever iterate the optimiser stops at -- on these objectives
that is 1e-3 .. 1e-2 (relative) away from the true optimum, so a backend can only agree with the reference to better than
that by walking the same iterates.  scipy (1.18.1 in this image; L-BFGS-B 3.0 of Zhu, Byrd, Lu, Nocedal, translated to C)
is a third-party dependency that is not part of PyDESeq2; this module restates its published algorithm for the case
the reference uses -- no bounds -- and is the specification the CUDA routine ``shrink_gene`` (pdq_gene.cuh) implements:

* direction: steepest descent while the memory is empty, otherwise the limited-memory BFGS step with ``m = 10`` pairs and
  ``H0 = (s'y / y'y) I`` of the newest pair (the subspace minimisation of L-BFGS-B with every variable free);
* line search: More-Thuente ``dcsrch``/``dcstep`` (MINPACK-2) with ``ftol = 1e-3, gtol = 0.9, xtol = 0.1``, first trial step
  ``1/|d|`` in the very first iteration and 1 afterwards, at most 20 evaluations, restart from steepest descent when it fails;
* pair update skipped when ``s'y <= eps * (-g'd * step)``;
* stop: ``max|g| <= pgtol`` (checked at the start point too) or ``(f_old - f) <= ftol * max(|f_old|, |f|, 1)``.

``tests/test_oracle_golden.py`` checks it against scipy itself (same iterates: equal iteration / evaluation counts, x to 1e-9).
"""
from __future__ import annotations

import numpy as np

EPS = np.finfo(float).eps
BIG = 1e10


def dcstep(stx, fx, dx, sty, fy, dy, stp, fp, dp, brackt, stpmin, stpmax):
    """MINPACK-2 dcstep: safeguarded cubic/quadratic step and interval update."""
    sgnd = dp * (dx / abs(dx))
    if fp > fx:  # case 1: higher function value -> minimum bracketed
        theta = 3.0 * (fx - fp) / (stp - stx) + dx + dp
        s = max(abs(theta), abs(dx), abs(dp))
        gamma = s * np.sqrt((theta / s) ** 2 - (dx / s) * (dp / s))
        if stp < stx:
            gamma = -gamma
        p = (gamma - dx) + theta
        q = ((gamma - dx) + gamma) + dp
        r = p / q
        stpc = stx + r * (stp - stx)
        stpq = stx + ((dx / ((fx - fp) / (stp - stx) + dx)) / 2.0) * (stp - stx)
        stpf = stpc if abs(stpc - stx) < abs(stpq - stx) else stpc + (stpq - stpc) / 2.0
        brackt = True
    elif sgnd < 0.0:  # case 2: derivatives of opposite sign -> bracketed
        theta = 3.0 * (fx - fp) / (stp - stx) + dx + dp
        s = max(abs(theta), abs(dx), abs(dp))
        gamma = s * np.sqrt((theta / s) ** 2 - (dx / s) * (dp / s))
        if stp > stx:
            gamma = -gamma
        p = (gamma - dp) + theta
        q = ((gamma - dp) + gamma) + dx
        r = p / q
        stpc = stp + r * (stx - stp)
        stpq = stp + (dp / (dp - dx)) * (stx - stp)
        stpf = stpc if abs(stpc - stp) > abs(stpq - stp) else stpq
        brackt = True
    elif abs(dp) < abs(dx):  # case 3: lower value, same sign, derivative magnitude decreases
        theta = 3.0 * (fx - fp) / (stp - stx) + dx + dp
        s = max(abs(theta), abs(dx), abs(dp))
        gamma = s * np.sqrt(max(0.0, (theta / s) ** 2 - (dx / s) * (dp / s)))
        if stp > stx:
            gamma = -gamma
        p = (gamma - dp) + theta
        q = (gamma + (dx - dp)) + gamma
        r = p / q
        if r < 0.0 and gamma != 0.0:
            stpc = stp + r * (stx - stp)
        elif stp > stx:
            stpc = stpmax
        else:
            stpc = stpmin
        stpq = stp + (dp / (dp - dx)) * (stx - stp)
        if brackt:
            stpf = stpc if abs(stpc - stp) < abs(stpq - stp) else stpq
            if stp > stx:
                stpf = min(stp + 0.66 * (sty - stp), stpf)
            else:
                stpf = max(stp + 0.66 * (sty - stp), stpf)
        else:
            stpf = stpc if abs(stpc - stp) > abs(stpq - stp) else stpq
            stpf = min(stpmax, stpf)
            stpf = max(stpmin, stpf)
    else:  # case 4: lower value, same sign, derivative magnitude does not decrease
        if brackt:
            theta = 3.0 * (fp - fy) / (sty - stp) + dy + dp
            s = max(abs(theta), abs(dy), abs(dp))
            gamma = s * np.sqrt((theta / s) ** 2 - (dy / s) * (dp / s))
            if stp > sty:
                gamma = -gamma
            p = (gamma - dp) + theta
            q = ((gamma - dp) + gamma) + dy
            r = p / q
            stpf = stp + r * (sty - stp)
        elif stp > stx:
            stpf = stpmax
        else:
            stpf = stpmin
    if fp > fx:
        sty, fy, dy = stp, fp, dp
    else:
        if sgnd < 0.0:
            sty, fy, dy = stx, fx, dx
        stx, fx, dx = stp, fp, dp
    return stx, fx, dx, sty, fy, dy, stpf, brackt


class Dcsrch:
    """MINPACK-2 dcsrch as a resumable object: ``start`` then ``step`` per evaluation; returns 'FG', 'CONV' or 'WARN'."""

    XTRAPL, XTRAPU = 1.1, 4.0

    def __init__(self, ftol=1e-3, gtol=0.9, xtol=0.1, stpmin=0.0, stpmax=BIG):
        self.ftol, self.gtol, self.xtol, self.stpmin, self.stpmax = ftol, gtol, xtol, stpmin, stpmax

    def start(self, stp, f, g):
        self.brackt, self.stage = False, 1
        self.finit, self.ginit = f, g
        self.gtest = self.ftol * g
        self.width = self.stpmax - self.stpmin
        self.width1 = self.width / 0.5
        self.stx, self.fx, self.gx = 0.0, f, g
        self.sty, self.fy, self.gy = 0.0, f, g
        self.stmin, self.stmax = 0.0, stp + self.XTRAPU * stp
        return stp

    def step(self, stp, f, g):
        ftest = self.finit + stp * self.gtest
        if self.stage == 1 and f <= ftest and g >= 0.0:
            self.stage = 2
        task = "FG"
        if self.brackt and (stp <= self.stmin or stp >= self.stmax):
            task = "WARN"  # rounding errors prevent progress
        if self.brackt and self.stmax - self.stmin <= self.xtol * self.stmax:
            task = "WARN"  # xtol test satisfied
        if stp == self.stpmax and f <= ftest and g <= self.gtest:
            task = "WARN"
        if stp == self.stpmin and (f > ftest or g >= self.gtest):
            task = "WARN"
        if f <= ftest and abs(g) <= self.gtol * (-self.ginit):
            task = "CONV"
        if task != "FG":
            return stp, task
        if self.stage == 1 and f <= self.fx and f > ftest:
            gt = self.gtest
            fm, fxm, fym = f - stp * gt, self.fx - self.stx * gt, self.fy - self.sty * gt
            gm, gxm, gym = g - gt, self.gx - gt, self.gy - gt
            self.stx, fxm, gxm, self.sty, fym, gym, stp, self.brackt = dcstep(self.stx, fxm, gxm, self.sty, fym, gym, stp, fm, gm,
                                                                            self.brackt, self.stmin, self.stmax)
            self.fx, self.fy = fxm + self.stx * gt, fym + self.sty * gt
            self.gx, self.gy = gxm + gt, gym + gt
        else:
            self.stx, self.fx, self.gx, self.sty, self.fy, self.gy, stp, self.brackt = dcstep(
                self.stx, self.fx, self.gx, self.sty, self.fy, self.gy, stp, f, g, self.brackt, self.stmin, self.stmax)
        if self.brackt:
            if abs(self.sty - self.stx) >= 0.66 * self.width1:
                stp = self.stx + 0.5 * (self.sty - self.stx)
            self.width1 = self.width
            self.width = abs(self.sty - self.stx)
        if self.brackt:
            self.stmin, self.stmax = min(self.stx, self.sty), max(self.stx, self.sty)
        else:
            self.stmin = stp + self.XTRAPL * (stp - self.stx)
            self.stmax = stp + self.XTRAPU * (stp - self.stx)
        stp = min(max(stp, self.stpmin), self.stpmax)
        if (self.brackt and (stp <= self.stmin or stp >= self.stmax)) or (
                self.brackt and self.stmax - self.stmin <= self.xtol * self.stmax):
            stp = self.stx
        return stp, "FG"


def minimize_lbfgsb_unbounded(fun, jac, x0, ftol=1e-8, gtol=1e-8, m=10, maxiter=15000, maxls=20):
    """Returns (x, success, nit, nfev)."""
    x = np.array(x0, dtype=float)
    f, g = float(fun(x)), np.array(jac(x), dtype=float)
    nfev, nit = 1, 0
    S, Y = [], []
    theta = 1.0
    if np.max(np.abs(g)) <= gtol:
        return x, True, nit, nfev
    while True:
        # ---- direction
        if not S:
            z = x + (1.0 / theta) * (-g)
        else:
            q = -g.copy()
            al = []
            for s, yv in zip(reversed(S), reversed(Y)):
                a = (s @ q) / (yv @ s)
                al.append(a)
                q = q - a * yv
            r = q / theta
            for (s, yv), a in zip(zip(S, Y), reversed(al)):
                b = (yv @ r) / (yv @ s)
                r = r + s * (a - b)
            z = x + r
        d = z - x
        # ---- line search
        dnorm = np.sqrt(d @ d)
        stp = min(1.0 / dnorm, BIG) if nit == 0 else 1.0
        t, r_old, fold = x.copy(), g.copy(), f
        gd = g @ d
        gdold = gd
        failed = gd >= 0.0
        iback = 0
        if not failed:
            ls = Dcsrch()
            stp = ls.start(stp, f, gd)
            while True:
                x = z.copy() if stp == 1.0 else stp * d + t
                f, g = float(fun(x)), np.array(jac(x), dtype=float)
                nfev += 1
                gd = g @ d
                stp, task = ls.step(stp, f, gd)
                if task != "FG":
                    break
                iback += 1
                if iback >= maxls:
                    failed = True
                    break
        if failed:
            x, g, f = t, r_old, fold
            if not S:
                return x, False, nit, nfev  # ABNORMAL_TERMINATION_IN_LNSRCH
            S, Y, theta = [], [], 1.0
            continue  # restart from steepest descent, same iteration count
        nit += 1
        if np.max(np.abs(g)) <= gtol:
            return x, True, nit, nfev
        if (fold - f) <= ftol * max(abs(fold), abs(f), 1.0):
            return x, True, nit, nfev
        if nit >= maxiter:
            return x, False, nit, nfev
        # ---- memory update
        yv = g - r_old
        rr = yv @ yv
        if stp == 1.0:
            dr, ddum, s = gd - gdold, -gdold, d
        else:
            dr, ddum, s = (gd - gdold) * stp, -gdold * stp, stp * d
        if dr <= EPS * ddum:
            continue
        S.append(s)
        Y.append(yv)
        if len(S) > m:
            S.pop(0)
            Y.pop(0)
        theta = rr / dr
