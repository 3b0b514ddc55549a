// pdq_fast.cuh -- FP64 log / exp / reciprocal tuned for the sm_90a FP64 pipe.
//
// Why not libdevice's `log`, `exp` and the `/` operator: their SASS materialises 64-bit polynomial coefficients with
// UMOV / IMAD.MOV pairs next to every DFMA and wraps each division's slow path in BSSY/BSYNC/branch scaffolding.  Here
//   * coefficients live in __constant__ memory, so DFMA takes them as constant-bank operands (no extra instruction);
//   * the reciprocal is MUFU.RCP64H + two Newton steps, branch-free (operands on this path are normal, finite);
//   * special cases (NaN, inf, zero, denormal, |x| huge) fall through to libdevice behind one predictable branch.
// Accuracy, worst case against mpmath over the inputs of tests/golden/math_ref.npz (scripts/make_math_golden.py), measured on the
// device branches (sm_90a, H100 80GB HBM3; tests/test_gpu_math.py) and the host branches (tests/test_math_ref.py) alike:
//   fast_log / fast_log_nb 1.75 ulp, fast_exp / fast_exp_nb 0.95 ulp, fast_rcp / fast_div 0.50 ulp;
// the tests assert <= 2 ulp for log/exp over the guarded range and <= 1 ulp for the reciprocal and the division.
#pragma once

#include <string.h>

#include "pdq_math.cuh"
#include "pdq_tables.h"

namespace pdq {

#if defined(__CUDA_ARCH__)
#define PDQ_CONST __constant__
#else
#define PDQ_CONST static const
#endif

// log(m) = 2f (1 + s g(s)),  f = (m-1)/(m+1), s = f^2, m in [sqrt(1/2), sqrt(2)];  g ~ degree-6 fit, |rel err| < 6e-18
PDQ_CONST double kLogG[7] = {0.3333333333333335, 0.1999999999994302, 0.14285714315994175, 0.11111105083699467,
                             0.09091479328268151, 0.07664720034027003, 0.073221513558091};
// e^r = 1 + r + r^2 q(r) on |r| <= ln2/2;  q ~ degree-9 fit, |abs err| < 1.5e-17
PDQ_CONST double kExpQ[10] = {0.5000000000000001, 0.1666666666666667, 0.04166666666662063, 0.008333333333325553,
                              0.0013888888918941061, 0.00019841269876841745, 2.480151863878229e-05,
                              2.7557252858587773e-06, 2.762133977167299e-07, 2.5106265298633842e-08};
PDQ_CONST double kLn2Hi = 6.93147180369123816490e-01;  // ln2 with the low 21 bits zero (fdlibm split)
PDQ_CONST double kLn2Lo = 1.90821492927058770002e-10;
PDQ_CONST double kLog2e = 1.44269504088896338700e+00;

// Polynomial tails.  Default: Horner (fewest instructions, one dependent DFMA per coefficient).  -DPDQ_ESTRIN=1 (experiment,
// default off): Estrin's scheme -- pairs, then powers of the square -- halves the dependent depth (log: 6 -> 4, exp: 9 -> 5) for two
// or three extra multiplications; the kernels stall on fixed-latency dependencies, not on FP64 issue slots (DESIGN.md §9.1).
#ifndef PDQ_ESTRIN
#define PDQ_ESTRIN 0
#endif

PDQ_HD double poly_log_g(double s) {
#if PDQ_ESTRIN
    const double s2 = s * s;
    const double p01 = fma(kLogG[1], s, kLogG[0]), p23 = fma(kLogG[3], s, kLogG[2]), p45 = fma(kLogG[5], s, kLogG[4]);
    const double s4 = s2 * s2;
    const double lo = fma(p23, s2, p01), hi = fma(kLogG[6], s2, p45);
    return fma(hi, s4, lo);
#else
    double g = kLogG[6];
    g = fma(g, s, kLogG[5]);
    g = fma(g, s, kLogG[4]);
    g = fma(g, s, kLogG[3]);
    g = fma(g, s, kLogG[2]);
    g = fma(g, s, kLogG[1]);
    return fma(g, s, kLogG[0]);
#endif
}

PDQ_HD double poly_exp_q(double r) {
#if PDQ_ESTRIN
    const double r2 = r * r;
    const double p01 = fma(kExpQ[1], r, kExpQ[0]), p23 = fma(kExpQ[3], r, kExpQ[2]), p45 = fma(kExpQ[5], r, kExpQ[4]);
    const double p67 = fma(kExpQ[7], r, kExpQ[6]), p89 = fma(kExpQ[9], r, kExpQ[8]);
    const double r4 = r2 * r2;
    const double q03 = fma(p23, r2, p01), q47 = fma(p67, r2, p45);
    const double r8 = r4 * r4;
    return fma(p89, r8, fma(q47, r4, q03));
#else
    double q = kExpQ[9];
    q = fma(q, r, kExpQ[8]);
    q = fma(q, r, kExpQ[7]);
    q = fma(q, r, kExpQ[6]);
    q = fma(q, r, kExpQ[5]);
    q = fma(q, r, kExpQ[4]);
    q = fma(q, r, kExpQ[3]);
    q = fma(q, r, kExpQ[2]);
    q = fma(q, r, kExpQ[1]);
    return fma(q, r, kExpQ[0]);
#endif
}

// 1/d for normal finite d (|d| in [2^-1000, 2^1000]): hardware seed + two Newton-Raphson steps
PDQ_HD double fast_rcp(double d) {
#if defined(__CUDA_ARCH__)
    double y;
    asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(d));
    double e = fma(-d, y, 1.0);
    y = fma(y, e, y);
    e = fma(-d, y, 1.0);
    return fma(y, e, y);
#else
    return 1.0 / d;
#endif
}

// a / b with one residual correction (<= 1 ulp for normal operands)
PDQ_HD double fast_div(double a, double b) {
#if defined(__CUDA_ARCH__)
    const double y = fast_rcp(b);
    const double q = a * y;
    return fma(fma(-b, q, a), y, q);
#else
    return a / b;
#endif
}

PDQ_HD double fast_log(double x) {
#if defined(__CUDA_ARCH__)
    int hi = __double2hiint(x);
    const int lo = __double2loint(x);
    if ((unsigned)(hi - 0x00100000) >= 0x7fe00000u) return log(x);  // <=0, denormal, inf, NaN: libdevice semantics
    int e = (hi >> 20) - 1023;
    hi = (hi & 0x000fffff) | 0x3ff00000;
    if (hi >= 0x3ff6a09f) {  // m > ~sqrt(2): halve it
        hi -= 0x00100000;
        e += 1;
    }
    const double m = __hiloint2double(hi, lo);
    const double ed = (double)e;
#else
    if (!(x > 2.2250738585072014e-308) || !(x < 1.7976931348623157e308)) return log(x);
    int e;
    double m = frexp(x, &e);  // m in [0.5, 1)
    m *= 2.0;
    e -= 1;
    if (m > 1.4142135623730951) {
        m *= 0.5;
        e += 1;
    }
    const double ed = (double)e;
#endif
    const double f = fast_div(m - 1.0, m + 1.0);
    const double s = f * f;
    const double g = poly_log_g(s);
    const double f2 = f + f;
    // e*ln2_hi is exact (|e| < 2^11, ln2_hi has 21 trailing zero bits)
    return fma(ed, kLn2Hi, f2 + fma(f2 * s, g, ed * kLn2Lo));
}

// Branch-free cores.  `fast_log_nb` needs a positive normal finite argument, `fast_exp_nb` needs |x| < 700; callers
// track violations in a flag and redo the (rare) affected gene through the guarded versions, so that the hot loops stay
// straight-line code in which the chains of two samples interleave.
PDQ_HD double fast_exp(double x);

PDQ_HD double fast_log_nb(double x) {
#if defined(__CUDA_ARCH__)
    int hi = __double2hiint(x);
    const int lo = __double2loint(x);
    int e = (hi >> 20) - 1023;
    hi = (hi & 0x000fffff) | 0x3ff00000;
    const bool big = hi >= 0x3ff6a09f;
    hi = big ? hi - 0x00100000 : hi;
    e = big ? e + 1 : e;
    const double m = __hiloint2double(hi, lo);
    const double ed = (double)e;
    const double f = fast_div(m - 1.0, m + 1.0);
    const double s = f * f;
    const double g = poly_log_g(s);
    const double f2 = f + f;
    return fma(ed, kLn2Hi, f2 + fma(f2 * s, g, ed * kLn2Lo));
#else
    return fast_log(x);
#endif
}

PDQ_HD double fast_exp_nb(double x) {
#if defined(__CUDA_ARCH__)
    const double kd = rint(x * kLog2e);
    const double r = fma(-kd, kLn2Lo, fma(-kd, kLn2Hi, x));
    const double q = poly_exp_q(r);
    const double p = fma(r * r, q, r) + 1.0;
    return p * __hiloint2double(((int)kd + 1023) << 20, 0);
#else
    return fast_exp(x);
#endif
}

PDQ_HD double fast_exp(double x) {
    if (!(fabs(x) < 700.0)) return exp(x);  // overflow/underflow edge, inf, NaN: libm/libdevice semantics
    const double kd = rint(x * kLog2e);
    const double r = fma(-kd, kLn2Lo, fma(-kd, kLn2Hi, x));
    const double q = poly_exp_q(r);
    const double p = fma(r * r, q, r) + 1.0;
    const int k = (int)kd;  // |k| <= 1010: 2^k is a normal double
#if defined(__CUDA_ARCH__)
    return p * __hiloint2double((k + 1023) << 20, 0);
#else
    return ldexp(p, k);
#endif
}

// ---------------------------------------------------------------------------------------------------------------------
// Table-driven logarithm / exponential (round 2).  The ncu captures of round 1 showed both heavy kernels bound by the FP64
// pipe with a third of its instructions spent inside fast_log (a division -- seed + 2 Newton steps + residual -- and a
// degree-6 polynomial: ~24 FP64 instructions).  With a 512-entry table of (c ~ 1/m, -log c) staged in shared memory the
// argument reduction is ONE fma, r = m c - 1 with |r| <= 2^-10 (first interval: [0, 2^-9)), and log1p(r) is its Taylor
// polynomial of degree 6: 10 FP64 instructions and one 16-byte shared-memory read.  Table construction and the sqrt(2) split
// that keeps the result relatively accurate around x = 1: scripts/gen_math_tables.py.  Worst case against mpmath over every
// table interval's ends and midpoint at four exponents (2^-1022, 1/2, 1, 2^1023), the split, powers of two and random fill:
// tlog / tlog_nb 1.38 ulp, texp / texp_nb 0.97 ulp, on the device (H100, tests/test_gpu_math.py) and the host (tests/test_math_ref.py); both assert
// <= 1.5 ulp.  tests/test_math_ref.py also checks the committed tables against the generator's definition.
// `tab` points at kMathTab (shared memory on the device, host_math_table() in the emulator).
// ---------------------------------------------------------------------------------------------------------------------
inline const double* host_math_table() {
    static const double t[kMathTabLen] = {PDQ_MATH_TABLE_VALUES};
    return t;
}

// x positive, normal, finite (callers track violations like for fast_log_nb)
PDQ_HD double tlog_nb(double x, const double* tab) {
#if defined(__CUDA_ARCH__)
    const int hi = __double2hiint(x);
    const int idx = (hi >> (20 - kLogTabBits)) & (kLogTabN - 1);
    // exponent, +1 when the mantissa lies at or above the table's sqrt(2) split: the bias makes exactly those mantissas carry
    const int e = (hi + (0x00100000 - (kLogTabSplit << (20 - kLogTabBits))) - 0x3ff00000) >> 20;
    const double m = __hiloint2double((hi & 0x000fffff) | 0x3ff00000, __double2loint(x));
    const double2 cl = reinterpret_cast<const double2*>(tab)[idx];
    const double c = cl.x, l = cl.y;
#else
    uint64_t u;
    memcpy(&u, &x, 8);
    const int hi = (int)(u >> 32);
    const int idx = (hi >> (20 - kLogTabBits)) & (kLogTabN - 1);
    const int e = ((hi >> 20) & 0x7ff) - 1023 + (idx >= kLogTabSplit ? 1 : 0);
    u = (u & 0x000fffffffffffffull) | 0x3ff0000000000000ull;
    double m;
    memcpy(&m, &u, 8);
    const double c = tab[2 * idx], l = tab[2 * idx + 1];
#endif
    const double r = fma(m, c, -1.0);
    // log1p(r) = r + r^2 (-1/2 + r (1/3 + r (-1/4 + r (1/5 - r/6))))
    double q = fma(r, -1.0 / 6.0, 0.2);
    q = fma(q, r, -0.25);
    q = fma(q, r, 1.0 / 3.0);
    q = fma(q, r, -0.5);
    const double t = fma(r * r, q, r) + l;
    const double ed = (double)e;
    return fma(ed, kLn2Hi, fma(ed, kLn2Lo, t));
}

// guarded version: <= 0, denormal, inf, NaN take the libm / libdevice path
PDQ_HD double tlog(double x, const double* tab) {
    if (!(x >= 2.2250738585072014e-308) || !(x <= 1.7976931348623157e308)) return log(x);
    return tlog_nb(x, tab);
}

PDQ_CONST double kLn2o64Hi = 6.93147180369123816490e-01 / 64.0;  // exact scalings of the fdlibm split
PDQ_CONST double kLn2o64Lo = 1.90821492927058770002e-10 / 64.0;
PDQ_CONST double k64oLn2 = 64.0 * 1.44269504088896338700e+00;

// e^x = 2^(k >> 6) * 2^((k & 63) / 64) * e^r,  k = rint(64 x / ln2), |r| <= ln2 / 128; needs |x| < 700
PDQ_HD double texp_nb(double x, const double* tab) {
    const double kd = rint(x * k64oLn2);
    const double r = fma(-kd, kLn2o64Lo, fma(-kd, kLn2o64Hi, x));
    const int k = (int)kd;
    const double T = tab[2 * kLogTabN + (k & 63)];
    // e^r - 1 = r + r^2 (1/2 + r (1/6 + r (1/24 + r (1/120 + r/720))))
    double q = fma(r, 1.0 / 720.0, 1.0 / 120.0);
    q = fma(q, r, 1.0 / 24.0);
    q = fma(q, r, 1.0 / 6.0);
    q = fma(q, r, 0.5);
    const double p = fma(r * r, q, r);
    const double v = fma(T, p, T);  // in [1, 2): scaling by 2^(k >> 6) is an exponent-field addition (result stays normal)
#if defined(__CUDA_ARCH__)
    return __hiloint2double(__double2hiint(v) + ((k >> 6) << 20), __double2loint(v));
#else
    return ldexp(v, k >> 6);
#endif
}

PDQ_HD double texp(double x, const double* tab) {
    if (!(fabs(x) < 700.0)) return exp(x);
    return texp_nb(x, tab);
}

}  // namespace pdq
