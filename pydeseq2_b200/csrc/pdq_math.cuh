// pdq_math.cuh -- FP64 building blocks shared by every per-gene routine.
//
// Everything here is `__host__ __device__` so that the exact same source is compiled (a) by nvcc
// for sm_90a and (b) by g++ into the host emulator used by the CPU test-suite
// (tests/emu/, test infrastructure only -- the product never loads it).
#pragma once

#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define PDQ_HD __host__ __device__ __forceinline__
// Loops over the p design columns: fully unrolled (register-resident p x p algebra) in the translation unit of p = 1..8; in the
// units of the wide designs (PDQ_TU_P = 9..16, see pdq_kernels.cu) they stay loops and the small matrices live in local
// memory -- slower per gene, but any design of up to 16 columns runs.  (A single `unroll (P <= 8 ? 64 : 1)` was tried first:
// a numeric factor made the base unit's kernels twice as large and its compilation seven times slower.)
#if defined(PDQ_TU_P) && PDQ_TU_P > 8
#define PDQ_UNROLL_P _Pragma("unroll 1")
#else
#define PDQ_UNROLL_P _Pragma("unroll")
#endif
#else
#define PDQ_HD inline
#define PDQ_UNROLL_P
#endif

namespace pdq {

constexpr double kRidge = 1e-6;          // utils.py:361 (ridge_factor of irls_solver)
constexpr double kHalfLog2Pi = 0.91893853320467274178;

PDQ_HD constexpr int tri(int i, int j) { return i * (i + 1) / 2 + j; }  // packed lower, j <= i

// ---------------------------------------------------------------------------------------------
// Packed lower-triangular Cholesky family for p x p SPD matrices held in registers.
// NaNs propagate (a non-positive pivot gives NaN through sqrt), mirroring how LAPACK failures
// surface as NaN/LinAlgError in the reference only for degenerate inputs.
// ---------------------------------------------------------------------------------------------
template <int P>
struct Sym {
    double a[P * (P + 1) / 2];
};

template <int P>
PDQ_HD void sym_zero(Sym<P>& s) {
PDQ_UNROLL_P
    for (int k = 0; k < P * (P + 1) / 2; ++k) s.a[k] = 0.0;
}

// s += w * x x^T
template <int P>
PDQ_HD void sym_rank1(Sym<P>& s, double w, const double (&x)[P]) {
PDQ_UNROLL_P
    for (int i = 0; i < P; ++i) {
        const double wx = w * x[i];
PDQ_UNROLL_P
        for (int j = 0; j <= i; ++j) s.a[tri(i, j)] = fma(wx, x[j], s.a[tri(i, j)]);
    }
}

// in-place L L^T = A
template <int P>
PDQ_HD void chol(Sym<P>& L) {
PDQ_UNROLL_P
    for (int j = 0; j < P; ++j) {
        double d = L.a[tri(j, j)];
PDQ_UNROLL_P
        for (int k = 0; k < j; ++k) d = fma(-L.a[tri(j, k)], L.a[tri(j, k)], d);
        d = sqrt(d);
        L.a[tri(j, j)] = d;
        const double inv = 1.0 / d;
PDQ_UNROLL_P
        for (int i = j + 1; i < P; ++i) {
            double s = L.a[tri(i, j)];
PDQ_UNROLL_P
            for (int k = 0; k < j; ++k) s = fma(-L.a[tri(i, k)], L.a[tri(j, k)], s);
            L.a[tri(i, j)] = s * inv;
        }
    }
}

// solve (L L^T) x = b in place
template <int P>
PDQ_HD void chol_solve(const Sym<P>& L, double (&b)[P]) {
PDQ_UNROLL_P
    for (int i = 0; i < P; ++i) {
        double s = b[i];
PDQ_UNROLL_P
        for (int k = 0; k < i; ++k) s = fma(-L.a[tri(i, k)], b[k], s);
        b[i] = s / L.a[tri(i, i)];
    }
PDQ_UNROLL_P
    for (int i = P - 1; i >= 0; --i) {
        double s = b[i];
PDQ_UNROLL_P
        for (int k = i + 1; k < P; ++k) s = fma(-L.a[tri(k, i)], b[k], s);
        b[i] = s / L.a[tri(i, i)];
    }
}

template <int P>
PDQ_HD double chol_logdet(const Sym<P>& L) {
    double s = 0.0;
PDQ_UNROLL_P
    for (int i = 0; i < P; ++i) s += log(L.a[tri(i, i)]);
    return 2.0 * s;
}

// inverse of (L L^T) as a packed symmetric matrix
template <int P>
PDQ_HD void chol_inverse(const Sym<P>& L, Sym<P>& Ainv) {
    Sym<P> Li;  // L^{-1}, lower
PDQ_UNROLL_P
    for (int j = 0; j < P; ++j) {
        Li.a[tri(j, j)] = 1.0 / L.a[tri(j, j)];
PDQ_UNROLL_P
        for (int i = j + 1; i < P; ++i) {
            double s = 0.0;
PDQ_UNROLL_P
            for (int k = j; k < i; ++k) s = fma(-L.a[tri(i, k)], Li.a[tri(k, j)], s);
            Li.a[tri(i, j)] = s / L.a[tri(i, i)];
        }
    }
    // Ainv = Li^T Li
PDQ_UNROLL_P
    for (int i = 0; i < P; ++i)
PDQ_UNROLL_P
        for (int j = 0; j <= i; ++j) {
            double s = 0.0;
PDQ_UNROLL_P
            for (int k = i; k < P; ++k) s = fma(Li.a[tri(k, i)], Li.a[tri(k, j)], s);
            Ainv.a[tri(i, j)] = s;
        }
}

// x^T S x for packed symmetric S
template <int P>
PDQ_HD double sym_quad(const Sym<P>& S, const double (&x)[P]) {
    double q = 0.0;
PDQ_UNROLL_P
    for (int i = 0; i < P; ++i) {
        double r = 0.0;
PDQ_UNROLL_P
        for (int j = 0; j < i; ++j) r = fma(S.a[tri(i, j)], x[j], r);
        q = fma(x[i], fma(2.0, r, S.a[tri(i, i)] * x[i]), q);
    }
    return q;
}

// y = S x
template <int P>
PDQ_HD void sym_matvec(const Sym<P>& S, const double (&x)[P], double (&y)[P]) {
PDQ_UNROLL_P
    for (int i = 0; i < P; ++i) {
        double r = 0.0;
PDQ_UNROLL_P
        for (int j = 0; j < P; ++j) r = fma(S.a[j <= i ? tri(i, j) : tri(j, i)], x[j], r);
        y[i] = r;
    }
}

// sum_ij S_ij T_ij  (= trace(S T) for symmetric S, T)
template <int P>
PDQ_HD double sym_dot(const Sym<P>& S, const Sym<P>& T) {
    double d = 0.0, o = 0.0;
PDQ_UNROLL_P
    for (int i = 0; i < P; ++i) {
        d = fma(S.a[tri(i, i)], T.a[tri(i, i)], d);
PDQ_UNROLL_P
        for (int j = 0; j < i; ++j) o = fma(S.a[tri(i, j)], T.a[tri(i, j)], o);
    }
    return fma(2.0, o, d);
}

// ---------------------------------------------------------------------------------------------
// Special functions for x > 0 (x = count + 1/alpha on this path).
// Stirling/Bernoulli asymptotics at z >= 10 with an exact upward shift of 10 below that; the shift
// uses the product P(x) = x (x+1) ... (x+9) and its derivative so that only ONE log and ONE
// division are spent on it:  lgamma(x) = lgamma(x+10) - log P(x),  psi(x) = psi(x+10) - P'(x)/P(x).
// Truncation error < 2e-16 absolute at z = 10 for both series (next omitted terms: 4.4e-17 / 1.2e-17).
// Worst error against mpmath over x in [1e-4, 1e9] (both sides of 10, the roots, integers), relative to max(|f|, 1), on the
// device (H100, tests/test_gpu_math.py) and the host (tests/test_math_ref.py) alike: lgamma_pos 6.9e-15, digamma_pos 1.4e-15,
// trigamma_pos 4.7e-16 (relative), lgamma_digamma_pos 6.4e-15 / 1.4e-15.  Asserted: |err| <= 3e-14 + 2e-14 |f| for lgamma /
// digamma, <= 4e-15 |f| for trigamma.
// ---------------------------------------------------------------------------------------------
PDQ_HD void shift10(double x, double& P, double& dP) {
    P = x;
    dP = 1.0;
#pragma unroll
    for (int k = 1; k < 10; ++k) {
        const double t = x + (double)k;
        dP = fma(dP, t, P);
        P *= t;
    }
}

PDQ_HD double fast_rcp(double d);  // pdq_fast.cuh
PDQ_HD double fast_div(double a, double b);
PDQ_HD double fast_log(double x);

PDQ_HD double digamma_asym(double z, double logz) {  // z >= 10
    const double iz = fast_rcp(z), w = iz * iz;
    // sum_k B_2k / (2k z^2k): 1/12, -1/120, 1/252, -1/240, 1/132, -691/32760, 1/12
    double s = 1.0 / 12.0;
    s = fma(s, w, -691.0 / 32760.0);
    s = fma(s, w, 1.0 / 132.0);
    s = fma(s, w, -1.0 / 240.0);
    s = fma(s, w, 1.0 / 252.0);
    s = fma(s, w, -1.0 / 120.0);
    s = fma(s, w, 1.0 / 12.0);
    return logz - 0.5 * iz - s * w;
}

PDQ_HD double lgamma_asym(double z, double logz) {  // z >= 10
    const double iz = fast_rcp(z), w = iz * iz;
    // sum_k B_2k / (2k (2k-1) z^(2k-1)): 1/12, -1/360, 1/1260, -1/1680, 1/1188, -691/360360, 1/156
    double s = 1.0 / 156.0;
    s = fma(s, w, -691.0 / 360360.0);
    s = fma(s, w, 1.0 / 1188.0);
    s = fma(s, w, -1.0 / 1680.0);
    s = fma(s, w, 1.0 / 1260.0);
    s = fma(s, w, -1.0 / 360.0);
    s = fma(s, w, 1.0 / 12.0);
    return fma(z - 0.5, logz, -z) + kHalfLog2Pi + s * iz;
}

// psi'(z), z >= 10: 1/z + 1/(2 z^2) + sum_k B_2k / z^(2k+1)   (next omitted term 3.6 z^-17)
PDQ_HD double trigamma_asym(double z) {
    const double iz = fast_rcp(z), w = iz * iz;
    double s = 7.0 / 6.0;
    s = fma(s, w, -691.0 / 2730.0);
    s = fma(s, w, 5.0 / 66.0);
    s = fma(s, w, -1.0 / 30.0);
    s = fma(s, w, 1.0 / 42.0);
    s = fma(s, w, -1.0 / 30.0);
    s = fma(s, w, 1.0 / 6.0);
    return fma(s * w, iz, fma(0.5, w, iz));
}

// psi'(x), x > 0: upward shift of 10 below z = 10, psi'(x) = psi'(x + 10) + sum_{k<10} (x + k)^-2
PDQ_HD double trigamma_pos(double x) {
    if (x >= 10.0) return trigamma_asym(x);
    double s = 0.0;
#pragma unroll
    for (int k = 0; k < 10; ++k) {
        const double i = fast_rcp(x + (double)k);
        s = fma(i, i, s);
    }
    return trigamma_asym(x + 10.0) + s;
}

PDQ_HD double digamma_pos(double x) {
    if (x >= 10.0) return digamma_asym(x, fast_log(x));
    double P, dP;
    shift10(x, P, dP);
    const double z = x + 10.0;
    return digamma_asym(z, fast_log(z)) - fast_div(dP, P);
}

PDQ_HD double lgamma_pos(double x) {
    if (x >= 10.0) return lgamma_asym(x, fast_log(x));
    double P, dP;
    shift10(x, P, dP);
    const double z = x + 10.0;
    return lgamma_asym(z, fast_log(z)) - fast_log(P);
}

// both at once (shares the log and the shift)
PDQ_HD void lgamma_digamma_pos(double x, double& lg, double& dg) {
    double z = x, corr_lg = 0.0, corr_dg = 0.0;
    if (x < 10.0) {
        double P, dP;
        shift10(x, P, dP);
        z = x + 10.0;
        corr_lg = log(P);
        corr_dg = dP / P;
    }
    const double lz = log(z);
    lg = lgamma_asym(z, lz) - corr_lg;
    dg = digamma_asym(z, lz) - corr_dg;
}

// two-sided normal tail helpers (scipy.stats.norm.sf(x) = 0.5 erfc(x / sqrt 2))
PDQ_HD double norm_sf(double x) { return 0.5 * erfc(x * 0.70710678118654752440); }

PDQ_HD double sgn(double x) { return (x != x) ? x : (double)((x > 0.0) - (x < 0.0)); }  // np.sign (NaN propagates)

}  // namespace pdq
