// pdq_padj.cuh -- the arithmetic of DeseqStats' multiple-testing step (ds.py:486-542): the base-mean cutoffs of the independent
// filter (np.quantile, numpy 2.3's "linear" method) and the Benjamini-Hochberg value of scipy.stats.false_discovery_control.
// Compiled for the device (pdq_padj.cu) and for the host emulator of the test-suite (same source).
//
// Every product and sum is written with an explicit rounding (__dmul_rn / __dadd_rn / __dsub_rn on the device, volatile
// temporaries on the host) so that neither nvcc nor g++ contracts `a + d * t` into an FMA: the results are numpy's and scipy's
// bit for bit.
#pragma once

#include <math.h>
#include <stdint.h>

#ifndef PDQ_HD  // as in pdq_math.cuh, which this header does not need
#if defined(__CUDACC__)
#define PDQ_HD __host__ __device__ __forceinline__
#else
#define PDQ_HD inline
#endif
#endif

namespace pdq {

constexpr int kPadjMaxTheta = 64;  // filter thresholds per call: one bit each in a gene's 64-bit membership mask

PDQ_HD double rn_mul(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dmul_rn(a, b);
#else
    volatile double r = a * b;
    return r;
#endif
}
PDQ_HD double rn_add(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dadd_rn(a, b);
#else
    volatile double r = a + b;
    return r;
#endif
}
PDQ_HD double rn_sub(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dsub_rn(a, b);
#else
    volatile double r = a - b;
    return r;
#endif
}
PDQ_HD double rn_div(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __ddiv_rn(a, b);
#else
    volatile double r = a / b;
    return r;
#endif
}

// np.quantile(x, theta) with method="linear" on `sorted` = np.sort(x) of n >= 1 values (numpy 2.3, _quantile): virtual index
// (n - 1) * theta; previous = floor, next = previous + 1, both replaced by the last index when the virtual index is >= n - 1 and
// by 0 when it is < 0; gamma = virtual index - previous (after that replacement); then _lerp with its `t >= 0.5` branch.  A NaN
// anywhere in x makes every quantile NaN (numpy checks the last sorted value; the caller passes `any_nan`).
PDQ_HD double quantile_linear(const double* sorted, int64_t n, double theta, bool any_nan) {
    if (any_nan) return NAN;
    const double vi = rn_mul((double)(n - 1), theta);
    int64_t prev, next;
    if (vi >= (double)(n - 1)) {
        prev = next = -1;
    } else if (vi < 0.0) {
        prev = next = 0;
    } else {
        prev = (int64_t)floor(vi);
        next = prev + 1;
    }
    const double gamma = rn_sub(vi, (double)prev);
    const double a = sorted[prev < 0 ? n + prev : prev], b = sorted[next < 0 ? n + next : next];
    const double d = rn_sub(b, a);
    if (gamma >= 0.5) return rn_sub(b, rn_mul(d, rn_sub(1.0, gamma)));
    return rn_add(a, rn_mul(d, gamma));
}

// scipy's BH value of the gene of rank r (1-based, in ascending p) among m tested p-values: p * (m / r), an IEEE division and
// then a multiply; for m <= 1 scipy returns p as it is.  The adjusted p-value is the minimum of this over ranks >= r, clipped to
// [0, 1] (m > 1 only).
PDQ_HD double bh_value(double p, int64_t r, int64_t m) {
    if (m <= 1) return p;
    return rn_mul(p, rn_div((double)m, (double)r));
}

// Is the adjusted p-value of rank r below alpha, given that it is the suffix minimum?  Only the count of such ranks matters for
// the rejection table: it is the largest r whose own value (clipped) is below alpha.  Decided from p * m against alpha * r when
// the two differ by far more than the roundings of either side, exactly through bh_value otherwise.
PDQ_HD bool bh_below(double p, int64_t r, int64_t m, double alpha) {
    if (m > 1 && alpha <= 1.0) {
        const double t = p * (double)m, u = alpha * (double)r;
        if (t < u * (1.0 - 1e-12)) return true;
        if (t > u * (1.0 + 1e-12)) return false;
    }
    const double q = bh_value(p, r, m);
    return (m > 1 ? fmin(q, 1.0) : q) < alpha;
}

// numpy's clip(x, 0, 1) of a non-NaN x: maximum then minimum, each `a > b ? a : b` (so -0.0 becomes +0.0)
PDQ_HD double clip01(double x) {
    x = x > 0.0 ? x : 0.0;
    return x < 1.0 ? x : 1.0;
}

// is a gene in the set of pdq_padj_bh's row with this cutoff: tested, and base mean >= cutoff; -inf takes every tested gene
// whatever its base mean (plain BH, _p_value_adjustment)
PDQ_HD bool padj_in_set(double p, double base_mean, double cutoff) {
    return !isnan(p) && (base_mean >= cutoff || cutoff == -INFINITY);
}

// bits i < n_theta: base_mean >= cutoff[i] (a NaN base mean or cutoff sets no bit)
PDQ_HD uint64_t padj_member_mask(double base_mean, const double* cutoffs, int n_theta) {
    uint64_t m = 0;
    for (int i = 0; i < n_theta; ++i)
        if (base_mean >= cutoffs[i]) m |= (uint64_t)1 << i;
    return m;
}

}  // namespace pdq
