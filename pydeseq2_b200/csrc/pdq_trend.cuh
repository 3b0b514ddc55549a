// pdq_trend.cuh -- parametric dispersion trend  alpha ~ a0 + a1 / mean  as a gamma GLM with identity link
// (reference: default_inference.py:200-230 for one fit, dds.py:1199-1275 for the outer loop that drops
// genes far from the curve and refits until the coefficients stop moving).
//
// The reference minimises  L(c) = mean(t/m + log m),  m = c0 + c1 x,  with scipy L-BFGS-B from (1, 1) under
// c >= 1e-12.  L-BFGS-B stops within ~4e-6 (relative) of the minimiser (measured, DESIGN.md §6); this code
// converges to the minimiser itself: Fisher scoring (expected Hessian, always positive definite) while the
// observed Hessian is indefinite, Newton steps once it is positive definite, backtracking on L, projection
// onto the bounds.  The whole fit -- all iterations of all outer rounds -- runs inside ONE kernel launch of
// one cooperative block; per iteration the G-length sums are block-reduced (warp shuffles + shared memory).
// Compiled for the host emulator as well (one "thread").
#pragma once

#include <string.h>

#include "pdq_fast.cuh"
#include "pdq_math.cuh"

namespace pdq {

struct TrendOut {
    double c0, c1;
    double status;   // 0 = ok, 1 = failed (not converged or a coefficient <= 1e-10) -> caller falls back to the mean trend
    double n_outer;  // outer rounds performed (dds.py:1236 loop)
    double n_used;   // genes left in the fit after outlier filtering
    double n_iter;   // inner iterations summed over rounds
    double loss;
    double last_converged;  // 1 when the most recent single fit converged (the reference's `res.success`)
    // dispersion prior (dds.py:840-884), filled by trend_prior(): squared scaled MAD of the log residuals of the genes
    // with genewise >= 100 * min_disp, the prior variance max(sq - trigamma((N-p)/2), 0.25), and the genes counted
    double squared_logres, prior_var, n_above;
    double pad[5];
};

// Reducer concept: tid(), nthreads(), sum(double) -> block-wide total visible to every thread.
struct SerialReducer {
    PDQ_HD int tid() const { return 0; }
    PDQ_HD int nthreads() const { return 1; }
    PDQ_HD double sum(double v) { return v; }
    PDQ_HD void sum_many(double*, int) {}  // in-place totals of k values, visible to every thread
    PDQ_HD void sync() {}
    // thread-private in the emulator; block-shared scratch on the device
    PDQ_HD int local_tid() const { return 0; }
    PDQ_HD int local_nthreads() const { return 1; }
    PDQ_HD void local_sync() {}
    PDQ_HD double max_one(double v) { return v; }
    PDQ_HD void hist_begin() {}
    PDQ_HD unsigned* hist_merge(unsigned* hist) { return hist; }
    PDQ_HD void find_bin(const unsigned* hist, unsigned*, size_t k, int& d, size_t& cum) {
        cum = 0;
        for (d = 0; d < 256; ++d) {
            const size_t c = hist[d];
            if (cum + c > k) break;
            cum += c;
        }
    }
};

// A per-gene vector as one thread of the fit sees it: a plain array indexed by gene (element i at v[i]), or the thread's own
// elements in its block's shared memory (LocalVec: its k-th gene, i = tid + k nthreads, at p[k stride]).  Every pass of the fit and
// of the prior visits the genes with the same map, so a thread only ever reads the elements it wrote itself.
struct LocalVec {
    double* p;
    unsigned stride;
};
PDQ_HD double& at(double* v, size_t i, size_t) { return v[i]; }
PDQ_HD double at(const double* v, size_t i, size_t) { return v[i]; }
PDQ_HD double& at(const LocalVec& v, size_t, size_t k) { return v.p[k * v.stride]; }

struct TrendSums {
    double L, g0, g1, h00, h01, h11, f00, f01, f11, n;
};

// xs[i]: covariate; ts[i]: target, NaN when the gene is not (or no longer) part of the fit.  Both are prepared once per
// launch by trend_prepare (clip, 1/mean, validity), so that a pass is: two loads, one reciprocal, one log, ten sums.
// The sums g1, h01, h11, f01, f11 are taken over the covariate less `xc` (see trend_fit_once); xc = 0 gives the plain sums.
template <class R, class VX, class VT>
PDQ_HD TrendSums trend_sums(R& red, const VX& xs, const VT& ts, size_t n, double c0, double c1, double xc = 0.0) {
    double L = 0, g0 = 0, g1 = 0, h00 = 0, h01 = 0, h11 = 0, f00 = 0, f01 = 0, f11 = 0, cnt = 0;
    for (size_t i = red.tid(), k = 0; i < n; i += red.nthreads(), ++k) {
        const double tv = at(ts, i, k);
        if (!(tv == tv)) continue;  // dropped gene / np.nanmean skips NaN targets
        const double xv = at(xs, i, k);
        const double m = fma(c1, xv, c0);
        const double im = fast_rcp(m);
        const double r = tv * im;
        L += r + fast_log(m);
        const double gi = -(r - 1.0) * im;             // d/dm (t/m + log m) = (1 - t/m)/m
        const double xd = xv - xc;
        g0 += gi;
        g1 += gi * xd;
        const double hi2 = (2.0 * r - 1.0) * im * im;  // d2/dm2
        h00 += hi2;
        h01 += hi2 * xd;
        h11 += hi2 * xd * xd;
        const double fi = im * im;                     // expected (Fisher) curvature
        f00 += fi;
        f01 += fi * xd;
        f11 += fi * xd * xd;
        cnt += 1.0;
    }
    double v[10] = {L, g0, g1, h00, h01, h11, f00, f01, f11, cnt};
    red.sum_many(v, 10);  // one packed reduction round for all ten sums
    TrendSums s;
    s.L = v[0]; s.g0 = v[1]; s.g1 = v[2];
    s.h00 = v[3]; s.h01 = v[4]; s.h11 = v[5];
    s.f00 = v[6]; s.f01 = v[7]; s.f11 = v[8];
    s.n = v[9];
    return s;
}

// One GLM fit; returns true when converged.  Starts from the incoming (c0, c1): (1, 1) for the first round like the
// reference (default_inference.py:221); later rounds of the outer loop warm-start from the previous optimum -- the
// minimiser does not depend on the start, only the iteration count does.  Every trial point costs ONE pass: the sums at
// the candidate serve both the Armijo test and, once accepted, the next Newton direction.
//
// When the covariate is (nearly) constant over the fitted genes, 1 and x are (nearly) collinear: the Fisher determinant
// f00 f11 - f01^2 is then cancellation, down to rounding noise, and a step through it can land anywhere (inf, or a point
// that is not a minimiser).  Below kSing f00 f11 the fit measures the covariate from its smallest fitted value xc, once,
// and solves for the step in (c0 + c1 xc, c1): the same point and the same steps in exact arithmetic, but the terms
// x - xc are small, and exact wherever x lies within a factor two of xc (Sterbenz), as it does for every nearly constant
// covariate, so the sums no longer cancel to rounding noise.  Their determinant a d - b^2 still
// cancels where most of the weight lies far from xc, to about 1/n relative at worst, which double precision resolves.
// kSing: the relative determinant is the weighted variance of x over its weighted mean square; real covariates (1 / mean over
// orders of magnitude) sit near 0.1-1, and a uniform spread of s relative gives about s^2 / 3.  1e-5 takes every spread below
// ~5e-3 (the plain solve failed to reach the minimiser at spreads of 1e-9 to 1e-3) and leaves every realistic fit, and every
// pinned record, on the plain path.
// A covariate that is exactly constant leaves only m = c0 + c1 x identified; the step then moves m to its optimum by the
// shortest step in (c0, c1), which makes the fit the minimiser nearest its start.
template <class R, class VX, class VT>
PDQ_HD bool trend_fit_once(R& red, const VX& xs, const VT& ts, size_t n, double& c0, double& c1, double& loss, int& iters) {
    const double kLB = 1e-12;    // bounds=[(1e-12, inf)] (default_inference.py:224)
    const double kSing = 1e-5;   // relative Fisher determinant below which 1 and x count as nearly collinear (see above)
    bool centred = false;
    double xc = 0.0;
    TrendSums s = trend_sums(red, xs, ts, n, c0, c1);
    ++iters;
    for (int it = 0; it < 200; ++it) {
        loss = s.L / s.n;
        if (!(s.L == s.L) || s.n < 2.0) return false;
        if (!centred && !(s.f00 * s.f11 - s.f01 * s.f01 > kSing * s.f00 * s.f11)) {
            double mx = -HUGE_VAL;
            for (size_t i = red.tid(), k = 0; i < n; i += red.nthreads(), ++k)
                if (at(ts, i, k) == at(ts, i, k)) mx = fmax(mx, -at(xs, i, k));
            xc = -red.max_one(mx);
            centred = true;
            s = trend_sums(red, xs, ts, n, c0, c1, xc);
            ++iters;
        }
        const double gc1 = centred ? fma(xc, s.g0, s.g1) : s.g1;  // dL/dc1
        // variables held at the lower bound with the gradient pushing outward are fixed
        const bool fix0 = (c0 <= kLB && s.g0 > 0.0), fix1 = (c1 <= kLB && gc1 > 0.0);
        double d0 = 0.0, d1 = 0.0;
        {
            double a = s.h00, b = s.h01, d = s.h11;
            const bool pd = (a > 0.0) && (a * d - b * b > 1e-12 * a * d);
            if (!pd) { a = s.f00; b = s.f01; d = s.f11; }  // Fisher scoring: always positive definite
            if (fix0 && fix1) return true;
            if (fix0) {
                d1 = -gc1 / (centred ? fma(xc, fma(xc, a, 2.0 * b), d) : d);  // curvature in c1 alone: sum w x^2
            } else if (fix1) {
                d0 = -s.g0 / a;
            } else if (centred && !(d > 0.0)) {  // every fitted x equals xc: the shortest step that moves m by -g0 / a
                const double dm = -s.g0 / a, w = 1.0 / fma(xc, xc, 1.0);
                d0 = dm * w;
                d1 = dm * xc * w;
            } else {
                const double det = a * d - b * b;
                d0 = -(d * s.g0 - b * s.g1) / det;
                d1 = -(a * s.g1 - b * s.g0) / det;
                if (centred) d0 = fma(-xc, d1, d0);  // the step in c0 + c1 xc, back to c0
            }
        }
        const double dec = -(s.g0 * d0 + gc1 * d1);             // Newton decrement (>= 0 for a descent direction)
        const bool endgame = dec <= 1e-9 * fabs(s.L);           // the summed loss no longer resolves progress in FP64
        // on a nearly constant covariate a step that carries a free coefficient across its bound stops there: projecting the
        // whole step instead keeps the other coefficient's share of a very long step, far from any minimiser
        const double a0 = (centred && c0 > kLB && c0 + d0 < kLB) ? (c0 - kLB) / -d0 : HUGE_VAL;
        const double a1 = (centred && c1 > kLB && c1 + d1 < kLB) ? (c1 - kLB) / -d1 : HUGE_VAL;
        double step = fmin(1.0, fmin(a0, a1)), n0 = c0, n1 = c1;
        TrendSums sn = s;
        bool acc = false;
        for (int ls = 0; ls < 40; ++ls) {
            n0 = step >= a0 ? kLB : fmax(fma(step, d0, c0), kLB);
            n1 = step >= a1 ? kLB : fmax(fma(step, d1, c1), kLB);
            sn = trend_sums(red, xs, ts, n, n0, n1, xc);
            ++iters;
            if (endgame || sn.L <= s.L + 1e-4 * (s.g0 * (n0 - c0) + gc1 * (n1 - c1))) {
                acc = true;
                break;
            }
            step *= 0.5;
        }
        if (!acc || !(sn.L == sn.L)) return false;
        const double rel = fmax(fabs(n0 - c0) / fmax(fabs(n0), 1e-300), fabs(n1 - c1) / fmax(fabs(n1), 1e-300));
        c0 = n0;
        c1 = n1;
        s = sn;
        loss = s.L / s.n;
        if (rel < 1e-12 || (endgame && rel < 1e-9 && it > 60)) return true;
    }
    return false;
}

// validity, clipping and the covariate are resolved once: xs / ts are n doubles of scratch each
template <class R, class V>
PDQ_HD void trend_prepare(R& red, const double* x, const double* t, size_t n, bool x_is_mean, double lo, double hi, const V& xs,
                          const V& ts) {
    for (size_t i = red.tid(), k = 0; i < n; i += red.nthreads(), ++k) {
        const double xv = x_is_mean ? 1.0 / x[i] : x[i];
        double tv = t[i];
        tv = (tv < lo) ? lo : ((tv > hi) ? hi : tv);
        const bool ok = (xv == xv) && (fabs(xv) <= 1.7976931348623157e308);  // drop inf / NaN covariates (dds.py:1225-1232)
        at(xs, i, k) = xv;
        at(ts, i, k) = ok ? tv : (0.0 / 0.0);
    }
    // no barrier: xs[i] / ts[i] are owned by the thread that writes them here -- every later pass of the fit (trend_sums, the
    // drop loop, the `used` count) visits i = tid, tid + nthreads, ... with the same map, so each thread reads only its own writes
}

// Full outer loop of dds.py:1199-1275 on the prepared vectors; ts[i] is set to NaN when gene i is dropped.  With
// `reduce_used` false, n_used is this thread's share of the count: the caller packs it into its next reduction.
template <class R, class VX, class VT>
PDQ_HD TrendOut trend_fit_outer(R& red, const VX& xs, const VT& ts, size_t n, bool outer, bool reduce_used = true) {
    double o0 = 0.1, o1 = 0.1, c0 = 1.0, c1 = 1.0, loss = 0.0;
    int rounds = 0, iters = 0;
    bool failed = false, last_conv = false;
    for (;;) {
        const double l0 = log(fabs(c0 / o0)), l1 = log(fabs(c1 / o1));
        if (!(c0 > 1e-10 && c1 > 1e-10) || !(l0 * l0 + l1 * l1 >= 1e-6)) break;  // dds.py:1236-1238
        o0 = c0;
        o1 = c1;
        const bool conv = trend_fit_once(red, xs, ts, n, c0, c1, loss, iters);
        ++rounds;
        last_conv = conv;
        if (!conv || c0 <= 1e-10 || c1 <= 1e-10) {  // dds.py:1243-1252 -> mean trend
            failed = true;
            break;
        }
        if (!outer) break;
        // drop genes far from the curve before refitting (dds.py:1255-1265)
        for (size_t i = red.tid(), k = 0; i < n; i += red.nthreads(), ++k) {
            const double tv = at(ts, i, k);
            if (!(tv == tv)) continue;
            const double ratio = tv / fma(c1, at(xs, i, k), c0);
            if (ratio < 1e-4 || ratio >= 15.0) at(ts, i, k) = 0.0 / 0.0;
        }
        // no barrier: ts[i] stays owned by its thread (see trend_prepare)
    }
    double used = 0.0;
    for (size_t i = red.tid(), k = 0; i < n; i += red.nthreads(), ++k) used += (at(ts, i, k) == at(ts, i, k)) ? 1.0 : 0.0;
    if (reduce_used) red.sum_many(&used, 1);
    TrendOut o;  // identical in every thread (all decisions were taken on block/cluster-wide sums), n_used aside (see above)
    o.c0 = c0;
    o.c1 = c1;
    o.status = failed ? 1.0 : 0.0;
    o.n_outer = (double)rounds;
    o.n_used = used;
    o.n_iter = (double)iters;
    o.loss = loss;
    o.last_converged = last_conv ? 1.0 : 0.0;
    o.squared_logres = o.prior_var = o.n_above = 0.0 / 0.0;
    for (int i = 0; i < 5; ++i) o.pad[i] = 0.0;
    return o;
}

// ---------------------------------------------------------------------------------------------------------
// Dispersion prior (dds.py:840-884): residuals r = log(genewise) - log(fitted) over the genes with
// genewise >= 100 * min_disp, squared scaled MAD (utils.py:1210-1227), prior_var = max(sq - trigamma((N-p)/2), 0.25).
// The two medians are exact order statistics found by an MSB-first radix select (8-bit digits, 256-bin histogram
// in block-shared memory) over an order-preserving integer image of the doubles; every block of the cluster runs
// the selection redundantly on the full vector (no cross-block traffic, identical results everywhere).
// ---------------------------------------------------------------------------------------------------------
PDQ_HD uint64_t f64_key(double v) {
    uint64_t u;
#if defined(__CUDA_ARCH__)
    u = (uint64_t)__double_as_longlong(v);
#else
    memcpy(&u, &v, 8);
#endif
    return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}
PDQ_HD double f64_from_key(uint64_t k) {
    const uint64_t u = (k >> 63) ? (k & 0x7fffffffffffffffull) : ~k;
#if defined(__CUDA_ARCH__)
    return __longlong_as_double((long long)u);
#else
    double v;
    memcpy(&v, &u, 8);
    return v;
#endif
}

// k-th smallest (0-based) of { |res[i] - center| or res[i] } over the non-NaN entries.  The blocks of the cluster
// histogram disjoint slices of the vector and merge their 256-bin histograms (reducer hist_* hooks); `hist` holds
// 256 local bins + 256 merged bins + 2 result slots.
template <class R, class V>
PDQ_HD double select_kth(R& red, const V& res, size_t n, bool absdev, double center, unsigned* hist, size_t k) {
    uint64_t prefix = 0, mask = 0;
    for (int shift = 56; shift >= 0; shift -= 8) {
        for (int b = red.local_tid(); b < 512; b += red.local_nthreads()) hist[b] = 0;
        red.hist_begin();
        for (size_t i = red.tid(), j = 0; i < n; i += red.nthreads(), ++j) {
            const double r = at(res, i, j);
            if (!(r == r)) continue;
            const uint64_t key = f64_key(absdev ? fabs(r - center) : r);
            if ((key & mask) == prefix) {
#if defined(__CUDA_ARCH__)
                atomicAdd(&hist[(key >> shift) & 0xff], 1u);
#else
                ++hist[(key >> shift) & 0xff];
#endif
            }
        }
        unsigned* tot = red.hist_merge(hist);  // totals over the cluster, identical in every block
        size_t cum = 0;
        int d = 0;
        red.find_bin(tot, hist + 512, k, d, cum);  // first bin whose cumulative count exceeds k, and the count before it
        k -= cum;
        prefix |= (uint64_t)d << shift;
        mask |= (uint64_t)0xff << shift;
        red.local_sync();
    }
    return f64_from_key(prefix);
}

template <class R, class V>
PDQ_HD double median_of(R& red, const V& res, size_t n, size_t cnt, bool absdev, double center, unsigned* hist) {
    if (cnt == 0) return 0.0 / 0.0;  // np.median([]) = nan
    const size_t k = cnt / 2;
    const double hi = select_kth(red, res, n, absdev, center, hist, k);  // upper median
    if (cnt & 1) return hi;
    // even count: the lower median is the largest value below `hi`, unless `hi` is duplicated down to rank k-1.  The running
    // maximum starts at -inf, not at the lowest finite double: held-out size factors take medians of log ratios that hold -inf
    // (a zero count in a gene of the fit), and a lower median of -inf must stay -inf, as in np.median
    double less = 0.0, mx = -HUGE_VAL;
    for (size_t i = red.tid(), j = 0; i < n; i += red.nthreads(), ++j) {
        const double r = at(res, i, j);
        if (!(r == r)) continue;
        const double v = absdev ? fabs(r - center) : r;
        if (v < hi) {
            less += 1.0;
            mx = v > mx ? v : mx;
        }
    }
    red.sum_many(&less, 1);
    mx = red.max_one(mx);
    const double lo = ((size_t)less >= k) ? mx : hi;
    return 0.5 * (lo + hi);
}

// Size-factor estimators (`kind` of pdq_size_factors_ex): median of ratios (preprocessing.py:31-102) and DESeq2's "poscounts"
// (dds.py:656-679)
enum { kSfRatio = 0, kSfPoscounts = 1 };

// One sample's term of a gene's log mean over ALL samples: log(count), -inf for a zero (ratio: the gene is then left out,
// preprocessing.py:52-54), or for poscounts the log of a positive count and 0 for a zero (dds.py:658-660)
PDQ_HD double log_mean_term(int64_t y, int kind) { return (kind == kSfPoscounts && y == 0) ? 0.0 : log((double)y); }

// The log mean a gene enters the medians with, or NaN when it is left out: not a control gene, a non-finite log mean, or for
// poscounts a log mean not above 0 -- every positive count 1, or an all-zero gene (dds.py:663-664, 696)
PDQ_HD double kept_logmean(double lm, int kind, bool control) {
    const bool keep = control && fabs(lm) <= 1.7976931348623157e308 && (kind != kSfPoscounts || lm > 0.0);
    return keep ? lm : (0.0 / 0.0);
}

// One entry of a sample's median of ratios (preprocessing.py:52-54, 89-97): log(count) - log mean of the gene, or NaN -- left out of
// the median -- for a gene whose log mean is not finite (~np.isinf(logmeans), or NaN from kept_logmean).  A zero count in a kept
// gene gives -inf, which takes part in the median as in numpy, unless `skip_zero` (poscounts: only positive counts enter,
// dds.py:668-669).  `keep` says whether the entry counts.
PDQ_HD double log_ratio_entry(int64_t y, double logmean, bool& keep, bool skip_zero = false) {
    keep = fabs(logmean) <= 1.7976931348623157e308 && !(skip_zero && y == 0);
    return keep ? log((double)y) - logmean : (0.0 / 0.0);
}

// Log residual of gene i against the fitted trend, or NaN when the gene is not part of the prior
PDQ_HD double prior_residual(const double* means, const double* t, size_t i, double c0, double c1, double lo, double hi,
                             double min_disp) {
    double tv = t[i];
    tv = (tv < lo) ? lo : ((tv > hi) ? hi : tv);
    const double fit = c0 + c1 / means[i];
    const bool use = (tv >= 100.0 * min_disp) && (means[i] == means[i]);
    return use ? (log(tv) - log(fit)) : (0.0 / 0.0);
}

PDQ_HD void prior_finish(double mad, double trigamma_c, double cnt, TrendOut& out) {
    const double sq = mad * mad;
    out.squared_logres = sq;
    const double pv = sq - trigamma_c;
    out.prior_var = (pv > 0.25 || pv != pv) ? pv : 0.25;  // np.maximum propagates NaN
    out.n_above = cnt;
}

// `res` : n doubles of scratch; `hist`: 514 unsigned in block-shared memory (see select_kth); `trigamma_c` = polygamma(1, (N-p)/2)
template <class R>
PDQ_HD void trend_prior(R& red, const double* means, const double* t, size_t n, double lo, double hi, double min_disp,
                        double trigamma_c, double* res, unsigned* hist, TrendOut& out) {
    const double c0 = out.c0, c1 = out.c1;
    double cnt = 0.0;
    // every thread fills (and later only ever reads) its own stride of the scratch vector: no barrier needed
    for (size_t i = red.tid(); i < n; i += red.nthreads()) {
        res[i] = prior_residual(means, t, i, c0, c1, lo, hi, min_disp);
        cnt += (res[i] == res[i]) ? 1.0 : 0.0;
    }
    red.sum_many(&cnt, 1);
    const size_t m = (size_t)cnt;
    const double med = median_of(red, res, n, m, false, 0.0, hist);
    const double mad = median_of(red, res, n, m, true, med, hist) * 1.4826022185056018;  // / (sqrt(2) erfinv(1/2))
    prior_finish(mad, trigamma_c, cnt, out);
}

#if defined(__CUDACC__)
// ---------------------------------------------------------------------------------------------------------
// The prior's medians on the device in a fixed number of cluster- / grid-wide rounds, whatever the key width:
//   1. the value range [vlo, vhi] comes with the count of prior genes (one packed sum + max reduction);
//   2. each block counts its slice into kVBins equal-width value bins -- bin(v) = clamp(floor((v - vlo) * scale)) is monotone
//      non-decreasing in v, so the k-th smallest value lies in the first bin b whose running count exceeds k -- and the blocks
//      merge their histograms in one round;
//   3. the values of bin b (their order-preserving keys) go to a global candidate buffer in one round; the same round brings
//      the largest value below bin b, which is the lower median of an even count when rank k opens bin b;
//   4. every block picks the exact ranks among the candidates with block-local barriers only.
// Too many candidates (heavy ties: genes clipped to max_disp), or a range of zero or non-finite width, fall back to the exact
// 8-digit radix walk of median_of.  Both give the exact order statistics, so the result does not depend on the path.
// Reducer hooks: sum_many(v, k, kmax) (the last kmax entries are maxima), vhist_merge(hist, slot), cand_index(slot),
// max_key(key) (integer maximum of 64-bit keys).
// ---------------------------------------------------------------------------------------------------------
constexpr int kVBins = 2048;
constexpr int kCandCap = 1024;

struct SelShared {                       // block-shared memory of median_bins
    unsigned hist[kVBins];               // the block's bins, then the merged bins
    unsigned long long keys[kCandCap];   // candidate keys of the chosen bin
    unsigned warp_sum[32];
    unsigned bin[3];                     // chosen bin, count before it, count in it
    unsigned long long pick[2];          // keys at the upper and lower rank
};

__device__ __forceinline__ int vbin(double v, double vlo, double scale) {
    const double x = (v - vlo) * scale;
    return x <= 0.0 ? 0 : (x >= (double)(kVBins - 1) ? kVBins - 1 : (int)x);
}

// first bin of `hist` whose running count exceeds k -> sh.bin = {bin, count before it, count in it}, visible to the block
__device__ inline void find_vbin(SelShared& sh, size_t k) {
    const int per = kVBins / blockDim.x, b0 = threadIdx.x * per;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned tot = 0;
    for (int j = 0; j < per; ++j) tot += sh.hist[b0 + j];
    unsigned inc = tot;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        const unsigned u = __shfl_up_sync(0xffffffffu, inc, off);
        if (lane >= off) inc += u;
    }
    if (lane == 31) sh.warp_sum[warp] = inc;
    __syncthreads();
    unsigned before = inc - tot;
    for (int w = 0; w < warp; ++w) before += sh.warp_sum[w];
    const unsigned kk = (unsigned)k;
    if (before <= kk && kk < before + tot) {  // exactly one thread owns the crossing
        unsigned run = before;
        int j = 0;
        for (; j < per; ++j) {
            if (run + sh.hist[b0 + j] > kk) break;
            run += sh.hist[b0 + j];
        }
        sh.bin[0] = (unsigned)(b0 + j);
        sh.bin[1] = run;
        sh.bin[2] = sh.hist[b0 + j];
    }
    __syncthreads();
}

// k-th smallest of { |res[i] - center| or res[i] } (0-based) over the non-NaN entries; when `lower`, also rank k - 1.  Returns
// the exact values, as median_of.  [vlo, vhi] bounds the values.  `cand`: kCandCap keys of global scratch no thread reads
// or writes meanwhile.  `slot` (0, 1) picks the reducer's merge buffers: the two medians of one launch use different slots.
template <class R, class V>
__device__ double median_bins(R& red, const V& res, size_t n, size_t cnt, bool absdev, double center, double vlo,
                              double vhi, int slot, unsigned long long* cand, SelShared& sh, unsigned* hist514) {
    if (cnt == 0) return 0.0 / 0.0;  // np.median([]) = nan
    const double width = vhi - vlo, scale = (double)kVBins / width;
    if (!(width > 0.0 && width <= 1.7976931348623157e308 && scale <= 1.7976931348623157e308))
        return median_of(red, res, n, cnt, absdev, center, hist514);  // equal values, or infinite ones
    const size_t k = cnt / 2;
    const bool even = !(cnt & 1);
    for (int b = threadIdx.x; b < kVBins; b += blockDim.x) sh.hist[b] = 0;
    __syncthreads();
    for (size_t i = red.tid(), j = 0; i < n; i += red.nthreads(), ++j) {
        const double r = at(res, i, j);
        if (!(r == r)) continue;
        atomicAdd(&sh.hist[vbin(absdev ? fabs(r - center) : r, vlo, scale)], 1u);
    }
    red.vhist_merge(sh.hist, slot);  // one round: sh.hist holds the totals, identical in every block
    find_vbin(sh, k);
    const int b = (int)sh.bin[0];
    const unsigned before = sh.bin[1], inbin = sh.bin[2];
    if (inbin > (unsigned)kCandCap) return median_of(red, res, n, cnt, absdev, center, hist514);
    const unsigned r_hi = (unsigned)k - before;
    const bool below = even && r_hi == 0;  // rank k - 1 is the largest value of the bins below b
    unsigned long long mx = 0ull;          // below every key of a non-NaN double
    for (size_t i = red.tid(), j = 0; i < n; i += red.nthreads(), ++j) {
        const double r = at(res, i, j);
        if (!(r == r)) continue;
        const double v = absdev ? fabs(r - center) : r;
        const int bi = vbin(v, vlo, scale);
        if (bi == b) {
            cand[red.cand_index(slot)] = f64_key(v);
        } else if (below && bi < b) {
            const unsigned long long key = f64_key(v);
            mx = key > mx ? key : mx;
        }
    }
    // one round: the candidates are written and visible, and every block learns the largest key below bin b.  The keys are
    // reduced as integers: key 0 (a thread that saw nothing below b) is below every key of a non-NaN double
    mx = red.max_key(mx);
    for (unsigned j = threadIdx.x; j < inbin; j += blockDim.x) sh.keys[j] = __ldcg(cand + j);
    __syncthreads();
    // exact ranks among the candidates: a key is at rank r when (#smaller) <= r < (#smaller) + (#equal)
    const bool lower_in_bin = even && !below;
    for (unsigned i = threadIdx.x; i < inbin; i += blockDim.x) {
        const unsigned long long key = sh.keys[i];
        unsigned less = 0, eq = 0;
        for (unsigned j = 0; j < inbin; ++j) {
            const unsigned long long o = sh.keys[j];
            less += o < key;
            eq += o == key;
        }
        if (less <= r_hi && r_hi < less + eq) sh.pick[0] = key;  // equal keys write equal values
        if (lower_in_bin && less <= r_hi - 1 && r_hi - 1 < less + eq) sh.pick[1] = key;
    }
    __syncthreads();
    const double hi = f64_from_key(sh.pick[0]);
    const double lo = !even ? hi : f64_from_key(below ? mx : sh.pick[1]);
    __syncthreads();  // sh is reused by the next selection
    return even ? 0.5 * (lo + hi) : hi;
}

// trend_prior on the device: the count of prior genes, the fit's `used` count (this thread's share in out.n_used, see
// trend_fit_outer) and the residuals' range share one reduction; the two medians run through median_bins.
template <class R, class V>
__device__ void trend_prior_dev(R& red, const double* means, const double* t, size_t n, double lo, double hi, double min_disp,
                                double trigamma_c, const V& res, unsigned long long* cand, SelShared& sh, unsigned* hist514,
                                TrendOut& out) {
    const double c0 = out.c0, c1 = out.c1;
    double v[4] = {0.0, out.n_used, -HUGE_VAL, -HUGE_VAL};  // count, used, max, -min
    for (size_t i = red.tid(), k = 0; i < n; i += red.nthreads(), ++k) {
        const double r = prior_residual(means, t, i, c0, c1, lo, hi, min_disp);
        at(res, i, k) = r;  // each thread later reads only its own stride of res: no barrier needed
        if (!(r == r)) continue;
        v[0] += 1.0;
        v[2] = fmax(v[2], r);
        v[3] = fmax(v[3], -r);
    }
    red.sum_many(v, 4, 2);
    out.n_used = v[1];
    const size_t m = (size_t)v[0];
    const double rmax = v[2], rmin = -v[3];
    const double med = median_bins(red, res, n, m, false, 0.0, rmin, rmax, 0, cand, sh, hist514);
    // |r - med| is largest at an end of the range (r - med is monotone in r); the smallest deviation is >= 0
    const double dmax = fmax(fabs(rmax - med), fabs(rmin - med));
    const double mad = median_bins(red, res, n, m, true, med, 0.0, dmax, 1, cand, sh, hist514) * 1.4826022185056018;
    prior_finish(mad, trigamma_c, v[0], out);
}
#endif

}  // namespace pdq
