// pdq_gene.cuh -- the per-gene routines of the hot path, one cooperative lane-group per gene.
//
// Work decomposition (DESIGN.md §3): a group of T = 1,2,4,...,32 lanes of one warp owns one gene;
// lane `si` of the group walks samples si, si+T, si+2T, ... so that, with 32/T adjacent genes per warp,
// every warp-wide load of the (N, G) sample-major arrays touches T rows x (32/T) contiguous genes.
// Per-gene sums (X^T W X, X^T W z, deviance, score terms) are butterfly-reduced across the group
// with warp shuffles; after the butterfly every lane of the group holds bit-identical totals, so the
// p x p Cholesky work and all control flow are replicated per lane without further communication.
//
// The same source is compiled for the device and for the host emulator (Group::sum is the identity
// there, T = 1), see pdq_math.cuh.
#pragma once

#include "pdq_fast.cuh"
#include "pdq_host_linalg.h"
#include "pdq_math.cuh"

#ifndef PDQ_PREFETCH
#define PDQ_PREFETCH 1
#endif
#ifndef PDQ_IRLS_UNROLL
#define PDQ_IRLS_UNROLL 2
#endif

#if defined(PDQ_EMU_LANES) && !defined(__CUDA_ARCH__)
// host emulator with T > 1 "lanes" (one std::thread each, tests/emu/pdq_emu.cpp): the same exchange patterns as the shuffles
namespace pdq_emu {
double lane_sum(int si, int T, double v);
double lane_excl_scan(int si, int T, double v);
bool lane_any(int si, int T, bool p);
void lane_sync(int T);
void lane_argmax(int si, int T, double& best, int& best_n, double& best_use);  // the butterfly of cooks_gene
int lane_argext(int si, int T, double v, bool want_max);                       // lane holding the group's min / max
}  // namespace pdq_emu
#endif

namespace pdq {

struct Group {
    int si;   // this lane's first sample
    int T;    // lanes per gene (sample stride)
    int gpw;  // genes per warp = 32 / T
    // exclusive prefix sum over the lanes of this gene ordered by si (host: single lane -> 0)
    PDQ_HD double excl_scan(double v) const {
#if defined(__CUDA_ARCH__)
        const int lane = threadIdx.x & 31;
        double inc = v;
        for (int off = gpw; off < 32; off <<= 1) {
            const double t = __shfl_up_sync(0xffffffffu, inc, off);
            if (lane >= off) inc += t;
        }
        return inc - v;
#elif defined(PDQ_EMU_LANES)
        return pdq_emu::lane_excl_scan(si, T, v);
#else
        (void)v;
        return 0.0;
#endif
    }
    PDQ_HD void sync() const {
#if defined(__CUDA_ARCH__)
        __syncwarp();
#elif defined(PDQ_EMU_LANES)
        pdq_emu::lane_sync(T);
#endif
    }
    PDQ_HD double sum(double v) const {
#if defined(__CUDA_ARCH__)
        for (int off = 16; off >= gpw; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
#elif defined(PDQ_EMU_LANES)
        v = pdq_emu::lane_sum(si, T, v);
#endif
        return v;
    }
    // lane index (si) of the group's smallest (largest) v, ties to the smaller si; identical in every lane of the group
    PDQ_HD int argext(double v, bool want_max) const {
#if defined(__CUDA_ARCH__)
        int who = si;
        for (int off = 16; off >= gpw; off >>= 1) {
            const double ov = __shfl_xor_sync(0xffffffffu, v, off);
            const int ow = __shfl_xor_sync(0xffffffffu, who, off);
            const bool better = want_max ? (ov > v) : (ov < v);
            if (better || (ov == v && ow < who)) {
                v = ov;
                who = ow;
            }
        }
        return who;
#elif defined(PDQ_EMU_LANES)
        return pdq_emu::lane_argext(si, T, v, want_max);
#else
        (void)v;
        (void)want_max;
        return 0;
#endif
    }
    // on the device a vote over the whole WARP (every gene of it), not just this group: a superset of the group's vote, so
    // the branches and loop exits it guards stay warp-uniform, as the full-mask shuffles inside them require (each gene masks
    // the extra work with its own flags).  The emulator runs one gene at a time and votes over its lanes.
    PDQ_HD bool any(bool p) const {
#if defined(__CUDA_ARCH__)
        return __any_sync(0xffffffffu, p) != 0;
#elif defined(PDQ_EMU_LANES)
        return pdq_emu::lane_any(si, T, p);
#else
        return p;
#endif
    }
};

// staged design pack (shared memory on the device; layout: design_pack): `sf` / `lsf` = X + p / X + p + 1, indexed [n * RS]
struct DesignS {
    const double* X;
    const double* sf;
    const double* lsf;
    int N;
    int RS;
    const double* mtab = nullptr;  // kMathTab of the table-driven log / exp (shared memory; set by the kernels that use it)
};

template <int P>
struct SmallMat {
    double v[P * P];
};

// A lane's walk over its samples n = si, si + T, ... of one (N, G) column, `p` pointing at the first of them and `step` = T * ld:
// four loads are issued before the first is used, so that a streaming pass keeps several requests in flight per lane (a
// one-load-per-trip walk is bound by the memory latency, not the bandwidth).  `f(n, value)` is called in increasing n.
template <class V, class F>
PDQ_HD void walk4(const Group& grp, int N, const V* p, int64_t step, F&& f) {
    int n = grp.si;
    const int T = grp.T;
    for (; n + 3 * T < N; n += 4 * T, p += 4 * step) {
        const V v0 = p[0], v1 = p[step], v2 = p[2 * step], v3 = p[3 * step];
        f(n, v0);
        f(n + T, v1);
        f(n + 2 * T, v2);
        f(n + 3 * T, v3);
    }
    for (; n < N; n += T, p += step) f(n, *p);
}

template <int P>
PDQ_HD void load_x(const DesignS& d, int n, double (&x)[P]) {
PDQ_UNROLL_P
    for (int j = 0; j < P; ++j) x[j] = d.X[n * design_row_stride(P) + j];
}

template <int P>
PDQ_HD void group_sum_sym(const Group& g, Sym<P>& s) {
PDQ_UNROLL_P
    for (int k = 0; k < P * (P + 1) / 2; ++k) s.a[k] = g.sum(s.a[k]);
}

template <int P>
PDQ_HD void group_sum_vec(const Group& g, double (&v)[P]) {
PDQ_UNROLL_P
    for (int k = 0; k < P; ++k) v[k] = g.sum(v[k]);
}

// =============================================================================================
// (a4) lin_reg_mu -- utils.py:682-715.  OLS of counts/sf on X, mu = max(sf * X beta, min_mu).
// `pinv` = (X^T X)^+ (host, from the SVD of X) so beta = pinv X^T (y / sf) is the least-squares
// (minimum-norm if rank deficient) solution sklearn's LinearRegression returns.
// =============================================================================================
template <int P>
PDQ_HD void linmu_gene(const Group& grp, const DesignS& d, const SmallMat<P>& pinv, const int64_t* y,
                       int64_t ld, double min_mu, double* mu_out, int64_t ld_out, bool valid) {
    double v[P];
PDQ_UNROLL_P
    for (int j = 0; j < P; ++j) v[j] = 0.0;
    walk4(grp, d.N, y + (int64_t)grp.si * ld, (int64_t)grp.T * ld, [&](int n, int64_t c) {
        double x[P];
        load_x<P>(d, n, x);
        const double t = (double)c / d.sf[n * d.RS];
PDQ_UNROLL_P
        for (int j = 0; j < P; ++j) v[j] = fma(x[j], t, v[j]);
    });
    group_sum_vec<P>(grp, v);
    double beta[P];
PDQ_UNROLL_P
    for (int i = 0; i < P; ++i) {
        double s = 0.0;
PDQ_UNROLL_P
        for (int j = 0; j < P; ++j) s = fma(pinv.v[i * P + j], v[j], s);
        beta[i] = s;
    }
    if (!valid) return;
    for (int n = grp.si; n < d.N; n += grp.T) {
        double x[P];
        load_x<P>(d, n, x);
        double e = 0.0;
PDQ_UNROLL_P
        for (int j = 0; j < P; ++j) e = fma(x[j], beta[j], e);
        const double m = d.sf[n * d.RS] * e;
        mu_out[n * ld_out] = (m < min_mu) ? min_mu : m;  // np.maximum (NaN propagates)
    }
}

// ---------------------------------------------------------------------------------------------
// Small-count tables shared by irls (lgamma) and alpha_mle (digamma): per gene, f(r + k) for k < kPsiK is built from
// f(r) by the recurrence (one log / reciprocal per entry, split over the gene's lanes and stitched with an exclusive
// scan); counts below kPsiK then cost one shared-memory read, and larger counts always satisfy the z >= 10
// precondition of the unshifted Stirling series.
// Accuracy (tests/test_gpu_math.py on an H100, tests/test_math_ref.py on the host; r in [1e-4, 1e8], every T in 1..32): each
// entry is within 0.07 (lgamma), 0.03 (psi) and 0.14 (psi') of the forward-error bound of its recurrence, start error +
// 4 eps (k + 1) (|f(r)| + sum_{j<k} |term_j|).  The largest absolute error, 3e-8 in psi' at r = 1e-4, is that conditioning:
// psi'(1e-4) ~ 1e8.
// ---------------------------------------------------------------------------------------------
constexpr int kPsiK = 32;

// log(k!) for k < kPsiK
PDQ_CONST double kLogFact[kPsiK] = {0.0, 0.0, 0.693147180559945, 1.7917594692280554, 3.178053830347945, 4.787491742782047, 6.579251212010102, 8.525161361065415, 10.604602902745249, 12.801827480081467, 15.104412573075514, 17.502307845873887, 19.987214495661885, 22.55216385312342, 25.191221182738683, 27.89927138384089, 30.671860106080672, 33.50507345013689, 36.39544520803305, 39.339884187199495, 42.335616460753485, 45.38013889847691, 48.47118135183522, 51.60667556776438, 54.78472939811232, 58.00360522298052, 61.26170176100201, 64.55753862700634, 67.88974313718153, 71.257038967168, 74.65823634883017, 78.0922235533153};

PDQ_HD void build_lgamma_table(const Group& grp, double* tab, double r, const double* mtab) {
    const int seg = kPsiK / grp.T;  // T in {1,...,32} divides 32
    const int k0 = grp.si * seg;
    double part = 0.0;
    for (int k = k0; k < k0 + seg; ++k) {
        const double lg = tlog(r + (double)k, mtab);
        tab[k] = lg;
        part += lg;
    }
    double run = lgamma_pos(r) + grp.excl_scan(part);
    for (int k = k0; k < k0 + seg; ++k) {
        const double lg = tab[k];
        tab[k] = run;  // lgamma(r + k) = lgamma(r) + sum_{j<k} log(r + j)
        run += lg;
    }
    grp.sync();
}

// =============================================================================================
// (a3) wald_test -- utils.py:718-811.
// =============================================================================================
template <int P>
struct WaldParams {
    double ridge[P * P];
    double contrast[P];
    double lfc_null;
    int alt;
};

// H = (M + ridge)^-1 for M = X^T W X (W from the caller's mu); `ridge` p x p row-major
template <int P>
PDQ_HD void wald_inverse(const Sym<P>& M, const double* ridge, Sym<P>& H) {
    Sym<P> L = M;
PDQ_UNROLL_P
    for (int i = 0; i < P; ++i)
PDQ_UNROLL_P
        for (int j = 0; j <= i; ++j) L.a[tri(i, j)] += ridge[i * P + j];
    chol<P>(L);
    chol_inverse<P>(L, H);
}

// one contrast against that factor: SE = sqrt(c' H M H c), the statistic and the p-value of alternative `alt` (PDQ_ALT_*)
template <int P>
PDQ_HD void wald_contrast(const Sym<P>& M, const Sym<P>& H, const double (&contrast)[P], double lfc_null, int alt, const double* lfc,
                          double& pv, double& stat, double& se) {
    double Hc[P], MHc[P];
    sym_matvec<P>(H, contrast, Hc);
    sym_matvec<P>(M, Hc, MHc);
    double q = 0.0;
PDQ_UNROLL_P
    for (int j = 0; j < P; ++j) q = fma(Hc[j], MHc[j], q);
    se = sqrt(q);
    double b[P];
PDQ_UNROLL_P
    for (int j = 0; j < P; ++j) b[j] = lfc[j];
    const double t0 = lfc_null;
    // each variant applies the elementwise transform to every coefficient, then dots with the contrast
    auto greater = [&](double t, double& s, double& p) {
        s = 0.0;
PDQ_UNROLL_P
        for (int j = 0; j < P; ++j) s = fma(contrast[j], fmax((b[j] - t) / se, 0.0), s);
        p = norm_sf(s);
    };
    auto less = [&](double t, double& s, double& p) {
        s = 0.0;
PDQ_UNROLL_P
        for (int j = 0; j < P; ++j) s = fma(contrast[j], fmin((b[j] - t) / se, 0.0), s);
        p = norm_sf(fabs(s));
    };
    if (alt == 0) {
        double s = 0.0;
PDQ_UNROLL_P
        for (int j = 0; j < P; ++j) s = fma(contrast[j], b[j] - t0, s);
        stat = s / se;
        pv = 2.0 * norm_sf(fabs(stat));
    } else if (alt == 1) {  // greaterAbs
        double s = 0.0;
PDQ_UNROLL_P
        for (int j = 0; j < P; ++j) s = fma(contrast[j], sgn(b[j]) * fmax((fabs(b[j]) - t0) / se, 0.0), s);
        stat = s;
        pv = 2.0 * norm_sf(fabs(s));
    } else if (alt == 2) {  // lessAbs
        double sa, pa, sb, pb;
        greater(-fabs(t0), sa, pa);
        less(fabs(t0), sb, pb);
        stat = (fabs(sb) < fabs(sa)) ? sb : sa;  // min(sa, sb, key=abs): first wins ties
        pv = (pb > pa) ? pb : pa;                // max(pa, pb)
    } else if (alt == 3) {
        greater(t0, stat, pv);
    } else {
        less(t0, stat, pv);
    }
}

// the per-gene algebra once M = X^T W X is known: H = (M + ridge)^-1, then the one contrast of `prm`
template <int P>
PDQ_HD void wald_finish(const Group& grp, const Sym<P>& M, const WaldParams<P>& prm, const double* lfc, double* p_out,
                        double* stat_out, double* se_out, bool valid) {
    Sym<P> H;
    wald_inverse<P>(M, prm.ridge, H);
    double pv, stat, se;
    wald_contrast<P>(M, H, prm.contrast, prm.lfc_null, prm.alt, lfc, pv, stat, se);
    if (valid && grp.si == 0) {
        *p_out = pv;
        *stat_out = stat;
        *se_out = se;
    }
}

template <int P>
PDQ_HD void wald_gene(const Group& grp, const DesignS& d, const WaldParams<P>& prm, double disp, const double* lfc,
                      const double* mu, int64_t ld_mu, double* p_out, double* stat_out, double* se_out, bool valid) {
    Sym<P> M;
    sym_zero<P>(M);
    walk4(grp, d.N, mu + (int64_t)grp.si * ld_mu, (int64_t)grp.T * ld_mu, [&](int n, double m) {
        double x[P];
        load_x<P>(d, n, x);
        sym_rank1<P>(M, m / fma(m, disp, 1.0), x);
    });
    group_sum_sym<P>(grp, M);
    wald_finish<P>(grp, M, prm, lfc, p_out, stat_out, se_out, valid);
}

// Wald tests of K contrasts from fitted coefficients (ds.py:303-360 once per contrast).  mu = sf * exp(x'beta) is built per
// sample -- the reference's exp(X @ LFC.T) * sf, as k_mu_from_lfc writes it -- so no (N, G) array is read; X^T W X is summed over
// the group and factored ONCE.  M and H are then replicated in every lane, so lane si evaluates contrasts si, si + T, ...: K
// contrasts cost ceil(K / T) rounds instead of K.  `tab` (K, P + 2) row-major: contrast, lfc_null, alt.  Outputs (K, ld_out).
template <int P>
PDQ_HD void wald_contrasts_gene(const Group& grp, const DesignS& d, const double* ridge, double disp, const double* lfc, int K,
                                const double* tab, double* p_out, double* stat_out, double* se_out, int64_t ld_out, bool valid) {
    double b[P];
PDQ_UNROLL_P
    for (int j = 0; j < P; ++j) b[j] = lfc[j];
    Sym<P> M;
    sym_zero<P>(M);
    for (int n = grp.si; n < d.N; n += grp.T) {
        double x[P];
        load_x<P>(d, n, x);
        double eta = 0.0;
PDQ_UNROLL_P
        for (int j = 0; j < P; ++j) eta = fma(x[j], b[j], eta);
        const double m = d.sf[n * d.RS] * exp(eta);
        sym_rank1<P>(M, m / fma(m, disp, 1.0), x);
    }
    group_sum_sym<P>(grp, M);
    Sym<P> H;
    wald_inverse<P>(M, ridge, H);
    // Every lane runs the same ceil(K / T) rounds and skips its slot when it has no contrast there.  A per-lane trip count
    // (k = si; k < K; k += T) gave wrong results from the second round on in the wide units (p = 9..16, ptxas -O1) on an H100.
    for (int k0 = 0; k0 < K; k0 += grp.T) {
        const int k = k0 + grp.si;
        if (!valid || k >= K) continue;
        const double* row = tab + (int64_t)k * (P + 2);
        double c[P];
PDQ_UNROLL_P
        for (int j = 0; j < P; ++j) c[j] = row[j];
        double pv, stat, se;
        wald_contrast<P>(M, H, c, row[P], (int)row[P + 1], b, pv, stat, se);
        p_out[k * ld_out] = pv;
        stat_out[k * ld_out] = stat;
        se_out[k * ld_out] = se;
    }
}

// =============================================================================================
// (a1) irls -- utils.py:273-438.
// =============================================================================================
struct IrlsParams {
    double min_mu, beta_tol, min_beta, max_beta;
    int maxiter;
    int full_rank;
    int few_rows;  // the design has few distinct rows (categorical factors): reuse exp(x'beta) while the row repeats
    int fail_optimizer;  // test hook (PDQ_DEBUG_FAIL_IRLS_OPTIMIZER): the optimiser branch reports `success = False`
};

// one fused sweep over the gene's samples at coefficient vector `beta`:
//   A = X^T W X, b = X^T W z  (utils.py:368-371, W and z from the CLAMPED mu)
//   S = sum (y + r) log(r + mu) - y log(mu)  -- the mu-dependent part of nb_nll (utils.py:220-234)
// contribution of one sample to the sweep.  NB = branch-free math cores; arguments outside their domain raise `odd`
// MEMO: a lane walks samples si, si+T, ...; with a categorical design consecutive ones usually share their design row, so
// eta = x'beta repeats bit for bit and exp(eta) -- a third of the body's instructions -- is carried over instead of recomputed
// (same value, results unchanged).  All lanes of a warp look at the same rows, so the skip is close to warp-uniform.
template <int P, bool NB, bool MEMO>
PDQ_HD void irls_sample(const double* xp, const double* mtab, double yv, const double (&beta)[P], double alpha,
                        double r, double min_mu, double log_min_mu, Sym<P>& A, double (&b)[P], double& S, bool& odd,
                        double& eta_prev, double& exp_prev) {
    double x[P];
PDQ_UNROLL_P
    for (int j = 0; j < P; ++j) x[j] = xp[j];
    const double sfn = xp[P], lsfn = xp[P + 1];                      // sf and log sf close the design row
    double eta = 0.0;
PDQ_UNROLL_P
    for (int j = 0; j < P; ++j) eta = fma(x[j], beta[j], eta);
    double ex;
    if (MEMO) {
        if (eta != eta_prev) {
            exp_prev = NB ? texp_nb(eta, mtab) : fast_exp(eta);
            eta_prev = eta;
        }
        ex = exp_prev;
    } else {
        ex = NB ? texp_nb(eta, mtab) : fast_exp(eta);
    }
    const double mu_raw = sfn * ex;
    const bool cl = mu_raw < min_mu;
    const double mu = cl ? min_mu : mu_raw;                            // np.maximum(sf*exp(X b), min_mu)
    const double lmu = cl ? log_min_mu : (eta + lsfn);                 // log(mu)
    const double lmu_sf = lmu - lsfn;                                  // log(mu / sf)
    const double den = fma(mu, alpha, 1.0);
    // W = mu / (1 + mu alpha);  W z = W log(mu/sf) + W (y - mu)/mu = W log(mu/sf) + (y - mu) / (1 + mu alpha)
    const double iden = NB ? fast_rcp(den) : 1.0 / den;
    const double W = mu * iden;
    const double Wz = fma(yv - mu, iden, W * lmu_sf);
    sym_rank1<P>(A, W, x);
PDQ_UNROLL_P
    for (int j = 0; j < P; ++j) b[j] = fma(Wz, x[j], b[j]);
    S += fma(yv + r, NB ? tlog_nb(r + mu, mtab) : fast_log(r + mu), -yv * lmu);
}

template <int P, bool NB, bool MEMO>
PDQ_HD bool irls_sweep_t(const Group& grp, const DesignS& d, const int64_t* y, int64_t ld, const double (&beta)[P],
                         double alpha, double r, double min_mu, double log_min_mu, Sym<P>& A, double (&b)[P], double& S) {
    sym_zero<P>(A);
PDQ_UNROLL_P
    for (int j = 0; j < P; ++j) b[j] = 0.0;
    S = 0.0;
    bool odd = false;
    const int T = grp.T;
    constexpr int RS = design_row_stride(P);
    const int64_t ystep = (int64_t)T * ld;
    const int64_t* yp = y + (int64_t)grp.si * ld;
    const double* xp = d.X + grp.si * RS;
    int n = grp.si;
    // NaN never compares equal: the first sample always computes its exponential
    double eta_prev = __builtin_nan(""), exp_prev = 0.0;
    // two samples per trip, straight-line: their exp / log / reciprocal chains interleave on the FP64 pipe.  The counts of the
    // NEXT trip are requested before this trip's arithmetic starts (register double buffer): the L1/L2 latency of the strided
    // column walk hides behind ~350 instructions instead of stalling the first use (long-scoreboard stalls were 22 %).
#if PDQ_IRLS_UNROLL == 4
    // experiment (default off): four samples per trip -- more independent exp / log / reciprocal chains in flight per lane
    // against the fixed-latency dependency stalls of the capture (DESIGN.md §9.1); costs registers
    for (; n + 3 * T < d.N; n += 4 * T, yp += 4 * ystep, xp += 4 * T * RS) {
        const double y0 = (double)yp[0], y1 = (double)yp[ystep], y2 = (double)yp[2 * ystep], y3 = (double)yp[3 * ystep];
        irls_sample<P, NB, MEMO>(xp, d.mtab, y0, beta, alpha, r, min_mu, log_min_mu, A, b, S, odd, eta_prev, exp_prev);
        irls_sample<P, NB, MEMO>(xp + T * RS, d.mtab, y1, beta, alpha, r, min_mu, log_min_mu, A, b, S, odd, eta_prev, exp_prev);
        irls_sample<P, NB, MEMO>(xp + 2 * T * RS, d.mtab, y2, beta, alpha, r, min_mu, log_min_mu, A, b, S, odd, eta_prev, exp_prev);
        irls_sample<P, NB, MEMO>(xp + 3 * T * RS, d.mtab, y3, beta, alpha, r, min_mu, log_min_mu, A, b, S, odd, eta_prev, exp_prev);
    }
    for (; n + T < d.N; n += 2 * T, yp += 2 * ystep, xp += 2 * T * RS) {
        const double y0 = (double)yp[0], y1 = (double)yp[ystep];
        irls_sample<P, NB, MEMO>(xp, d.mtab, y0, beta, alpha, r, min_mu, log_min_mu, A, b, S, odd, eta_prev, exp_prev);
        irls_sample<P, NB, MEMO>(xp + T * RS, d.mtab, y1, beta, alpha, r, min_mu, log_min_mu, A, b, S, odd, eta_prev, exp_prev);
    }
#elif PDQ_PREFETCH
    int64_t c0 = (n + T < d.N) ? yp[0] : 0, c1 = (n + T < d.N) ? yp[ystep] : 0;
    for (; n + T < d.N; n += 2 * T, yp += 2 * ystep, xp += 2 * T * RS) {
        const double y0 = (double)c0, y1 = (double)c1;
        if (n + 3 * T < d.N) {
            c0 = yp[2 * ystep];
            c1 = yp[3 * ystep];
        }
        irls_sample<P, NB, MEMO>(xp, d.mtab, y0, beta, alpha, r, min_mu, log_min_mu, A, b, S, odd, eta_prev, exp_prev);
        irls_sample<P, NB, MEMO>(xp + T * RS, d.mtab, y1, beta, alpha, r, min_mu, log_min_mu, A, b, S, odd, eta_prev, exp_prev);
    }
#else
    for (; n + T < d.N; n += 2 * T, yp += 2 * ystep, xp += 2 * T * RS) {
        const double y0 = (double)yp[0], y1 = (double)yp[ystep];
        irls_sample<P, NB, MEMO>(xp, d.mtab, y0, beta, alpha, r, min_mu, log_min_mu, A, b, S, odd, eta_prev, exp_prev);
        irls_sample<P, NB, MEMO>(xp + T * RS, d.mtab, y1, beta, alpha, r, min_mu, log_min_mu, A, b, S, odd, eta_prev, exp_prev);
    }
#endif
    if (n < d.N)
        irls_sample<P, NB, MEMO>(xp, d.mtab, (double)yp[0], beta, alpha, r, min_mu, log_min_mu, A, b, S, odd, eta_prev, exp_prev);
    return odd;
}

template <int P>
PDQ_HD void irls_sweep(const Group& grp, const DesignS& d, const int64_t* y, int64_t ld, const double (&beta)[P],
                       double alpha, double r, double min_mu, double log_min_mu, Sym<P>& A, double (&b)[P],
                       double& S, bool few_rows) {
#if defined(PDQ_EMU_COUNT_EVALS) && !defined(__CUDA_ARCH__)
    if (grp.si == 0) ++g_emu_irls_sweeps;  // host emulator instrumentation only
#endif
    // the branch-free cores need r = 1/alpha positive finite, a positive clamp and |x'beta| < 300 for every sample; the last
    // is checked once per sweep through |x'beta| <= sum_j |beta_j| max_n |x_nj| (the column maxima close the design pack)
    bool odd = !(alpha > 0.0 && r > 0.0 && r < 1e300 && min_mu > 0.0);
    {
        double bound = 0.0;
PDQ_UNROLL_P
        for (int j = 0; j < P; ++j) bound = fma(fabs(beta[j]), d.X[d.N * design_row_stride(P) + j], bound);
        odd = odd || !(bound < 300.0);
    }
    if (!odd) {
        odd = few_rows ? irls_sweep_t<P, true, true>(grp, d, y, ld, beta, alpha, r, min_mu, log_min_mu, A, b, S)
                       : irls_sweep_t<P, true, false>(grp, d, y, ld, beta, alpha, r, min_mu, log_min_mu, A, b, S);
    }
    if (grp.any(odd))  // rare (diverging beta, NaN dispersion): guarded libdevice path, IEEE semantics of the reference
        irls_sweep_t<P, false, false>(grp, d, y, ld, beta, alpha, r, min_mu, log_min_mu, A, b, S);
    group_sum_sym<P>(grp, A);
    group_sum_vec<P>(grp, b);
    S = grp.sum(S);
}

// status codes written per gene
constexpr int kIrlsOk = 0;
constexpr int kIrlsNeedsOptimizer = 1;  // left through utils.py:374 (|beta|>max_beta or i>=maxiter)

template <int P>
PDQ_HD void irls_gene(const Group& grp, const DesignS& d, const SmallMat<P>& pinv, const IrlsParams& prm,
                      const int64_t* y, int64_t ld, double alpha, double* beta_out, double* mu_out,
                      double* hat_out, int64_t ld_out, double* conv_out, int* status_out, bool valid, double* lg_tab,
                      const double* logfact, const WaldParams<P>* wald = nullptr, double* wald_p = nullptr,
                      double* wald_stat = nullptr, double* wald_se = nullptr) {
    // wald != nullptr: also the Wald test of this fit (ds.py:303-360 / utils.py:718-811) from the sums of the last sweep -- the
    // caller would otherwise re-read the mu written below (8 N G bytes) just to rebuild X^T W X
    // lg_tab: kPsiK doubles of per-gene scratch (shared memory); logfact: log(k!) table, k < kPsiK (shared memory)
    const double r = 1.0 / alpha;
    const double Nd = (double)d.N;
    const double log_min_mu = log(prm.min_mu);
    const bool tab_ok = (r > 0.0) && (r < 1e300);  // NaN / non-positive dispersion: plain lgamma path, IEEE semantics
    grp.sync();
    if (tab_ok) build_lgamma_table(grp, lg_tab, r, d.mtab);

    // ---- start value (utils.py:349-357) and the mu-independent part of nb_nll ----------------
    double v[P];
PDQ_UNROLL_P
    for (int j = 0; j < P; ++j) v[j] = 0.0;
    double lgsum = 0.0, logmean = 0.0;
    const int trips = (d.N + grp.T - 1) / grp.T;  // uniform across the warp: the loop body votes
    // this pass is the gene tile's first touch (DRAM / L2 latency): the counts of the next two trips are already requested
    // while a trip computes (the capture of round 2 showed 9.5 % of the kernel's stall samples on this one load)
    const int64_t ystep = (int64_t)grp.T * ld;
    const int64_t* yp = y + (int64_t)grp.si * ld;
    long long c_cur = (grp.si < d.N) ? yp[0] : 0, c_nxt = (grp.si + grp.T < d.N) ? yp[ystep] : 0;
    for (int it = 0, n = grp.si; it < trips; ++it, n += grp.T, yp += ystep) {
        const bool in = n < d.N;
        const int nn = in ? n : 0;
        double x[P];
        load_x<P>(d, nn, x);
        const long long yi = c_cur;
        c_cur = c_nxt;
        c_nxt = (n + 2 * grp.T < d.N) ? yp[2 * ystep] : 0;
        const double yv = (double)yi;
        const double q = fast_div(yv, d.sf[nn * d.RS]);
        double t;
        if (prm.full_rank) {
            t = tlog(q + 0.1, d.mtab);
PDQ_UNROLL_P
            for (int j = 0; j < P; ++j) v[j] = fma(x[j], in ? t : 0.0, v[j]);
        } else {
            t = tlog(q, d.mtab);
            logmean += in ? t : 0.0;
        }
        // lgamma(y + 1) - lgamma(y + r): table reads for small counts, unshifted Stirling series otherwise
        const bool small = tab_ok && yi >= 0 && yi < kPsiK;
        double term = small ? logfact[(int)(yi & (kPsiK - 1))] - lg_tab[(int)(yi & (kPsiK - 1))] : 0.0;
        if (grp.any(in && !small)) {
            const double z1 = small ? 40.0 : yv + 1.0, zr = small ? 40.0 : yv + r;
            const double big = tab_ok ? lgamma_asym(z1, tlog(z1, d.mtab)) - lgamma_asym(zr, tlog(zr, d.mtab))
                                      : lgamma_pos(yv + 1.0) - lgamma_pos(yv + r);
            term = small ? term : big;
        }
        lgsum += in ? term : 0.0;
    }
    group_sum_vec<P>(grp, v);
    lgsum = grp.sum(lgsum);
    double beta[P];
    if (prm.full_rank) {
PDQ_UNROLL_P
        for (int i = 0; i < P; ++i) {
            double s = 0.0;
PDQ_UNROLL_P
            for (int j = 0; j < P; ++j) s = fma(pinv.v[i * P + j], v[j], s);
            beta[i] = s;
        }
    } else {
        logmean = grp.sum(logmean);
PDQ_UNROLL_P
        for (int i = 0; i < P; ++i) beta[i] = 0.0;
        beta[0] = logmean / Nd;
    }
    // nb_nll = C + S(mu):  C = N r log(alpha) + N lgamma(r) + sum lgamma(y+1) - lgamma(y+r)
    const double C = Nd * r * log(alpha) + Nd * lgamma_pos(r) + lgsum;

    // ---- IRLS loop (utils.py:359-421) ---------------------------------------------------------
    // ONE call site of the sweep (the kernel's instruction footprint decides its instruction-cache behaviour: 15 % of the stall
    // samples of the p = 3 capture were instruction fetches): the trip of the start value skips the deviance bookkeeping.
    Sym<P> A;
    double b[P], S;
    double dev = 1000.0, ratio = 1.0;
    int it = 0, status = kIrlsOk;
    bool active = true, first = true;
    for (;;) {
        // frozen groups recompute the same sums (keeps the warp's shuffles uniform)
        irls_sweep<P>(grp, d, y, ld, beta, alpha, r, prm.min_mu, log_min_mu, A, b, S, prm.few_rows != 0);
        if (active && !first) {
            const double old = dev;
            dev = -2.0 * (C + S);
            ratio = fabs(dev - old) / (fabs(dev) + 0.1);
        }
        first = false;
        if (active && !(ratio > prm.beta_tol)) active = false;  // `while dev_ratio > beta_tol` (NaN exits)
        if (!grp.any(active)) break;
        Sym<P> L = A;
PDQ_UNROLL_P
        for (int i = 0; i < P; ++i) L.a[tri(i, i)] += kRidge;
        chol<P>(L);
        double bh[P];
PDQ_UNROLL_P
        for (int j = 0; j < P; ++j) bh[j] = b[j];
        chol_solve<P>(L, bh);
        if (active) {
            ++it;
            bool div = it >= prm.maxiter;
PDQ_UNROLL_P
            for (int j = 0; j < P; ++j) div = div || (fabs(bh[j]) > prm.max_beta);
            if (div) {
                status = kIrlsNeedsOptimizer;
                active = false;
            } else {
PDQ_UNROLL_P
                for (int j = 0; j < P; ++j) beta[j] = bh[j];
            }
        }
    }

    // ---- outputs: hat diagonal from the clamped mu, mu itself unclamped (utils.py:423-438) -----
    Sym<P> Hinv;
    {
        Sym<P> L = A;
PDQ_UNROLL_P
        for (int i = 0; i < P; ++i) L.a[tri(i, i)] += kRidge;
        chol<P>(L);
        chol_inverse<P>(L, Hinv);
    }
    double eta_prev = __builtin_nan(""), exp_prev = 0.0;
    Sym<P> Dc;  // run_wald_test uses the UNCLAMPED mu (ds.py:320-324): correction of A for the samples on the min_mu clamp
    sym_zero<P>(Dc);
    bool clamped = false;
    for (int n = grp.si; n < d.N; n += grp.T) {
        double x[P];
        load_x<P>(d, n, x);
        double eta = 0.0;
PDQ_UNROLL_P
        for (int j = 0; j < P; ++j) eta = fma(x[j], beta[j], eta);
        if (eta != eta_prev) {  // same carry-over as the sweeps: equal design rows share their exponential
            exp_prev = texp(eta, d.mtab);
            eta_prev = eta;
        }
        const double mu_raw = d.sf[n * d.RS] * exp_prev;
        const bool cl = mu_raw < prm.min_mu;
        const double mu = cl ? prm.min_mu : mu_raw;
        const double W = fast_div(mu, fma(mu, alpha, 1.0));
        if (valid) {
            mu_out[(int64_t)n * ld_out] = mu_raw;
            hat_out[(int64_t)n * ld_out] = W * sym_quad<P>(Hinv, x);
        }
        if (wald && cl) {
            clamped = true;
            sym_rank1<P>(Dc, mu_raw / fma(mu_raw, alpha, 1.0) - W, x);
        }
    }
    if (wald) {
        Sym<P> M = A;
        if (grp.any(clamped)) {
            group_sum_sym<P>(grp, Dc);
PDQ_UNROLL_P
            for (int k = 0; k < P * (P + 1) / 2; ++k) M.a[k] += Dc.a[k];
        }
        wald_finish<P>(grp, M, *wald, beta, wald_p, wald_stat, wald_se, valid);
    }
    if (valid && grp.si == 0) {
PDQ_UNROLL_P
        for (int j = 0; j < P; ++j) beta_out[j] = beta[j];
        *conv_out = 1.0;  // IRLS exits are "converged" (utils.py:365); the optimiser branch overwrites
        *status_out = status;
    }
}

// ---------------------------------------------------------------------------------------------
// Optimiser branch of irls (utils.py:374-413): minimise f(beta) = nb_nll(y, max(sf e^{X beta}, min_mu), disp)
// + 0.5 * 1e-6 |beta|^2 over the box [min_beta, max_beta]^p, started from the IRLS start value.
// The reference uses scipy L-BFGS-B; f is convex in X beta wherever the clamp is inactive, so any
// descent method reaches the same minimiser: here a projected Newton iteration with the exact
// Hessian and Armijo backtracking.  Called for the (rare) genes flagged kIrlsNeedsOptimizer.
// =============================================================================================
template <int P>
PDQ_HD void irls_obj_sweep(const Group& grp, const DesignS& d, const int64_t* y, int64_t ld, const double (&beta)[P],
                           double alpha, double r, double min_mu, double log_min_mu, double& f, double (&g)[P],
                           Sym<P>& H) {
    sym_zero<P>(H);
PDQ_UNROLL_P
    for (int j = 0; j < P; ++j) g[j] = 0.0;
    f = 0.0;
    for (int n = grp.si; n < d.N; n += grp.T) {
        double x[P];
        load_x<P>(d, n, x);
        const double yv = (double)y[n * ld];
        double eta = 0.0;
PDQ_UNROLL_P
        for (int j = 0; j < P; ++j) eta = fma(x[j], beta[j], eta);
        const double mu_raw = d.sf[n * d.RS] * exp(eta);
        const bool cl = mu_raw < min_mu;
        const double mu = cl ? min_mu : mu_raw;
        const double lmu = cl ? log_min_mu : (eta + d.lsf[n * d.RS]);
        f += fma(yv + r, log(r + mu), -yv * lmu);
        // df of the reference: -X^T y + ((r + y) mu / (r + mu)) X  (treats d mu / d eta = mu everywhere)
        const double t = (r + yv) * mu / (r + mu);
        const double gi = t - yv;
        const double hi = t * r / (r + mu);  // d t / d eta where the clamp is inactive
PDQ_UNROLL_P
        for (int j = 0; j < P; ++j) g[j] = fma(gi, x[j], g[j]);
        sym_rank1<P>(H, hi, x);
    }
    f = grp.sum(f);
    group_sum_vec<P>(grp, g);
    group_sum_sym<P>(grp, H);
PDQ_UNROLL_P
    for (int j = 0; j < P; ++j) {
        f = fma(0.5 * kRidge * beta[j], beta[j], f);
        g[j] = fma(kRidge, beta[j], g[j]);
        H.a[tri(j, j)] += kRidge;
    }
}

// numpy.linspace node i of n: arange(n) * step + start with step = (stop - start) / (n - 1), two roundings (no FMA contraction,
// so the nodes are the reference's bit for bit); the last node is `stop` exactly
PDQ_HD double linspace_at(double lo, double hi, int n, int i) {
    if (i == n - 1) return hi;
    const double step = (hi - lo) / (double)(n - 1);
#if defined(__CUDA_ARCH__)
    return __dadd_rn(__dmul_rn((double)i, step), lo);
#else
    volatile double prod = (double)i * step;
    return prod + lo;
#endif
}

// grid_fit_beta (grid_search.py:145-221), the reference's last resort for two-column designs when its optimiser reports failure
// (utils.py:402-409): 60 x 60 nodes on [-30, 30]^2, then 60 x 60 on one coarse cell either side of the best node; loss =
// nb_nll(y, max(sf exp(X b), 0.5), alpha) + 0.5e-6 |b|^2 -- the CALLER's min_mu and bounds are not passed on (`grid_fit_beta(counts,
// size_factors, X, disp)`) --, np.argmin's first minimum in row-major order (a NaN node counts as the minimum, like np.argmin).
// Only the part of the likelihood that depends on b is summed; the rest is the same number at every node.
PDQ_HD void irls_grid_gene(const Group& grp, const DesignS& d, const int64_t* y, int64_t ld, double r, double (&out)[2]) {
    constexpr int K = 60;
    const double min_mu = 0.5, log_min_mu = log(0.5);
    double lo0 = -30.0, hi0 = 30.0, lo1 = -30.0, hi1 = 30.0;
    for (int pass = 0; pass < 2; ++pass) {
        double best = 0.0;
        int bi = 0, bj = 0;
        bool best_nan = false;
        for (int i = 0; i < K; ++i) {
            const double b0 = linspace_at(lo0, hi0, K, i);
            for (int j = 0; j < K; ++j) {
                const double b1 = linspace_at(lo1, hi1, K, j);
                double f = 0.0;
                for (int n = grp.si; n < d.N; n += grp.T) {
                    const double* row = d.X + (size_t)n * d.RS;
                    const double yv = (double)y[n * ld];
                    const double eta = fma(row[1], b1, row[0] * b0);
                    const double mu_raw = d.sf[n * d.RS] * exp(eta);
                    const bool cl = mu_raw < min_mu;
                    const double mu = cl ? min_mu : mu_raw;
                    const double lmu = cl ? log_min_mu : log(mu);
                    f += fma(yv + r, log(r + mu), -yv * lmu);
                }
                f = grp.sum(f);
                f = fma(0.5 * kRidge, fma(b0, b0, b1 * b1), f);
                const bool first = (i == 0 && j == 0);
                const bool is_nan = !(f == f);
                if (first || (!best_nan && (is_nan || f < best))) {
                    best = f;
                    best_nan = is_nan;
                    bi = i;
                    bj = j;
                }
            }
        }
        out[0] = linspace_at(lo0, hi0, K, bi);
        out[1] = linspace_at(lo1, hi1, K, bj);
        if (pass == 0) {
            const double delta = linspace_at(-30.0, 30.0, K, 1) - (-30.0);
            lo0 = out[0] - delta; hi0 = out[0] + delta;
            lo1 = out[1] - delta; hi1 = out[1] + delta;
        }
    }
}

template <int P>
PDQ_HD void irls_optimizer_gene(const Group& grp, const DesignS& d, const SmallMat<P>& pinv, const IrlsParams& prm,
                                const int64_t* y, int64_t ld, double alpha, double* beta_out, double* mu_out,
                                double* hat_out, int64_t ld_out, double* conv_out, bool valid, const WaldParams<P>* wald = nullptr,
                                double* wald_p = nullptr, double* wald_stat = nullptr, double* wald_se = nullptr) {
    const double r = 1.0 / alpha;
    const double log_min_mu = log(prm.min_mu);
    // start value: same as irls_gene (utils.py:349-357, `beta_init`)
    double v[P];
PDQ_UNROLL_P
    for (int j = 0; j < P; ++j) v[j] = 0.0;
    double logmean = 0.0;
    for (int n = grp.si; n < d.N; n += grp.T) {
        double x[P];
        load_x<P>(d, n, x);
        const double q = (double)y[n * ld] / d.sf[n * d.RS];
        if (prm.full_rank) {
            const double t = log(q + 0.1);
PDQ_UNROLL_P
            for (int j = 0; j < P; ++j) v[j] = fma(x[j], t, v[j]);
        } else {
            logmean += log(q);
        }
    }
    group_sum_vec<P>(grp, v);
    double beta[P];
    if (prm.full_rank) {
PDQ_UNROLL_P
        for (int i = 0; i < P; ++i) {
            double s = 0.0;
PDQ_UNROLL_P
            for (int j = 0; j < P; ++j) s = fma(pinv.v[i * P + j], v[j], s);
            beta[i] = s;
        }
    } else {
        logmean = grp.sum(logmean);
PDQ_UNROLL_P
        for (int i = 0; i < P; ++i) beta[i] = 0.0;
        beta[0] = logmean / (double)d.N;
    }
PDQ_UNROLL_P
    for (int j = 0; j < P; ++j) beta[j] = fmin(fmax(beta[j], prm.min_beta), prm.max_beta);

    double f, g[P];
    Sym<P> H;
    irls_obj_sweep<P>(grp, d, y, ld, beta, alpha, r, prm.min_mu, log_min_mu, f, g, H);
    bool ok = false, active = valid;  // `valid` = this gene was flagged and is in range
    for (int it = 0; it < 100; ++it) {
        // projected-gradient norm (free variables only)
        double pg = 0.0;
        bool fixed[P];
PDQ_UNROLL_P
        for (int j = 0; j < P; ++j) {
            fixed[j] = (beta[j] <= prm.min_beta && g[j] > 0.0) || (beta[j] >= prm.max_beta && g[j] < 0.0);
            if (!fixed[j]) pg = fmax(pg, fabs(g[j]));
        }
        if (active && (pg <= 1e-9 * (1.0 + fabs(f)) || !(pg == pg))) {
            ok = (pg == pg);
            active = false;
        }
        if (!grp.any(active)) break;
        // Newton direction on the free set
        Sym<P> L = H;
        double dir[P];
PDQ_UNROLL_P
        for (int i = 0; i < P; ++i) {
            dir[i] = fixed[i] ? 0.0 : -g[i];
            if (fixed[i]) {
PDQ_UNROLL_P
                for (int j = 0; j < P; ++j)
                    if (j != i) L.a[j <= i ? tri(i, j) : tri(j, i)] = 0.0;
                L.a[tri(i, i)] = 1.0;
            }
        }
        chol<P>(L);
        chol_solve<P>(L, dir);
        double slope = 0.0;
PDQ_UNROLL_P
        for (int j = 0; j < P; ++j) slope = fma(g[j], dir[j], slope);
        if (!(slope < 0.0)) {  // not a descent direction (indefinite/NaN): steepest descent on the free set
            slope = 0.0;
PDQ_UNROLL_P
            for (int j = 0; j < P; ++j) {
                dir[j] = fixed[j] ? 0.0 : -g[j];
                slope = fma(g[j], dir[j], slope);
            }
        }
        // backtracking line search with projection onto the box
        double step = 1.0, fn = f, gn[P], bn[P];
        Sym<P> Hn = H;
        bool accepted = false;
PDQ_UNROLL_P
        for (int j = 0; j < P; ++j) { gn[j] = g[j]; bn[j] = beta[j]; }
        for (int ls = 0; ls < 30; ++ls) {
            double bt[P], dec = 0.0;
PDQ_UNROLL_P
            for (int j = 0; j < P; ++j) {
                bt[j] = fmin(fmax(fma(step, dir[j], beta[j]), prm.min_beta), prm.max_beta);
                dec = fma(g[j], bt[j] - beta[j], dec);
            }
            double ft, gt[P];
            Sym<P> Ht;
            irls_obj_sweep<P>(grp, d, y, ld, bt, alpha, r, prm.min_mu, log_min_mu, ft, gt, Ht);
            const bool good = ft <= f + 1e-4 * dec;
            if (active && !accepted && good) {
                accepted = true;
                fn = ft;
                Hn = Ht;
PDQ_UNROLL_P
                for (int j = 0; j < P; ++j) { gn[j] = gt[j]; bn[j] = bt[j]; }
            }
            if (!grp.any(active && !accepted)) break;
            step *= 0.5;
        }
        if (active) {
            if (!accepted) {  // line search failed: declare failure like res.success == False
                active = false;
                ok = false;
            } else {
                const double df = f - fn;
                f = fn;
                H = Hn;
PDQ_UNROLL_P
                for (int j = 0; j < P; ++j) { g[j] = gn[j]; beta[j] = bn[j]; }
                if (df <= 1e-15 * (1.0 + fabs(f))) {  // no further decrease possible in FP64
                    active = false;
                    ok = true;
                }
            }
        }
    }
    if (prm.fail_optimizer) ok = false;
    if constexpr (P == 2) {
        // utils.py:402-409: `not res.success and num_vars <= 2` -> grid_fit_beta; `converged` stays False.  (With one column the
        // reference's grid_fit_beta raises on the shape of `beta.T`; nothing to mirror.)
        const bool need = valid && !ok;
        if (grp.any(need)) {
            double gb[2];
            irls_grid_gene(grp, d, y, ld, r, gb);
            if (need) {
                beta[0] = gb[0];
                beta[1] = gb[1];
            }
        }
    }
    // outputs exactly like the tail of irls_solver: W from clamped mu, ridge 1e-6, mu unclamped
    Sym<P> A, M;  // M: the Wald test's X^T W X, W from the unclamped mu
    sym_zero<P>(A);
    sym_zero<P>(M);
    for (int n = grp.si; n < d.N; n += grp.T) {
        double x[P];
        load_x<P>(d, n, x);
        double eta = 0.0;
PDQ_UNROLL_P
        for (int j = 0; j < P; ++j) eta = fma(x[j], beta[j], eta);
        const double mu_raw = d.sf[n * d.RS] * exp(eta);
        const double mu = (mu_raw < prm.min_mu) ? prm.min_mu : mu_raw;
        sym_rank1<P>(A, mu / fma(mu, alpha, 1.0), x);
        if (wald) sym_rank1<P>(M, mu_raw / fma(mu_raw, alpha, 1.0), x);
    }
    group_sum_sym<P>(grp, A);
    if (wald) {
        group_sum_sym<P>(grp, M);
        wald_finish<P>(grp, M, *wald, beta, wald_p, wald_stat, wald_se, valid);
    }
    Sym<P> Hinv;
PDQ_UNROLL_P
    for (int i = 0; i < P; ++i) A.a[tri(i, i)] += kRidge;
    chol<P>(A);
    chol_inverse<P>(A, Hinv);
    if (!valid) return;
    for (int n = grp.si; n < d.N; n += grp.T) {
        double x[P];
        load_x<P>(d, n, x);
        double eta = 0.0;
PDQ_UNROLL_P
        for (int j = 0; j < P; ++j) eta = fma(x[j], beta[j], eta);
        const double mu_raw = d.sf[n * d.RS] * exp(eta);
        const double mu = (mu_raw < prm.min_mu) ? prm.min_mu : mu_raw;
        mu_out[n * ld_out] = mu_raw;
        hat_out[n * ld_out] = mu / fma(mu, alpha, 1.0) * sym_quad<P>(Hinv, x);
    }
    if (grp.si == 0) {
PDQ_UNROLL_P
        for (int j = 0; j < P; ++j) beta_out[j] = beta[j];
        *conv_out = ok ? 1.0 : 0.0;
    }
}

// =============================================================================================
// (a2) alpha_mle -- utils.py:441-564.
// The objective in x = log(alpha) (utils.py:509-520) and its derivative (utils.py:522-544):
//   loss  = nb_nll(y, mu, a) + [cr] 0.5 logdet(X^T W X) + [prior] (x - xhat)^2 / (2 var),   W = mu/(1+mu a)
//   dloss = a dnb_nll + [cr] -0.5 a tr((X^T W X)^-1 X^T W^2 X) + [prior] (x - xhat)/var
// =============================================================================================
struct AlphaParams {
    double lo, hi;  // log(min_disp), log(max_disp)
    double prior_var;
    int cr_reg, prior_reg;
};

// psi(r + k), k < kPsiK, per gene and per evaluation: psi(r+k) = psi(r) + sum_{j<k} 1/(r+j)  (see the table note above)
PDQ_HD void build_psi_table(const Group& grp, double* tab, double r) {
    const int seg = kPsiK / grp.T;              // T in {1,...,32} divides 32
    const int k0 = grp.si * seg;
    double part = 0.0;
    for (int k = k0; k < k0 + seg; ++k) {
        const double inv = fast_rcp(r + (double)k);
        tab[k] = inv;
        part += inv;
    }
    double run = digamma_pos(r) + grp.excl_scan(part);
    for (int k = k0; k < k0 + seg; ++k) {
        const double inv = tab[k];
        tab[k] = run;
        run += inv;
    }
    grp.sync();
}

// the same for psi and psi' together (first evaluation of a gene, which also returns the curvature of the NB part):
// psi'(r + k) = psi'(r) - sum_{j<k} (r + j)^-2.  `tab` holds 2 * kPsiK doubles: psi first, psi' behind it.
PDQ_HD void build_psi_tri_tables(const Group& grp, double* tab, double r) {
    const int seg = kPsiK / grp.T;
    const int k0 = grp.si * seg;
    double part = 0.0, part2 = 0.0;
    for (int k = k0; k < k0 + seg; ++k) {
        const double inv = fast_rcp(r + (double)k);
        tab[k] = inv;
        part += inv;
        part2 = fma(inv, inv, part2);
    }
    double run = digamma_pos(r) + grp.excl_scan(part);
    double run2 = trigamma_pos(r) - grp.excl_scan(part2);
    for (int k = k0; k < k0 + seg; ++k) {
        const double inv = tab[k];
        tab[k] = run;
        tab[kPsiK + k] = run2;
        run += inv;
        run2 = fma(-inv, inv, run2);
    }
    grp.sync();
}

// contribution of two samples (or one, when !two) to the derivative sums; NB as in irls_sample.
// CURV: also S2 = sum 1/(r+mu) - psi'(y+r) - (y-mu)/(r+mu)^2, the r-derivative of the summand of Sg.
template <int P, bool NB, bool CURV>
PDQ_HD void alpha_pair(const Group& grp, const double* xp0, const double* xp1, const double* mtab, long long yi0, long long yi1,
                       double m0, double m1, bool one, bool two, double r, bool cr_reg, const double* psi_tab, double& Sg,
                       Sym<P>& A, Sym<P>& B, bool& odd, double& S2) {
    // `one` / `two`: which of the two samples exist for this lane (masked-out slots carry y = 0, mu = 1)
    const double yv0 = (double)yi0, yv1 = (double)yi1;
    const bool big0 = one && ((yi0 >= kPsiK) || (yi0 < 0)), big1 = two && ((yi1 >= kPsiK) || (yi1 < 0));
#if defined(__CUDA_ARCH__)
    // means outside [+0, ~1e300) (negative, NaN, inf) send the gene to the guarded path: one integer compare on the high word
    if (NB) odd = odd || ((unsigned)__double2hiint(m0) >= 0x7e300000u) || ((unsigned)__double2hiint(m1) >= 0x7e300000u);
#else
    if (NB) odd = odd || !(m0 >= 0.0 && m0 < 1e300) || !(m1 >= 0.0 && m1 < 1e300);
#endif
    const double rm0 = r + m0, rm1 = r + m1;
    const double inv0 = NB ? fast_rcp(rm0) : 1.0 / rm0, inv1 = NB ? fast_rcp(rm1) : 1.0 / rm1;
    const double lg0 = NB ? tlog_nb(rm0, mtab) : fast_log(rm0), lg1 = NB ? tlog_nb(rm1, mtab) : fast_log(rm1);
    double dg0 = psi_tab[(int)(yi0 & (kPsiK - 1))], dg1 = psi_tab[(int)(yi1 & (kPsiK - 1))];
    double tg0 = 0.0, tg1 = 0.0;
    if (CURV) {
        tg0 = psi_tab[kPsiK + (int)(yi0 & (kPsiK - 1))];
        tg1 = psi_tab[kPsiK + (int)(yi1 & (kPsiK - 1))];
    }
    if (grp.any(big0 || big1)) {  // warp-uniform: the unshifted series only when some lane holds a count >= kPsiK
        const double z0 = big0 ? yv0 + r : r + (double)kPsiK, z1 = big1 ? yv1 + r : r + (double)kPsiK;
        const double a0 = digamma_asym(z0, NB ? tlog_nb(z0, mtab) : fast_log(z0));
        const double a1 = digamma_asym(z1, NB ? tlog_nb(z1, mtab) : fast_log(z1));
        dg0 = big0 ? a0 : dg0;
        dg1 = big1 ? a1 : dg1;
        if (CURV) {
            const double b0 = trigamma_asym(z0), b1 = trigamma_asym(z1);
            tg0 = big0 ? b0 : tg0;
            tg1 = big1 ? b1 : tg1;
        }
    }
    const double t0 = lg0 - dg0 + (yv0 - m0) * inv0, t1 = lg1 - dg1 + (yv1 - m1) * inv1;
    Sg += (one ? t0 : 0.0) + (two ? t1 : 0.0);
    if (CURV) {
        const double u0 = fma(-(yv0 - m0) * inv0, inv0, inv0 - tg0), u1 = fma(-(yv1 - m1) * inv1, inv1, inv1 - tg1);
        S2 += (one ? u0 : 0.0) + (two ? u1 : 0.0);
    }
    if (cr_reg) {
        double xv[P];
PDQ_UNROLL_P
        for (int j = 0; j < P; ++j) xv[j] = xp0[j];
        const double W0 = one ? m0 * r * inv0 : 0.0;
        sym_rank1<P>(A, W0, xv);
        sym_rank1<P>(B, W0 * W0, xv);
PDQ_UNROLL_P
        for (int j = 0; j < P; ++j) xv[j] = xp1[j];
        const double W1 = two ? m1 * r * inv1 : 0.0;
        sym_rank1<P>(A, W1, xv);
        sym_rank1<P>(B, W1 * W1, xv);
    }
}

template <int P, bool NB, bool CURV>
PDQ_HD bool alpha_sweep_t(const Group& grp, const DesignS& d, bool cr_reg, const int64_t* y, int64_t ld, const double* mu,
                          int64_t ld_mu, double r, const double* psi_tab, double& Sg, Sym<P>& A, Sym<P>& B, double& S2) {
    Sg = 0.0;
    S2 = 0.0;
    sym_zero<P>(A);
    sym_zero<P>(B);
    bool odd = false;
    const int T = grp.T;
    const int64_t ystep = (int64_t)T * ld, mstep = (int64_t)T * ld_mu;
    const int64_t* yp = y + (int64_t)grp.si * ld;
    const double* mp = mu + (int64_t)grp.si * ld_mu;
    constexpr int RS = design_row_stride(P);
    const double* xp = d.X + grp.si * RS;
    // the trip count is made uniform across the warp (lanes past N contribute a masked dummy) because alpha_pair votes
    const int trips = (d.N + 2 * T - 1) / (2 * T);
    int n = grp.si;
#if PDQ_PREFETCH
    // register triple buffer: the counts and means of the NEXT TWO trips are in flight while this trip computes -- one trip of
    // cover (~150 instructions) hides an L2 hit, not a DRAM access (first evaluation of a gene; 9 % long-scoreboard samples at
    // 60 000 x 500 with one trip of cover)
    bool v0 = n < d.N, v1 = n + T < d.N, w0 = n + 2 * T < d.N, w1 = n + 3 * T < d.N;
    long long yi0 = v0 ? yp[0] : 0, yi1 = v1 ? yp[ystep] : 0, ny0 = w0 ? yp[2 * ystep] : 0, ny1 = w1 ? yp[3 * ystep] : 0;
    double m0 = v0 ? mp[0] : 1.0, m1 = v1 ? mp[mstep] : 1.0, nm0 = w0 ? mp[2 * mstep] : 1.0, nm1 = w1 ? mp[3 * mstep] : 1.0;
    for (int it = 0; it < trips; ++it, n += 2 * T, yp += 2 * ystep, mp += 2 * mstep, xp += 2 * T * RS) {
        const bool u0 = n + 4 * T < d.N, u1 = n + 5 * T < d.N;
        const long long fy0 = u0 ? yp[4 * ystep] : 0, fy1 = u1 ? yp[5 * ystep] : 0;
        const double fm0 = u0 ? mp[4 * mstep] : 1.0, fm1 = u1 ? mp[5 * mstep] : 1.0;
        // one call site: every lane of the warp reaches the vote inside alpha_pair together
        alpha_pair<P, NB, CURV>(grp, v0 ? xp : d.X, v1 ? xp + T * RS : d.X, d.mtab, yi0, yi1, m0, m1, v0, v1, r, cr_reg, psi_tab,
                                Sg, A, B, odd, S2);
        v0 = w0; v1 = w1; yi0 = ny0; yi1 = ny1; m0 = nm0; m1 = nm1;
        w0 = u0; w1 = u1; ny0 = fy0; ny1 = fy1; nm0 = fm0; nm1 = fm1;
    }
#else
    for (int it = 0; it < trips; ++it, n += 2 * T, yp += 2 * ystep, mp += 2 * mstep, xp += 2 * T * RS) {
        const bool v0 = n < d.N, v1 = n + T < d.N;
        const long long yi0 = v0 ? yp[0] : 0, yi1 = v1 ? yp[ystep] : 0;
        const double m0 = v0 ? mp[0] : 1.0, m1 = v1 ? mp[mstep] : 1.0;
        // one call site: every lane of the warp reaches the vote inside alpha_pair together
        alpha_pair<P, NB, CURV>(grp, v0 ? xp : d.X, v1 ? xp + T * RS : d.X, d.mtab, yi0, yi1, m0, m1, v0, v1, r, cr_reg, psi_tab,
                                Sg, A, B, odd, S2);
    }
#endif
    return odd;
}

// derivative only (the minimiser is located as a root of dloss).  `curv` (first evaluation of a gene): also the second
// derivative of the NB part (+ prior) with respect to x = log(alpha), used for ONE Newton step from the start value:
//   a dnb_nll = -r F(r),  F = N (psi(r) + x) + Sg,  dr/dx = -r   =>   d/dx = r F + r^2 F',  F' = N (psi'(r) - 1/r) + S2.
// The Cox-Reid term's curvature is left out (the secant steps that follow see the whole function); NaN when unavailable.
template <int P>
PDQ_HD double alpha_dloss(const Group& grp, const DesignS& d, const AlphaParams& prm, const int64_t* y, int64_t ld,
                          const double* mu, int64_t ld_mu, double x, double xhat, double* psi_tab, double* curv = nullptr) {
#if defined(PDQ_EMU_COUNT_EVALS) && !defined(__CUDA_ARCH__)
    if (grp.si == 0) ++g_emu_alpha_evals;  // host emulator instrumentation only
#endif
    const double a = fast_exp(x), r = fast_rcp(a), Nd = (double)d.N;
    grp.sync();  // previous evaluation's table reads are done
    double Sg, S2 = 0.0;
    Sym<P> A, B;
    // every lane of the warp runs the same sequence (the sweeps vote and the table builders scan across the warp); a gene
    // whose r is unusable only marks itself `odd` and the whole warp repeats the sweep on the guarded libdevice path
    bool odd;
    if (curv != nullptr) {
        build_psi_tri_tables(grp, psi_tab, r);
        odd = alpha_sweep_t<P, true, true>(grp, d, prm.cr_reg != 0, y, ld, mu, ld_mu, r, psi_tab, Sg, A, B, S2);
    } else {
        build_psi_table(grp, psi_tab, r);
        odd = alpha_sweep_t<P, true, false>(grp, d, prm.cr_reg != 0, y, ld, mu, ld_mu, r, psi_tab, Sg, A, B, S2);
    }
    odd = odd || !(r > 0.0 && r < 1e300);
    const bool any_odd = grp.any(odd);
    if (any_odd) alpha_sweep_t<P, false, false>(grp, d, prm.cr_reg != 0, y, ld, mu, ld_mu, r, psi_tab, Sg, A, B, S2);
    const bool have_curv = (curv != nullptr) && !any_odd;
    Sg = grp.sum(Sg);
    // a * dnb_nll = -r * sum[psi(r) - psi(y+r) + log(1 + mu a) + (y - mu)/(mu + r)],  log(1+mu a) = x + log(r+mu)
    const double F = Nd * (psi_tab[0] + x) + Sg;
    double g = -r * F;
    if (curv != nullptr) {
        double h = __builtin_nan("");
        if (have_curv) {  // warp-uniform
            S2 = grp.sum(S2);
            const double Fp = Nd * (psi_tab[kPsiK] - a) + S2;
            h = r * (F + r * Fp) + (prm.prior_reg ? 1.0 / prm.prior_var : 0.0);
        }
        *curv = h;
    }
    if (prm.cr_reg) {
        group_sum_sym<P>(grp, A);
        group_sum_sym<P>(grp, B);
        Sym<P> Ainv;
        chol<P>(A);
        chol_inverse<P>(A, Ainv);
        g -= 0.5 * a * sym_dot<P>(Ainv, B);
    }
    if (prm.prior_reg) g += (x - xhat) / prm.prior_var;
    return g;
}

// loss value up to the alpha-independent constant  sum lgamma(y+1) - y log(mu)  (irrelevant to argmin)
template <int P>
PDQ_HD double alpha_loss(const Group& grp, const DesignS& d, int cr_reg, int prior_reg, double prior_var,
                         const int64_t* y, int64_t ld, const double* mu, int64_t ld_mu, double x, double xhat) {
    const double a = exp(x), r = 1.0 / a, Nd = (double)d.N;
    double Sf = 0.0;
    Sym<P> A;
    sym_zero<P>(A);
    for (int n = grp.si; n < d.N; n += grp.T) {
        const double yv = (double)y[n * ld];
        const double m = mu[n * ld_mu];
        const double rm = r + m;
        Sf += fma(yv + r, log(rm), -lgamma_pos(yv + r));
        if (cr_reg) {
            double xv[P];
            load_x<P>(d, n, xv);
            sym_rank1<P>(A, m * r / rm, xv);
        }
    }
    Sf = grp.sum(Sf);
    double f = Nd * (r * x + lgamma_pos(r)) + Sf;
    if (cr_reg) {
        group_sum_sym<P>(grp, A);
        chol<P>(A);
        f += 0.5 * chol_logdet<P>(A);
    }
    if (prior_reg) f += (x - xhat) * (x - xhat) / (2.0 * prior_var);
    return f;
}

constexpr int kAlphaOk = 0;
constexpr int kAlphaNeedsGrid = 1;  // the reference's `res.success == False` branch (utils.py:556-564)

// Bounded root search on dloss, shaped after what 1-D L-BFGS-B does from the same start: project x0 into
// the box, take a unit step against the gradient, then secant (= 1-D BFGS) steps; once the root is
// bracketed the secant point is safeguarded by the bracket (bisection when it leaves it or stalls).
// `dloss(x, xhat, curv)` evaluates d loss / d log(alpha) at x (alpha_dloss; curv != nullptr on the first evaluation): the search
// is the same for every layout of the per-gene sums (the wide-design kernels pass their own, pdq_wide.cu)
template <class DLoss>
PDQ_HD void alpha_search(const Group& grp, const AlphaParams& prm, double alpha_hat, DLoss&& dloss, double* alpha_out, double* conv_out,
                         int* status_out, bool valid, const double* hint_in = nullptr, double* hint_out = nullptr) {
    // hint_in = [x*, h*] of an EARLIER search on the same counts and means without the prior (the genewise fit, whose optimum x*
    // = log alpha and curvature h* of its loss there carry over): the MAP objective is that loss plus (x - xhat)^2 / (2 var), so
    // one Newton step of it from x* lands within ~1e-3 of the MAP optimum, and a second one, with the curvature h* + 1/var,
    // usually ends the search: ~2.2 evaluations instead of 3.5.  The start point x0 = log(alpha_hat) is still evaluated first:
    // the rules that keep a gene AT its start (flat tail, bounds; see below) are the reference's and do not depend on the hint.
    // hint_out receives [x, h] of this search (h = slope of dloss between its last two evaluations, NaN when unavailable).
    const double xhat = log(alpha_hat);
    const double tolx = 1e-5;   // last secant step is taken unevaluated: final error << tolx
    // scipy's L-BFGS-B declares convergence as soon as the projected gradient is <= pgtol = 1e-5 (checked at the
    // start point too).  This matters for parity, not accuracy: on the flat left tail of the objective (alpha -> 1e-8,
    // |dloss| ~ 1e-7) the reference therefore never leaves its start value, and neither may we.
    const double pgtol = 1e-5;
    double xb = fmin(fmax(xhat, prm.lo), prm.hi);
    double h0;
    double gb = dloss(xb, xhat, &h0);
    double xa = xb, ga = gb;
    double bl = prm.lo, br = prm.hi;  // bracket ends (valid when have_br)
    bool have_br = false, active = true, fail = false;
    double xres = xb, xt = xb;
    int stall = 0;
    bool use_hint = false;
    double hint_h = 0.0;
    // decide the first trial point
    if (!(gb == gb)) {
        fail = true;
        active = false;
    } else if (fabs(gb) <= pgtol || (gb > 0.0 && xb <= prm.lo) || (gb < 0.0 && xb >= prm.hi)) {
        active = false;  // stationary to L-BFGS-B's tolerance, or the projected gradient vanishes at a bound
    } else {
        // first trial point: one Newton step with the curvature of the NB part (+ prior) when it is shorter than 1 in
        // log(alpha), else (or where that curvature is not positive / not available) the unit step against the gradient that
        // L-BFGS-B opens with.  The root is polished by the safeguarded secant below either way, but the Newton point
        // usually lands within a few percent of it: 3.2-3.8 evaluations per gene instead of 5.1-5.3.
        double step = -sgn(gb);
        if (h0 > 0.0) {
            // a Newton step longer than L-BFGS-B's unit step means the start is far from the root or on a flat tail: there the
            // stopping point (first evaluated point with |dloss| <= pgtol) depends on the sequence of trial points, so the
            // reference's own opening move is kept
            const double s = -gb / h0;
            if (fabs(s) < 1.0) step = s;
        }
        xt = fmin(fmax(xb + step, prm.lo), prm.hi);
        if (hint_in != nullptr) {
            const double hx = hint_in[0];
            hint_h = hint_in[1] + (prm.prior_reg ? 1.0 / prm.prior_var : 0.0);
            const double xp = hx - (prm.prior_reg ? (hx - xhat) / prm.prior_var : 0.0) / hint_h;
            // usable: finite, positive curvature, inside the box, and on the downhill side of the start point
            use_hint = (hint_h > 0.0) && (hint_h < 1e300) && (xp > prm.lo) && (xp < prm.hi) && ((xp - xb) * gb < 0.0);
            if (use_hint) xt = xp;
        }
        if (fabs(xt - xb) <= tolx) {  // already there: take the step unevaluated, like the last secant step
            xres = xt;
            active = false;
        }
    }
    for (int ev = 0; ev < 60; ++ev) {
        if (!grp.any(active)) break;
        const double gt = dloss(xt, xhat, (double*)nullptr);
        if (!active) continue;
        if (!(gt == gt)) {
            fail = true;
            active = false;
            continue;
        }
        // bracket bookkeeping: the minimum lies where dloss goes from - (left end) to + (right end)
        if (have_br) {
            if (gt < 0.0) bl = xt; else br = xt;
        } else if ((gt < 0.0) != (gb < 0.0) && gt != 0.0) {
            have_br = true;
            bl = (gt < 0.0) ? xt : xb;
            br = (gt < 0.0) ? xb : xt;
        }
        const double prev_step = fabs(xb - xa);
        xa = xb; ga = gb;
        xb = xt; gb = gt;
        xres = xb;
        if (fabs(gt) <= pgtol) {
            // stationary to L-BFGS-B's tolerance.  The secant through the last two points is free: take it unevaluated when it
            // is a small correction (on a flat stretch, where it would jump, the evaluated point stands)
            const double dgs = gb - ga, xs = xb - gb * (xb - xa) / dgs;
            if (dgs != 0.0 && fabs(xs - xb) <= 1e-3 && xs >= prm.lo && xs <= prm.hi) xres = xs;
            active = false;
            continue;
        }
        if (!have_br && ((gb > 0.0 && xb <= prm.lo) || (gb < 0.0 && xb >= prm.hi))) {
            active = false;  // pushed against a bound: L-BFGS-B stops with zero projected gradient
            continue;
        }
        // next point
        const double dx = xb - xa, dg = gb - ga;
        double xn;
        if (use_hint && ev == 0) {
            // the hinted point has just been evaluated: Newton step with the carried-over curvature (the secant through the far
            // start point would be a poor slope); inside a bracket it must stay inside, else bisect like below
            xn = fmin(fmax(xb - gb / hint_h, prm.lo), prm.hi);
            if (have_br && !((xn > bl) && (xn < br))) xn = 0.5 * (bl + br);
        } else if (have_br) {
            xn = xb - gb * dx / dg;
            // Brent-style safeguard: fall back to bisection when the secant point leaves the bracket or
            // the steps have not been shrinking for two evaluations in a row
            if (ev > 0 && fabs(dx) > 0.5 * prev_step) ++stall; else stall = 0;
            const bool inside = (xn > bl) && (xn < br);
            if (!inside || !(dg != 0.0) || stall >= 2) {
                xn = 0.5 * (bl + br);
                stall = 0;
            }
            if (br - bl <= tolx) {  // bracket already tight: finish at the interpolated point
                xres = xn;
                active = false;
                continue;
            }
        } else {
            if (dg * dx > 0.0) {
                xn = xb - gb * dx / dg;                      // secant = 1-D BFGS step
                const double cap = 8.0 * fabs(dx);           // keep extrapolation bounded
                if (fabs(xn - xb) > cap) xn = xb - sgn(gb) * cap;
            } else {
                xn = xb - sgn(gb) * 2.0 * fabs(dx);          // non-convex stretch: keep walking downhill
            }
            xn = fmin(fmax(xn, prm.lo), prm.hi);
        }
        if (fabs(xn - xb) <= tolx) {
            xres = xn;
            active = false;
            continue;
        }
        xt = xn;
    }
    if (active) fail = true;  // evaluation budget exhausted
    if (hint_out != nullptr && valid && grp.si == 0) {
        hint_out[0] = xres;
        hint_out[1] = (xb != xa) ? (gb - ga) / (xb - xa) : __builtin_nan("");
    }
    if (valid && grp.si == 0) {
        *alpha_out = exp(xres);
        *conv_out = fail ? 0.0 : 1.0;
        *status_out = fail ? kAlphaNeedsGrid : kAlphaOk;
    }
}

template <int P>
PDQ_HD void alpha_gene(const Group& grp, const DesignS& d, const AlphaParams& prm, const int64_t* y, int64_t ld,
                       const double* mu, int64_t ld_mu, double alpha_hat, double* alpha_out, double* conv_out,
                       int* status_out, bool valid, double* psi_tab, const double* hint_in = nullptr, double* hint_out = nullptr) {
    alpha_search(
        grp, prm, alpha_hat,
        [&](double x, double xhat, double* curv) { return alpha_dloss<P>(grp, d, prm, y, ld, mu, ld_mu, x, xhat, psi_tab, curv); },
        alpha_out, conv_out, status_out, valid, hint_in, hint_out);
}

// grid fallback (grid_search.py:54-142): 100-point grid on [lo, hi], then 100 points on +-1 cell around the
// best; always cr_reg=True, prior_reg=False because the reference's call drops those flags (utils.py:558-562).
// `loss(x)` = alpha_loss with cr_reg on and no prior
template <class Loss>
PDQ_HD void alpha_grid_search(const Group& grp, double lo, double hi, Loss&& loss, double* alpha_out, bool valid) {
    const int K = 100;
    const double delta = (hi - lo) / (double)(K - 1);
    double best = 0.0, bestx = lo;
    for (int k = 0; k < K; ++k) {
        const double x = (k == K - 1) ? hi : fma((double)k, delta, lo);
        const double f = loss(x);
        if (k == 0 || f < best) { best = f; bestx = x; }  // np.argmin: first minimum, NaN-free case
    }
    const double flo = bestx - delta, fhi = bestx + delta;
    const double fd = (fhi - flo) / (double)(K - 1);
    double bestf = flo;
    for (int k = 0; k < K; ++k) {
        const double x = (k == K - 1) ? fhi : fma((double)k, fd, flo);
        const double f = loss(x);
        if (k == 0 || f < best) { best = f; bestf = x; }
    }
    if (valid && grp.si == 0) *alpha_out = exp(bestf);
}

template <int P>
PDQ_HD void alpha_grid_gene(const Group& grp, const DesignS& d, double lo, double hi, const int64_t* y, int64_t ld,
                            const double* mu, int64_t ld_mu, double* alpha_out, bool valid) {
    alpha_grid_search(
        grp, lo, hi, [&](double x) { return alpha_loss<P>(grp, d, 1, 0, 1.0, y, ld, mu, ld_mu, x, 0.0); }, alpha_out, valid);
}

// final dispersion of one gene (dds.py:918-932): the clipped MAP estimate, but a gene whose genewise estimate lies more than
// 2 sd of the log residuals above the trend keeps its (clipped) genewise value.  The one statement of the rule: the elementwise
// kernel and the fused MAP -> LFC launch both call it.
PDQ_HD double select_disp(double gw, double mp, double fitted, double squared_logres, double lo, double hi, bool& outlier) {
    double g = gw, m = mp;
    g = (g < lo) ? lo : ((g > hi) ? hi : g);
    m = (m < lo) ? lo : ((m > hi) ? hi : m);
    outlier = log(g) > log(fitted) + 2.0 * sqrt(squared_logres);
    return outlier ? g : m;
}

// =============================================================================================
// (a5) fit_rough_dispersions (utils.py:814-853) / fit_moments_dispersions (utils.py:856-885)
// `Y` abstracts where normalised counts come from: a float64 (N,G) array (the plugin call) or raw
// int64 counts divided by the staged size factors on the fly (resident pipeline).
// =============================================================================================
struct NormedF64 {
    const double* p;
    int64_t ld;
    PDQ_HD double at(const DesignS&, int n) const { return p[n * ld]; }
};
struct NormedFromCounts {
    const int64_t* p;
    int64_t ld;
    PDQ_HD double at(const DesignS& d, int n) const { return (double)p[n * ld] / d.sf[n * d.RS]; }
};

template <int P, class Y>
PDQ_HD double rough_disp_gene(const Group& grp, const DesignS& d, const SmallMat<P>& pinv, const Y& yy) {
    double v[P];
PDQ_UNROLL_P
    for (int j = 0; j < P; ++j) v[j] = 0.0;
    for (int n = grp.si; n < d.N; n += grp.T) {
        double x[P];
        load_x<P>(d, n, x);
        const double t = yy.at(d, n);
PDQ_UNROLL_P
        for (int j = 0; j < P; ++j) v[j] = fma(x[j], t, v[j]);
    }
    group_sum_vec<P>(grp, v);
    double beta[P];
PDQ_UNROLL_P
    for (int i = 0; i < P; ++i) {
        double s = 0.0;
PDQ_UNROLL_P
        for (int j = 0; j < P; ++j) s = fma(pinv.v[i * P + j], v[j], s);
        beta[i] = s;
    }
    double acc = 0.0;
    for (int n = grp.si; n < d.N; n += grp.T) {
        double x[P];
        load_x<P>(d, n, x);
        double yh = 0.0;
PDQ_UNROLL_P
        for (int j = 0; j < P; ++j) yh = fma(x[j], beta[j], yh);
        yh = (yh < 1.0) ? 1.0 : yh;  // np.maximum(y_hat, 1)
        const double e = yy.at(d, n) - yh;
        acc += (e * e - yh) / (yh * yh);
    }
    acc = grp.sum(acc) / (double)(d.N - P);
    return (acc < 0.0) ? 0.0 : acc;  // np.maximum(alpha_rde, 0)
}

// Resident pipeline: rough + moments estimators, their min/clip (dds.py:1140-1162), the normalised mean (dds.py:708) and --
// because lin_reg_mu is the SAME least-squares projection of counts/sf (utils.py:711-713 vs :846-848) -- optionally the
// initial mu_hat = max(sf * X beta, min_mu) (utils.py:682-715), in two sweeps over the gene instead of six.  Returns the clipped
// start value, the same in every lane of the group (k_mom_alpha hands it to the dispersion search in registers).
template <int P>
PDQ_HD double mom_fused_gene(const Group& grp, const DesignS& d, const SmallMat<P>& pinv, const int64_t* y, int64_t ld,
                           double s_mean_inv, double min_disp, double max_disp, double min_mu, double* alpha_out,
                           double* mean_out, double* mu_out, int64_t ld_out, bool valid) {
    double v[P];
PDQ_UNROLL_P
    for (int j = 0; j < P; ++j) v[j] = 0.0;
    double s = 0.0;
    const int64_t ystep = (int64_t)grp.T * ld;
    const int64_t* yp = y + (int64_t)grp.si * ld;
    walk4(grp, d.N, yp, ystep, [&](int n, int64_t c) {
        double x[P];
        load_x<P>(d, n, x);
        const double t = fast_div((double)c, d.sf[n * d.RS]);  // <= 1 ulp from counts / sf
        s += t;
PDQ_UNROLL_P
        for (int j = 0; j < P; ++j) v[j] = fma(x[j], t, v[j]);
    });
    group_sum_vec<P>(grp, v);
    const double m = grp.sum(s) / (double)d.N;
    double beta[P];
PDQ_UNROLL_P
    for (int i = 0; i < P; ++i) {
        double acc = 0.0;
PDQ_UNROLL_P
        for (int j = 0; j < P; ++j) acc = fma(pinv.v[i * P + j], v[j], acc);
        beta[i] = acc;
    }
    double rough = 0.0, ss = 0.0;
    walk4(grp, d.N, yp, ystep, [&](int n, int64_t c) {
        double x[P];
        load_x<P>(d, n, x);
        double fit = 0.0;
PDQ_UNROLL_P
        for (int j = 0; j < P; ++j) fit = fma(x[j], beta[j], fit);
        const double t = fast_div((double)c, d.sf[n * d.RS]);  // <= 1 ulp from counts / sf
        const double yh = (fit < 1.0) ? 1.0 : fit;  // np.maximum(y_hat, 1)
        const double e = t - yh;
        rough += fast_div(e * e - yh, yh * yh);
        const double dm = t - m;
        ss = fma(dm, dm, ss);
        if (mu_out && valid) {
            const double mu = d.sf[n * d.RS] * fit;
            mu_out[(int64_t)n * ld_out] = (mu < min_mu) ? min_mu : mu;
        }
    });
    rough = grp.sum(rough) / (double)(d.N - P);
    rough = (rough < 0.0) ? 0.0 : rough;  // np.maximum(alpha_rde, 0)
    const double var = grp.sum(ss) / (double)(d.N - 1);
    double mde = (var - s_mean_inv * m) / (m * m);
    if (!(mde == mde)) mde = 0.0;  // np.nan_to_num
    else if (mde > 1.7976931348623157e308) mde = 1.7976931348623157e308;
    else if (mde < -1.7976931348623157e308) mde = -1.7976931348623157e308;
    double a = (mde < rough) ? mde : rough;                                // np.minimum (dds.py:1158)
    a = (a < min_disp) ? min_disp : ((a > max_disp) ? max_disp : a);       // np.clip (dds.py:1161)
    if (valid && grp.si == 0) {
        *alpha_out = a;
        *mean_out = m;
    }
    return a;
}

// returns the moments estimate; `mean_out` = per-gene mean of the normalised counts, `all_zero` flag
template <class Y>
PDQ_HD double moments_disp_gene(const Group& grp, const DesignS& d, const Y& yy, double s_mean_inv, double& mean_out,
                                bool& all_zero) {
    double s = 0.0;
    bool nz = false;
    for (int n = grp.si; n < d.N; n += grp.T) {
        const double t = yy.at(d, n);
        s += t;
        nz = nz || (t != 0.0);
    }
    s = grp.sum(s);
    all_zero = !(grp.sum(nz ? 1.0 : 0.0) > 0.0);
    const double m = s / (double)d.N;
    double ss = 0.0;
    for (int n = grp.si; n < d.N; n += grp.T) {
        const double e = yy.at(d, n) - m;
        ss = fma(e, e, ss);
    }
    const double var = grp.sum(ss) / (double)(d.N - 1);  // ddof=1
    mean_out = m;
    double a = (var - s_mean_inv * m) / (m * m);
    // np.nan_to_num: NaN -> 0, +-inf -> +-DBL_MAX
    if (!(a == a)) a = 0.0;
    else if (a > 1.7976931348623157e308) a = 1.7976931348623157e308;
    else if (a < -1.7976931348623157e308) a = -1.7976931348623157e308;
    return a;
}

}  // namespace pdq

namespace pdq {

// =============================================================================================
// (f-1) Cook's distances -- dds.py:986-1040 with the trimmed-moments dispersion of utils.py:567-679, 914-960,
// and the two per-gene decisions the orchestrator derives from them (dds.py:1066-1110, :1320-1323).
// Cells = groups of samples with identical design rows that hold >= 3 replicates; `order` lists the samples of those
// cells cell by cell, `cell_start` (n_cells + 1 entries) delimits them.  When no cell qualifies the whole sample set is
// one "cell" with the fixed trim 1/8 (utils.py:650-679 `trimmed_variance`).
// Trimmed means are exact order-statistic sums: the rank of every value inside its cell is counted against all other
// members (ties broken by position, like a stable sort); O(n_c^2 / T) comparisons per lane, values staged in shared memory.
// =============================================================================================
struct CellPlan {
    const int* order;       // [n_in_cells] sample indices, grouped by cell
    const int* cell_start;  // [n_cells + 1]
    int n_cells;
    int global_mode;        // 1: no cell has 3 replicates -> single cell, trim 1/8, scale 1.51
};

PDQ_HD void trim_class(int nc, bool global_mode, int& ntrim, double& scale) {
    if (global_mode) {
        ntrim = (int)floor((double)nc * 0.125);
        scale = 1.51;
        return;
    }
    const int k = (nc >= 23.5) ? 2 : ((nc >= 3.5) ? 1 : 0);             // utils.py:621-623
    const double ratio = (k == 2) ? (1.0 / 8.0) : ((k == 1) ? (1.0 / 4.0) : (1.0 / 3.0));
    ntrim = (int)floor((double)nc * ratio);
    scale = (k == 2) ? 1.51 : ((k == 1) ? 1.86 : 2.04);
}

// mean of v[s:e) after dropping the ntrim smallest and ntrim largest entries (np.sort + slice + mean), by SELECTION: every lane
// sorts its own strided share of the cell in place (insertion sort, m = n_c / T entries), then the group pops the smallest and
// the largest remaining head ntrim times (one argmin / argmax butterfly each); what is left between the lanes' cursors is the
// kept set, summed directly.  O(m^2 + ntrim log T) per lane instead of the O(n_c^2 / T) rank counting of round 1.  Ties carry equal values, so which of them is dropped does not matter.
// The cell is left permuted (callers only need it as a multiset).
PDQ_HD double trimmed_mean_cell(const Group& grp, double* v, int s, int e, int ntrim) {
    const int nc = e - s, T = grp.T;
    const int m = (nc - grp.si + T - 1) / T;        // this lane's entries: v[s + si + k T], k < m   (m <= 0: none)
    double* mine = v + s + grp.si;
    for (int i = 1; i < m; ++i) {
        const double x = mine[i * T];
        int j = i - 1;
        while (j >= 0 && mine[j * T] > x) {
            mine[(j + 1) * T] = mine[j * T];
            --j;
        }
        mine[(j + 1) * T] = x;
    }
    int lo = 0, hi = m > 0 ? m : 0;
    for (int k = 0; k < ntrim; ++k) {                // uniform trip count across the warp: the butterflies vote
        const double head = lo < hi ? mine[lo * T] : 1.7976931348623157e308 * 10.0;
        if (grp.argext(head, false) == grp.si) ++lo;
        const double tail = lo < hi ? mine[(hi - 1) * T] : -1.7976931348623157e308 * 10.0;
        if (grp.argext(tail, true) == grp.si) --hi;
    }
    double part = 0.0;
    for (int k = lo; k < hi; ++k) part += mine[k * T];
    return grp.sum(part) / (double)(nc - 2 * ntrim);
}

// `p` design columns (cooks_gene<P> for the narrow kernels, the wide-design kernels pass theirs)
PDQ_HD void cooks_gene_cols(const Group& grp, const DesignS& d, int p, const CellPlan& plan, const int64_t* y, int64_t ld,
                            const double* mu, const double* hat, int64_t ld2, double cutoff, double* vals /* smem: n_in_cells */,
                            double* sq /* smem: n_in_cells */, double* cooks_out, int64_t ld_out, double* disp_out,
                            double* outlier_out, double* replaced_out, bool valid) {
    const int nf = plan.cell_start[plan.n_cells];
    // normalised counts: mean over ALL samples, and the grouped copy of the samples that sit in cells
    double msum = 0.0;
    for (int n = grp.si; n < d.N; n += grp.T) msum += (double)y[n * ld] / d.sf[n * d.RS];
    const double m_all = grp.sum(msum) / (double)d.N;
    grp.sync();
    for (int i = grp.si; i < nf; i += grp.T) {
        const int n = plan.order[i];
        vals[i] = (double)y[n * ld] / d.sf[n * d.RS];
    }
    grp.sync();
    double v = -1.7976931348623157e308;
    for (int c = 0; c < plan.n_cells; ++c) {
        const int s = plan.cell_start[c], e = plan.cell_start[c + 1];
        int ntrim;
        double scale;
        trim_class(e - s, plan.global_mode != 0, ntrim, scale);
        const double tm = trimmed_mean_cell(grp, vals, s, e, ntrim);
        for (int i = s + grp.si; i < e; i += grp.T) {
            const double dlt = vals[i] - tm;
            sq[i] = dlt * dlt;
        }
        grp.sync();
        const double tv = scale * trimmed_mean_cell(grp, sq, s, e, ntrim);
        v = (tv > v || tv != tv) ? tv : v;  // np.max propagates NaN
    }
    double alpha = (v - m_all) / (m_all * m_all);
    alpha = (alpha < 0.04) ? 0.04 : alpha;  // np.maximum(alpha, 0.04): NaN stays NaN
    // Cook's distance per sample, running maximum (first occurrence) and the cutoff tests
    double best = -1.0, best_use = -1.0;
    int best_n = 0x7fffffff;
    bool any_all = false;
    for (int n = grp.si; n < d.N; n += grp.T) {
        const double yv = (double)y[n * ld], m = mu[n * ld2], h = hat[n * ld2];
        const double V = fma(m * m, alpha, m);
        const double omh = 1.0 - h;
        const double ck = (yv - m) * (yv - m) / V / (double)p * (h / (omh * omh));
        if (valid && cooks_out) cooks_out[n * ld_out] = ck;
        any_all = any_all || (ck > cutoff);
        if (ck > best) {  // lanes visit their samples in increasing n: strict > keeps the first maximum
            best = ck;
            best_n = n;
        }
    }
    // samples in qualifying cells decide the p-value filter (dds.py:1077-1092)
    if (!plan.global_mode) {
        for (int i = grp.si; i < nf; i += grp.T) {
            const int n = plan.order[i];
            const double yv = (double)y[n * ld], m = mu[n * ld2], h = hat[n * ld2];
            const double V = fma(m * m, alpha, m);
            const double omh = 1.0 - h;
            const double ck = (yv - m) * (yv - m) / V / (double)p * (h / (omh * omh));
            best_use = ck > best_use ? ck : best_use;
        }
    }
    // group-wide argmax (value, then smaller sample index) and flags
#if defined(__CUDA_ARCH__)
    for (int off = 16; off >= grp.gpw; off >>= 1) {
        const double ob = __shfl_xor_sync(0xffffffffu, best, off);
        const int on = __shfl_xor_sync(0xffffffffu, best_n, off);
        if (ob > best || (ob == best && on < best_n)) {
            best = ob;
            best_n = on;
        }
        const double ou = __shfl_xor_sync(0xffffffffu, best_use, off);
        best_use = ou > best_use ? ou : best_use;
    }
#elif defined(PDQ_EMU_LANES)
    pdq_emu::lane_argmax(grp.si, grp.T, best, best_n, best_use);
#endif
    const bool replaced = grp.sum(any_all ? 1.0 : 0.0) > 0.0;
    bool outlier = best_use > cutoff;
    // a gene is not an outlier when 3 or more samples have larger counts than the sample with the largest distance
    const long long ypos = y[(int64_t)(best_n == 0x7fffffff ? 0 : best_n) * ld];
    double larger = 0.0;
    for (int n = grp.si; n < d.N; n += grp.T) larger += (y[n * ld] > ypos) ? 1.0 : 0.0;
    larger = grp.sum(larger);
    outlier = outlier && (larger < 3.0);
    if (valid && grp.si == 0) {
        *disp_out = alpha;
        *outlier_out = outlier ? 1.0 : 0.0;
        *replaced_out = replaced ? 1.0 : 0.0;
    }
}

template <int P>
PDQ_HD void cooks_gene(const Group& grp, const DesignS& d, const CellPlan& plan, const int64_t* y, int64_t ld, const double* mu,
                       const double* hat, int64_t ld2, double cutoff, double* vals, double* sq, double* cooks_out, int64_t ld_out,
                       double* disp_out, double* outlier_out, double* replaced_out, bool valid) {
    cooks_gene_cols(grp, d, P, plan, y, ld, mu, hat, ld2, cutoff, vals, sq, cooks_out, ld_out, disp_out, outlier_out, replaced_out, valid);
}

}  // namespace pdq
