// pdq_wide.cu -- per-gene kernels and their launchers (`_wide`) for designs of PDQ_MAX_P + 1 .. PDQ_MAX_P_WIDE columns (opt-in
// per context: pdq_set_wide_designs) and of PDQ_MAX_P_WIDE + 1 .. PDQ_MAX_P_LARGE columns (a second opt-in on top of it:
// pdq_set_large_designs).
//
// The kernels of pdq_kernels.cu keep one gene's p x p state per LANE: in registers for p <= 8, in local memory for 9..16.  At
// p = 64 one packed symmetric matrix is 16.6 KB, so that layout does not scale.  Here one TEAM of W warps owns one gene (one team
// per block, one gene per block), and the gene's matrices live once, in the block's dynamic shared memory (DESIGN.md §3):
//   * per-sample work is split over the team's threads: chunks of 32 W samples, thread t takes sample n0 + t and stages its
//     weight (and working response) in shared memory;
//   * the rank-(32 W) update of a packed matrix from one chunk is split over its entries (thread t owns entries t, t + 32 W, ...);
//     vectors such as X^T W z are split over their components;
//   * the Cholesky factorisation, the triangular solves and the inverse are cooperative, one team barrier per column step;
//   * sums and votes are warp butterflies, combined across the warps through per-warp slots in shared memory.
// These building blocks (Team<W>, the workspace, the chunk accumulators, the Cholesky family, the Wald SE, wdot / wmaxabs) are in
// pdq_team.cuh, where the GPU probe's team unit tests them directly at every team width.
// The 17..64 tier runs W = 1 (a warp barrier is enough).  At p = 128 the workspace is ~204 KB, so one block fits per SM: the
// 65..128 tier runs W = 2, 4 or 8 warps per gene (large_warps, from each kernel's workspace) to keep the SM's FP64 pipes busy.
// with_warps picks W for a design.  apeGLM shrinkage of that tier is a further opt-in (pdq_set_large_shrink).
// At every width the kernels read the Wald ridge and contrast from a device buffer next to the design pack
// (DesignDev::wald_dev; at 128 columns they exceed the 32 KB kernel-parameter limit).  Passes whose work does not grow with p
// (moments, mu from LFCs, Cook's distances) run the W = 1 kernels at every width.
// The design pack is read from global memory (it stays in L1 / L2).  The per-gene semantics are those of pdq_gene.cuh -- start
// values, ridge, stopping rules, optimiser branch, dispersion search and grid, Wald alternatives, Cook's distances -- written
// against libdevice's exp / log and the series of pdq_math.cuh instead of the table-driven cores; parity is to the reference's
// tolerances, not bit for bit with the narrow kernels (which never run the same designs).
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "pdq_gene.cuh"
#include "pdq_internal.h"
#include "pdq_launch.cuh"
#include "pdq_shrink.cuh"
#include "pdq_team.cuh"

namespace pdq {
namespace {

// ---------------------------------------------------------------------------------------------
// Wald test from M = X^T W X (wald_inverse + wald_contrast of pdq_gene.cuh)
// ---------------------------------------------------------------------------------------------
// ridge (lower triangle of the caller's p x p matrix, packed: the only part wald_inverse reads) and contrast in device memory
// (DesignDev::wald_dev, written by put_wald)
struct WaldRef {
    const double* ridge;
    const double* contrast;
    double lfc_null;
    int alt;
};

// statistic and p-value of alternative `alt` given SE (every lane, replicated; the same expressions as wald_contrast)
__device__ void wald_alt(const double* c, const double* b, int p, double se, double t0, int alt, double& pv, double& stat) {
    auto greater = [&](double t, double& s, double& q) {
        s = 0.0;
        for (int j = 0; j < p; ++j) s = fma(c[j], fmax((b[j] - t) / se, 0.0), s);
        q = norm_sf(s);
    };
    auto less = [&](double t, double& s, double& q) {
        s = 0.0;
        for (int j = 0; j < p; ++j) s = fma(c[j], fmin((b[j] - t) / se, 0.0), s);
        q = norm_sf(fabs(s));
    };
    if (alt == 0) {
        double s = 0.0;
        for (int j = 0; j < p; ++j) s = fma(c[j], b[j] - t0, s);
        stat = s / se;
        pv = 2.0 * norm_sf(fabs(stat));
    } else if (alt == 1) {
        double s = 0.0;
        for (int j = 0; j < p; ++j) s = fma(c[j], sgn(b[j]) * fmax((fabs(b[j]) - t0) / se, 0.0), s);
        stat = s;
        pv = 2.0 * norm_sf(fabs(s));
    } else if (alt == 2) {
        double sa, pa, sb, pb;
        greater(-fabs(t0), sa, pa);
        less(fabs(t0), sb, pb);
        stat = (fabs(sb) < fabs(sa)) ? sb : sa;
        pv = (pb > pa) ? pb : pa;
    } else if (alt == 3) {
        greater(t0, stat, pv);
    } else {
        less(t0, stat, pv);
    }
}

template <int W>
__device__ void wald_finish_w(const double* M, const WaldRef& w, const double* beta, Ws& ws, double* p_out, double* stat_out,
                              double* se_out) {
    using T = Team<W>;
    wald_inverse_w<W>(M, w.ridge, ws);
    const double se = wald_se_w<W>(M, w.contrast, ws);
    double pv, stat;
    wald_alt(w.contrast, beta, ws.p, se, w.lfc_null, w.alt, pv, stat);
    if (T::tid() == 0) {
        *p_out = pv;
        *stat_out = stat;
        *se_out = se;
    }
}

// ---------------------------------------------------------------------------------------------
// kernels: one team of W warps per block, one gene per block
// ---------------------------------------------------------------------------------------------
struct WideBase {
    const double* pack;  // design pack (global)
    const double* pinv;  // (X^T X)^+ p x p row-major (global)
    int N, p, G;
};

struct LinArgs {
    WideBase b;
    const int64_t* counts;
    int64_t ld;
    double min_mu;
    double* mu;
    int64_t ld_out;
};

// v = X^T t with t = y / sf per sample (the projection lin_reg_mu / fit_rough_dispersions start from); returns sum t
template <int W, class Y>
__device__ double project(const DesignS& d, int p, const Y& yy, Ws& ws, double* v) {
    using T = Team<W>;
    wfill<W>(v, p, 0.0);
    double s = 0.0;
    for (int n0 = 0; n0 < d.N; n0 += T::NT) {
        const int n = n0 + T::tid();
        const double t = n < d.N ? yy.at(d, n) : 0.0;
        s += t;
        T::sync();
        ws.cz[T::tid()] = t;
        T::sync();
        vec_chunk<W>(d, p, n0, min(T::NT, d.N - n0), ws.cz, v);
    }
    T::sync();
    return T::sum(s);
}

template <int W>
__global__ void __launch_bounds__(32 * W, W == 1 ? 0 : 1) k_wide_lin_reg_mu(const __grid_constant__ LinArgs a) {
    using T = Team<W>;
    extern __shared__ __align__(16) double wsm[];
    Ws ws = carve<W>(wsm, a.b.p);
    const int g = blockIdx.x, p = a.b.p;
    const DesignS d = design_of(a.b.pack, a.b.N, p);
    project<W>(d, p, NormedFromCounts{a.counts + g, a.ld}, ws, ws.v[0]);
    apply_pinv<W>(a.b.pinv, ws.v[0], ws.v[1], p);
    for (int n = T::tid(); n < d.N; n += T::NT) {
        const double m = d.sf[n * d.RS] * xdot(row_of(d, n), ws.v[1], p);
        a.mu[(int64_t)n * a.ld_out + g] = (m < a.min_mu) ? a.min_mu : m;  // np.maximum (NaN propagates)
    }
}

struct MomArgsW {
    WideBase b;
    const double* normed;   // rough / moments: (N, G) normalised counts
    const int64_t* counts;  // mom_from_counts: raw counts
    int64_t ld;
    double s_mean_inv, min_disp, max_disp, min_mu;
    double *alpha, *aux;    // aux: all-zero flags (moments) or normalised means (mom_from_counts)
    double* mu;             // mom_from_counts: initial mu_hat, or nullptr
    int64_t ld_mu;
};

// fit_rough_dispersions (rough_disp_gene); `fit` receives nothing, beta stays in ws.v[1]
template <int W, class Y>
__device__ double rough_w(const DesignS& d, const double* pinv, int p, const Y& yy, Ws& ws, double* mean, double* mu_out,
                          int64_t ld_mu, double min_mu) {
    using T = Team<W>;
    const double s = project<W>(d, p, yy, ws, ws.v[0]);
    apply_pinv<W>(pinv, ws.v[0], ws.v[1], p);
    const double m = s / (double)d.N;
    double acc = 0.0, ss = 0.0;
    for (int n = T::tid(); n < d.N; n += T::NT) {
        const double fit = xdot(row_of(d, n), ws.v[1], p);
        const double t = yy.at(d, n);
        const double yh = (fit < 1.0) ? 1.0 : fit;  // np.maximum(y_hat, 1)
        const double e = t - yh;
        acc += (e * e - yh) / (yh * yh);
        const double dm = t - m;
        ss = fma(dm, dm, ss);
        if (mu_out) {
            const double mu = d.sf[n * d.RS] * fit;
            mu_out[(int64_t)n * ld_mu] = (mu < min_mu) ? min_mu : mu;
        }
    }
    acc = T::sum(acc) / (double)(d.N - p);
    if (mean) *mean = T::sum(ss);  // sum of squared deviations from the mean (mom_from_counts)
    return (acc < 0.0) ? 0.0 : acc;  // np.maximum(alpha_rde, 0)
}

template <int W>
__global__ void __launch_bounds__(32 * W, W == 1 ? 0 : 1) k_wide_rough(const __grid_constant__ MomArgsW a) {
    using T = Team<W>;
    extern __shared__ __align__(16) double wsm[];
    Ws ws = carve<W>(wsm, a.b.p);
    const int g = blockIdx.x;
    const DesignS d = design_of(a.b.pack, a.b.N, a.b.p);
    const double r = rough_w<W>(d, a.b.pinv, a.b.p, NormedF64{a.normed + g, a.ld}, ws, nullptr, nullptr, 0, 0.0);
    if (T::tid() == 0) a.alpha[g] = r;
}

__global__ void __launch_bounds__(32) k_wide_moments(const __grid_constant__ MomArgsW a) {
    const int g = blockIdx.x;
    const DesignS d = design_of(a.b.pack, a.b.N, a.b.p);
    const Group grp{lane_id(), 32, 1};
    double mean;
    bool all_zero;
    const double m = moments_disp_gene(grp, d, NormedF64{a.normed + g, a.ld}, a.s_mean_inv, mean, all_zero);
    if (lane_id() == 0) {
        a.alpha[g] = m;
        if (a.aux) a.aux[g] = all_zero ? 1.0 : 0.0;
    }
}

// rough + moments, their min / clip, the normalised mean and (lin_reg_mu branch) mu_hat: mom_fused_gene
template <int W>
__global__ void __launch_bounds__(32 * W, W == 1 ? 0 : 1) k_wide_mom_from_counts(const __grid_constant__ MomArgsW a) {
    using T = Team<W>;
    extern __shared__ __align__(16) double wsm[];
    Ws ws = carve<W>(wsm, a.b.p);
    const int g = blockIdx.x;
    const DesignS d = design_of(a.b.pack, a.b.N, a.b.p);
    double ss;
    const NormedFromCounts yy{a.counts + g, a.ld};
    // the mean is needed inside the sweep: one projection pass for it first (rough_w recomputes the same sums)
    const double m = project<W>(d, a.b.p, yy, ws, ws.v[0]) / (double)d.N;
    const double rough = rough_w<W>(d, a.b.pinv, a.b.p, yy, ws, &ss, a.mu ? a.mu + g : nullptr, a.ld_mu, a.min_mu);
    const double var = ss / (double)(d.N - 1);
    double mde = (var - a.s_mean_inv * m) / (m * m);
    if (!(mde == mde)) mde = 0.0;  // np.nan_to_num
    else if (mde > 1.7976931348623157e308) mde = 1.7976931348623157e308;
    else if (mde < -1.7976931348623157e308) mde = -1.7976931348623157e308;
    if (T::tid() == 0) {
        double al = (mde < rough) ? mde : rough;                                    // np.minimum (dds.py:1158)
        al = (al < a.min_disp) ? a.min_disp : ((al > a.max_disp) ? a.max_disp : al);  // np.clip (dds.py:1161)
        a.alpha[g] = al;
        a.aux[g] = m;
    }
}

struct MuLfcArgsW {
    WideBase b;
    const double* lfc;
    double* mu;
    int64_t ld_out;
};

__global__ void __launch_bounds__(32) k_wide_mu_from_lfc(const __grid_constant__ MuLfcArgsW a) {
    const int g = blockIdx.x, p = a.b.p;
    const DesignS d = design_of(a.b.pack, a.b.N, p);
    const double* b = a.lfc + (int64_t)g * p;
    for (int n = lane_id(); n < d.N; n += 32) a.mu[(int64_t)n * a.ld_out + g] = exp(xdot(row_of(d, n), b, p)) * d.sf[n * d.RS];
}

// ---------------------------------------------------------------------------------------------
// irls (irls_gene + irls_optimizer_gene)
// ---------------------------------------------------------------------------------------------
struct IrlsArgsW {
    WideBase b;
    IrlsParams prm;
    const int64_t* counts;
    int64_t ld;
    const double* disp;
    double *beta, *mu, *hat, *conv;
    int64_t ld_out;
    int* status;
    int* n_fallback;
    int force;
    int with_wald;
    WaldRef wald;
    double *wald_p, *wald_stat, *wald_se;
};

// start value (utils.py:349-357) into `beta`; also returns sum lgamma(y + 1) - lgamma(y + r) through lgsum when asked
template <int W = 1>
__device__ void irls_start(const DesignS& d, const double* pinv, int p, int full_rank, const int64_t* y, int64_t ld, double r,
                           Ws& ws, double* beta, double* lgsum) {
    using T = Team<W>;
    double* v = ws.v[0];
    wfill<W>(v, p, 0.0);
    double logmean = 0.0, lg = 0.0;
    for (int n0 = 0; n0 < d.N; n0 += T::NT) {
        const int n = n0 + T::tid();
        double t = 0.0;
        if (n < d.N) {
            const double yv = (double)y[(int64_t)n * ld];
            const double q = yv / d.sf[n * d.RS];
            if (full_rank) t = log(q + 0.1);
            else logmean += log(q);
            if (lgsum) lg += lgamma_pos(yv + 1.0) - lgamma_pos(yv + r);
        }
        T::sync();
        ws.cz[T::tid()] = t;
        T::sync();
        if (full_rank) vec_chunk<W>(d, p, n0, min(T::NT, d.N - n0), ws.cz, v);
    }
    T::sync();
    if (lgsum) *lgsum = T::sum(lg);
    if (full_rank) {
        apply_pinv<W>(pinv, v, beta, p);
    } else {
        logmean = T::sum(logmean);
        wfill<W>(beta, p, 0.0);
        T::sync();
        if (T::tid() == 0) beta[0] = logmean / (double)d.N;
        T::sync();
    }
}

// one IRLS sweep at `beta`: A = X^T W X, b = X^T W z (W, z from the clamped mu); returns S = sum (y + r) log(r + mu) - y log(mu)
template <int W = 1>
__device__ double irls_sweep_w(const DesignS& d, int p, const int64_t* y, int64_t ld, const double* beta, double alpha, double r,
                               double min_mu, double log_min_mu, Ws& ws, double* A, double* b) {
    using T = Team<W>;
    wfill<W>(A, p * (p + 1) / 2, 0.0);
    wfill<W>(b, p, 0.0);
    double S = 0.0;
    for (int n0 = 0; n0 < d.N; n0 += T::NT) {
        const int n = n0 + T::tid();
        double wt = 0.0, Wz = 0.0;
        if (n < d.N) {
            const double* x = row_of(d, n);
            const double yv = (double)y[(int64_t)n * ld];
            const double eta = xdot(x, beta, p);
            const double sfn = x[p], lsfn = x[p + 1];
            const double mu_raw = sfn * exp(eta);
            const bool cl = mu_raw < min_mu;
            const double mu = cl ? min_mu : mu_raw;
            const double lmu = cl ? log_min_mu : (eta + lsfn);
            const double iden = 1.0 / fma(mu, alpha, 1.0);
            wt = mu * iden;
            Wz = fma(yv - mu, iden, wt * (lmu - lsfn));
            S += fma(yv + r, log(r + mu), -yv * lmu);
        }
        T::sync();
        ws.cw[T::tid()] = wt;
        ws.cz[T::tid()] = Wz;
        T::sync();
        const int cnt = min(T::NT, d.N - n0);
        rank_chunk<W>(d, p, n0, cnt, ws.cw, A);
        vec_chunk<W>(d, p, n0, cnt, ws.cz, b);
    }
    T::sync();
    return T::sum(S);
}

// mu (unclamped) and hat = W x^T H x with H = (A + ridge)^-1 (A: W from the clamped mu of `beta`); H ends in ws.L
template <int W = 1>
__device__ void irls_outputs(const DesignS& d, int p, const double* beta, double alpha, double min_mu, Ws& ws, const double* A,
                             double* mu_out, double* hat_out, int64_t ld_out) {
    using T = Team<W>;
    factor_ridged<W>(A, ws.L, p, kRidge, nullptr);
    chol_inverse_w<W>(ws.L, ws.Li, ws.L, p);
    for (int n = T::tid(); n < d.N; n += T::NT) {
        const double* x = row_of(d, n);
        const double mu_raw = x[p] * exp(xdot(x, beta, p));
        const double mu = (mu_raw < min_mu) ? min_mu : mu_raw;
        mu_out[(int64_t)n * ld_out] = mu_raw;
        hat_out[(int64_t)n * ld_out] = mu / fma(mu, alpha, 1.0) * quad_w(ws.L, x, p);
    }
}

// M = sum w x x^T with w = mu / (1 + mu alpha) of the UNCLAMPED (clamped = false) or clamped mu of `beta`
template <int W = 1>
__device__ void weight_matrix(const DesignS& d, int p, const double* beta, double alpha, double min_mu, bool clamp, Ws& ws,
                              double* M) {
    using T = Team<W>;
    wfill<W>(M, p * (p + 1) / 2, 0.0);
    for (int n0 = 0; n0 < d.N; n0 += T::NT) {
        const int n = n0 + T::tid();
        double wt = 0.0;
        if (n < d.N) {
            const double* x = row_of(d, n);
            const double mu_raw = x[p] * exp(xdot(x, beta, p));
            const double mu = (clamp && mu_raw < min_mu) ? min_mu : mu_raw;
            wt = mu / fma(mu, alpha, 1.0);
        }
        T::sync();
        ws.cw[T::tid()] = wt;
        T::sync();
        rank_chunk<W>(d, p, n0, min(T::NT, d.N - n0), ws.cw, M);
    }
    T::sync();
}

// f(beta) = nb_nll (mu-dependent part) + 0.5 ridge |beta|^2, its gradient g and Hessian H (irls_obj_sweep)
template <int W = 1>
__device__ double obj_sweep_w(const DesignS& d, int p, const int64_t* y, int64_t ld, const double* beta, double alpha, double r,
                              double min_mu, double log_min_mu, Ws& ws, double* g, double* H) {
    using T = Team<W>;
    wfill<W>(H, p * (p + 1) / 2, 0.0);
    wfill<W>(g, p, 0.0);
    double f = 0.0;
    for (int n0 = 0; n0 < d.N; n0 += T::NT) {
        const int n = n0 + T::tid();
        double gi = 0.0, hi = 0.0;
        if (n < d.N) {
            const double* x = row_of(d, n);
            const double yv = (double)y[(int64_t)n * ld];
            const double eta = xdot(x, beta, p);
            const double mu_raw = x[p] * exp(eta);
            const bool cl = mu_raw < min_mu;
            const double mu = cl ? min_mu : mu_raw;
            const double lmu = cl ? log_min_mu : (eta + x[p + 1]);
            f += fma(yv + r, log(r + mu), -yv * lmu);
            const double t = (r + yv) * mu / (r + mu);
            gi = t - yv;
            hi = t * r / (r + mu);
        }
        T::sync();
        ws.cw[T::tid()] = hi;
        ws.cz[T::tid()] = gi;
        T::sync();
        const int cnt = min(T::NT, d.N - n0);
        rank_chunk<W>(d, p, n0, cnt, ws.cw, H);
        vec_chunk<W>(d, p, n0, cnt, ws.cz, g);
    }
    T::sync();
    f = T::sum(f);
    for (int j = 0; j < p; ++j) f = fma(0.5 * kRidge * beta[j], beta[j], f);
    for (int j = T::tid(); j < p; j += T::NT) {
        g[j] = fma(kRidge, beta[j], g[j]);
        H[tri(j, j)] += kRidge;
    }
    T::sync();
    return f;
}

__device__ __forceinline__ bool is_fixed(double b, double g, double lo, double hi) { return (b <= lo && g > 0.0) || (b >= hi && g < 0.0); }

// the reference's L-BFGS-B branch (utils.py:374-413) as projected Newton: irls_optimizer_gene, every output written here
template <int W = 1>
__device__ void irls_optimizer_w(const IrlsArgsW& a, const DesignS& d, Ws& ws, int g) {
    using T = Team<W>;
    const int p = a.b.p, lane = T::tid();
    const IrlsParams& prm = a.prm;
    const int64_t* y = a.counts + g;
    const double alpha = a.disp[g], r = 1.0 / alpha, log_min_mu = log(prm.min_mu);
    double *beta = ws.v[1], *dir = ws.v[2], *gr = ws.v[3], *bt = ws.v[4], *gt = ws.v[5];
    irls_start<W>(d, a.b.pinv, p, prm.full_rank, y, a.ld, r, ws, beta, nullptr);
    for (int j = lane; j < p; j += T::NT) beta[j] = fmin(fmax(beta[j], prm.min_beta), prm.max_beta);
    T::sync();
    double f = obj_sweep_w<W>(d, p, y, a.ld, beta, alpha, r, prm.min_mu, log_min_mu, ws, gr, ws.A);
    bool ok = false;
    for (int it = 0; it < 100; ++it) {
        double pg = 0.0;
        for (int j = 0; j < p; ++j)
            if (!is_fixed(beta[j], gr[j], prm.min_beta, prm.max_beta)) pg = fmax(pg, fabs(gr[j]));
        if (pg <= 1e-9 * (1.0 + fabs(f)) || !(pg == pg)) {
            ok = (pg == pg);
            break;
        }
        // Newton direction on the free set: fixed rows / columns of H replaced by the identity
        T::sync();
        for (int i = lane; i < p; i += T::NT) {
            const bool fi = is_fixed(beta[i], gr[i], prm.min_beta, prm.max_beta);
            dir[i] = fi ? 0.0 : -gr[i];
            for (int j = 0; j <= i; ++j) {
                const bool fj = is_fixed(beta[j], gr[j], prm.min_beta, prm.max_beta);
                ws.L[tri(i, j)] = (i == j) ? (fi ? 1.0 : ws.A[tri(i, i)]) : ((fi || fj) ? 0.0 : ws.A[tri(i, j)]);
            }
        }
        chol_w<W>(ws.L, p);
        chol_solve_w<W>(ws.L, dir, p);
        double slope = 0.0;
        for (int j = 0; j < p; ++j) slope = fma(gr[j], dir[j], slope);
        if (!(slope < 0.0)) {  // not a descent direction (indefinite / NaN): steepest descent on the free set
            T::sync();
            for (int j = lane; j < p; j += T::NT) dir[j] = is_fixed(beta[j], gr[j], prm.min_beta, prm.max_beta) ? 0.0 : -gr[j];
            T::sync();
        }
        // backtracking line search with projection onto the box; the trial Hessian goes to ws.Li
        double step = 1.0, fn = f;
        bool accepted = false;
        for (int ls = 0; ls < 30; ++ls) {
            T::sync();
            for (int j = lane; j < p; j += T::NT) bt[j] = fmin(fmax(fma(step, dir[j], beta[j]), prm.min_beta), prm.max_beta);
            T::sync();
            double dec = 0.0;
            for (int j = 0; j < p; ++j) dec = fma(gr[j], bt[j] - beta[j], dec);
            const double ft = obj_sweep_w<W>(d, p, y, a.ld, bt, alpha, r, prm.min_mu, log_min_mu, ws, gt, ws.Li);
            if (ft <= f + 1e-4 * dec) {
                accepted = true;
                fn = ft;
                break;
            }
            step *= 0.5;
        }
        if (!accepted) {  // line search failed: res.success == False
            ok = false;
            break;
        }
        const double df = f - fn;
        f = fn;
        wcopy<W>(ws.A, ws.Li, p * (p + 1) / 2);
        wcopy<W>(gr, gt, p);
        wcopy<W>(beta, bt, p);
        T::sync();
        if (df <= 1e-15 * (1.0 + fabs(f))) {  // no further decrease possible in FP64
            ok = true;
            break;
        }
    }
    if (prm.fail_optimizer) ok = false;
    // (the two-column grid_fit_beta of utils.py:402-409 is never reached: p > 16 here)
    if (a.with_wald) {
        weight_matrix<W>(d, p, beta, alpha, prm.min_mu, false, ws, ws.A);
        wald_finish_w<W>(ws.A, a.wald, beta, ws, a.wald_p + g, a.wald_stat + g, a.wald_se + g);
    }
    weight_matrix<W>(d, p, beta, alpha, prm.min_mu, true, ws, ws.A);
    irls_outputs<W>(d, p, beta, alpha, prm.min_mu, ws, ws.A, a.mu + g, a.hat + g, a.ld_out);
    for (int j = lane; j < p; j += T::NT) a.beta[(int64_t)g * p + j] = beta[j];
    if (lane == 0) a.conv[g] = ok ? 1.0 : 0.0;
}

template <int W>
__global__ void __maxnreg__(224) k_wide_irls(const __grid_constant__ IrlsArgsW a) {
    using T = Team<W>;
    extern __shared__ __align__(16) double wsm[];
    Ws ws = carve<W>(wsm, a.b.p);
    const int g = blockIdx.x, p = a.b.p, lane = T::tid();
    const DesignS d = design_of(a.b.pack, a.b.N, p);
    const IrlsParams& prm = a.prm;
    const int64_t* y = a.counts + g;
    const double alpha = a.disp[g], r = 1.0 / alpha, Nd = (double)d.N, log_min_mu = log(prm.min_mu);
    double *b = ws.v[0], *beta = ws.v[1], *bh = ws.v[2];
    double lgsum;
    irls_start<W>(d, a.b.pinv, p, prm.full_rank, y, a.ld, r, ws, beta, &lgsum);
    const double C = Nd * r * log(alpha) + Nd * lgamma_pos(r) + lgsum;  // nb_nll = C + S(mu)
    double dev = 1000.0, ratio = 1.0;
    int it = 0, status = kIrlsOk;
    bool first = true;
    for (;;) {
        const double S = irls_sweep_w<W>(d, p, y, a.ld, beta, alpha, r, prm.min_mu, log_min_mu, ws, ws.A, b);
        if (!first) {
            const double old = dev;
            dev = -2.0 * (C + S);
            ratio = fabs(dev - old) / (fabs(dev) + 0.1);
        }
        first = false;
        if (!(ratio > prm.beta_tol)) break;  // `while dev_ratio > beta_tol` (NaN exits)
        factor_ridged<W>(ws.A, ws.L, p, kRidge, nullptr);
        wcopy<W>(bh, b, p);
        chol_solve_w<W>(ws.L, bh, p);
        ++it;
        bool div = false;
        for (int j = lane; j < p; j += T::NT) div = div || (fabs(bh[j]) > prm.max_beta);
        if (T::any(div) || it >= prm.maxiter) {
            status = kIrlsNeedsOptimizer;
            break;
        }
        wcopy<W>(beta, bh, p);
        T::sync();
    }
    if (a.force) status = kIrlsNeedsOptimizer;
    if (status != kIrlsOk) {
        if (lane == 0) {
            a.status[g] = status;
            if (a.n_fallback) atomicAdd(a.n_fallback, 1);
        }
        irls_optimizer_w<W>(a, d, ws, g);
        return;
    }
    irls_outputs<W>(d, p, beta, alpha, prm.min_mu, ws, ws.A, a.mu + g, a.hat + g, a.ld_out);
    if (a.with_wald) {
        // run_wald_test uses the UNCLAMPED mu (ds.py:320-324): A + the correction of the samples on the min_mu clamp
        for (int n0 = 0; n0 < d.N; n0 += T::NT) {
            const int n = n0 + lane;
            double wd = 0.0;
            if (n < d.N) {
                const double* x = row_of(d, n);
                const double mu_raw = x[p] * exp(xdot(x, beta, p));
                if (mu_raw < prm.min_mu) wd = mu_raw / fma(mu_raw, alpha, 1.0) - prm.min_mu / fma(prm.min_mu, alpha, 1.0);
            }
            if (!T::any(wd != 0.0)) continue;
            T::sync();
            ws.cw[lane] = wd;
            T::sync();
            rank_chunk<W>(d, p, n0, min(T::NT, d.N - n0), ws.cw, ws.A);
        }
        T::sync();
        wald_finish_w<W>(ws.A, a.wald, beta, ws, a.wald_p + g, a.wald_stat + g, a.wald_se + g);
    }
    for (int j = lane; j < p; j += T::NT) a.beta[(int64_t)g * p + j] = beta[j];
    if (lane == 0) {
        a.conv[g] = 1.0;  // IRLS exits are "converged" (utils.py:365)
        a.status[g] = kIrlsOk;
    }
}

// ---------------------------------------------------------------------------------------------
// alpha_mle (alpha_dloss / alpha_loss with the search and grid of pdq_gene.cuh)
// ---------------------------------------------------------------------------------------------
struct AlphaArgsW {
    WideBase b;
    AlphaParams prm;
    const int64_t* counts;
    int64_t ld;
    const double* mu;
    int64_t ld_mu;
    const double* alpha_hat;
    double *alpha, *conv;
    int* status;
    const double* prior_var_dev;
    int force;
    const double* hint_in;
    double* hint_out;
};

// d loss / d log(alpha) at x (curv: also the NB part's curvature, see alpha_dloss)
template <int W = 1>
__device__ double dloss_w(const DesignS& d, int p, const AlphaParams& prm, const int64_t* y, int64_t ld, const double* mu,
                          int64_t ld_mu, double x, double xhat, double* curv, Ws& ws) {
    using T = Team<W>;
    const double a = exp(x), r = 1.0 / a, Nd = (double)d.N;
    const bool cr = prm.cr_reg != 0;
    if (cr) {
        wfill<W>(ws.A, p * (p + 1) / 2, 0.0);
        wfill<W>(ws.Li, p * (p + 1) / 2, 0.0);
    }
    double Sg = 0.0, S2 = 0.0;
    for (int n0 = 0; n0 < d.N; n0 += T::NT) {
        const int n = n0 + T::tid();
        double wt = 0.0;
        if (n < d.N) {
            const double yv = (double)y[(int64_t)n * ld], m = mu[(int64_t)n * ld_mu];
            const double inv = 1.0 / (r + m);
            Sg += log(r + m) - digamma_pos(yv + r) + (yv - m) * inv;
            if (curv) S2 += fma(-(yv - m) * inv, inv, inv - trigamma_pos(yv + r));
            wt = m * r * inv;
        }
        if (!cr) continue;
        T::sync();
        ws.cw[T::tid()] = wt;
        ws.cz[T::tid()] = wt * wt;
        T::sync();
        const int cnt = min(T::NT, d.N - n0);
        rank_chunk<W>(d, p, n0, cnt, ws.cw, ws.A);
        rank_chunk<W>(d, p, n0, cnt, ws.cz, ws.Li);
    }
    T::sync();
    Sg = T::sum(Sg);
    const double F = Nd * (digamma_pos(r) + x) + Sg;
    double g = -r * F;
    if (curv) {
        S2 = T::sum(S2);
        const double Fp = Nd * (trigamma_pos(r) - a) + S2;
        *curv = r * (F + r * Fp) + (prm.prior_reg ? 1.0 / prm.prior_var : 0.0);
    }
    if (cr) {
        // tr((X^T W X)^-1 X^T W^2 X): A is factored in ws.L and inverted back into ws.L; ws.Li holds X^T W^2 X, so A's own buffer
        // is the inverse's scratch
        wcopy<W>(ws.L, ws.A, p * (p + 1) / 2);
        chol_w<W>(ws.L, p);
        chol_inverse_w<W>(ws.L, ws.A, ws.L, p);
        g -= 0.5 * a * symdot_w<W>(ws.L, ws.Li, p);
    }
    if (prm.prior_reg) g += (x - xhat) / prm.prior_var;
    return g;
}

// loss up to an alpha-independent constant, cr_reg on, no prior (the grid's objective, alpha_loss)
template <int W = 1>
__device__ double loss_w(const DesignS& d, int p, const int64_t* y, int64_t ld, const double* mu, int64_t ld_mu, double x, Ws& ws) {
    using T = Team<W>;
    const double a = exp(x), r = 1.0 / a, Nd = (double)d.N;
    wfill<W>(ws.A, p * (p + 1) / 2, 0.0);
    double Sf = 0.0;
    for (int n0 = 0; n0 < d.N; n0 += T::NT) {
        const int n = n0 + T::tid();
        double wt = 0.0;
        if (n < d.N) {
            const double yv = (double)y[(int64_t)n * ld], m = mu[(int64_t)n * ld_mu];
            const double rm = r + m;
            Sf += fma(yv + r, log(rm), -lgamma_pos(yv + r));
            wt = m * r / rm;
        }
        T::sync();
        ws.cw[T::tid()] = wt;
        T::sync();
        rank_chunk<W>(d, p, n0, min(T::NT, d.N - n0), ws.cw, ws.A);
    }
    T::sync();
    double f = Nd * (r * x + lgamma_pos(r)) + T::sum(Sf);
    chol_w<W>(ws.A, p);
    double ld2 = 0.0;
    for (int i = 0; i < p; ++i) ld2 += log(ws.A[tri(i, i)]);
    return f + 0.5 * (2.0 * ld2);
}

template <int W>
__global__ void __launch_bounds__(32 * W, W == 1 ? 0 : 1) k_wide_alpha_mle(const __grid_constant__ AlphaArgsW a) {
    using T = Team<W>;
    extern __shared__ __align__(16) double wsm[];
    Ws ws = carve<W>(wsm, a.b.p);
    const int g = blockIdx.x, p = a.b.p;
    const DesignS d = design_of(a.b.pack, a.b.N, p);
    AlphaParams prm = a.prm;
    if (a.prior_var_dev) prm.prior_var = *a.prior_var_dev;
    const int64_t* y = a.counts + g;
    const double* mu = a.mu + g;
    // alpha_search / alpha_grid_search vote through Group::any (a single-warp __any_sync) and write through grp.si == 0 (thread
    // 0 of the block).  At W > 1 that is right only because every value dloss_w / loss_w return is a Team<W>::sum, bit-identical
    // in every thread of the block, so every warp takes the same branches and reaches the __syncthreads inside T::sum together.
    // A change that lets a per-thread value reach the search's control flow breaks that uniformity.
    const Group grp{T::tid(), T::NT, 1};
    alpha_search(grp, prm, a.alpha_hat[g],
                 [&](double x, double xhat, double* curv) { return dloss_w<W>(d, p, prm, y, a.ld, mu, a.ld_mu, x, xhat, curv, ws); },
                 a.alpha + g, a.conv + g, a.status + g, true, a.hint_in ? a.hint_in + 2 * (int64_t)g : nullptr,
                 a.hint_out ? a.hint_out + 2 * (int64_t)g : nullptr);
    T::sync();
    if (a.force && T::tid() == 0) {
        a.status[g] = kAlphaNeedsGrid;
        a.conv[g] = 0.0;
    }
    T::sync();
    if (a.status[g] == kAlphaNeedsGrid)
        alpha_grid_search(grp, prm.lo, prm.hi, [&](double x) { return loss_w<W>(d, p, y, a.ld, mu, a.ld_mu, x, ws); }, a.alpha + g, true);
}

// ---------------------------------------------------------------------------------------------
// Wald tests
// ---------------------------------------------------------------------------------------------
struct WaldArgsW {
    WideBase b;
    WaldRef w;
    const double *disp, *lfc, *mu;
    int64_t ld_mu;
    double *pv, *stat, *se;
};

template <int W>
__global__ void __launch_bounds__(32 * W, W == 1 ? 0 : 1) k_wide_wald(const __grid_constant__ WaldArgsW a) {
    using T = Team<W>;
    extern __shared__ __align__(16) double wsm[];
    Ws ws = carve<W>(wsm, a.b.p);
    const int g = blockIdx.x, p = a.b.p;
    const DesignS d = design_of(a.b.pack, a.b.N, p);
    const double disp = a.disp[g];
    wfill<W>(ws.A, p * (p + 1) / 2, 0.0);
    for (int n0 = 0; n0 < d.N; n0 += T::NT) {
        const int n = n0 + T::tid();
        double wt = 0.0;
        if (n < d.N) {
            const double m = a.mu[(int64_t)n * a.ld_mu + g];
            wt = m / fma(m, disp, 1.0);
        }
        T::sync();
        ws.cw[T::tid()] = wt;
        T::sync();
        rank_chunk<W>(d, p, n0, min(T::NT, d.N - n0), ws.cw, ws.A);
    }
    T::sync();
    wcopy<W>(ws.v[1], a.lfc + (int64_t)g * p, p);
    T::sync();
    wald_finish_w<W>(ws.A, a.w, ws.v[1], ws, a.pv + g, a.stat + g, a.se + g);
}

struct WaldKArgsW {
    WideBase b;
    const double* ridge;  // packed, DesignDev::wald_dev
    const double *disp, *lfc, *tab;  // tab (K, p + 2): contrast | lfc_null | alt
    int K;
    double *pv, *stat, *se;
    int64_t ld_out;
};

template <int W>
__global__ void __launch_bounds__(32 * W, W == 1 ? 0 : 1) k_wide_wald_contrasts(const __grid_constant__ WaldKArgsW a) {
    using T = Team<W>;
    extern __shared__ __align__(16) double wsm[];
    Ws ws = carve<W>(wsm, a.b.p);
    const int g = blockIdx.x, p = a.b.p;
    const DesignS d = design_of(a.b.pack, a.b.N, p);
    double* beta = ws.v[1];
    wcopy<W>(beta, a.lfc + (int64_t)g * p, p);
    T::sync();
    weight_matrix<W>(d, p, beta, a.disp[g], 0.0, false, ws, ws.A);  // mu = sf exp(x'beta), as k_mu_from_lfc writes it
    wald_inverse_w<W>(ws.A, a.ridge, ws);
    for (int k = 0; k < a.K; ++k) {
        const double* row = a.tab + (int64_t)k * (p + 2);
        const double se = wald_se_w<W>(ws.A, row, ws);
        double pv, stat;
        wald_alt(row, beta, p, se, row[p], (int)row[p + 1], pv, stat);
        if (T::tid() == 0) {
            a.pv[(int64_t)k * a.ld_out + g] = pv;
            a.stat[(int64_t)k * a.ld_out + g] = stat;
            a.se[(int64_t)k * a.ld_out + g] = se;
        }
    }
}

// ---------------------------------------------------------------------------------------------
// Cook's distances (cooks_gene with the warp as the gene's lane group)
// ---------------------------------------------------------------------------------------------
struct CooksArgsW {
    WideBase b;
    const int* plan;  // [n_cells, global_mode, starts (n_cells + 1), order (n_in_cells)]
    int n_cells, n_in_cells;
    const int64_t* counts;
    int64_t ld;
    const double *mu, *hat;
    int64_t ld2;
    double cutoff;
    double* cooks;
    int64_t ld_out;
    double *disp, *outlier, *replaced;
    double* ws;  // null: the gene's cell members in shared memory; else in ws, one slot per gene (cooks_in_smem)
};

__global__ void __launch_bounds__(32) k_wide_cooks(const __grid_constant__ CooksArgsW a) {
    extern __shared__ __align__(16) double wsm[];
    const int g = blockIdx.x;
    const DesignS d = design_of(a.b.pack, a.b.N, a.b.p);
    const CellPlan plan{a.plan + 2 + a.n_cells + 1, a.plan + 2, a.n_cells, a.plan[1]};
    const Group grp{lane_id(), 32, 1};
    double* st = a.ws ? a.ws + (size_t)g * 2 * a.n_in_cells : wsm;
    cooks_gene_cols(grp, d, a.b.p, plan, a.counts + g, a.ld, a.mu + g, a.hat + g, a.ld2, a.cutoff, st, st + a.n_in_cells,
                    a.cooks ? a.cooks + g : nullptr, a.ld_out, a.disp + g, a.outlier + g, a.replaced + g, true);
}

// ---------------------------------------------------------------------------------------------
// apeGLM shrinkage (shrink_gene / shrink_eval / shrink_inv_hessian of pdq_shrink.cuh)
// ---------------------------------------------------------------------------------------------
// The narrow driver keeps its vectors in per-lane register arrays indexed by unrolled loops; here they are shared-memory vectors
// split over the lanes, so the driver below restates shrink_gene step for step (the line search, dcsrch_start / dcsrch_step /
// dcstep, is shared as is).  One team of W warps owns one gene, as in the fit kernels: W = 1 for 17..64 columns, W = 2, 4 or 8
// above.  Every scalar of the optimiser (line-search state, theta, the memory's head and size, the convergence tests) is computed
// redundantly in every thread of the team from Team<W>::sum / max totals or shared vectors, so it is bit-identical everywhere
// and all branches are team-uniform; that is what lets the W > 1 barriers inside those totals be reached by the whole block.
//
// Workspace of one gene: two packed p x p matrices (X'FX and its inverse's scratch), kShrinkVecs vectors of p, the L-BFGS memory
// S, Y (2 kShrinkMem p) with s'y and the two-loop's alphas (kShrinkMem each), two chunk buffers of 32 W.
constexpr int kShrinkVecs = 9;
__host__ __device__ constexpr size_t shrink_ws_doubles(int p, int W = 1) {
    return 2 * (size_t)tri_count(p) + (size_t)(kShrinkVecs + 2 * kShrinkMem) * p + 2 * kShrinkMem + 64 * W;
}

struct ShrinkWs {
    double *A, *Li;
    double *x, *g, *t, *r, *dir, *z, *xt, *gt, *q;
    double *S, *Y, *sy, *al;
    double *cw, *cz;
};

template <int W>
__device__ __forceinline__ ShrinkWs carve_shrink(double* s, int p) {
    ShrinkWs w;
    const int t = tri_count(p);
    w.A = s;
    w.Li = s + t;
    double* v = s + 2 * t;
    double** vecs[kShrinkVecs] = {&w.x, &w.g, &w.t, &w.r, &w.dir, &w.z, &w.xt, &w.gt, &w.q};
    for (int k = 0; k < kShrinkVecs; ++k) *vecs[k] = v + k * p;
    w.S = v + kShrinkVecs * p;
    w.Y = w.S + kShrinkMem * p;
    w.sy = w.Y + kShrinkMem * p;
    w.al = w.sy + kShrinkMem;
    w.cw = w.al + kShrinkMem;
    w.cz = w.cw + Team<W>::NT;
    return w;
}

// unscaled f (returned) and, when `grad`, its gradient: shrink_eval
template <int W>
__device__ double shrink_eval_w(const DesignS& d, int p, const ShrinkParams& prm, const int64_t* y, int64_t ld, double size,
                                double lsize, const double* beta, double* grad, ShrinkWs& ws) {
    using T = Team<W>;
    if (grad) wfill<W>(grad, p, 0.0);
    double nll = 0.0;
    for (int n0 = 0; n0 < d.N; n0 += T::NT) {
        const int n = n0 + T::tid();
        double gi = 0.0;
        if (n < d.N) {
            const double* x = row_of(d, n);
            const double yv = (double)y[(int64_t)n * ld];
            const double xb = xdot(x, beta, p);
            const double e = xb + x[p + 1];
            const double dd = e - lsize;
            const double t = exp(-fabs(dd));               // in (0, 1]
            const double lae = fmax(e, lsize) + log1p(t);  // logaddexp(e, log s)
            const double ys = yv + size;
            nll += yv * xb - ys * lae;
            const double q = ((dd >= 0.0) ? 1.0 : t) / (1.0 + t);  // 1 / (1 + s exp(-e)) without overflow
            gi = ys * q - yv;
        }
        if (!grad) continue;
        T::sync();
        ws.cz[T::tid()] = gi;
        T::sync();
        vec_chunk<W>(d, p, n0, min(T::NT, d.N - n0), ws.cz, grad);
    }
    nll = T::sum(nll);
    double prior = 0.0;
    for (int j = 0; j < p; ++j)
        prior += (j == prm.k) ? log1p(beta[j] * beta[j] / prm.scale2) : 0.5 * beta[j] * beta[j] * prm.inv_var0;
    if (grad) {
        T::sync();
        for (int j = T::tid(); j < p; j += T::NT)
            grad[j] += (j == prm.k) ? 2.0 * beta[j] / (prm.scale2 + beta[j] * beta[j]) : beta[j] * prm.inv_var0;
    }
    T::sync();
    return prior - nll;
}

// shrink_inv_hessian: (X'FX + 1 h')^-1 through Sherman-Morrison on the Cholesky factor of A = X'FX, written to ih (p x p)
template <int W>
__device__ void shrink_inv_hessian_w(const DesignS& d, int p, const ShrinkParams& prm, const int64_t* y, int64_t ld, double size,
                                     double lsize, const double* beta, double* ih, ShrinkWs& ws) {
    using T = Team<W>;
    wfill<W>(ws.A, p * (p + 1) / 2, 0.0);
    for (int n0 = 0; n0 < d.N; n0 += T::NT) {
        const int n = n0 + T::tid();
        double w = 0.0;
        if (n < d.N) {
            const double* x = row_of(d, n);
            const double yv = (double)y[(int64_t)n * ld];
            const double dd = xdot(x, beta, p) + x[p + 1] - lsize;
            const double t = exp(-fabs(dd));
            w = (yv + size) * (t / ((1.0 + t) * (1.0 + t)));  // (y+s) q (1-q)
        }
        T::sync();
        ws.cw[T::tid()] = w;
        T::sync();
        rank_chunk<W>(d, p, n0, min(T::NT, d.N - n0), ws.cw, ws.A);
    }
    chol_w<W>(ws.A, p);
    chol_inverse_w<W>(ws.A, ws.Li, ws.A, p);  // A^-1 in ws.A
    double *h = ws.t, *u = ws.r, *v = ws.q;  // the optimiser's vectors are free now
    const double bk = beta[prm.k], den = prm.scale2 + bk * bk;
    for (int j = T::tid(); j < p; j += T::NT) h[j] = (j == prm.k) ? 2.0 * (prm.scale2 - bk * bk) / (den * den) : prm.inv_var0;
    T::sync();
    for (int i = T::tid(); i < p; i += T::NT) {
        double su = 0.0, sv = 0.0;
        for (int j = 0; j < p; ++j) {
            const double aij = ws.A[j <= i ? tri(i, j) : tri(j, i)];
            su += aij;
            sv = fma(aij, h[j], sv);
        }
        u[i] = su;
        v[i] = sv;
    }
    T::sync();
    const double inv = 1.0 / (1.0 + wdot<W>(h, u, p));
    for (int k = T::tid(); k < p * p; k += T::NT) {
        const int i = k / p, j = k - i * p;
        ih[k] = ws.A[j <= i ? tri(i, j) : tri(j, i)] - u[i] * v[j] * inv;
    }
}

// z = x + (L-BFGS step), with an empty memory z = x - g / theta: lbfgs_point
template <int W>
__device__ void lbfgs_point_w(int p, int col, int head, double theta, ShrinkWs& ws) {
    using T = Team<W>;
    const int lane = T::tid();
    for (int j = lane; j < p; j += T::NT) ws.q[j] = -ws.g[j];
    T::sync();
    if (col == 0) {
        for (int j = lane; j < p; j += T::NT) ws.z[j] = ws.x[j] + (1.0 / theta) * ws.q[j];
        T::sync();
        return;
    }
    for (int i = col - 1; i >= 0; --i) {  // newest -> oldest
        const int s = (head + i) % kShrinkMem;
        const double a = wdot<W>(ws.S + s * p, ws.q, p) / ws.sy[s];
        if (lane == 0) ws.al[i] = a;
        for (int j = lane; j < p; j += T::NT) ws.q[j] = ws.q[j] - a * ws.Y[s * p + j];
        T::sync();
    }
    for (int j = lane; j < p; j += T::NT) ws.q[j] = ws.q[j] / theta;
    T::sync();
    for (int i = 0; i < col; ++i) {  // oldest -> newest
        const int s = (head + i) % kShrinkMem;
        const double b = wdot<W>(ws.Y + s * p, ws.q, p) / ws.sy[s];
        for (int j = lane; j < p; j += T::NT) ws.q[j] = ws.q[j] + ws.S[s * p + j] * (ws.al[i] - b);
        T::sync();
    }
    for (int j = lane; j < p; j += T::NT) ws.z[j] = ws.x[j] + ws.q[j];
    T::sync();
}

struct ShrinkArgsW {
    WideBase b;
    ShrinkParams prm;
    const int64_t* counts;
    int64_t ld;
    const double* size;
    double *beta, *ih, *conv;
    int* status;
};

// shrink_gene: beta_init +-0.1, scale max(f(0), 1), m = 10 two-loop direction, dcsrch with maxls 20, the update skip, the restarts,
// ftol = gtol = 1e-8 and the evaluation budget; no grid fallback (two-column designs only)
template <int W>
__global__ void __launch_bounds__(32 * W, W == 1 ? 0 : 1) k_wide_lfc_shrink(const __grid_constant__ ShrinkArgsW a) {
    using T = Team<W>;
    extern __shared__ __align__(16) double wsm[];
    const int g = blockIdx.x, p = a.b.p, lane = T::tid();
    ShrinkWs ws = carve_shrink<W>(wsm, p);
    const DesignS d = design_of(a.b.pack, a.b.N, p);
    const ShrinkParams prm = a.prm;
    const int64_t* y = a.counts + g;
    const double size = a.size[g], lsize = log(size);
    const double ftol = 1e-8, gtol = 1e-8;
    wfill<W>(ws.x, p, 0.0);
    T::sync();
    double f = shrink_eval_w<W>(d, p, prm, y, a.ld, size, lsize, ws.x, nullptr, ws);
    const double cnst = (f < 1.0) ? 1.0 : f;  // np.maximum(scale_cnst, 1)
    for (int j = lane; j < p; j += T::NT) ws.x[j] = (j & 1) ? -0.1 : 0.1;
    T::sync();
    f = shrink_eval_w<W>(d, p, prm, y, a.ld, size, lsize, ws.x, ws.g, ws) / cnst;
    for (int j = lane; j < p; j += T::NT) ws.g[j] = ws.g[j] / cnst;
    T::sync();

    int col = 0, head = 0;
    double theta = 1.0;
    LineSearch ls;
    double fold = f, gdold = 0.0, stp = 1.0;
    int nit = 0, iback = 0;
    bool active = true, ok = false;

    auto set_trial = [&]() {  // xt = t + stp dir (z itself at stp = 1)
        for (int j = lane; j < p; j += T::NT) ws.xt[j] = (stp == 1.0) ? ws.z[j] : fma(stp, ws.dir[j], ws.t[j]);
        T::sync();
    };
    // prepares the next line search from (x, f, g); returns false on ABNORMAL_TERMINATION_IN_LNSRCH
    auto begin_iteration = [&]() -> bool {
        for (;;) {
            lbfgs_point_w<W>(p, col, head, theta, ws);
            for (int j = lane; j < p; j += T::NT) ws.dir[j] = ws.z[j] - ws.x[j];
            T::sync();
            const double dtd = wdot<W>(ws.dir, ws.dir, p), gd = wdot<W>(ws.g, ws.dir, p);
            stp = (nit == 0) ? fmin(1.0 / sqrt(dtd), kLsStpMax) : 1.0;
            wcopy<W>(ws.t, ws.x, p);
            wcopy<W>(ws.r, ws.g, p);
            T::sync();
            fold = f;
            gdold = gd;
            iback = 0;
            if (!(gd < 0.0)) {  // not a descent direction: drop the memory and retry, or give up
                if (col == 0) return false;
                col = 0;
                head = 0;
                theta = 1.0;
                continue;
            }
            dcsrch_start(ls, stp, f, gd);
            set_trial();
            return true;
        }
    };

    if (wmaxabs<W>(ws.g, p) <= gtol) {
        ok = true;
        active = false;
    }
    if (active && !begin_iteration()) active = false;
    for (int ev = 0; ev < kShrinkMaxEval && active; ++ev) {
        const double ft = shrink_eval_w<W>(d, p, prm, y, a.ld, size, lsize, ws.xt, ws.gt, ws);
        f = ft / cnst;
        for (int j = lane; j < p; j += T::NT) {
            ws.g[j] = ws.gt[j] / cnst;
            ws.x[j] = ws.xt[j];
        }
        T::sync();
        const double gd = wdot<W>(ws.g, ws.dir, p);
        if (dcsrch_step(ls, stp, f, gd)) {  // another trial point
            if (++iback >= kShrinkMaxLs) {  // line search failed: restore, restart from steepest descent or give up
                wcopy<W>(ws.x, ws.t, p);
                wcopy<W>(ws.g, ws.r, p);
                T::sync();
                f = fold;
                if (col == 0) {
                    active = false;
                    continue;
                }
                col = 0;
                head = 0;
                theta = 1.0;
                if (!begin_iteration()) active = false;
                continue;
            }
            set_trial();
            continue;
        }
        // ---- new iterate
        ++nit;
        if (wmaxabs<W>(ws.g, p) <= gtol || (fold - f) <= ftol * fmax(fmax(fabs(fold), fabs(f)), 1.0)) {
            ok = true;
            active = false;
            continue;
        }
        if (nit >= kShrinkMaxIter) {
            active = false;
            continue;
        }
        // memory update (skipped when the curvature s'y is not safely positive); y = g - r
        double rr = 0.0;
        for (int j = lane; j < p; j += T::NT) {
            const double yj = ws.g[j] - ws.r[j];
            rr = fma(yj, yj, rr);
        }
        rr = T::sum(rr);
        const double dr = (stp == 1.0) ? (gd - gdold) : (gd - gdold) * stp;
        const double ddum = (stp == 1.0) ? -gdold : -gdold * stp;
        if (dr > 2.220446049250313e-16 * ddum) {
            int slot;
            if (col < kShrinkMem) {
                slot = (head + col) % kShrinkMem;
                ++col;
            } else {
                slot = head;
                head = (head + 1) % kShrinkMem;
            }
            double *Ss = ws.S + slot * p, *Ys = ws.Y + slot * p;
            for (int j = lane; j < p; j += T::NT) {
                Ss[j] = (stp == 1.0) ? ws.dir[j] : stp * ws.dir[j];
                Ys[j] = ws.g[j] - ws.r[j];
            }
            T::sync();
            const double sy = wdot<W>(Ys, Ss, p);
            if (lane == 0) ws.sy[slot] = sy;
            T::sync();
            theta = rr / dr;
        }
        if (!begin_iteration()) active = false;
    }
    // `active` still set: evaluation budget exhausted -> not converged
    shrink_inv_hessian_w<W>(d, p, prm, y, a.ld, size, lsize, ws.x, a.ih + (int64_t)g * p * p, ws);
    for (int j = lane; j < p; j += T::NT) a.beta[(int64_t)g * p + j] = ws.x[j];
    if (lane == 0) {
        a.conv[g] = ok ? 1.0 : 0.0;
        a.status[g] = kShrinkOk;
    }
}
// instantiated here, not at its launcher, so that the module lists the kernels in the order ptxas was given them before the team
// widths existed: ptxas's register assignment depends on that order, and with it every other kernel keeps its code
template __global__ void k_wide_lfc_shrink<1>(const __grid_constant__ ShrinkArgsW a);

// ---------------------------------------------------------------------------------------------
// launch helpers
// ---------------------------------------------------------------------------------------------
inline size_t ws_bytes(int p, int W = 1) { return wide_ws_doubles(p, W) * sizeof(double); }
inline WideBase base_of(const DesignDev& d, int G) { return WideBase{d.pack, d.pinv_dev, d.N, d.p, G}; }

void pack_lower(const double* full, int p, double* tri_out) {
    for (int i = 0; i < p; ++i)
        for (int j = 0; j <= i; ++j) tri_out[tri(i, j)] = full[i * p + j];
}

// host values -> device memory as kernel parameters, in chunks that fit the parameter space: stream-ordered behind the kernels
// that read the previous values, and a captured graph keeps the values of its capture
constexpr int kPutChunk = 3968;
struct PutArgs {
    double v[kPutChunk];
    double* dst;
    int n;
};
__global__ void __launch_bounds__(256) k_wide_put(const __grid_constant__ PutArgs a) {
    for (int i = threadIdx.x; i < a.n; i += blockDim.x) a.dst[i] = a.v[i];
}

// uploads `n` doubles; returns the number of launches or a negative pdq_status
int put_dev(const LaunchCfg& c, const double* h, int n, double* dst) {
    int launches = 0;
    for (int o = 0; o < n; o += kPutChunk) {
        PutArgs a;
        a.n = (n - o < kPutChunk) ? n - o : kPutChunk;
        a.dst = dst + o;
        for (int i = 0; i < a.n; ++i) a.v[i] = h[o + i];
        k_wide_put<<<1, 256, 0, c.stream>>>(a);
        if (int e = check_launch()) return e;
        ++launches;
    }
    return launches;
}

// ridge (packed lower triangle) and contrast into DesignDev::wald_dev; contrast may be null.  The host-buffer calls launch once
// per gene block, and with the gene-block pipeline the upload of block b + 1 (on the other stream) can write wald_dev while block
// b's kernel reads it.  That is safe because every upload within one call writes the same bytes.
int put_wald(const LaunchCfg& c, const DesignDev& d, const double* ridge, const double* contrast, WaldRef& w) {
    const int p = d.p, t = tri_count(p);
    double buf[PDQ_MAX_P_LARGE * (PDQ_MAX_P_LARGE + 1) / 2 + 1 + PDQ_MAX_P_LARGE];
    pack_lower(ridge, p, buf);
    if (t > p * (p + 1) / 2) buf[t - 1] = 0.0;  // the pad slot of an odd p(p+1)/2: never read, uploaded as zero
    if (contrast)
        for (int j = 0; j < p; ++j) buf[t + j] = contrast[j];
    w.ridge = d.wald_dev;
    w.contrast = d.wald_dev + t;
    return put_dev(c, buf, contrast ? t + p : t, d.wald_dev);
}

inline size_t shrink_ws_bytes(int p, int W) { return shrink_ws_doubles(p, W) * sizeof(double); }
using WsBytes = size_t (*)(int p, int W);

// warps per gene of the 65..128 tier for a kernel whose workspace takes ws(p, W) bytes: the fewest of 2, 4, 8 that keep 8 warps
// on an SM, given how many blocks the workspace lets share one (228 KB of shared memory per SM, 1 KB of it reserved per block).
// For the fit kernels (ws_bytes) that is 2 at p = 65 (four blocks), 4 at p = 81 (two) and 8 from p = 101 on (one): the fastest of
// the three at each of those widths (DESIGN.md §5).  For apeGLM shrinkage (shrink_ws_bytes) it is 2 at p = 65, 4 at 81 and 101,
// 8 at 128.
int large_warps(int p, WsBytes ws) {
    for (int W = 2; W < 8; W *= 2)
        if ((int)(228 * 1024 / (ws(p, W) + 1024)) * W >= 8) return W;
    return 8;
}

// the team width of a design: one warp up to PDQ_MAX_P_WIDE columns, above that DesignDev::warps (a tuning hook) or large_warps
// for the kernel's workspace
template <class F>
int with_warps(const DesignDev& d, F&& f, WsBytes ws = ws_bytes) {
    if (d.p <= PDQ_MAX_P_WIDE) return f(std::integral_constant<int, 1>{});
    switch (d.warps ? d.warps : large_warps(d.p, ws)) {
        case 2: return f(std::integral_constant<int, 2>{});
        case 4: return f(std::integral_constant<int, 4>{});
        default: return f(std::integral_constant<int, 8>{});
    }
}

// one block of W warps per gene with its workspace of ws(p, W) bytes; returns the number of launches, the `puts` Wald uploads included
template <int W, class A>
int launch_team(const LaunchCfg& c, const DesignDev& d, int G, void (*kernel)(A), const A& a, int puts = 0, WsBytes ws = ws_bytes) {
    const size_t smem = ws(d.p, W);
    if (int e = prep(kernel, smem)) return e;
    kernel<<<G, 32 * W, smem, c.stream>>>(a);
    if (int e = check_launch()) return e;
    return 1 + puts;
}

}  // namespace

int launch_lin_reg_mu_wide(const LaunchCfg& c, const DesignDev& d, const int64_t* counts, int64_t ld, int G, double min_mu, double* mu_out,
                           int64_t ld_out) {
    const LinArgs a{base_of(d, G), counts, ld, min_mu, mu_out, ld_out};
    return with_warps(d, [&](auto w) { return launch_team<decltype(w)::value>(c, d, G, k_wide_lin_reg_mu<decltype(w)::value>, a); });
}

int launch_irls_wide(const LaunchCfg& c, const DesignDev& d, const int64_t* counts, int64_t ld, int G, const double* disp, const IrlsHost& h,
                     double* beta, double* mu, double* hat, int64_t ld_out, double* conv, int* status, int* n_fallback, const WaldHost* w) {
    if (n_fallback && cudaMemsetAsync(n_fallback, 0, sizeof(int), c.stream) != cudaSuccess) return PDQ_ERR_CUDA;
    int puts = 0;
    IrlsArgsW a{};
    a.b = base_of(d, G);
    a.prm = irls_params(h, d, c.debug);
    a.counts = counts; a.ld = ld; a.disp = disp;
    a.beta = beta; a.mu = mu; a.hat = hat; a.conv = conv; a.ld_out = ld_out;
    a.status = status; a.n_fallback = n_fallback;
    a.force = hook(c.debug, PDQ_DEBUG_FORCE_IRLS_OPTIMIZER);
    a.with_wald = w ? 1 : 0;
    if (w) {
        if ((puts = put_wald(c, d, w->ridge, w->contrast, a.wald)) < 0) return puts;
        a.wald.lfc_null = w->lfc_null;
        a.wald.alt = w->alt;
        a.wald_p = w->pv; a.wald_stat = w->stat; a.wald_se = w->se;
    }
    return with_warps(d, [&](auto tw) { return launch_team<decltype(tw)::value>(c, d, G, k_wide_irls<decltype(tw)::value>, a, puts); });
}

int launch_alpha_mle_wide(const LaunchCfg& c, const DesignDev& d, const int64_t* counts, int64_t ld, int G, const double* mu, int64_t ld_mu,
                          const double* alpha_hat, double min_disp, double max_disp, double prior_var, const double* prior_var_dev, int cr_reg,
                          int prior_reg, double* alpha, double* conv, int* status, const double* hint_in, double* hint_out) {
    const AlphaArgsW a{base_of(d, G), alpha_params(min_disp, max_disp, prior_var, cr_reg, prior_reg), counts, ld, mu, ld_mu,
                       alpha_hat, alpha, conv, status, prior_var_dev, hook(c.debug, PDQ_DEBUG_FORCE_ALPHA_GRID), hint_in, hint_out};
    return with_warps(d, [&](auto w) { return launch_team<decltype(w)::value>(c, d, G, k_wide_alpha_mle<decltype(w)::value>, a); });
}

int launch_wald_wide(const LaunchCfg& c, const DesignDev& d, const double* disp, const double* lfc, const double* mu, int64_t ld_mu, int G,
                     const double* ridge, const double* contrast, double lfc_null, int alt, double* pv, double* stat, double* se) {
    WaldArgsW a{};
    a.b = base_of(d, G);
    const int puts = put_wald(c, d, ridge, contrast, a.w);
    if (puts < 0) return puts;
    a.w.lfc_null = lfc_null;
    a.w.alt = alt;
    a.disp = disp; a.lfc = lfc; a.mu = mu; a.ld_mu = ld_mu;
    a.pv = pv; a.stat = stat; a.se = se;
    return with_warps(d, [&](auto w) { return launch_team<decltype(w)::value>(c, d, G, k_wide_wald<decltype(w)::value>, a, puts); });
}

int launch_wald_contrasts_wide(const LaunchCfg& c, const DesignDev& d, const double* disp, const double* lfc, int G, const double* ridge, int K,
                               const double* tab, double* pv, double* stat, double* se, int64_t ld_out) {
    WaldRef r;
    const int puts = put_wald(c, d, ridge, nullptr, r);
    if (puts < 0) return puts;
    const WaldKArgsW a{base_of(d, G), r.ridge, disp, lfc, tab, K, pv, stat, se, ld_out};
    return with_warps(d, [&](auto w) { return launch_team<decltype(w)::value>(c, d, G, k_wide_wald_contrasts<decltype(w)::value>, a, puts); });
}

int launch_rough_wide(const LaunchCfg& c, const DesignDev& d, const double* normed, int64_t ld, int G, double* alpha) {
    const MomArgsW a{base_of(d, G), normed, nullptr, ld, d.s_mean_inv, 0.0, 0.0, 0.0, alpha, nullptr, nullptr, 0};
    return with_warps(d, [&](auto w) { return launch_team<decltype(w)::value>(c, d, G, k_wide_rough<decltype(w)::value>, a); });
}

// the passes whose work does not grow with p (moments, mu from LFCs, Cook's distances) run one warp per gene at every width
int launch_moments_wide(const LaunchCfg& c, const DesignDev& d, const double* normed, int64_t ld, int G, double* alpha, double* all_zero) {
    const MomArgsW a{base_of(d, G), normed, nullptr, ld, d.s_mean_inv, 0.0, 0.0, 0.0, alpha, all_zero, nullptr, 0};
    k_wide_moments<<<G, 32, 0, c.stream>>>(a);
    if (int e = check_launch()) return e;
    return 1;
}

int launch_mom_from_counts_wide(const LaunchCfg& c, const DesignDev& d, const int64_t* counts, int64_t ld, int G, double min_disp,
                                double max_disp, double* alpha, double* normed_mean, double min_mu, double* mu_hat, int64_t ld_mu) {
    const MomArgsW a{base_of(d, G), nullptr, counts, ld, d.s_mean_inv, min_disp, max_disp, min_mu, alpha, normed_mean, mu_hat, ld_mu};
    return with_warps(d, [&](auto w) { return launch_team<decltype(w)::value>(c, d, G, k_wide_mom_from_counts<decltype(w)::value>, a); });
}

int launch_mu_from_lfc_wide(const LaunchCfg& c, const DesignDev& d, const double* lfc, int G, double* mu, int64_t ld_out) {
    const MuLfcArgsW a{base_of(d, G), lfc, mu, ld_out};
    k_wide_mu_from_lfc<<<G, 32, 0, c.stream>>>(a);
    if (int e = check_launch()) return e;
    return 1;
}

int launch_cooks_wide(const LaunchCfg& c, const DesignDev& d, const int64_t* counts, int64_t ld, int G, const double* mu, const double* hat,
                      int64_t ld2, double cutoff, double* cooks, int64_t ld_out, double* disp, double* outlier, double* replaced, double* ws) {
    const bool global = !cooks_in_smem(d);
    const int chunk = global ? cooks_chunk(d) : G;
    if (global && (!ws || chunk < 1)) return PDQ_ERR_UNSUPPORTED;
    const size_t smem = global ? 0 : cooks_gene_bytes(d);
    if (int e = prep(k_wide_cooks, smem)) return e;
    int launches = 0;
    for (int g0 = 0; g0 < G; g0 += chunk, ++launches) {
        const int n = G - g0 < chunk ? G - g0 : chunk;
        const CooksArgsW a{base_of(d, n), d.cell_plan, d.n_cells, d.n_in_cells, counts + g0, ld, mu + g0, hat + g0, ld2, cutoff,
                           cooks ? cooks + g0 : nullptr, ld_out, disp + g0, outlier + g0, replaced + g0, global ? ws : nullptr};
        k_wide_cooks<<<n, 32, smem, c.stream>>>(a);
    }
    if (int e = check_launch()) return e;
    return launches;
}

int launch_lfc_shrink_wide(const LaunchCfg& c, const DesignDev& d, const int64_t* counts, int64_t ld, int G, const double* size,
                           double prior_no_shrink_scale, double prior_scale, int shrink_index, double* beta, double* inv_hessian,
                           double* conv, int* status) {
    if (shrink_index < 0 || shrink_index >= d.p) return PDQ_ERR_INVALID;
    const ShrinkArgsW a{base_of(d, G), ShrinkParams{1.0 / (prior_no_shrink_scale * prior_no_shrink_scale), prior_scale * prior_scale, shrink_index},
                        counts, ld, size, beta, inv_hessian, conv, status};
    return with_warps(
        d, [&](auto w) { return launch_team<decltype(w)::value>(c, d, G, k_wide_lfc_shrink<decltype(w)::value>, a, 0, shrink_ws_bytes); },
        shrink_ws_bytes);
}

}  // namespace pdq
