// pdq_host_linalg.h -- host-only design-matrix preprocessing and input packing, shared by the C ABI and the host emulator (hoisted
// out of the per-gene work: the reference recomputes matrix_rank / QR of the SAME X for every gene, utils.py:349-352).
#pragma once

#include <math.h>
#include <string.h>

#include <vector>

#ifndef PDQ_MAX_P
#define PDQ_MAX_P 16
#endif
#ifndef PDQ_MAX_P_WIDE
#define PDQ_MAX_P_WIDE 64
#endif
#ifndef PDQ_MAX_P_LARGE
#define PDQ_MAX_P_LARGE 128
#endif

namespace pdq {

// Design pack of X (N x p; DesignS, pdq_gene.cuh), ROW-major: row n = [ x_n0 .. x_n,p-1 | sf_n | log sf_n | pad ] of RS = p + 2
// rounded up to even doubles (16-byte aligned rows: a sample's design row + size factor is one or two 128-bit shared-memory reads),
// then row N of the column maxima max_n |x_nj| (to bound |x'beta| once per sweep).  `sf` NULL = all ones; `offsets`: `sf` holds LOG
// size factors (the apeGLM call receives them so, and exp/log is not the identity in FP64).  Returns mean(1 / sf) (utils.py:880).
constexpr int design_row_stride(int p) { return (p + 3) & ~1; }
inline double design_pack(const double* X, const double* sf, bool offsets, int N, int p, std::vector<double>& pack) {
    const int RS = design_row_stride(p);
    pack.assign((size_t)(N + 1) * RS, 0.0);
    double inv_sum = 0.0;
    for (int n = 0; n < N; ++n) {
        double* row = pack.data() + (size_t)n * RS;
        for (int j = 0; j < p; ++j) {
            row[j] = X[(size_t)n * p + j];
            double& mx = pack[(size_t)N * RS + j];
            mx = !(fabs(row[j]) <= mx) ? fabs(row[j]) : mx;  // NaN propagates into the bound
        }
        const double s = sf ? (offsets ? exp(sf[n]) : sf[n]) : 1.0;
        row[p] = s;
        row[p + 1] = (sf && offsets) ? sf[n] : log(s);
        inv_sum += 1.0 / s;
    }
    return inv_sum / N;
}

// wald_contrasts_gene's (K, p + 2) rows [contrast | lfc_null | alt]; returns the first contrast whose alternative is not 0..4, or -1
inline int wald_contrast_table(int K, int p, const double* contrasts, const double* lfc_null, const int* alt, double* tab) {
    for (int k = 0; k < K; ++k) {
        if (alt[k] < 0 || alt[k] > 4) return k;
        memcpy(tab + (size_t)k * (p + 2), contrasts + (size_t)k * p, (size_t)p * 8);
        tab[(size_t)k * (p + 2) + p] = lfc_null[k];
        tab[(size_t)k * (p + 2) + p + 1] = (double)alt[k];
    }
    return -1;
}

// One-sided Jacobi SVD of X (N x p, p <= PDQ_MAX_P_LARGE): the right singular vectors V and singular values give
//   rank(X)   with numpy.linalg.matrix_rank's tolerance  s_max * max(N, p) * eps     (utils.py:349)
//   (X^T X)^+ = V diag(1/s_i^2 for s_i > tol) V^T        (least-squares / minimum-norm projector)
// number of distinct rows of X (capped at `cap + 1`): categorical designs have a handful, continuous covariates ~N
inline int design_distinct_rows(const double* X, int N, int p, int cap) {
    std::vector<int> reps;
    for (int n = 0; n < N; ++n) {
        bool seen = false;
        for (int r : reps)
            if (memcmp(X + (size_t)r * p, X + (size_t)n * p, (size_t)p * sizeof(double)) == 0) { seen = true; break; }
        if (!seen) {
            reps.push_back(n);
            if ((int)reps.size() > cap) break;
        }
    }
    return (int)reps.size();
}

inline void design_linear_algebra(const double* X, int N, int p, double* pinv, int* full_rank) {
    std::vector<double> U((size_t)N * p);
    for (size_t i = 0; i < (size_t)N * p; ++i) U[i] = X[i];
    std::vector<double> Vs((size_t)p * p, 0.0);
    auto V = [&](int k, int a) -> double& { return Vs[(size_t)k * p + a]; };
    for (int i = 0; i < p; ++i) V(i, i) = 1.0;
    for (int sweep = 0; sweep < 60; ++sweep) {
        double off = 0.0;
        for (int a = 0; a < p - 1; ++a)
            for (int b = a + 1; b < p; ++b) {
                double aa = 0, bb = 0, ab = 0;
                for (int n = 0; n < N; ++n) {
                    const double ua = U[(size_t)n * p + a], ub = U[(size_t)n * p + b];
                    aa += ua * ua;
                    bb += ub * ub;
                    ab += ua * ub;
                }
                if (ab == 0.0) continue;
                off = fmax(off, fabs(ab) / sqrt(aa * bb + 1e-300));
                const double zeta = (bb - aa) / (2.0 * ab);
                const double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
                const double cs = 1.0 / sqrt(1.0 + t * t), sn = cs * t;
                for (int n = 0; n < N; ++n) {
                    const double ua = U[(size_t)n * p + a], ub = U[(size_t)n * p + b];
                    U[(size_t)n * p + a] = cs * ua - sn * ub;
                    U[(size_t)n * p + b] = sn * ua + cs * ub;
                }
                for (int k = 0; k < p; ++k) {
                    const double va = V(k, a), vb = V(k, b);
                    V(k, a) = cs * va - sn * vb;
                    V(k, b) = sn * va + cs * vb;
                }
            }
        if (off < 1e-15) break;
    }
    std::vector<double> s(p);
    double smax = 0.0;
    for (int j = 0; j < p; ++j) {
        double q = 0;
        for (int n = 0; n < N; ++n) q += U[(size_t)n * p + j] * U[(size_t)n * p + j];
        s[j] = sqrt(q);
        smax = fmax(smax, s[j]);
    }
    const double tol = smax * (double)(N > p ? N : p) * 2.220446049250313e-16;
    int rank = 0;
    for (int j = 0; j < p; ++j) rank += s[j] > tol;
    *full_rank = (rank == p);
    for (int i = 0; i < p; ++i)
        for (int k = 0; k < p; ++k) {
            double acc = 0;
            for (int j = 0; j < p; ++j)
                if (s[j] > tol) acc += V(i, j) * V(k, j) / (s[j] * s[j]);
            pinv[i * p + k] = acc;
        }
}


// Cells of the design (SURVEY.md §8 f-1): samples with identical design rows, kept when they hold >= 3 replicates
// (utils.py:888-912 + the groupby of utils.py:935-941, cells numbered by first appearance among the kept samples).
// plan = [n_cells, global_mode, start_0 .. start_ncells, order_0 .. order_{nf-1}]
inline std::vector<int> design_cell_plan(const double* X, int N, int p) {
    std::vector<int> rep(N, -1);  // representative (first sample with the same row)
    std::vector<int> count(N, 0);
    for (int i = 0; i < N; ++i) {
        for (int j = 0; j < i && rep[i] < 0; ++j) {
            if (rep[j] != j) continue;
            bool same = true;
            for (int k = 0; k < p && same; ++k) same = X[(size_t)i * p + k] == X[(size_t)j * p + k];
            if (same) rep[i] = j;
        }
        if (rep[i] < 0) rep[i] = i;
        ++count[rep[i]];
    }
    std::vector<int> cells;  // representatives of the kept cells, by first appearance
    for (int i = 0; i < N; ++i)
        if (rep[i] == i && count[i] >= 3) cells.push_back(i);
    std::vector<int> plan;
    if (cells.empty()) {  // no replicates anywhere: one global cell (utils.py:942-945)
        plan.push_back(1);
        plan.push_back(1);
        plan.push_back(0);
        plan.push_back(N);
        for (int i = 0; i < N; ++i) plan.push_back(i);
        return plan;
    }
    plan.push_back((int)cells.size());
    plan.push_back(0);
    int acc = 0;
    for (int c : cells) {
        plan.push_back(acc);
        acc += count[c];
    }
    plan.push_back(acc);
    for (int c : cells)
        for (int i = 0; i < N; ++i)
            if (rep[i] == c) plan.push_back(i);
    return plan;
}

}  // namespace pdq
