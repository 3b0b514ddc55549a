// pdq_emu.cpp -- HOST EMULATOR of the device per-gene routines.  TEST INFRASTRUCTURE ONLY.
//
// Compiles pydeseq2_b200/csrc/pdq_gene.cuh, pdq_trend.cuh, pdq_shrink.cuh and pdq_vst.cuh (the exact sources the sm_90a kernels
// are built from) with g++, one "lane" per gene (T = 1, Group::sum is the identity), so that the CPU test-suite can
// check the algorithmic content of the kernels -- IRLS control flow, the bounded root search for
// the dispersion, Cholesky algebra, special functions, size factors, the vst, Wald tests of K contrasts -- against the oracle
// without a GPU.  The design pack and the contrast table are written by the product's own host code (pdq_host_linalg.h).
// It is built by tests/emu/build.py into tests/emu/_build/ and loaded only by tests/; the product
// (pydeseq2_b200) never loads it and has no CPU fallback.
//
// emu_set_lanes(T) switches to T = 2..32 cooperating "lanes" per gene, one std::thread each: Group::sum / excl_scan / any /
// sync then exchange through a shared board with the device's own patterns (xor butterfly over the lane index, Hillis-Steele
// scan), so the lane-cooperative code paths -- strided sample walks, split table builds, replicated control flow -- and the
// device's summation ORDER are exercised on the CPU as well.
#include <stdint.h>
#include <string.h>

#include <barrier>
#include <thread>
#include <vector>

extern long g_emu_alpha_evals;
extern long g_emu_irls_sweeps;
#define PDQ_EMU_COUNT_EVALS 1
#define PDQ_EMU_LANES 1
#include "../../pydeseq2_b200/csrc/pdq_gene.cuh"
#include "../../pydeseq2_b200/csrc/pdq_host_linalg.h"
#include "../../pydeseq2_b200/csrc/pdq_trend.cuh"
#include "../../pydeseq2_b200/csrc/pdq_shrink.cuh"
#include "../../pydeseq2_b200/csrc/pdq_vst.cuh"
#include "../gpu_probe/math_ops.h"

long g_emu_alpha_evals = 0;
long g_emu_irls_sweeps = 0;
using namespace pdq;

// ---- lane team: what a warp's shuffles and votes become on the host ------------------------------------------------------
namespace {
struct LaneTeam {
    explicit LaneTeam(int T) : bar(T) {}
    std::barrier<> bar;
    double board[32], board2[32];
    int flags[32];
};
thread_local LaneTeam* t_team = nullptr;
int g_lanes = 1;
}  // namespace

namespace pdq_emu {
// every lane ends with the same total, accumulated in the order of the device's xor butterfly (largest stride first)
double lane_sum(int si, int T, double v) {
    if (T == 1 || !t_team) return v;
    for (int s = T >> 1; s >= 1; s >>= 1) {
        t_team->board[si] = v;
        t_team->bar.arrive_and_wait();
        const double o = t_team->board[si ^ s];
        t_team->bar.arrive_and_wait();
        v += o;
    }
    return v;
}
double lane_excl_scan(int si, int T, double v) {
    if (T == 1 || !t_team) return 0.0;
    double inc = v;
    for (int s = 1; s < T; s <<= 1) {
        t_team->board[si] = inc;
        t_team->bar.arrive_and_wait();
        const double o = (si >= s) ? t_team->board[si - s] : 0.0;
        t_team->bar.arrive_and_wait();
        if (si >= s) inc += o;
    }
    return inc - v;
}
bool lane_any(int si, int T, bool p) {
    if (T == 1 || !t_team) return p;
    t_team->flags[si] = p ? 1 : 0;
    t_team->bar.arrive_and_wait();
    int any = 0;
    for (int i = 0; i < T; ++i) any |= t_team->flags[i];
    t_team->bar.arrive_and_wait();
    return any != 0;
}
void lane_sync(int T) {
    if (T == 1 || !t_team) return;
    t_team->bar.arrive_and_wait();
}
int lane_argext(int si, int T, double v, bool want_max) {
    if (T == 1 || !t_team) return 0;
    int who = si;
    for (int s = T >> 1; s >= 1; s >>= 1) {
        t_team->board[si] = v;
        t_team->flags[si] = who;
        t_team->bar.arrive_and_wait();
        const double ov = t_team->board[si ^ s];
        const int ow = t_team->flags[si ^ s];
        t_team->bar.arrive_and_wait();
        const bool better = want_max ? (ov > v) : (ov < v);
        if (better || (ov == v && ow < who)) {
            v = ov;
            who = ow;
        }
    }
    return who;
}
void lane_argmax(int si, int T, double& best, int& best_n, double& best_use) {
    if (T == 1 || !t_team) return;
    for (int s = T >> 1; s >= 1; s >>= 1) {
        t_team->board[si] = best;
        t_team->flags[si] = best_n;
        t_team->board2[si] = best_use;
        t_team->bar.arrive_and_wait();
        const double ob = t_team->board[si ^ s], ou = t_team->board2[si ^ s];
        const int on = t_team->flags[si ^ s];
        t_team->bar.arrive_and_wait();
        if (ob > best || (ob == best && on < best_n)) {
            best = ob;
            best_n = on;
        }
        best_use = ou > best_use ? ou : best_use;
    }
}
}  // namespace pdq_emu

namespace {

struct Pack {
    std::vector<double> buf;
    DesignS d;
    double pinv[PDQ_MAX_P * PDQ_MAX_P];
    int full_rank;
    double s_mean_inv;
};

// the pack of design_create (pdq_api.cu): `offsets` as there, for the apeGLM call
Pack make_pack(const double* X, const double* sf, int N, int p, bool offsets = false) {
    Pack k;
    k.s_mean_inv = design_pack(X, sf, offsets, N, p, k.buf);
    k.d = DesignS{k.buf.data(), k.buf.data() + p, k.buf.data() + p + 1, N, design_row_stride(p), host_math_table()};
    design_linear_algebra(X, N, p, k.pinv, &k.full_rank);
    return k;
}

// k_size_factor_median, one "thread": each sample's median of log ratios against the log means `lm` (a non-finite entry leaves
// the gene out), exponentiated; `skip_zero` for poscounts
void size_factor_medians(const int64_t* counts, int64_t ld, int N, int G, const double* lm, bool skip_zero, double* sf) {
    std::vector<double> row((size_t)G);
    unsigned hist[514];
    SerialReducer red;
    for (int n = 0; n < N; ++n) {
        size_t cnt = 0;
        for (int g = 0; g < G; ++g) {
            bool keep;
            row[g] = log_ratio_entry(counts[(size_t)n * ld + g], lm[g], keep, skip_zero);
            cnt += keep;
        }
        sf[n] = exp(median_of(red, row.data(), (size_t)G, cnt, false, 0.0, hist));
    }
}

template <int P>
SmallMat<P> pinv_of(const Pack& k) {
    SmallMat<P> m;
    for (int i = 0; i < P * P; ++i) m.v[i] = k.pinv[i];
    return m;
}

const Group kOne{0, 1, 32};

// runs f(Group) once per lane of one gene: directly for one lane, on T threads sharing a LaneTeam otherwise
template <class F>
void with_lanes(F&& f) {
    const int T = g_lanes;
    if (T <= 1) {
        t_team = nullptr;
        f(kOne);
        return;
    }
    LaneTeam team(T);
    std::vector<std::thread> th;
    th.reserve((size_t)T);
    for (int si = 0; si < T; ++si)
        th.emplace_back([&team, &f, si, T] {
            t_team = &team;
            f(Group{si, T, 32 / T});
        });
    for (auto& t : th) t.join();
}

#define EMU_DISPATCH(p, ...)                               \
    switch (p) {                                           \
        case 1: { constexpr int P = 1; __VA_ARGS__; } break; \
        case 2: { constexpr int P = 2; __VA_ARGS__; } break; \
        case 3: { constexpr int P = 3; __VA_ARGS__; } break; \
        case 4: { constexpr int P = 4; __VA_ARGS__; } break; \
        case 5: { constexpr int P = 5; __VA_ARGS__; } break; \
        case 6: { constexpr int P = 6; __VA_ARGS__; } break; \
        case 7: { constexpr int P = 7; __VA_ARGS__; } break; \
        case 8: { constexpr int P = 8; __VA_ARGS__; } break; \
        case 9: { constexpr int P = 9; __VA_ARGS__; } break; \
        case 10: { constexpr int P = 10; __VA_ARGS__; } break; \
        case 11: { constexpr int P = 11; __VA_ARGS__; } break; \
        case 12: { constexpr int P = 12; __VA_ARGS__; } break; \
        case 13: { constexpr int P = 13; __VA_ARGS__; } break; \
        case 14: { constexpr int P = 14; __VA_ARGS__; } break; \
        case 15: { constexpr int P = 15; __VA_ARGS__; } break; \
        case 16: { constexpr int P = 16; __VA_ARGS__; } break; \
        default: return -3;                                \
    }

}  // namespace

extern "C" {

int emu_lin_reg_mu(const int64_t* counts, int64_t ld, int N, int G, const double* sf, const double* X, int p, double min_mu,
                   double* mu) {
    Pack k = make_pack(X, sf, N, p);
    EMU_DISPATCH(p, {
        const SmallMat<P> pi = pinv_of<P>(k);
        for (int g = 0; g < G; ++g)
            with_lanes([&](const Group& grp) { linmu_gene<P>(grp, k.d, pi, counts + g, ld, min_mu, mu + g, G, true); });
    });
    return 0;
}

int emu_irls(const int64_t* counts, int64_t ld, int N, int G, const double* sf, const double* X, int p, const double* disp,
             double min_mu, double beta_tol, double min_beta, double max_beta, int maxiter, double* beta, double* mu,
             double* hat, double* conv, int* status, int force_optimizer) {
    Pack k = make_pack(X, sf, N, p);
    EMU_DISPATCH(p, {
        const SmallMat<P> pi = pinv_of<P>(k);
        // force_optimizer: bit 0 = every gene takes the optimiser branch, bit 1 = that branch reports failure (grid_fit_beta at p = 2)
        const IrlsParams prm{min_mu, beta_tol, min_beta, max_beta, maxiter, k.full_rank, design_distinct_rows(X, N, p, 16) <= 16,
                             (force_optimizer >> 1) & 1};
        double lg_tab[kPsiK];
        for (int g = 0; g < G; ++g) {
            with_lanes([&](const Group& grp) {
                irls_gene<P>(grp, k.d, pi, prm, counts + g, ld, disp[g], beta + (size_t)g * P, mu + g, hat + g, G, conv + g,
                             status + g, true, lg_tab, kLogFact);
            });
            if (force_optimizer & 1) status[g] = kIrlsNeedsOptimizer;
            if (status[g] == kIrlsNeedsOptimizer)
                with_lanes([&](const Group& grp) {
                    irls_optimizer_gene<P>(grp, k.d, pi, prm, counts + g, ld, disp[g], beta + (size_t)g * P, mu + g, hat + g, G,
                                           conv + g, true);
                });
        }
    });
    return 0;
}

int emu_alpha_mle_hint(const int64_t* counts, int64_t ld, int N, int G, const double* X, int p, const double* mu, int64_t ld_mu,
                       const double* alpha_hat, double min_disp, double max_disp, double prior_var, int cr_reg, int prior_reg,
                       double* alpha, double* conv, int* status, int force_grid, const double* hint_in, double* hint_out);

int emu_alpha_mle(const int64_t* counts, int64_t ld, int N, int G, const double* X, int p, const double* mu, int64_t ld_mu,
                  const double* alpha_hat, double min_disp, double max_disp, double prior_var, int cr_reg, int prior_reg,
                  double* alpha, double* conv, int* status, int force_grid) {
    return emu_alpha_mle_hint(counts, ld, N, G, X, p, mu, ld_mu, alpha_hat, min_disp, max_disp, prior_var, cr_reg, prior_reg, alpha, conv,
                              status, force_grid, nullptr, nullptr);
}

// hint_in / hint_out: [G][2], see alpha_gene
int emu_alpha_mle_hint(const int64_t* counts, int64_t ld, int N, int G, const double* X, int p, const double* mu, int64_t ld_mu,
                       const double* alpha_hat, double min_disp, double max_disp, double prior_var, int cr_reg, int prior_reg,
                       double* alpha, double* conv, int* status, int force_grid, const double* hint_in, double* hint_out) {
    Pack k = make_pack(X, nullptr, N, p);
    EMU_DISPATCH(p, {
        const AlphaParams prm{log(min_disp), log(max_disp), prior_var, cr_reg, prior_reg};
        double psi[2 * kPsiK];
        for (int g = 0; g < G; ++g) {
            with_lanes([&](const Group& grp) {
                alpha_gene<P>(grp, k.d, prm, counts + g, ld, mu + g, ld_mu, alpha_hat[g], alpha + g, conv + g, status + g, true, psi,
                              hint_in ? hint_in + 2 * g : nullptr, hint_out ? hint_out + 2 * g : nullptr);
            });
            if (force_grid) {
                status[g] = kAlphaNeedsGrid;
                conv[g] = 0.0;
            }
            if (status[g] == kAlphaNeedsGrid)
                with_lanes([&](const Group& grp) {
                    alpha_grid_gene<P>(grp, k.d, prm.lo, prm.hi, counts + g, ld, mu + g, ld_mu, alpha + g, true);
                });
        }
    });
    return 0;
}

int emu_lfc_shrink(const double* X, const int64_t* counts, int64_t ld, int N, int G, int p, const double* size, const double* offset,
                   double prior_no_shrink_scale, double prior_scale, int shrink_index, double* lfcs, double* inv_hessians, double* conv,
                   int* status, int force_grid) {
    Pack k = make_pack(X, offset, N, p, true);
    const ShrinkParams prm{1.0 / (prior_no_shrink_scale * prior_no_shrink_scale), prior_scale * prior_scale, shrink_index};
    EMU_DISPATCH(p, {
        for (int g = 0; g < G; ++g)
            with_lanes([&](const Group& grp) {
                shrink_gene<P>(grp, k.d, prm, counts + g, ld, size[g], lfcs + (size_t)g * P, inv_hessians + (size_t)g * P * P,
                               conv + g, status + g, true, force_grid != 0);
            });
    });
    if (p == 2)
        for (int g = 0; g < G; ++g)
            if (status[g] == kShrinkNeedsGrid)
                with_lanes([&](const Group& grp) {
                    shrink_grid_gene(grp, k.d, prm, counts + g, ld, size[g], lfcs + (size_t)g * 2, inv_hessians + (size_t)g * 4, true);
                });
    return 0;
}

int emu_wald_test(const double* X, int N, int p, const double* disp, const double* lfc, const double* mu, int64_t ld_mu, int G,
                  const double* ridge, const double* contrast, double lfc_null, int alt, double* pv, double* stat,
                  double* se) {
    Pack k = make_pack(X, nullptr, N, p);
    EMU_DISPATCH(p, {
        WaldParams<P> prm;
        for (int i = 0; i < P * P; ++i) prm.ridge[i] = ridge[i];
        for (int i = 0; i < P; ++i) prm.contrast[i] = contrast[i];
        prm.lfc_null = lfc_null;
        prm.alt = alt;
        for (int g = 0; g < G; ++g)
            with_lanes([&](const Group& grp) {
                wald_gene<P>(grp, k.d, prm, disp[g], lfc + (size_t)g * P, mu + g, ld_mu, pv + g, stat + g, se + g, true);
            });
    });
    return 0;
}

int emu_rough(const double* normed, int64_t ld, int N, int G, const double* X, int p, double* alpha) {
    Pack k = make_pack(X, nullptr, N, p);
    EMU_DISPATCH(p, {
        const SmallMat<P> pi = pinv_of<P>(k);
        for (int g = 0; g < G; ++g)
            with_lanes([&](const Group& grp) {
                const double a = rough_disp_gene<P>(grp, k.d, pi, NormedF64{normed + g, ld});
                if (grp.si == 0) alpha[g] = a;
            });
    });
    return 0;
}

int emu_moments(const double* normed, int64_t ld, int N, int G, const double* sf, double* alpha, double* all_zero) {
    std::vector<double> ones((size_t)N, 1.0);
    Pack k = make_pack(ones.data(), sf, N, 1);
    for (int g = 0; g < G; ++g) {
        with_lanes([&](const Group& grp) {
            double mean;
            bool az;
            const double a = moments_disp_gene(grp, k.d, NormedF64{normed + g, ld}, k.s_mean_inv, mean, az);
            if (grp.si == 0) {
                alpha[g] = a;
                all_zero[g] = az ? 1.0 : 0.0;
            }
        });
    }
    return 0;
}

int emu_mom_from_counts(const int64_t* counts, int64_t ld, int N, int G, const double* sf, const double* X, int p,
                        double min_disp, double max_disp, double* alpha, double* normed_mean, double min_mu, double* mu_hat) {
    Pack k = make_pack(X, sf, N, p);
    EMU_DISPATCH(p, {
        const SmallMat<P> pi = pinv_of<P>(k);
        for (int g = 0; g < G; ++g)
            with_lanes([&](const Group& grp) {
                mom_fused_gene<P>(grp, k.d, pi, counts + g, ld, k.s_mean_inv, min_disp, max_disp, min_mu, alpha + g, normed_mean + g,
                                  mu_hat ? mu_hat + g : nullptr, G, true);
            });
    });
    return 0;
}

int emu_trend_fit(const double* x, const double* t, size_t n, int x_is_mean, double lo, double hi, int outer, double min_disp,
                  double trigamma_c, int with_prior, double* out16) {
    std::vector<double> xs(n), ts(n), res(n);
    unsigned hist[514];
    SerialReducer red;
    trend_prepare(red, x, t, n, x_is_mean != 0, lo, hi, xs.data(), ts.data());
    TrendOut o = trend_fit_outer(red, xs.data(), ts.data(), n, outer != 0);
    if (with_prior && o.status == 0.0) trend_prior(red, x, t, n, lo, hi, min_disp, trigamma_c, res.data(), hist, o);
    memcpy(out16, &o, sizeof o);
    return 0;
}

int emu_cooks(const int64_t* counts, int64_t ld, int N, int G, const double* sf, const double* X, int p, const double* mu,
              const double* hat, int64_t ld2, double cutoff, double* cooks, double* disp, double* outlier, double* replaced) {
    Pack k = make_pack(X, sf, N, p);
    const std::vector<int> plan = design_cell_plan(X, N, p);
    const int n_cells = plan[0];
    const int nf = (int)plan.size() - (2 + n_cells + 1);
    const CellPlan cp{plan.data() + 2 + n_cells + 1, plan.data() + 2, n_cells, plan[1]};
    std::vector<double> vals((size_t)2 * nf);
    EMU_DISPATCH(p, {
        for (int g = 0; g < G; ++g)
            with_lanes([&](const Group& grp) {
                cooks_gene<P>(grp, k.d, cp, counts + g, ld, mu + g, hat + g, ld2, cutoff, vals.data(), vals.data() + nf,
                              cooks ? cooks + g : nullptr, G, disp + g, outlier + g, replaced + g, true);
            });
    });
    return 0;
}

// k_wide_cooks: cooks_gene_cols with the design width `p` at run time (any p >= 1, no template width), at the lane count of
// emu_set_lanes (the device runs it at 32)
int emu_cooks_cols(const int64_t* counts, int64_t ld, int N, int G, const double* sf, const double* X, int p, const double* mu,
                   const double* hat, int64_t ld2, double cutoff, double* cooks, double* disp, double* outlier, double* replaced) {
    if (p < 1) return -2;
    std::vector<double> buf;
    design_pack(X, sf, false, N, p, buf);
    const DesignS d{buf.data(), buf.data() + p, buf.data() + p + 1, N, design_row_stride(p), host_math_table()};
    const std::vector<int> plan = design_cell_plan(X, N, p);
    const int n_cells = plan[0];
    const int nf = (int)plan.size() - (2 + n_cells + 1);
    const CellPlan cp{plan.data() + 2 + n_cells + 1, plan.data() + 2, n_cells, plan[1]};
    std::vector<double> vals((size_t)2 * nf);
    for (int g = 0; g < G; ++g)
        with_lanes([&](const Group& grp) {
            cooks_gene_cols(grp, d, p, cp, counts + g, ld, mu + g, hat + g, ld2, cutoff, vals.data(), vals.data() + nf,
                            cooks ? cooks + g : nullptr, G, disp + g, outlier + g, replaced + g, true);
        });
    return 0;
}

// pdq_size_factors_ex (k_log_means, k_size_factor_median, k_size_factor_geomean; one "thread"): `control` and `logmeans` (G,), the
// raw log means, may be NULL; -2 (PDQ_ERR_INVALID) for an unknown kind
int emu_size_factors_ex(const int64_t* counts, int64_t ld, int N, int G, int kind, const uint8_t* control, double* sf, double* logmeans) {
    if (kind != kSfRatio && kind != kSfPoscounts) return -2;
    std::vector<double> lm((size_t)G), kept((size_t)G);
    for (int g = 0; g < G; ++g) {
        double s = 0.0;
        for (int n = 0; n < N; ++n) s += log_mean_term(counts[(size_t)n * ld + g], kind);
        lm[g] = s / (double)N;
        kept[g] = kept_logmean(lm[g], kind, control == nullptr || control[g] != 0);
    }
    if (logmeans) memcpy(logmeans, lm.data(), (size_t)G * sizeof(double));
    size_factor_medians(counts, ld, N, G, kept.data(), kind == kSfPoscounts, sf);
    if (kind == kSfPoscounts) {
        double s = 0.0;
        for (int n = 0; n < N; ++n) s += log(sf[n]);
        const double gm = exp(s / (double)N);
        for (int n = 0; n < N; ++n) sf[n] = sf[n] / gm;
    }
    return 0;
}

// pdq_size_factors: median of ratios over every gene
int emu_size_factors(const int64_t* counts, int64_t ld, int N, int G, double* sf, double* logmeans) {
    return emu_size_factors_ex(counts, ld, N, G, kSfRatio, nullptr, sf, logmeans);
}

// pdq_size_factors_from_logmeans: held-out samples against the caller's log means
int emu_size_factors_from_logmeans(const int64_t* counts, int64_t ld, int N, int G, const double* lm, double* sf) {
    size_factor_medians(counts, ld, N, G, lm, false, sf);
    return 0;
}

int emu_vst_transform(const int64_t* counts, int64_t ld, int N, int G, const double* sf, int kind, double c0, double c1, double* out,
                      int64_t ld_out) {
    if (kind != kVstParametric && kind != kVstMean) return -2;
    const VstParams prm{kind, c0, c1};
    for (int n = 0; n < N; ++n)
        for (int g = 0; g < G; ++g) out[(size_t)n * ld_out + g] = vst_value(counts[(size_t)n * ld + g], sf[n], prm);
    return 0;
}

// pdq_wald_contrasts: K contrasts of fitted coefficients, mu built from them (wald_contrasts_gene); outputs (K, ld_out).
// -2 (PDQ_ERR_INVALID) for K <= 0, ld_out < G or an unknown alternative, -3 for p > 16.
int emu_wald_contrasts(const double* X, const double* sf, int N, int p, const double* disp, const double* lfc, int G, const double* ridge,
                       int K, const double* contrasts, const double* lfc_null, const int* alt, double* pv, double* stat, double* se,
                       int64_t ld_out) {
    if (K <= 0 || ld_out < G) return -2;
    std::vector<double> tab((size_t)K * (p + 2));
    if (wald_contrast_table(K, p, contrasts, lfc_null, alt, tab.data()) >= 0) return -2;
    Pack k = make_pack(X, sf, N, p);
    EMU_DISPATCH(p, {
        for (int g = 0; g < G; ++g)
            with_lanes([&](const Group& grp) {
                wald_contrasts_gene<P>(grp, k.d, ridge, disp[g], lfc + (size_t)g * P, K, tab.data(), pv + g, stat + g, se + g, ld_out, true);
            });
    });
    return 0;
}

int emu_set_lanes(int lanes) {
    if (lanes != 1 && lanes != 2 && lanes != 4 && lanes != 8 && lanes != 16 && lanes != 32) return -1;
    g_lanes = lanes;
    return 0;
}

long emu_sweep_count(int reset) {
    long v = g_emu_irls_sweeps;
    if (reset) g_emu_irls_sweeps = 0;
    return v;
}
long emu_eval_count(int reset) {
    long v = g_emu_alpha_evals;
    if (reset) g_emu_alpha_evals = 0;
    return v;
}
double emu_fast_log(double x) { return fast_log(x); }
double emu_fast_exp(double x) { return fast_exp(x); }
double emu_lgamma(double x) { return lgamma_pos(x); }
double emu_digamma(double x) { return digamma_pos(x); }
// the host branches of every primitive, with the GPU probe's op codes (tests/gpu_probe/math_ops.h)
int emu_math(int op, const double* x, const double* y, double* out, int n) {
    if (op < 0 || op >= pdq_probe::kNumOps) return -1;
    for (int i = 0; i < n; ++i) out[i] = pdq_probe::apply(op, x[i], y[i], host_math_table());
    return 0;
}
// the per-gene tables of G genes, each built by T lanes (threads) with the device's exchange patterns: [G][4 kPsiK]
int emu_tables(const double* r, int G, int T, double* out) {
    const int saved = g_lanes;
    if (emu_set_lanes(T) != 0) return -1;
    for (int g = 0; g < G; ++g) {
        double tab[pdq_probe::kTabOut];
        with_lanes([&](const Group& grp) { pdq_probe::build_tables(grp, tab, r[g], host_math_table()); });
        memcpy(out + (size_t)g * pdq_probe::kTabOut, tab, sizeof tab);
    }
    g_lanes = saved;
    return 0;
}
// kMathTab as the emulator (and the device, from the same initialiser) sees it; layout[] = {kLogTabBits, kLogTabN, kLogTabSplit,
// kExpTabN}; returns kMathTabLen
int emu_math_table(double* out, int* layout) {
    memcpy(out, host_math_table(), sizeof(double) * kMathTabLen);
    layout[0] = kLogTabBits;
    layout[1] = kLogTabN;
    layout[2] = kLogTabSplit;
    layout[3] = kExpTabN;
    return kMathTabLen;
}
int emu_design_rank_pinv(const double* X, int N, int p, double* pinv) {
    int fr;
    design_linear_algebra(X, N, p, pinv, &fr);
    return fr;
}

}  // extern "C"
