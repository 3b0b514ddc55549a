// pdq_internal.h -- host-side declarations shared by pdq_api.cu (C ABI) and pdq_kernels.cu (launchers).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/pydeseq2_b200.h"

namespace pdq {

struct DesignDev {
    double* pack;       // device; layout: design_pack (pdq_host_linalg.h), DESIGN.md §2
    int N, RS, p;
    int full_rank;      // np.linalg.matrix_rank(X) == p  (utils.py:349)
    int few_rows;       // X has at most 16 distinct rows (categorical design): k_irls reuses exp(x'beta) across equal rows
    double pinv[PDQ_MAX_P * PDQ_MAX_P];  // (X^T X)^+ row-major p x p (host copy, passed by value to kernels)
    double s_mean_inv;  // mean(1 / size_factors)  (utils.py:880)
    int staged;         // the pack is small enough to be copied into shared memory by every block (else read from global / L1)
    size_t smem_bytes;  // dynamic shared memory the kernels need for the design: staged pack + mbarrier, or the mbarrier alone
    int* cell_plan;     // device: [n_cells, global_mode, starts (n_cells + 1), order (n_in_cells)]  (Cook's distances)
    int n_cells, n_in_cells, plan_len;
};

constexpr size_t kGridScratchBytes = 32768;  // LaunchCfg::grid_scratch (accumulators and value bins of k_trend_prior_grid)

struct LaunchCfg {
    cudaStream_t stream;
    int lgT;       // log2(lanes per gene)
    int sm_count;
    int* tickets;  // device ints: tile counters of the persistent kernels
    int debug;     // PDQ_DEBUG_* test hooks
    void* grid_scratch = nullptr;  // device scratch of the grid-wide trend fit (launch_trend_fit), kGridScratchBytes
};

struct IrlsHost {
    double min_mu, beta_tol, min_beta, max_beta;
    int maxiter;
};

// Wald test fused into the IRLS launch (resident pipeline): host copies of the small parameters, device outputs
struct WaldHost {
    const double* ridge;     // p x p row-major (host)
    const double* contrast;  // p (host)
    double lfc_null;
    int alt;
    double *pv, *stat, *se;  // device, one per gene
};

// launchers (pdq_kernels.cu); each returns the number of kernels launched or a negative pdq_status
int launch_lin_reg_mu(const LaunchCfg&, const DesignDev&, const int64_t* counts, int64_t ld, int G, double min_mu,
                      double* mu_out, int64_t ld_out);
int launch_irls(const LaunchCfg&, const DesignDev&, const int64_t* counts, int64_t ld, int G, const double* disp,
                const IrlsHost& prm, double* beta, double* mu, double* hat, int64_t ld_out, double* conv, int* status,
                int* n_fallback, const WaldHost* wald = nullptr);
int launch_alpha_mle(const LaunchCfg&, const DesignDev&, const int64_t* counts, int64_t ld, int G, const double* mu,
                     int64_t ld_mu, const double* alpha_hat, double min_disp, double max_disp, double prior_var,
                     const double* prior_var_dev, int cr_reg, int prior_reg, double* alpha, double* conv, int* status,
                     const double* hint_in = nullptr, double* hint_out = nullptr);
int launch_wald(const LaunchCfg&, const DesignDev&, const double* disp, const double* lfc, const double* mu,
                int64_t ld_mu, int G, const double* ridge, const double* contrast, double lfc_null, int alt,
                double* pv, double* stat, double* se);
// K contrasts from fitted coefficients: `ridge` p x p (host), `tab` (K, p + 2) device rows [contrast | lfc_null | alt]
int launch_wald_contrasts(const LaunchCfg&, const DesignDev&, const double* disp, const double* lfc, int G, const double* ridge, int K,
                          const double* tab, double* pv, double* stat, double* se, int64_t ld_out);
int launch_rough(const LaunchCfg&, const DesignDev&, const double* normed, int64_t ld, int G, double* alpha);
int launch_moments(const LaunchCfg&, const DesignDev&, const double* normed, int64_t ld, int G, double* alpha,
                   double* all_zero);
int launch_mom_from_counts(const LaunchCfg&, const DesignDev&, const int64_t* counts, int64_t ld, int G,
                           double min_disp, double max_disp, double* alpha, double* normed_mean, double min_mu, double* mu_hat,
                           int64_t ld_mu);
int launch_mu_from_lfc(const LaunchCfg&, const DesignDev&, const double* lfc, int G, double* mu, int64_t ld_out);

int launch_trend_fit(const LaunchCfg&, const double* x, const double* t, double* scratch3n, size_t n, int x_is_mean,
                     double lo, double hi, int outer, double min_disp, double trigamma_c, int with_prior, double* out16);
int launch_trend_eval(const LaunchCfg&, const double* means, size_t n, const double* out16, double* fitted);
int launch_cooks(const LaunchCfg&, const DesignDev&, const int64_t* counts, int64_t ld, int G, const double* mu, const double* hat,
                 int64_t ld2, double cutoff, double* cooks, int64_t ld_out, double* disp, double* outlier, double* replaced);
int launch_lfc_shrink(const LaunchCfg&, const DesignDev&, const int64_t* counts, int64_t ld, int G, const double* size,
                      double prior_no_shrink_scale, double prior_scale, int shrink_index, double* beta, double* inv_hessian,
                      double* conv, int* status);
int launch_gather_cols(cudaStream_t stream, const double* in, int64_t ld_in, int N, const int* idx, int R, double* out, int64_t ld_out);
int launch_column_sums(cudaStream_t stream, const int64_t* counts, int64_t ld, int N, int G, double* sums);
int launch_scatter_rows(cudaStream_t stream, const double* in, double* out, const int* perm, int n, int nvec, int64_t stride, int width);
int launch_hash(cudaStream_t stream, int sm_count, const void* dptr, size_t words, uint64_t* out2 /* device, zeroed */);
int launch_fp64_peak(const LaunchCfg&, double* out /* sm_count * 8 * 256 doubles */, int iters, double* flop);
int launch_size_factors(const LaunchCfg&, const int64_t* counts, int64_t ld, int N, int G, double* logmeans,
                        double* scratch, double* sf_out);
// kind kSfRatio / kSfPoscounts (pdq_trend.cuh); `control` (G,) may be NULL; `kept` (G,) scratch, NULL only for ratio over every gene
int launch_size_factors_ex(const LaunchCfg&, const int64_t* counts, int64_t ld, int N, int G, int kind, const uint8_t* control,
                           double* logmeans, double* kept, double* scratch, double* sf_out);
int launch_size_factors_from_logmeans(const LaunchCfg&, const int64_t* counts, int64_t ld, int N, int G, const double* logmeans,
                                      double* scratch, double* sf_out);
// kind 0 parametric (c0 = a0, c1 = a1), 1 mean (c0 = mean dispersion); see pdq_vst.cuh
int launch_vst_transform(const LaunchCfg&, const int64_t* counts, int64_t ld, int N, int G, const double* sf, int kind, double c0,
                         double c1, double* out, int64_t ld_out);
int launch_select_disp(const LaunchCfg&, const double* gw, const double* mp, const double* fitted, const double* out16,
                       size_t n, double lo, double hi, double* disp, double* outlier);

// largest dynamic shared memory a kernel of this library may ask for (H100: 227 KB per CTA)
constexpr size_t kMaxDynSmem = 227 * 1024;

}  // namespace pdq
