// pdq_internal.h -- host-side declarations shared by pdq_api.cu (C ABI) and the kernel units (launchers).
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
    double pinv[PDQ_MAX_P * PDQ_MAX_P];  // (X^T X)^+ row-major p x p (host copy, passed by value to kernels), p <= PDQ_MAX_P
    double* pinv_dev = nullptr;          // device copy of (X^T X)^+ for wide designs (p > PDQ_MAX_P), read by pdq_wide.cu
    double* wald_dev = nullptr;          // p > PDQ_MAX_P: the Wald ridge (packed) and contrast of the latest launch, read by pdq_wide.cu
    int warps = 0;                       // p > PDQ_MAX_P_WIDE: warps per gene (0: the built-in choice; PDQ_LARGE_WARPS tuning hook);
                                         // unused below, where with_warps (pdq_wide.cu) always picks one
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

// launchers: those that take a DesignDev route by width (pdq_dispatch.cu) to pdq_kernels.cu or pdq_wide.cu, the others are in
// pdq_common.cu; each returns the number of kernels launched or a negative pdq_status
int launch_lin_reg_mu(const LaunchCfg&, const DesignDev&, const int64_t* counts, int64_t ld, int G, double min_mu,
                      double* mu_out, int64_t ld_out);
int launch_irls(const LaunchCfg&, const DesignDev&, const int64_t* counts, int64_t ld, int G, const double* disp,
                const IrlsHost& prm, double* beta, double* mu, double* hat, int64_t ld_out, double* conv, int* status,
                int* n_fallback, const WaldHost* wald = nullptr);
int launch_alpha_mle(const LaunchCfg&, const DesignDev&, const int64_t* counts, int64_t ld, int G, const double* mu,
                     int64_t ld_mu, const double* alpha_hat, double min_disp, double max_disp, double prior_var,
                     const double* prior_var_dev, int cr_reg, int prior_reg, double* alpha, double* conv, int* status,
                     const double* hint_in = nullptr, double* hint_out = nullptr);
// MAP dispersion search -> final dispersions -> LFC fit + Wald test as one persistent launch (k_map_irls): device pointers of the
// stages' inputs and outputs, everything but the counts and the small host parameters (IrlsHost, WaldHost)
struct TailHost {
    const double* mu;          // (N, G) means the dispersion search runs on
    int64_t ld_mu;
    const double *fitted, *gw, *hint_in;  // trend values, genewise dispersions, [G][2] hints of the genewise search
    const double* trend16;     // trend record (TrendOut)
    double min_disp, max_disp, prior_var;
    const double* prior_var_dev;  // overrides prior_var when set
    double *map, *map_conv, *disp, *outlier;
    double *beta, *mu_out, *hat, *conv;
    int64_t ld_out;
    int *status_map, *status_irls;  // G ints each
    unsigned* tile_done;       // >= number of warp tiles words, zeroed when allocated and owned by these launches since
    unsigned long long* err;   // device address of a mapped host word: non-zero after a tile wait gave up
};
// LaunchCfg::tickets must hold 32 ints, all zero when the context is created (ints 16.. are the launch's control words)
int launch_map_irls(const LaunchCfg&, const DesignDev&, const int64_t* counts, int64_t ld, int G, const TailHost&, const IrlsHost&,
                    const WaldHost&);
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
// the lin_reg_mu branch's start values and the genewise dispersion search in one persistent launch (k_mom_alpha, then k_alpha_grid):
// what launch_mom_from_counts followed by launch_alpha_mle (cr_reg on, no prior, alpha_hat = mom) writes, bit for bit.  `mu_hat`
// is required.  LaunchCfg::tickets as for launch_map_irls.
int launch_mom_alpha(const LaunchCfg&, const DesignDev&, const int64_t* counts, int64_t ld, int G, double min_disp, double max_disp,
                     double min_mu, double* mom, double* normed_mean, double* mu_hat, int64_t ld_mu, double* alpha, double* conv,
                     int* status, double* hint_out);
int launch_mu_from_lfc(const LaunchCfg&, const DesignDev&, const double* lfc, int G, double* mu, int64_t ld_out);

// `fitted` (may be null, x_is_mean only): c0 + c1 / x[i] from the final coefficients, written by the same launch
int launch_trend_fit(const LaunchCfg&, const double* x, const double* t, double* scratch3n, size_t n, int x_is_mean,
                     double lo, double hi, int outer, double min_disp, double trigamma_c, int with_prior, double* out16,
                     double* fitted = nullptr);
// `ws`: cooks_ws_bytes(d, G) bytes of device workspace, null when that is 0
int launch_cooks(const LaunchCfg&, const DesignDev&, const int64_t* counts, int64_t ld, int G, const double* mu, const double* hat,
                 int64_t ld2, double cutoff, double* cooks, int64_t ld_out, double* disp, double* outlier, double* replaced, double* ws);
// bytes of the global workspace launch_cooks stages the genes' cell members in: 0 where they fit in shared memory (see
// cooks_in_smem, pdq_launch.cuh)
size_t cooks_ws_bytes(const DesignDev& d, int G);
int launch_lfc_shrink(const LaunchCfg&, const DesignDev&, const int64_t* counts, int64_t ld, int G, const double* size,
                      double prior_no_shrink_scale, double prior_scale, int shrink_index, double* beta, double* inv_hessian,
                      double* conv, int* status);
int launch_gather_cols(cudaStream_t stream, const double* in, int64_t ld_in, int N, const int* idx, int R, double* out, int64_t ld_out);
int launch_column_sums(cudaStream_t stream, const int64_t* counts, int64_t ld, int N, int G, double* sums);
int launch_scatter_rows(cudaStream_t stream, const double* in, double* out, const int* perm, int n, int nvec, int64_t stride, int width);
// `seg` (host): nseg rows of (offset in doubles, rows, width, permuted); see pdq_scatter_segments_dev
constexpr int kMaxScatterSegs = 16;
int launch_scatter_segments(cudaStream_t stream, const double* in, double* out, const int* src, int nseg, const int64_t* seg);
int launch_hash(cudaStream_t stream, int sm_count, const void* dptr, size_t words, uint64_t* out2 /* device, zeroed */);
int launch_fp64_peak(const LaunchCfg&, double* out /* sm_count * 8 * 256 doubles */, int iters, double* flop);
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

// multiple testing (pdq_padj.cu): device scratch of one call over K rows of G p-values, carved by padj_layout from one buffer
struct PadjScratch {
    uint64_t *keys_in, *keys;  // (K, G): the p-values as uploaded, then the sort keys; sorted.  keys_in takes pdq_padj_bh's output
    int *vals_in, *vals;       // (K, G) gene indices, sorted with the keys
    double *bm, *bm_sorted;    // (G,) base means
    uint64_t* masks;           // (G,) bit i: base mean >= cutoff i
    int* counters;             // K set sizes, then the count of p-values outside [0, 1]
    double *theta, *cutoffs;   // kPadjMaxTheta each
    double* row_cutoff;        // (K,) pdq_padj_bh's cutoffs
    int *num_rej, *totals;     // (K, n_theta)
    int* chunk_counts;         // (K, n_theta, chunks)
    double *chunk_min, *suffix;  // (K, chunks)
    void* temp;                // cub's temporary storage
    size_t temp_bytes;
};
// bytes of the scratch (base may be NULL: sizes only); fills `s` with pointers into `base`
size_t padj_layout(int G, int K, int n_theta, void* base, PadjScratch* s);
// inputs in s.bm, s.keys_in (raw p-values), s.theta; outputs s.cutoffs, s.num_rej, s.counters[K] (p-values outside [0, 1])
int launch_padj_rejections(cudaStream_t, const PadjScratch& s, int G, int K, int n_theta, double alpha);
// inputs in s.bm, s.keys_in, s.row_cutoff; output `padj` (K, ld_out) device, which may be s.keys_in
int launch_padj_bh(cudaStream_t, const PadjScratch& s, int G, int K, double* padj, int64_t ld_out);

// largest dynamic shared memory a kernel of this library may ask for (H100: 227 KB per CTA)
constexpr size_t kMaxDynSmem = 227 * 1024;

}  // namespace pdq
