/*
 * pydeseq2_b200 -- C ABI of the H100 (sm_90a) backend for PyDESeq2's per-gene NB-GLM hot path.
 *
 * Every `pdq_*` compute entry point replaces one method of the reference's plugin interface
 * `pydeseq2.inference.Inference` (reference file:line cited per function).  The reference binds
 * to it with the ctypes stub shown in INTEGRATION.md (`pydeseq2_b200/_lib.py` is that stub).
 *
 * Conventions
 *   - extern "C", plain pointers + sizes, caller-allocated outputs, no ownership crosses the ABI.
 *   - Every function returns 0 on success or a negative `pdq_status`; `pdq_last_error(ctx)` gives text.
 *   - (N, G) arrays are the reference's native layout: C-contiguous, sample-major, the gene index
 *     is the fastest-varying one (`dds.py:752,759,779,902,954`: `self.X[:, self.non_zero_idx]`).
 *     `ld` arguments are the row pitch in ELEMENTS (ld == G for a contiguous array).
 *   - counts are int64, everything else float64 (`dds.py:245-249`); `converged` flags are returned
 *     as float64 0/1 (the caller stores them in a NaN-initialised float column, `dds.py:796-797`).
 *   - Two flavours of each hot call: `pdq_<op>` takes HOST buffers (the drop-in boundary: copies
 *     in, launches, copies out, synchronises) and `pdq_<op>_dev` takes DEVICE buffers allocated
 *     with `pdq_malloc` (resident pipeline; asynchronous on the context's stream).
 *   - One context per backend object, not re-entrant (the reference's caller is single-threaded).
 */
#ifndef PYDESEQ2_B200_H
#define PYDESEQ2_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct pdq_ctx pdq_ctx;       /* device, stream, scratch, NCCL communicator */
typedef struct pdq_design pdq_design; /* device-resident design pack: X (N x p), size factors, (XtX)^+ */

typedef enum pdq_status {
    PDQ_OK = 0,
    PDQ_ERR_CUDA = -1,        /* a CUDA runtime call failed */
    PDQ_ERR_INVALID = -2,     /* bad argument (null pointer, N<=0, p<1, ld<G, ...) */
    PDQ_ERR_UNSUPPORTED = -3, /* p > PDQ_MAX_P */
    PDQ_ERR_NCCL = -4,        /* NCCL missing or a collective failed */
    PDQ_ERR_NO_DEVICE = -5    /* no CUDA device / not an sm_90 part */
} pdq_status;

#define PDQ_MAX_P 16 /* design columns supported (p <= 8: register-resident p x p solvers; 9..16: the same code with the small matrices in local memory) */

/* alt_hypothesis codes of Inference.wald_test (utils.py:778-806) */
#define PDQ_ALT_NONE 0
#define PDQ_ALT_GREATER_ABS 1
#define PDQ_ALT_LESS_ABS 2
#define PDQ_ALT_GREATER 3
#define PDQ_ALT_LESS 4

/* ----------------------------------------------------------------- context / memory */
int pdq_ctx_create(int device, pdq_ctx** out);
void pdq_ctx_destroy(pdq_ctx* ctx);
const char* pdq_last_error(const pdq_ctx* ctx);
const char* pdq_version(void);
int pdq_device_count(void);
/* name, SM count, global memory bytes of the context's device */
int pdq_device_info(const pdq_ctx* ctx, char* name, size_t name_len, int* sm_count, size_t* mem_bytes);
/* lanes cooperating on one gene (1,2,4,8,16,32); 0 = choose from G (default) */
int pdq_set_lanes_per_gene(pdq_ctx* ctx, int lanes);
/* Test hook: PDQ_DEBUG_FORCE_IRLS_OPTIMIZER sends every gene of pdq_irls through the optimiser branch
 * (utils.py:374-413) and PDQ_DEBUG_FORCE_ALPHA_GRID every gene of pdq_alpha_mle through the grid fallback
 * (grid_search.py:54-142), so that the rarely taken kernels are exercised by the GPU test-suite ... */
#define PDQ_DEBUG_FORCE_IRLS_OPTIMIZER 1
#define PDQ_DEBUG_FORCE_ALPHA_GRID 2
/* ... and PDQ_DEBUG_FORCE_SHRINK_GRID every gene of pdq_lfc_shrink_nbinom_glm (two-column designs) through
 * grid_fit_shrink_beta (grid_search.py:224-318). */
#define PDQ_DEBUG_FORCE_SHRINK_GRID 4
/* PDQ_DEBUG_FAIL_IRLS_OPTIMIZER: the optimiser branch of pdq_irls behaves as if its minimiser had reported failure
 * (`res.success == False`, utils.py:402): two-column designs then take the reference's grid_fit_beta (grid_search.py:145-221). */
#define PDQ_DEBUG_FAIL_IRLS_OPTIMIZER 8
int pdq_set_debug_flags(pdq_ctx* ctx, int flags);
/* Measured FP64 FMA throughput of the context's device in TFLOP/s (dependent-free DFMA chains on every SM, CUDA-event timed):
 * the arithmetic roofline bench.py reports next to the HBM one -- the per-gene kernels are FP64-pipe bound (DESIGN.md §5). */
int pdq_fp64_peak_tflops(pdq_ctx* ctx, double* tflops_out);
/* number of kernel launches issued through this context so far (bench.py `gpu_launches`) */
int64_t pdq_launch_count(const pdq_ctx* ctx);
/* Number of times a context-owned scratch buffer has been re-allocated.  A CUDA graph captured with pdq_capture_begin / _end
 * holds pointers into that scratch: compare the value at capture time with the current one before pdq_graph_launch and
 * re-capture when it changed. */
int64_t pdq_buffer_epoch(const pdq_ctx* ctx);

/* Residency of the host-buffer entry points: (samples, genes) inputs of at least 1 MB are keyed on a 128-bit checksum of their
 * full content (computed by a few host threads at memory bandwidth) and kept on the device, (samples, genes) outputs are kept
 * under the same checksum computed on the device; a later call that is handed the same CONTENT -- the orchestrator passes the
 * same counts to four calls and feeds mu_hat / mu back (dds.py:752-779, 902, 954; ds.py:338), always as fresh host copies --
 * skips the upload.  Never keyed on pointers.  Environment: PDQ_RESIDENCY=0 disables, PDQ_RESIDENCY_BYTES caps the device bytes
 * (default: a quarter of device memory, at most 16 GB). */
int pdq_residency_stats(const pdq_ctx* ctx, int64_t* hits, int64_t* misses, int64_t* hit_bytes, int64_t* resident_bytes);
int pdq_residency_clear(pdq_ctx* ctx);

/* ---- count-matrix ingestion (SURVEY.md §8 f-4; the reference: pandas.read_csv(..., index_col=0).T,
 * examples/plot_pandas_io_example.py:57-66).  Host code, no device needed.  A CSV whose header line holds the column labels and
 * whose lines start with a row label, the remaining fields read counts (non-negative integers; labels may be double-quoted).
 * pdq_csv_scan: number of data rows / columns and the bytes the labels need.  pdq_csv_read_counts: parse with `threads` host
 * threads (0 = all, at most 32) into `out` -- with `transpose` the file's rows become the matrix' columns (the shipped datasets are
 * genes x samples, the hot path consumes (samples, genes) int64, dds.py:245-249) -- e.g. a page-locked buffer from pdq_host_alloc.
 * `labels` (may be NULL): column labels '\n'-separated, '\0', row labels '\n'-separated, '\0'.  A field that is not a non-negative
 * integer fails the call with PDQ_ERR_INVALID and its position in bad_row / bad_col. */
int pdq_csv_scan(const char* path, char sep, int64_t* n_rows, int64_t* n_cols, size_t* label_bytes);
int pdq_csv_read_counts(const char* path, char sep, int transpose, int64_t* out, int64_t ld_out, int64_t n_rows, int64_t n_cols,
                        char* labels, size_t label_cap, int threads, int64_t* bad_row, int64_t* bad_col);

int pdq_malloc(pdq_ctx* ctx, size_t bytes, void** dptr);
int pdq_free(pdq_ctx* ctx, void* dptr);
int pdq_host_alloc(pdq_ctx* ctx, size_t bytes, void** hptr); /* pinned host memory */
int pdq_host_free(pdq_ctx* ctx, void* hptr);
int pdq_memcpy_h2d(pdq_ctx* ctx, void* dst, const void* src, size_t bytes); /* async on ctx stream */
int pdq_memcpy_d2h(pdq_ctx* ctx, void* dst, const void* src, size_t bytes); /* async on ctx stream */
int pdq_memcpy_d2d(pdq_ctx* ctx, void* dst, const void* src, size_t bytes); /* async on ctx stream */
int pdq_memset(pdq_ctx* ctx, void* dst, int value, size_t bytes);
int pdq_sync(pdq_ctx* ctx);
/* CUDA-event timing on the context's stream (bench.py): record slot 0/1, elapsed ms between them */
int pdq_event_record(pdq_ctx* ctx, int slot);
int pdq_event_elapsed_ms(pdq_ctx* ctx, int slot_start, int slot_stop, float* ms);

/* CUDA-graph capture of a sequence of `*_dev` calls (the resident pipeline enqueues ~20 launches + copies per pass and
 * never synchronises in between: replaying them as ONE graph removes the per-launch host cost).  Everything enqueued on the
 * context between begin and end is recorded instead of executed; all buffers must already exist (run the sequence once
 * eagerly first).  `pdq_graph_launch` replays it on the context's stream. */
typedef struct pdq_graph pdq_graph;
int pdq_capture_begin(pdq_ctx* ctx);
int pdq_capture_end(pdq_ctx* ctx, pdq_graph** out);
int pdq_graph_launch(pdq_ctx* ctx, pdq_graph* g);
void pdq_graph_destroy(pdq_ctx* ctx, pdq_graph* g);

/* Design pack.  X is (N x p) row-major as the reference passes `design_matrix`
 * (`dds.py:740`), size_factors (N,) may be NULL for calls that take none (alpha_mle, wald_test). */
int pdq_design_create(pdq_ctx* ctx, const double* X, const double* size_factors, int N, int p,
                      pdq_design** out);
void pdq_design_destroy(pdq_ctx* ctx, pdq_design* d);

/* ----------------------------------------------------------------- hot path, host buffers
 * Inference.lin_reg_mu  (inference.py:12-43; default_inference.py:58-81; utils.py:682-715) */
int pdq_lin_reg_mu(pdq_ctx* ctx, const int64_t* counts, int64_t ld, int N, int G,
                   const double* size_factors, const double* X, int p, double min_mu,
                   double* mu_out /* (N,G) ld=G */);

/* Inference.irls  (inference.py:45-118; default_inference.py:83-124; utils.py:273-438).
 * `mu_out` is the UNclamped mean, `hat_out` the hat-matrix diagonal, both (N,G) with ld=G.
 * `n_fallback` (may be NULL) receives how many genes left the IRLS loop through the reference's
 * optimiser branch (utils.py:374-413). */
int pdq_irls(pdq_ctx* ctx, const int64_t* counts, int64_t ld, int N, int G,
             const double* size_factors, const double* X, int p, const double* disp,
             double min_mu, double beta_tol, double min_beta, double max_beta, int maxiter,
             double* beta_out /* (G,p) */, double* mu_out, double* hat_out,
             double* converged_out /* (G,) 0/1 */, int* n_fallback);

/* Inference.alpha_mle  (inference.py:120-177; default_inference.py:126-161; utils.py:441-564;
 * fallback grid_search.py:54-142).  `prior_disp_var` is ignored unless prior_reg != 0. */
int pdq_alpha_mle(pdq_ctx* ctx, const int64_t* counts, int64_t ld, int N, int G,
                  const double* X, int p, const double* mu, int64_t ld_mu,
                  const double* alpha_hat, double min_disp, double max_disp,
                  double prior_disp_var, int cr_reg, int prior_reg,
                  double* alpha_out /* (G,) */, double* converged_out /* (G,) 0/1 */);

/* Inference.wald_test  (inference.py:179-234; default_inference.py:163-198; utils.py:718-811).
 * `ridge` is (p,p) row-major, `contrast` (p,), `lfc_null` in natural log, `alt` a PDQ_ALT_* code. */
int pdq_wald_test(pdq_ctx* ctx, const double* X, int N, int p, const double* disp,
                  const double* lfc /* (G,p) */, const double* mu, int64_t ld_mu, int G,
                  const double* ridge, const double* contrast, double lfc_null, int alt,
                  double* pvalue_out, double* stat_out, double* se_out);

/* Inference.fit_rough_dispersions  (inference.py:236-258; utils.py:814-853) */
int pdq_fit_rough_dispersions(pdq_ctx* ctx, const double* normed_counts, int64_t ld, int N, int G,
                              const double* X, int p, double* alpha_out);
/* Inference.fit_moments_dispersions  (inference.py:260-281; utils.py:856-885).  Computes every
 * column; `all_zero_out[g]` = 1 marks the all-zero columns the reference drops (utils.py:878). */
int pdq_fit_moments_dispersions(pdq_ctx* ctx, const double* normed_counts, int64_t ld, int N, int G,
                                const double* size_factors, double* alpha_out, double* all_zero_out);

/* Inference.dispersion_trend_gamma_glm  (inference.py:283-307; default_inference.py:200-230): ONE gamma-GLM
 * fit  targets ~ c0 + c1 * covariates  (identity link) from (1, 1) under c >= 1e-12.  `coeffs_out` (2,),
 * `pred_out` (n,) = c0 + c1 * covariates, `converged_out` 0/1.  The reference's scipy L-BFGS-B stops within
 * ~4e-6 of the minimiser; this converges to the minimiser itself (DESIGN.md §6). */
int pdq_dispersion_trend_gamma_glm(pdq_ctx* ctx, const double* covariates, const double* targets, size_t n,
                                   double* coeffs_out, double* pred_out, int* converged_out);
/* Dispersion trend AND dispersion prior in one launch, host vectors: the whole outer loop of
 * DeseqDataSet.fit_dispersion_trend (dds.py:1199-1275: gamma-GLM fit, drop genes far from the curve, refit until the
 * coefficients settle) followed by fit_dispersion_prior (dds.py:840-884).  `out16` receives the record
 * [c0, c1, status (0 ok / 1 -> fall back to the mean trend), n_outer, n_used, n_iter, loss, last_converged, squared_logres,
 * prior_var, n_above, ...]; `fitted_out` (may be NULL) the fitted curve c0 + c1 / mean per gene.  NaN means are skipped. */
int pdq_trend_prior(pdq_ctx* ctx, const double* normed_means, const double* genewise, size_t n, double min_disp,
                    double max_disp, double trigamma_c, double* out16, double* fitted_out);

/* apeGLM LFC shrinkage -- Inference.lfc_shrink_nbinom_glm (inference.py:309-362) -> DefaultInference (default_inference.py:232-264)
 * -> utils.nbinomGLM (utils.py:990-1145), grid fallback grid_search.py:224-318; caller DeseqStats.lfc_shrink (ds.py:363-443).
 * SURVEY.md §8 f-3.  MAP coefficients under a normal(0, prior_no_shrink_scale) prior on every coefficient but `shrink_index`,
 * which gets the Cauchy-type prior of scale `prior_scale`; the optimiser is the reference's (unconstrained L-BFGS-B, ftol =
 * gtol = 1e-8 on the objective scaled by max(f(0), 1), start 0.1 * (-1)^j), iterate for iterate.  `size` (G,) = 1 / dispersion,
 * `offset` (N,) = log size factors.  Outputs: `lfcs_out` (G,p), `inv_hessians_out` (G,p,p) = inverse of the reference's Hessian
 * expression at the result (utils.py:1091-1108, 1143), `converged_out` (G,) 0/1 = scipy's `res.success`; genes that did not
 * converge are refitted on the 2-D grid when p == 2 (their flag stays 0), `*n_grid` (may be NULL) counts them. */
int pdq_lfc_shrink_nbinom_glm(pdq_ctx* ctx, const double* X, const int64_t* counts, int64_t ld, int N, int G, int p,
                              const double* size, const double* offset, double prior_no_shrink_scale, double prior_scale,
                              int shrink_index, double* lfcs_out, double* inv_hessians_out, double* converged_out, int* n_grid);

/* Median-of-ratios size factors -- preprocessing.deseq2_norm_fit/transform (preprocessing.py:31-102), the step before the
 * plugin calls (SURVEY.md §8 f-2): per-gene mean of log counts, genes holding a zero dropped, per-sample exact median
 * of log(count) - gene mean (radix select), exponentiated.  `sf_out` (N,).  All entries NaN when every gene holds a zero
 * (the reference then switches to its iterative fallback, dds.py:682-690). */
int pdq_size_factors(pdq_ctx* ctx, const int64_t* counts, int64_t ld, int N, int G, double* sf_out, double* logmeans_out /* per-gene mean log count (-inf when the gene holds a zero), may be NULL */);

/* Cook's distances -- DeseqDataSet.calculate_cooks (dds.py:986-1040) with the trimmed-moments dispersion
 * (utils.py:914-960; cells = identical design rows with >= 3 replicates) -- and the two per-gene decisions derived from them:
 * `outlier_out` = the p-value filter of cooks_outlier() (dds.py:1066-1110, no prior refit), `replaced_out` = any distance above
 * `cutoff` (dds.py:1320-1323).  `cutoff` = F.ppf(0.99, p, N - p).  `mu`/`hat` are the outputs of pdq_irls.  `cooks_out` (N,G)
 * may be NULL when only the per-gene results are wanted (saves the 8*N*G-byte copy).  SURVEY.md §8 f-1. */
int pdq_calculate_cooks(pdq_ctx* ctx, const int64_t* counts, int64_t ld, int N, int G, const double* size_factors,
                        const double* X, int p, const double* mu, const double* hat, int64_t ld2, double cutoff,
                        double* cooks_out, double* robust_disp_out, double* outlier_out, double* replaced_out);

/* ----------------------------------------------------------------- hot path, device-resident
 * Same semantics; every pointer except `design` is device memory from pdq_malloc.  Asynchronous. */
int pdq_lin_reg_mu_dev(pdq_ctx* ctx, const pdq_design* design, const int64_t* counts, int64_t ld, int G,
                       double min_mu, double* mu_out, int64_t ld_out);
int pdq_irls_dev(pdq_ctx* ctx, const pdq_design* design, const int64_t* counts, int64_t ld, int G,
                 const double* disp, double min_mu, double beta_tol, double min_beta, double max_beta,
                 int maxiter, double* beta_out, double* mu_out, double* hat_out, int64_t ld_out,
                 double* converged_out, int* n_fallback_dev /* device int, may be NULL */);
/* pdq_irls_dev + pdq_wald_test_dev in one launch: the Wald test (ds.py:303-360 -> utils.py:718-811) of the coefficients the
 * fit returns, built from the X^T W X of the last IRLS sweep (corrected for samples on the min_mu clamp, because the
 * orchestrator's test uses mu = sf * exp(X beta) unclamped, ds.py:320-324) instead of a second pass over mu.  `disp` serves
 * both.  Results equal calling the two entry points in sequence up to rounding. */
int pdq_irls_wald_dev(pdq_ctx* ctx, const pdq_design* design, const int64_t* counts, int64_t ld, int G,
                      const double* disp, double min_mu, double beta_tol, double min_beta, double max_beta,
                      int maxiter, double* beta_out, double* mu_out, double* hat_out, int64_t ld_out,
                      double* converged_out, int* n_fallback_dev, const double* ridge_host,
                      const double* contrast_host, double lfc_null, int alt, double* pvalue_out,
                      double* stat_out, double* se_out);
int pdq_alpha_mle_dev(pdq_ctx* ctx, const pdq_design* design, const int64_t* counts, int64_t ld, int G,
                      const double* mu, int64_t ld_mu, const double* alpha_hat, double min_disp,
                      double max_disp, double prior_disp_var,
                      const double* prior_var_dev /* device double overriding prior_disp_var, may be NULL */,
                      int cr_reg, int prior_reg, double* alpha_out, double* converged_out);
/* pdq_alpha_mle_dev with a carried-over search state.  `hint_out` (device, [G][2], may be NULL) receives per gene the optimum
 * x* = log(alpha) this search found and the curvature h* of its loss there; `hint_in` (may be NULL) takes such a record from an
 * earlier search on the SAME counts and means WITHOUT the prior -- the genewise fit, dds.py:778 -- so that the MAP search
 * (dds.py:901; objective = that loss + (x - log alpha_hat)^2 / (2 var)) opens with a Newton step of the MAP objective from x*
 * instead of walking in from log(alpha_hat): ~2.2 evaluations per gene instead of ~3.5, same optimum (the start point is still
 * evaluated first: the reference's rules that keep a gene at its start value are applied unchanged). */
int pdq_alpha_mle_hint_dev(pdq_ctx* ctx, const pdq_design* design, const int64_t* counts, int64_t ld, int G,
                           const double* mu, int64_t ld_mu, const double* alpha_hat, double min_disp,
                           double max_disp, double prior_disp_var, const double* prior_var_dev, int cr_reg,
                           int prior_reg, double* alpha_out, double* converged_out, const double* hint_in,
                           double* hint_out);
int pdq_wald_test_dev(pdq_ctx* ctx, const pdq_design* design, const double* disp, const double* lfc,
                      const double* mu, int64_t ld_mu, int G, const double* ridge_host,
                      const double* contrast_host, double lfc_null, int alt, double* pvalue_out,
                      double* stat_out, double* se_out);
/* Method-of-moments start values straight from raw counts (fuses `counts / size_factors`,
 * fit_rough_dispersions, fit_moments_dispersions, the min() and clip of dds.py:1140-1162) and the
 * per-gene normalised mean (`dds.py:708`).  Device-resident pipeline only. */
int pdq_mom_dispersions_dev(pdq_ctx* ctx, const pdq_design* design, const int64_t* counts, int64_t ld,
                            int G, double min_disp, double max_disp, double* alpha_out,
                            double* normed_mean_out, double min_mu,
                            double* mu_hat_out /* (N,G), may be NULL: also the lin_reg_mu result, same projection */,
                            int64_t ld_mu);
/* Parametric dispersion trend INCLUDING the caller's outer loop (dds.py:1199-1275: fit, drop genes with
 * genewise/fitted outside [1e-4, 15), refit until sum(log(c/c_old)^2) < 1e-6) AND the dispersion prior
 * (dds.py:840-884: squared scaled MAD of the log residuals, prior variance), entirely on the device in one launch of
 * one thread-block cluster.  `normed_means`, `genewise` (n,) device; genewise is clipped to [min_disp, max_disp] on
 * the fly (dds.py:792); NaN entries (padding of ragged gene shards) are ignored.  `trigamma_c` = polygamma(1, (N-p)/2).
 * `out16` (16 doubles, device): c0, c1, status (0 ok / 1 = caller must fall back to the mean trend), outer rounds,
 * genes used, inner iterations, loss, last fit converged, squared_logres, prior_var, genes above 100*min_disp, 0...
 * `fitted_out` (n,) device, may be NULL: c0 + c1 / mean. */
int pdq_trend_fit_dev(pdq_ctx* ctx, const double* normed_means, const double* genewise, size_t n, double min_disp,
                      double max_disp, double trigamma_c, double* out16, double* fitted_out);
int pdq_cooks_dev(pdq_ctx* ctx, const pdq_design* design, const int64_t* counts, int64_t ld, int G, const double* mu,
                  const double* hat, int64_t ld2, double cutoff, double* cooks_out, int64_t ld_out,
                  double* robust_disp_out, double* outlier_out, double* replaced_out);
/* device-resident flavour of pdq_lfc_shrink_nbinom_glm: the offsets are the log size factors of `design`;
 * `status_out` (G,) ints, 1 = refitted on the grid */
int pdq_lfc_shrink_dev(pdq_ctx* ctx, const pdq_design* design, const int64_t* counts, int64_t ld, int G, const double* size,
                       double prior_no_shrink_scale, double prior_scale, int shrink_index, double* lfcs_out,
                       double* inv_hessians_out, double* converged_out, int* status_out);
/* device-resident flavour of pdq_size_factors; `logmeans_out` (G,) may be NULL */
int pdq_size_factors_dev(pdq_ctx* ctx, const int64_t* counts, int64_t ld, int N, int G, double* sf_out,
                         double* logmeans_out);
/* Final dispersions (dds.py:918-932): clip(MAP), except genes with log(genewise) > log(fitted) + 2 sqrt(squared_logres)
 * which keep their clipped genewise value; `trend_out16` is the record written by pdq_trend_fit_dev.
 * `outlier_out` (n,) 0/1 may be NULL. */
/* out[n, j] = in[n, idx[j]] for j < R: selected gene columns of a resident (samples, genes) array as a compact (samples, R)
 * array -- what the Cook's outlier refit (dds.py:1301-1458) needs from the device for the few replaced genes. */
int pdq_gather_columns_dev(pdq_ctx* ctx, const double* in, int64_t ld_in, int N, const int* idx_dev, int R, double* out,
                           int64_t ld_out);
/* Gene order of a resident shard.  pdq_column_sums_dev: per-gene total count (device, G doubles).  pdq_scatter_rows_dev:
 * out[v][perm[j]][k] = in[v][j][k] for `nvec` blocks of `stride` rows of `width` doubles -- per-gene results computed in a
 * device-friendly gene order (ResidentFit sorts the columns by total count at upload: the four genes a warp iterates in lock
 * step then need similar iteration counts) returned to the caller's order. */
int pdq_column_sums_dev(pdq_ctx* ctx, const int64_t* counts, int64_t ld, int N, int G, double* sums_out);
int pdq_scatter_rows_dev(pdq_ctx* ctx, const double* in, double* out, const int* perm_dev, int n, int nvec, int64_t stride,
                         int width);
int pdq_select_dispersions_dev(pdq_ctx* ctx, const double* genewise, const double* map, const double* fitted,
                               const double* trend_out16, size_t n, double min_disp, double max_disp,
                               double* disp_out, double* outlier_out);
/* mu = size_factor * exp(X beta) for the Wald stage (ds.py:320-324), device-resident */
int pdq_mu_from_lfc_dev(pdq_ctx* ctx, const pdq_design* design, const double* lfc, int G,
                        double* mu_out, int64_t ld_out);

/* ----------------------------------------------------------------- multi-GPU (gene shards)
 * One process per GPU.  Rank 0 calls pdq_comm_unique_id and ships the 128 bytes to the other ranks
 * (any out-of-band channel); every rank then calls pdq_comm_init.  The only exchange on the path is
 * the all-gather of per-gene vectors (genewise dispersions + normalised means before the trend fit,
 * final per-gene results at the end).  `count` doubles are contributed per rank. */
#define PDQ_UNIQUE_ID_BYTES 128
int pdq_comm_unique_id(pdq_ctx* ctx, void* id_out);
int pdq_comm_init(pdq_ctx* ctx, const void* id, int world_size, int rank);
int pdq_allgather_f64_dev(pdq_ctx* ctx, const double* send, double* recv, size_t count);
/* k (<= 16) equal-count all-gathers issued as one NCCL group -- a single fused launch on the context's stream.  `send` / `recv`
 * are HOST arrays of k device pointers; recv[i] receives world * count doubles in rank order. */
int pdq_allgather_multi_f64_dev(pdq_ctx* ctx, int k, const double* const* send, double* const* recv, size_t count);
int pdq_comm_destroy(pdq_ctx* ctx);

/* Peer-memory flavour of the same two exchanges (ranks of ONE node; CUDA IPC + NVLink peer stores, no NCCL on the data path).
 * Every rank allocates a window (`data_bytes` of payload, identical on all ranks), ships the 64-byte handle to its peers through any
 * out-of-band channel, and opens the group with the `world` handles in rank order.  `pdq_peer_push_dev` is ONE kernel on the
 * context's stream: it stores segment i (`count` doubles) of this rank at payload offset recv_off_bytes[i] + rank * count * 8 of
 * EVERY rank's window and completes once all ranks' segments have arrived in the own window (copy + barrier; k = 0: barrier
 * only); capturable into a CUDA graph.  A peer that never arrives is reported through `pdq_peer_status` (1 + its rank) after
 * PDQ_PEER_TIMEOUT_MS (default 30 000) instead of hanging the device.  Every rank must close its group before any rank frees
 * its window.  Replaces, like the NCCL calls above, the host-side concatenation of per-shard results a multi-process caller of the
 * reference would do (the reference itself is single-process: `default_inference.py:18-41` fans genes out over joblib workers). */
#define PDQ_PEER_HANDLE_BYTES 64
typedef struct pdq_peer_group pdq_peer_group;
int pdq_peer_window_alloc(pdq_ctx* ctx, size_t data_bytes, void** window_out, void** data_out, void* handle_out);
int pdq_peer_window_free(pdq_ctx* ctx, void* window);
int pdq_peer_group_open(pdq_ctx* ctx, void* own_window, int world_size, int rank, const void* handles, pdq_peer_group** group_out);
int pdq_peer_push_dev(pdq_ctx* ctx, pdq_peer_group* group, int k, const double* const* send, const unsigned long long* recv_off_bytes,
                      size_t count);
int pdq_peer_status(pdq_ctx* ctx, pdq_peer_group* group, unsigned long long* status_out);
int pdq_peer_group_close(pdq_ctx* ctx, pdq_peer_group* group);

#ifdef __cplusplus
}
#endif
#endif /* PYDESEQ2_B200_H */
